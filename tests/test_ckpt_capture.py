"""The checkpointer's device mode (``train._AsyncCheckpointer`` with an engine) on the CPU, against a fake engine: pending and
landed captures, a failed capture retried at the next step, host arenas not reused while the saver thread holds them, and
the blocking final save with its timeout."""
import os
import threading

import pytest
import torch

from distributedmnist_b200.checkpoint import Saver, get_checkpoint_state
from distributedmnist_b200.train import _AsyncCheckpointer


class _Spec:
    def to_state_dict(self, flat):
        return {"w": flat.clone()}


class _FakeEngine:
    """Captures land when the test says so (``land``) or when waited for; capture i reports ``outcomes[i]`` as its step
    (-1: no consistent snapshot), by default 10 * seq.  A capture fills its host arena with its step."""

    def __init__(self, outcomes=(), then=None):
        self.then = then                                   # step of every capture after ``outcomes`` (None: 10 * seq)
        self.ckpt_host = [torch.zeros(4) for _ in range(2)]
        self.outcomes = list(outcomes)
        self.inflight = None
        self.landed = False
        self.enqueued = []
        self.seq = 0

    def enqueue_checkpoint(self, buf):
        assert self.inflight is None, "two captures in flight"
        self.seq += 1
        step = self.outcomes.pop(0) if self.outcomes else (10 * self.seq if self.then is None else self.then)
        self.ckpt_host[buf].fill_(float(step))
        self.inflight, self.landed = (self.seq, buf, step), False
        self.enqueued.append(buf)
        return self.seq

    def land(self):
        self.landed = True

    def checkpoint_poll(self):
        if self.inflight is None or not self.landed:
            return None
        rec, self.inflight = self.inflight, None
        return rec

    def checkpoint_wait(self):
        if self.inflight is None:
            return None
        self.landed = True
        return self.checkpoint_poll()


def _files(d):
    return sorted(f for f in os.listdir(d) if f.endswith(".index")) if os.path.isdir(d) else []


def _ckpt(tmp_path, eng, interval_s=0.0, timeout_s=1.0):
    return _AsyncCheckpointer(str(tmp_path / "train"), _Spec(), interval_s, engine=eng, timeout_s=timeout_s)


def test_a_capture_is_enqueued_polled_and_written_once_it_has_landed(tmp_path):
    eng = _FakeEngine()
    ck = _ckpt(tmp_path, eng, interval_s=1000.0)
    ck._next = 0.0                                         # due now
    ck.maybe_save(None, 0)
    assert eng.enqueued == [0]
    for _ in range(3):                                     # pending: polled, nothing new enqueued, nothing written
        ck.maybe_save(None, 0)
    assert eng.enqueued == [0] and eng.inflight is not None
    eng.land()
    ck.maybe_save(None, 0)                                 # landed: handed to the saver thread; not due again for 1000 s
    ck._queue.join()
    assert eng.enqueued == [0] and eng.inflight is None
    assert _files(tmp_path / "train") == ["model.ckpt-10.index"]
    state, step = Saver.restore(Saver.latest(str(tmp_path / "train")))
    assert step == 10 and torch.equal(state["w"], torch.full((4,), 10.0))
    ck.close()


def test_a_failed_capture_writes_nothing_and_is_retried_at_the_next_step(tmp_path):
    eng = _FakeEngine(outcomes=[-1, -1, 7])
    ck = _ckpt(tmp_path, eng, interval_s=1000.0)
    ck._next = 0.0
    ck.maybe_save(None, 0)
    for n in (2, 3):
        eng.land()
        ck.maybe_save(None, 0)                             # failure seen -> the retry is enqueued in the same call
        assert len(eng.enqueued) == n and ck.failed == n - 1
    ck._queue.join()
    assert _files(tmp_path / "train") == []
    eng.land()
    ck.maybe_save(None, 0)
    ck.maybe_save(None, 0)                                 # accepted: no retry, and the interval has not passed
    ck._queue.join()
    assert len(eng.enqueued) == 3 and ck.failed == 2
    assert _files(tmp_path / "train") == ["model.ckpt-7.index"]
    ck.close()


def test_a_host_arena_is_not_reused_while_the_saver_thread_holds_it(tmp_path):
    eng = _FakeEngine()
    ck = _ckpt(tmp_path, eng, interval_s=0.0)
    gate, inside = threading.Event(), threading.Event()
    real = ck.saver.save

    def slow_save(train_dir, state, step):
        inside.set()
        assert gate.wait(10.0)
        return real(train_dir, state, step)
    ck.saver.save = slow_save
    ck.maybe_save(None, 0)                                 # capture 1 -> arena 0
    eng.land()
    ck.maybe_save(None, 0)                                 # arena 0 to the (blocked) saver, capture 2 -> arena 1
    assert inside.wait(10.0)
    assert eng.enqueued == [0, 1]
    eng.land()
    for _ in range(3):                                     # arena 1 queued behind arena 0: no arena is free
        ck.maybe_save(None, 0)
    assert eng.enqueued == [0, 1] and eng.inflight is None
    assert ck.engine.ckpt_host[0][0] == 10.0 and ck.engine.ckpt_host[1][0] == 20.0     # untouched while held
    gate.set()
    ck._queue.join()
    ck.maybe_save(None, 0)
    assert eng.enqueued == [0, 1, 0]
    assert _files(tmp_path / "train") == ["model.ckpt-10.index", "model.ckpt-20.index"]
    eng.land()
    ck.save(None, 0)
    ck.close()
    assert get_checkpoint_state(str(tmp_path / "train")).model_checkpoint_path == "model.ckpt-40"


def test_the_final_save_blocks_and_retries_until_a_capture_is_accepted(tmp_path):
    eng = _FakeEngine(outcomes=[-1, -1, 9])
    ck = _ckpt(tmp_path, eng, interval_s=1000.0)
    ck.save(None, 0)
    assert ck.failed == 2 and len(eng.enqueued) == 3
    assert _files(tmp_path / "train") == ["model.ckpt-9.index"]          # written before save() returned
    ck.close()


def test_the_final_save_writes_a_periodic_capture_still_in_flight_first(tmp_path):
    eng = _FakeEngine(outcomes=[5, 6])
    ck = _ckpt(tmp_path, eng, interval_s=0.0)
    ck.maybe_save(None, 0)
    ck.save(None, 0)
    ck.close()
    assert _files(tmp_path / "train") == ["model.ckpt-5.index", "model.ckpt-6.index"]
    assert Saver.restore(Saver.latest(str(tmp_path / "train")))[1] == 6


def test_the_final_save_fails_after_its_timeout_without_writing_anything(tmp_path):
    eng = _FakeEngine(then=-1)
    ck = _ckpt(tmp_path, eng, interval_s=1000.0, timeout_s=0.05)
    with pytest.raises(RuntimeError, match="no consistent snapshot"):
        ck.save(None, 0)
    ck.close()
    assert ck.failed >= 1 and _files(tmp_path / "train") == []
