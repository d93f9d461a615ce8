"""Fused allreduce+scale+SGD kernel vs `NCCL allreduce -> /N -> torch SGD` (SURVEY §4 item 4)."""
import json
import os

import pytest
import torch

from distributedmnist_b200.parallel.launcher import run_replicas

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_single_rank_is_plain_sgd():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    be = FusedBackend(ctx)
    n = 1 << 16
    params, grads = be.allocate(n), be.allocate(n)
    be.attach_shadow(params)
    params.copy_(torch.randn(n, device="cuda"))
    ref = params.clone()
    for step in range(4):
        grads.copy_(torch.randn(n, device="cuda"))
        ref -= 0.25 * grads
        info = be.sync_step(params, grads, 0.25, step, 1)
        assert info.global_step == step + 1 and info.accepted and info.mask == 1 and info.count == 1
        assert torch.allclose(params, ref, atol=1e-6)
        assert (be.shadow.float() - params).abs().max().item() < 0.02 * params.abs().max().item()
    # device-side LR schedule: staircase decay evaluated from the device step counter
    be.enqueue(params, grads, 1, lr0=1.0, decay_rate=0.5, decay_steps=2)   # epoch 4 -> lr = 0.25
    ref -= 0.25 * grads
    torch.cuda.synchronize()
    assert torch.allclose(params, ref, atol=1e-6)
    be.check_error()


def test_gradient_drop_connect_mask_in_the_load_stage():
    """reference distributed_train.py:194-196,414-416: Bernoulli(p) 0/1 mask on every gradient element, no 1/p rescale."""
    from distributedmnist_b200.models import dropout_keep_mask
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    n = 1 << 14
    params, grads = be.allocate(n), be.allocate(n)
    params.copy_(torch.randn(n, device="cuda"))
    grads.copy_(torch.randn(n, device="cuda"))
    be.drop_connect_(grads, 0.9, 0)
    ref = params.clone()
    for step in range(3):
        mix = (be.drop_seed + step * 0x9E3779B9 + 0 * 0x85EBCA77) & 0xFFFFFFFF
        keep = dropout_keep_mask(mix, 1, n, 0.9, device="cuda").view(-1)
        ref -= 0.5 * grads * keep
        be.sync_step(params, grads, 0.5, step, 1)
        assert torch.allclose(params, ref, atol=1e-6)
        assert 0.85 < keep.float().mean().item() < 0.95


@pytest.mark.multigpu
def test_k_of_n_training_through_the_reference_entrypoint(tmp_path):
    """2 replicas, K=1, rank 1 delayed on the device every step: training proceeds at rank 0's pace,
    rank 1's gradients are dropped, both logs show the same global steps."""
    import re
    import sys

    from distributedmnist_b200.parallel.launcher import run_replicas
    root = os.path.dirname(HERE)
    codes = run_replicas([os.path.join(root, "src", "mnist_distributed_train.py"), "--job_name=worker",
                          "--batch_size=64", "--max_steps=400", "--num_replicas_to_aggregate=1",
                          "--inject_straggler=1:1.0:1000", "--initial_learning_rate=0.02",
                          "--train_dir=" + str(tmp_path / "train_dir"), "--save_interval_secs=1000"],
                         2, timeout=300, out_dir=str(tmp_path / "out"))
    logs = {f: open(os.path.join(tmp_path, "out", f)).read() for f in sorted(os.listdir(tmp_path / "out"))}
    assert codes == [0, 0], "\n".join(v[-1500:] for v in logs.values())
    s0 = [int(x) for x in re.findall(r"Worker 0: .*: step ([0-9]+),", logs["out_master"])]
    s1 = [int(x) for x in re.findall(r"Worker 1: .*: step ([0-9]+),", logs["out_worker_0"])]
    # Each replica logs the global steps it took part in or woke up in.  With K = 1 whoever arrives first commits the
    # step and the other one's gradient is dropped: its next iteration fast-forwards to the newest committed step
    # (reference: stale push dropped, worker proceeds, ...modified.py:59-62,87-90), so at least one replica logs fewer
    # local iterations than global steps, and nobody ever goes backwards.
    assert s0 and s1 and max(max(s0), max(s1)) >= 400, (s0, s1)
    assert s0 == sorted(set(s0)) and s1 == sorted(set(s1)), (s0, s1)
    assert len(s0) < max(s0) or len(s1) < max(s1), (s0, s1)
    assert os.path.exists(tmp_path / "train_dir" / "checkpoint")


@pytest.mark.multigpu
def test_multi_rank_matches_nccl_and_masks_straggler(tmp_path):
    n = min(torch.cuda.device_count(), 8)
    worker = os.path.join(HERE, "_fused_worker.py")
    codes = run_replicas([worker, str(tmp_path / "res_RANK.json"), str(1665024)], n, timeout=300,
                         out_dir=str(tmp_path / "out"))
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    res = [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(n)]
    full_mask = (1 << n) - 1
    for s in range(6):
        rows = [r["full"][s] for r in res]
        assert all(x["mask"] == full_mask and x["count"] == n and x["accepted"] for x in rows)
        assert all(x["err"] < 1e-5 for x in rows), rows         # tolerance: reduction order only
        assert len({x["fp"] for x in rows}) == 1                  # replicas bit-identical
        assert all(x["shadow_err"] < 0.05 for x in rows)
    for s in range(6):
        rows = [r["kofn"][s] for r in res]
        assert len({x["mask"] for x in rows}) == 1                # same contributor set everywhere
        m = rows[0]["mask"]
        assert bin(m).count("1") >= n - 1 and all(x["count"] == bin(m).count("1") for x in rows)
        assert not (m >> (n - 1)) & 1                             # the delayed rank is masked out
        assert not rows[n - 1]["accepted"] and all(rows[q]["accepted"] for q in range(n - 1))
        assert all(x["err"] < 1e-5 for x in rows), rows         # divisor = accepted count
        assert len({x["fp"] for x in rows}) == 1


def _check_bucket_unit(res, n):
    for s in range(5):
        rows = [r["rows"][s] for r in res]
        assert all(x["step"] == s + 1 and x["count"] == n and x["mask"] == (1 << n) - 1 for x in rows), rows
        assert len({x["fp"] for x in rows}) == 1, ("replicas differ", s)          # bit-identical weights everywhere
        assert len({x["fp_g16"] for x in rows}) == 1, ("reduced gradients differ", s)
        assert all(x["late_err"] < 2e-6 for x in rows), rows                      # fp32 rank-ordered sum vs NCCL
        assert all(x["fc1_bad"] == 0 for x in rows), rows                         # bf16 wire: one rounding of the sum
        assert all(x["sum_rel_err"] < 2.0 ** -7 for x in rows), rows
        assert all(x["shadow_err"] <= 0.01 * x["pmax"] + 1e-6 for x in rows), rows


def test_bucket_kernels_single_replica(tmp_path):
    """One replica: no exchange, the early kernel applies SGD to fc1 from the bf16 gradient, the late kernel the rest."""
    worker = os.path.join(HERE, "_bucket_unit_worker.py")
    codes = run_replicas([worker, str(tmp_path / "res_RANK.json")], 1, timeout=300, out_dir=str(tmp_path / "out"))
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0], logs
    _check_bucket_unit([json.load(open(tmp_path / "res_0.json"))], 1)


@pytest.mark.multigpu
def test_bucket_kernels_match_nccl_oracle(tmp_path):
    """csrc/fused_bucket.cu against NCCL directly: early bucket = in-place bf16 reduce (NVLS multimem / peer loads) + local
    SGD, late bucket = pushed inbox + rank-ordered fp32 sum; own VMM/NVLS allocator (csrc/symm_mem.cu) and torch's."""
    n = min(torch.cuda.device_count(), 8)
    worker = os.path.join(HERE, "_bucket_unit_worker.py")
    for tag, env in (("p2p", {"DMNIST_NVLS": "0"}), ("nvls_own", {"DMNIST_NVLS": "1", "DMNIST_SYMM": "own"}),
                     ("nvls_torch", {"DMNIST_NVLS": "1", "DMNIST_SYMM": "torch"})):
        out = tmp_path / tag
        codes = run_replicas([worker, str(out / "res_RANK.json")], n, timeout=300, out_dir=str(out / "out"), env=env)
        logs = "\n".join(open(os.path.join(out, "out", f)).read()[-1500:] for f in sorted(os.listdir(out / "out")))
        assert codes == [0] * n, tag + "\n" + logs
        res = [json.load(open(out / ("res_%d.json" % r))) for r in range(n)]
        _check_bucket_unit(res, n)
        if tag == "nvls_own":
            # the product path: multicast mapping created by our own driver-API code
            assert all(r["alloc"] == "VmmBuffer" for r in res), [r["alloc"] for r in res]
            assert all(r["nvls"] and r["mc_ptr"] for r in res), "own NVLS multicast set-up did not come up"


@pytest.mark.multigpu
def test_bucketed_overlapped_aggregation_matches_single_kernel(tmp_path):
    """The bucketed path (early fc bucket next to the backward kernels + one-shot late conv bucket) must leave every
    replica with bit-identical weights, and with the same weights as the single-kernel path (peer loads sum in rank
    order on both; the NVLS run may differ by the switch's reduction order only)."""
    n = min(torch.cuda.device_count(), 8)
    worker = os.path.join(HERE, "_bucket_worker.py")
    res = {}
    for tag, env in (("bucket", {"DMNIST_BUCKET": "1", "DMNIST_NVLS": "0"}), ("single", {"DMNIST_BUCKET": "0", "DMNIST_NVLS": "0"}),
                     ("bucket_nvls", {"DMNIST_BUCKET": "1", "DMNIST_NVLS": "1"}),
                     ("v2", {"DMNIST_BUCKET": "2", "DMNIST_NVLS": "0"}), ("v2_nvls", {"DMNIST_BUCKET": "2", "DMNIST_NVLS": "1"})):
        out = tmp_path / tag
        codes = run_replicas([worker, str(out / "res_RANK.json"), "8"], n, timeout=300, out_dir=str(out / "out"), env=env)
        logs = "\n".join(open(os.path.join(out, "out", f)).read()[-1500:] for f in sorted(os.listdir(out / "out")))
        assert codes == [0] * n, tag + "\n" + logs
        res[tag] = [json.load(open(out / ("res_%d.json" % r))) for r in range(n)]
    assert all(r["bucketed"] for r in res["bucket"]) and not any(r["bucketed"] for r in res["single"])
    assert all(r["bucketed"] and r["v2"] for r in res["v2"]) and all(r["v2"] for r in res["v2_nvls"])
    for tag in res:
        for s in range(8):
            rows = [r["rows"][s] for r in res[tag]]
            assert len({x["fp"] for x in rows}) == 1, (tag, s)                   # replicas bit-identical
            assert all(x["step"] == s + 1 and x["count"] == n and x["mask"] == (1 << n) - 1 for x in rows), (tag, rows)
            assert all(x["shadow_err"] <= 0.01 * x["pmax"] + 1e-6 for x in rows), (tag, rows)
    # the aggregation paths do not apply bit-identical updates: they add the replicas' gradients in different orders, and
    # the bucketed v2 path sends its late bucket (everything but fc1's weights) as bf16 by default (DMNIST_LATE_BF16=1), as it
    # does fc1's gradient.  So they are compared tightly after the first update and loosely after eight, once ReLU /
    # max-pool / dropout decisions have amplified the differences
    first = {t: torch.tensor(res[t][0]["rows"][0]["sample"]) for t in res}
    last = {t: torch.tensor(res[t][0]["rows"][-1]["sample"]) for t in res}
    assert (first["bucket"] - first["single"]).abs().max().item() < 2e-6
    assert (first["bucket_nvls"] - first["bucket"]).abs().max().item() < 2e-6
    assert (last["bucket"] - last["single"]).abs().max().item() < 2e-2
    assert (last["bucket_nvls"] - last["bucket"]).abs().max().item() < 2e-2
    # bf16 wire (csrc/fused_bucket.cu): fc1's gradient is rounded to bf16 before and after the reduction -> the first update
    # differs from the fp32 path by <= lr * 2^-8 * |g|
    assert (first["v2"] - first["single"]).abs().max().item() < 2e-5
    assert (first["v2_nvls"] - first["v2"]).abs().max().item() < 2e-5
    assert (last["v2"] - last["single"]).abs().max().item() < 2e-2
    assert (last["v2_nvls"] - last["v2"]).abs().max().item() < 2e-2
    assert res["bucket"][0]["rows"][-1]["loss"] == res["bucket"][0]["rows"][-1]["loss"]      # not NaN


def _run_interval(tmp_path, n, interval_ms, iters, delay_us):
    worker = os.path.join(HERE, "_interval_worker.py")
    codes = run_replicas([worker, str(tmp_path / "res_RANK.json"), str(interval_ms), str(iters), str(delay_us)], n,
                         timeout=300, out_dir=str(tmp_path / "out"))
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    return [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(n)]


def test_interval_mode_single_replica_ticks_on_the_device_clock(tmp_path):
    """Mode C on the device (csrc/fused_interval.cu), one replica: gradients accumulate locally, a tick applies their mean
    when the %globaltimer deadline has passed -- ~0.2 ms per iteration and 2 ms ticks: far fewer steps than iterations."""
    (res,) = _run_interval(tmp_path, 1, 2.0, 150, 0)
    assert 3 <= res["steps"] <= 40, res["steps"]
    assert res["err"] < 1e-5 * max(1.0, res["pmax"]), res["err"]
    assert res["dropped"] == 0 and res["accepted"] == 150
    assert all(row[2] == 1 for row in res["rows"] if row[0] > 0)          # mask = {0} on every committed tick
    assert max(row[3] for row in res["rows"]) >= 3                        # several gradients per tick: divisor = their number


@pytest.mark.multigpu
def test_interval_mode_device_deadline_masks_the_late_replica(tmp_path):
    """Several replicas free-run; the last one needs 3 ticks per iteration.  Nobody waits for it: ticks commit with the
    replicas that have something accumulated (it is missing from those masks), its stale gradients are dropped, and all
    replicas end with bit-identical weights = w0 - steps * lr * g."""
    n = min(torch.cuda.device_count(), 8)
    res = _run_interval(tmp_path, n, 2.0, 120, 6000.0)
    steps = {r["steps"] for r in res}
    assert len(steps) == 1 and 3 <= res[0]["steps"] <= 80, [r["steps"] for r in res]
    assert len({r["fp"] for r in res}) == 1                               # replicas bit-identical once quiescent
    assert all(r["err"] < 1e-5 * max(1.0, r["pmax"]) for r in res), [r["err"] for r in res]
    assert all(r["shadow_err"] <= 0.01 * r["pmax"] + 1e-6 for r in res)
    masks = {row[2] for r in res for row in r["rows"] if row[0] > 0}
    late_bit = 1 << (n - 1)
    assert any(m and not (m & late_bit) for m in masks), masks           # some tick committed without the delayed replica
    assert res[n - 1]["dropped"] > 0                                      # ... whose stale gradients were discarded
    assert sum(r["ticks_committed"] for r in res) == res[0]["steps"]     # every step has exactly one committer


@pytest.mark.multigpu
def test_message_passing_litmus_over_nvlink_and_nvls(tmp_path):
    """The ordering pattern of every aggregation kernel, 20 000 rounds inside one launch on two GPUs: weak stores ->
    bar.sync -> fence.sys + st.release.sys(flag on the peer) || ld.acquire.sys(flag) -> bar.sync -> peer loads and
    multimem.ld_reduce of the data.  Any stale value is a violation."""
    worker = os.path.join(HERE, "_litmus_worker.py")
    codes = run_replicas([worker, str(tmp_path / "res_RANK.json"), "20000"], 2, timeout=300, out_dir=str(tmp_path / "out"))
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0, 0], logs
    w, r = (json.load(open(tmp_path / ("res_%d.json" % q))) for q in range(2))
    assert not w["aborted"] and not r["aborted"], (w, r)
    assert w["rounds"] == 20000 and r["rounds"] == 20000, (w, r)
    assert r["bad_p2p"] == 0 and r["bad_mc"] == 0, r
