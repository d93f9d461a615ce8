"""Back-to-back training steps checked stage by stage against the float64 references.

:class:`StepRecorder` clones, after each enqueued step and on that step's stream (no host synchronisation), the buffers
every stage of the step wrote, and the gradients, weights, bf16 shadow and (loss, accuracy) it left.
:func:`lenet_trajectory_results` / :func:`mlp_trajectory_results` then judge each step from the records alone, with the
bounds the kernel checks use (``ops/selfcheck.py``):

* each stage from its recorded inputs, on the weights the previous step committed (the initial arena for the first);
  the bf16 shadow a step reads is RNE of those weights, the dropout mask the one of the epoch word the step read;
* the update bit for bit against ``ops/aggrefs.py``, and the recorded shadow as RNE of the recorded weights (with K > N
  and in interval mode: of the weights the step adopted);
* with random affine augmentation (and elastic distortion) armed, the recorded augmented buffer against the float64 warp
  of the fed batch with the draws of the step's own iteration, the iteration counter after every step, and every reader of the images
  (conv1 forward and wgrad, the MLP's x16) against that step's recorded buffer;
* in interval mode (and with K > N, and with the cdf telemetry stamps) the replica's control block after every step.  An
  interval step commits when its close finds the wall-clock deadline passed, which no host-side model can predict; the
  block holds every decision the device took, so the checker reads the commits from it (:func:`interval_trace`), judges
  the update bit for bit against the ticks that happened, and checks the decisions against the device's own
  ``%globaltimer`` stamps (:func:`control_results`).

The input slots are not recorded: the copy stream may refill a slot as soon as the step that read it is done.  The caller
passes what it fed each step, so a step that computed on another batch fails its stage checks.
"""
from __future__ import annotations

import re
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ..lr_plateau import NO_CUT
from ..models import dropout_keep_mask, dropout_seed_mix
from . import aggrefs as A
from . import refs as R
from . import selfcheck as S

Result = S.Result
LENET_BUFFERS = ("a1", "code1", "a2", "code2", "h_part", "dh", "h_act", "dlogits", "dy2", "dx1")
MLP_BUFFERS = ("x16", "h", "dh", "dl_pad")
# the control-block words the checks read (csrc/fused_sync.cuh, SyncCtrl), and the length of its stamp rings
CTRL_U32 = ("epoch", "error", "accepted_steps", "dropped_steps", "last_count", "iv_ticks_committed")
CTRL_U64 = ("iv_state", "iv_deadline")
TIMING_RING = 1024


class StepRecorder:
    """Call :meth:`record` right after each step is enqueued (``train_step``, ``step_packed``, ``step_indices``), on the
    stream the step was enqueued on: the clones then run after the step and before the next one.  The native runner
    launches on the stream that was current when it was created, so this holds for its steps too.

    In interval mode, with K > N and with the cdf stamps, the replica's control block is recorded too (raw bytes, decoded
    by :func:`ctrl_words`): once now, so arm the interval clock before creating the recorder, and after every step."""

    def __init__(self, eng):
        self.eng = eng
        # asynchronous SGD: ``params`` is the master copy, which the update changes (with one replica the next step pulls
        # it as it is); the working arena is recorded as ``pulled``
        self._async = getattr(eng, "_async", False)
        self.init = dict(params=(eng._master if self._async else eng.params).clone(), shadow=eng.shadow.clone())
        if getattr(eng, "_aug", None) is not None:
            self.init["aug_counter"] = eng._aug_counter.clone()
        self._ctrl = getattr(eng, "_interval", False) or getattr(eng, "_stamp", False)
        if self._ctrl:
            self.init["ctrl"] = eng.backend._ctrl_bytes.clone()
        self.records: List[Dict[str, object]] = []

    def record(self) -> None:
        e = self.eng
        r: Dict[str, object] = {}
        for name in (LENET_BUFFERS if hasattr(e, "h_part") else MLP_BUFFERS):
            v = getattr(e, name)
            r[name] = [t.clone() for t in v] if isinstance(v, list) else v.clone()
        r.update(grads=e.grads.clone(), params=(e._master if self._async else e.params).clone(), shadow=e.shadow.clone(),
                 loss_acc=e.d_loss_acc.clone())
        if self._async:
            r["pulled"] = e.params.clone()
        if e._bucket_v2:
            r["g16"] = e._g16_view.clone()
        if getattr(e, "_decay", 0.0):
            r["decay_ws"] = e._decay_ws.clone()         # the W^2 partials of both weight-gradient kernels, then R
        if getattr(e, "_aug", None) is not None:        # the next step's augmentation node overwrites both
            r["aug_images"] = e._aug_images.clone()
            r["aug_counter"] = e._aug_counter.clone()
        if self._ctrl:
            r["ctrl"] = e.backend._ctrl_bytes.clone()
        self.records.append(r)


def ctrl_words(raw, off: Dict[str, int], stamp_step: Optional[int] = None) -> Dict[str, int]:
    """The words of a recorded control block (``raw``: its bytes, a tensor or an array) at the byte offsets ``off``
    (``FusedBackend._off``): CTRL_U32 and CTRL_U64, and ``t_start`` / ``t_arrive`` of step ``stamp_step`` (default: the
    block's epoch word) from the stamp rings."""
    b = (raw.detach().cpu().numpy() if isinstance(raw, torch.Tensor) else np.asarray(raw)).view(np.uint8)

    def word(o: int, n: int) -> int:
        return int(b[o:o + n].view("<u%d" % n)[0])
    w = {f: word(off[f], 4) for f in CTRL_U32}
    w.update({f: word(off[f], 8) for f in CTRL_U64})
    s = (w["epoch"] if stamp_step is None else stamp_step) % TIMING_RING
    w["t_start"], w["t_arrive"] = word(off["t_start"] + 8 * s, 8), word(off["t_arrive"] + 8 * s, 8)
    return w


def update_of(eng, sched, step0: int, aug_start: int = 0) -> dict:
    """How ``eng`` applies its gradients: ``mode`` "fused" (fused_sync_sgd), "bucket" (the bf16-wire bucketed kernels),
    "kgtn" (K > N: every k-th iteration commits), "interval" (a tick commits when its deadline has passed; ``interval_ns``
    the armed period), "async" (asynchronous SGD on one replica: every step pulls the master copy and adds its update),
    "local" (local SGD on one replica: every step applies its own update, every ``period``-th global step is averaged) or
    "gossip" (gossip SGD on one replica: every step mixes its own half step, a neighbourhood of one), the schedule and the global step of the first step.  ``drop``:
    (seed, keep probability) of the drop-connect mask the fused kernel applies, None without it.  With a cut table armed
    (``arm_lr_cuts``), ``sched`` must name the same cuts (raises ValueError otherwise): the step sizes are then those of
    the schedule with the cuts (synchronises the device to read the table).  ``aug``: (ranges, seed mix) of the armed
    augmentation, None without it; ``aug_start`` the iteration the run's first step draws from (see
    :func:`augment_stage_results`); ``elastic`` the armed ``augment.Elastic``, None without elastic distortion.
    ``ctrl_off``: the control block's byte offsets, for the recorded blocks (see :func:`ctrl_words`)."""
    be = eng.backend
    e0, e1 = eng._bucket_early
    if getattr(eng, "_async", False):
        mode = "async"
    elif getattr(eng, "_local", 0):
        mode = "local"
    elif getattr(eng, "_gossip", False):
        mode = "gossip"
    elif eng._kgtn_k:
        mode = "kgtn"
    elif getattr(eng, "_interval", False):
        mode = "interval"
    else:
        mode = "bucket" if eng._bucket_v2 else "fused"
    if getattr(eng, "_lr_table", None) is not None:
        table = sorted(c for c in eng.lr_cut_table() if c != NO_CUT)
        if table != sorted(getattr(sched, "cuts", ())):
            raise ValueError("the engine's cut table holds %s, the schedule's cuts are %s" % (table, sched.cuts))
    return dict(mode=mode, sched=sched, step0=step0, k=max(eng._kgtn_k, 1), early=(e0, e1),
                late_bf16=A.late_bucket_rounds_bf16(eng.spec.arena_numel, e1 - e0, be.late_ll, be.late_bf16),
                drop=(be.drop_seed, be.drop_keep) if be.drop_keep > 0.0 else None,
                aug=getattr(eng, "_aug", None), aug_start=int(aug_start), elastic=getattr(eng, "_aug_elastic", None),
                interval_ns=be.interval_ns if mode == "interval" else None, ctrl_off=dict(be._off),
                period=getattr(eng, "_local", 0))


def epoch_of(upd: dict, t: int) -> int:
    """The epoch word step t reads: the global step, which with K > N stays put over the k iterations of a commit.  Not
    for interval mode, whose commits follow the clock: see :func:`epochs_of`."""
    assert upd["mode"] != "interval"
    return upd["step0"] + t // upd["k"]


def interval_trace(upd: dict, init: dict, records: Sequence[dict]) -> dict:
    """Interval mode: what the recorded control blocks say the device did.  ``words``: the decoded block before the first
    step and after each step (``words[t + 1]`` after step t); ``commit[t]``: step t committed its tick (iv_ticks_committed
    went up during it); ``count[t]``: the low word of iv_state after step t, the gradients accumulated in the open tick
    (T of a committing step); ``epoch[t]``: the epoch word step t read, STEP0 + the commits before step t."""
    words = [ctrl_words(init["ctrl"], upd["ctrl_off"])] + [ctrl_words(r["ctrl"], upd["ctrl_off"]) for r in records]
    commit = [b["iv_ticks_committed"] != a["iv_ticks_committed"] for a, b in zip(words, words[1:])]
    epoch = [upd["step0"] + sum(commit[:t]) for t in range(len(records))]
    return dict(words=words, commit=commit, count=[w["iv_state"] & 0xFFFFFFFF for w in words[1:]], epoch=epoch)


def epochs_of(upd: dict, init: dict, records: Sequence[dict]) -> List[int]:
    """The epoch word each recorded step read (its dropout mask and its step size are those of that global step)."""
    if upd["mode"] == "interval":
        return interval_trace(upd, init, records)["epoch"]
    return [epoch_of(upd, t) for t in range(len(records))]


def augment_iteration_of(upd: dict, t: int) -> int:
    """The iteration whose draws step t uses: one per step in every mode, K > N included (the counter advances once per
    iteration, unlike the epoch word), modulo 2^32."""
    return (upd["aug_start"] + t) & 0xFFFFFFFF


def _words(t: torch.Tensor) -> List[int]:
    return [int(v) for v in t.detach().cpu().numpy().view("<u4")]


def augment_stage_results(tag: str, init: dict, records: Sequence[dict], batches: Sequence, upd: dict) -> List[Result]:
    """With augmentation armed (``upd["aug"]``): each step's recorded buffer against the warp of the batch it was fed
    (:func:`selfcheck.augment_results`; with ``upd["elastic"]`` the elastic warp) with the draws of
    :func:`augment_iteration_of`, and the counter words: the
    iteration before the first step, and after step t the next one with the ticket back at 0."""
    if upd.get("aug") is None:
        return []
    ranges, mix = upd["aug"]
    start = augment_iteration_of(upd, 0)
    res: List[Result] = [(tag + ".init.aug_counter_differs", float(_words(init["aug_counter"]) != [start, 0]), 0.0)]
    for t, (r, (x, _y)) in enumerate(zip(records, batches)):
        it = augment_iteration_of(upd, t)
        res += S.augment_results("%s.step%d.augment" % (tag, t), x, r["aug_images"], mix, it, ranges, upd.get("elastic"))
        res.append(("%s.step%d.aug_counter_differs" % (tag, t),
                    float(_words(r["aug_counter"]) != [(it + 1) & 0xFFFFFFFF, 0]), 0.0))
    return res


def _images_read(upd: dict, r: dict, fed):
    """The images a step's image readers must have read: its recorded augmented buffer, or the batch it was fed."""
    return r["aug_images"] if upd.get("aug") is not None else fed


def _shadow_bits(t: torch.Tensor):
    return t.detach().cpu().view(torch.int16).numpy().view("<u2")


def update_results(tag: str, init: dict, records: Sequence[dict], upd: dict) -> List[Result]:
    """Each step's weights from the previous record (or ``init``) and the step's recorded gradients, bit for bit; with
    K > N the weights stay put until the k-th iteration, which applies the accumulated k gradients.  In interval mode a
    step that did not commit leaves the weights unchanged, and a committing one applies the T gradients of its tick
    (T from its recorded count word, see :func:`interval_trace`), accumulated in iteration order, at the step size of
    the epoch word it read over T.  With drop-connect the fused kernel masks the gradient with the mask of the step's
    global step.

    The shadow: RNE of the step's own weights where the aggregation kernel refreshes it (K <= N); with K > N and in
    interval mode the next iteration's adoption refreshes it, so after step t it is RNE of the weights step t adopted,
    those recorded after step t - 1."""
    res: List[Result] = []
    mode, k, drop = upd["mode"], upd["k"], upd.get("drop")
    res.append((tag + ".init.shadow_bits_differ", float((_shadow_bits(init["shadow"]) != A.bf16_bits(init["params"])).sum()), 0.0))
    iv = interval_trace(upd, init, records) if mode == "interval" else None
    epochs = epochs_of(upd, init, records)
    w, acc = A.f32(init["params"]), []
    for t, r in enumerate(records):
        scale = A.step_scale(upd["sched"], epochs[t], k)
        g = A.f32(r["grads"])
        if mode == "kgtn":
            acc.append(g)
            want = A.sgd(w, A.interval_accumulate(acc), scale) if len(acc) == k else w
            acc = [] if len(acc) == k else acc
        elif mode == "interval":
            acc.append(g)
            want = w
            if iv["commit"][t]:
                T = max(iv["count"][t], 1)          # a count of 0 fails its own check (control_results)
                want = A.fused_sync_step(w, [A.interval_accumulate(acc)], 1, A.step_scale(upd["sched"], epochs[t], T))
                acc = []
        elif mode == "async":
            want = A.async_apply(w, [A.async_update(g, scale)])
            res.append(("%s.step%d.pull_bits_differ" % (tag, t), float((A.bits(r["pulled"]) != A.bits(w)).sum()), 0.0))
        elif mode == "local":
            want = A.sgd(w, g, scale)
            if (epochs[t] + 1) % upd["period"] == 0:
                want = A.local_average([want])
        elif mode == "gossip":
            want = A.gossip_mix([A.sgd(w, g, scale)], 0)
        elif mode == "bucket":
            want = A.bucket_step(w, [g], [A.f32(r["g16"].float()).reshape(-1)], upd["early"], scale, upd["late_bf16"])
        else:
            want = A.fused_sync_step(w, [g], 1, scale,
                                     drop=None if drop is None else (drop[0], epochs[t], drop[1]))
        got = A.bits(r["params"])
        res.append(("%s.step%d.update_bits_differ" % (tag, t), float((got != A.bits(want)).sum()), 0.0))
        adopted = (init if t == 0 else records[t - 1])["params"] if mode in ("kgtn", "interval", "async") else r["params"]
        res.append(("%s.step%d.shadow_bits_differ" % (tag, t),
                    float((_shadow_bits(r["shadow"]) != A.bf16_bits(adopted)).sum()), 0.0))
        w = A.f32(r["params"])
    return res


def control_results(tag: str, init: dict, records: Sequence[dict], upd: dict) -> List[Result]:
    """The recorded control blocks (none recorded: no checks).  Every mode: each step's ``%globaltimer`` stamps are its
    own, t_arrive(t - 1) <= t_start(t) <= t_arrive(t) and t_start(t) > 0.  The stamps of step t sit in the rings at the
    epoch word it read.

    Interval mode, d_t = iv_deadline after step t, I = ``upd["interval_ns"]``:

    * before the first step the clock is armed at STEP0 (iv_state = (STEP0 + 1) << 32: arming it before
      ``set_global_step`` would leave the step half behind and every tick would commit an empty accumulator);
    * after step t the epoch word is the one step t read (STEP0 + the commits before it), iv_state's step half that + 1,
      its count the gradients since the last commit, at most one more tick committed, one more accepted gradient and
      none dropped (one replica: nothing is stale), and after the adoption of a tick of T gradients last_count = T;
    * deadlines: a step that did not commit closed before its deadline (t_arrive(t) < d_t, the gate runs before the
      close) and leaves it armed (d_{t+1} = d_t, d_0 = the armed one); a commit came after it (t_start(t + 1) >= d_t) and
      the next step's adoption re-armed it: t_arrive(t) < d_{t+1} - I <= t_start(t + 1)."""
    if "ctrl" not in init:
        return []
    res: List[Result] = []
    interval = upd["mode"] == "interval"
    if interval:
        iv = interval_trace(upd, init, records)
        words, commit, count, epochs = iv["words"], iv["commit"], iv["count"], iv["epoch"]
    else:
        off, epochs = upd["ctrl_off"], epochs_of(upd, init, records)
        words = [ctrl_words(init["ctrl"], off)] + [ctrl_words(r["ctrl"], off, e) for r, e in zip(records, epochs)]
    step0, I = upd["step0"], upd.get("interval_ns")
    c0 = words[0]
    if interval:
        res.append((tag + ".init.clock_armed_before_global_step",
                    float(c0["iv_state"] != (step0 + 1) << 32 or c0["epoch"] != step0), 0.0))
    n, T_prev = 0, None
    for t in range(len(records)):
        a, c = words[t], words[t + 1]
        name = "%s.step%d." % (tag, t)
        bad = c["t_start"] == 0 or c["t_start"] > c["t_arrive"] or (t > 0 and a["t_arrive"] > c["t_start"])
        res.append((name + "stamps_out_of_order", float(bad), 0.0))
        if not interval:
            continue
        n += 1
        res.append((name + "ticks_committed_jump", float(c["iv_ticks_committed"] - a["iv_ticks_committed"] not in (0, 1)), 0.0))
        res.append((name + "epoch_differs", float(c["epoch"] != epochs[t] or c["iv_state"] >> 32 != epochs[t] + 1), 0.0))
        res.append((name + "count_differs", float(count[t] != n), 0.0))
        res.append((name + "accepted_dropped_differ", float(c["accepted_steps"] != c0["accepted_steps"] + t + 1
                                                            or c["dropped_steps"] != c0["dropped_steps"]), 0.0))
        if T_prev is not None:
            res.append((name + "last_count_differs", float(c["last_count"] != T_prev), 0.0))
        if not commit[t]:
            res.append((name + "open_tick_past_deadline", float(c["t_arrive"] >= c["iv_deadline"]), 0.0))
        if t == 0 or not commit[t - 1]:
            res.append((name + "deadline_moved_without_commit", float(c["iv_deadline"] != a["iv_deadline"]), 0.0))
        else:
            res.append(("%s.step%d.commit_before_deadline" % (tag, t - 1), float(c["t_start"] < a["iv_deadline"]), 0.0))
            res.append((name + "deadline_not_rearmed_at_adoption",
                        float(not a["t_arrive"] < c["iv_deadline"] - I <= c["t_start"]), 0.0))
        T_prev, n = (count[t], 0) if commit[t] else (None, n)
    return res


def _inputs(spec, init: dict, records: Sequence[dict], t: int, dev):
    """(fp32 views, bf16 shadow views) of the weights step t read: RNE of the previous step's committed weights."""
    p = (init if t == 0 else records[t - 1])["params"].to(dev)
    return spec.views(p), spec.views(p.to(torch.bfloat16))


def lenet_step_results(tag: str, spec, r: dict, p, pb, images, labels, mask, keep_prob: float,
                       lam: float = 0.0) -> List[Result]:
    """One LeNet training step from its record ``r``: every stage from the recorded inputs of that stage.  ``p`` / ``pb``:
    the fp32 / bf16 weights the step read, ``images`` [B,28,28] / ``labels`` what it was fed, ``mask`` its dropout mask.

    ``lam``: L2 weight decay armed.  The fc weight gradients are then checked elementwise against the plain reference +
    lambda v, v from ``p`` (the wire buffer as RNE of that value), the recorded R against float64 R of ``p``, and the loss
    word against CE + lambda R."""
    kind = "rand"
    B = labels.shape[0]
    decay_loss = None
    if lam:
        r_ref = R.weight_decay_terms(spec, p, lam)[0]
        decay_loss = S._lam32(lam) * float(r_ref)
    x = images.reshape(B, 28, 28)
    a2 = r["a2"]
    g = spec.views(r["grads"])
    res = S.conv1_fwd_results(tag + ".conv1_fwd", kind, x, p["conv1_weights"], p["conv1_biases"], r["a1"], r["code1"])
    res += S.conv2_fwd_results(tag + ".conv2_fwd", kind, r["a1"], pb["conv2_weights"], p["conv2_biases"],
                               a2.view(B, 7, 7, 64), r["code2"].view(B, 7, 7, 64))
    res += S.fc1_fwd_results(tag + ".fc1_fwd", kind, a2, pb["fc1_weights"], r["h_part"])
    w1 = pb["fc1_weights"].double()
    hsum = a2.double() @ w1
    ref = R.fc2_fwd_bwd(hsum, p["fc1_biases"], p["fc2_weights"], p["fc2_biases"], labels, mask, keep_prob)
    o = dict(la=r["loss_acc"], h=r["h_act"], dl=r["dlogits"], dh=r["dh"])
    res += S._fc2_results(tag + ".fc2_fwd_bwd", kind, o, ref, p["fc2_weights"], B, True, decay_loss=decay_loss)
    b1 = p["fc1_biases"].double()
    # the kernel's pre-activation: 7 fp32 GEMM partials of 448 products each, summed with the bias in fp32
    res += S.keep_pattern_results(tag + ".fc2_fwd_bwd.keep_pattern", r["h_act"], ref["h"], hsum + b1,
                                  R.fp32_slack(a2.double().abs() @ w1.abs() + b1.abs(), 3136 + 8))
    if lam:
        ws = r["decay_ws"]
        res += S.decay_partials_results(tag + ".decay_R", ws[-1:], r_ref.reshape(1).to(ws.device))
        res += S.fc2_wgrad_decay_results(tag + ".fc2_wgrad", kind, r["h_act"], r["dlogits"], r["dh"], g["fc2_weights"],
                                         g["fc2_biases"], g["fc1_biases"], lam, p["fc2_weights"], p["fc2_biases"],
                                         p["fc1_biases"])
        res += S.fc1_wgrad_decay_results(tag + ".fc1_wgrad", kind, a2, r["dh"], r.get("g16", g["fc1_weights"]), lam,
                                         p["fc1_weights"])
    else:
        res += S.fc2_wgrad_results(tag + ".fc2_wgrad", r["h_act"], r["dlogits"], r["dh"], g["fc2_weights"],
                                   g["fc2_biases"], g["fc1_biases"])
        res += S.fc1_wgrad_results(tag + ".fc1_wgrad", kind, a2, r["dh"], r.get("g16", g["fc1_weights"]))
    res += S.fc1_dgrad_results(tag + ".fc1_dgrad_unpool", kind, r["dh"], pb["fc1_weights"], r["code2"], r["dy2"],
                               g["conv2_biases"])
    res += S.conv2_dgrad_results(tag + ".conv2_dgrad", kind, r["dy2"], pb["conv2_weights"], r["dx1"])
    res += S.conv2_wgrad_results(tag + ".conv2_wgrad", kind, r["a1"], r["dy2"], g["conv2_weights"])
    res += S.conv1_wgrad_results(tag + ".conv1_wgrad", kind, x, r["dx1"], r["code1"], g["conv1_weights"].reshape(25, 32),
                                 g["conv1_biases"])
    valid = spec.valid_mask().to(r["grads"].device)
    res.append((tag + ".grad_padding", float(r["grads"][~valid].abs().max()), 0.0))
    return res


def lenet_trajectory_results(tag: str, spec, init: dict, records: Sequence[dict], batches: Sequence, upd: dict,
                             seed: int, rank: int, keep_prob: float, lam: float = 0.0) -> List[Result]:
    """Every step of a LeNet run (``batches[t]`` = (images, labels) fed to step t) and every update.  ``lam``: the L2
    weight decay the run was armed with (see :func:`lenet_step_results`).  With augmentation armed, the augment stage is
    checked against the fed batch and conv1 forward and conv1 wgrad against the step's recorded augmented images.  The
    recorded control blocks, if any, through :func:`control_results`."""
    res = update_results(tag, init, records, upd) + augment_stage_results(tag, init, records, batches, upd)
    res += control_results(tag, init, records, upd)
    epochs = epochs_of(upd, init, records)
    for t, (r, (x, y)) in enumerate(zip(records, batches)):
        dev = r["a1"].device
        p, pb = _inputs(spec, init, records, t, dev)
        y = torch.as_tensor(y).to(dev)
        mask = dropout_keep_mask(dropout_seed_mix(seed, epochs[t], rank), y.shape[0], 512, keep_prob, device=dev)
        res += lenet_step_results("%s.step%d" % (tag, t), spec, r, p, pb, torch.as_tensor(_images_read(upd, r, x)).to(dev),
                                  y, mask, keep_prob, lam)
    return res


def mlp_trajectory_results(tag: str, spec, init: dict, records: Sequence[dict], batches: Sequence,
                           upd: dict) -> List[Result]:
    """Every step of an MLP run through :func:`selfcheck._mlp_step_results`, and every update.  With the bucketed
    aggregation the early layer's weight gradient is the bf16 wire buffer.  With augmentation armed, the augment stage is
    checked against the fed batch and x16 against the step's recorded augmented images."""
    res = update_results(tag, init, records, upd) + augment_stage_results(tag, init, records, batches, upd)
    res += control_results(tag, init, records, upd)
    n_layers = len(spec.params) // 2
    early = next(q.name for q in spec.params if q.offset == upd["early"][0])
    for t, (r, (x, y)) in enumerate(zip(records, batches)):
        dev = r["x16"].device
        p, pb = _inputs(spec, init, records, t, dev)
        g = dict(spec.views(r["grads"]))
        if "g16" in r:
            g[early] = r["g16"]
        B = r["x16"].shape[0]
        rec = SimpleNamespace(p=p, pb=pb, g=g, n_layers=n_layers, batch_size=B, x16=r["x16"], h=r["h"], dh=r["dh"],
                              dl_pad=r["dl_pad"], d_loss_acc=r["loss_acc"], grads=r["grads"], spec=spec)
        res += S._mlp_step_results("%s.step%d" % (tag, t), "rand", rec,
                                   torch.as_tensor(_images_read(upd, r, x)).to(dev).reshape(B, 784),
                                   torch.as_tensor(y).to(dev))
    return res


def failures(results: Sequence[Result]) -> List[Result]:
    return [(n, e, b) for (n, e, b) in results if not e <= b]


def worst_by_stage(tag: str, results: Sequence[Result]) -> Dict[str, float]:
    """Largest error-to-bound ratio of each check over all steps (its name without ``tag`` and ``stepN``); checks with a
    zero bound count as 0 when they pass."""
    out: Dict[str, float] = {}
    for n, e, b in results:
        stage = re.sub(r"^step\d+\.", "", n[len(tag) + 1:] if n.startswith(tag + ".") else n)
        ratio = e / b if b > 0 else (0.0 if e <= b else float("inf"))
        out[stage] = max(out.get(stage, 0.0), ratio)
    return out
