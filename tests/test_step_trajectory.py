"""The trajectory checker (ops/trajectory.py) on CPU-built records: small LeNet and MLP runs emulated from the float64
references in the engine's storage formats pass unchanged, and each seeded ordering fault fails."""
import numpy as np
import pytest
import torch

from distributedmnist_b200 import augment as AU
from distributedmnist_b200 import weight_decay as W
from distributedmnist_b200.models import dropout_keep_mask, dropout_seed_mix, get_model
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.ops import refs as R
from distributedmnist_b200.ops import trajectory as T
from distributedmnist_b200.schedule import LearningRateSchedule

BF = torch.bfloat16
SEED, RANK, KEEP = 5, 0, 0.5
# a large step size, so that one step's update moves the bf16 shadow and the activations visibly
SCHED = LearningRateSchedule(4.0, 1, 0.999)
STEP0 = 3001
# augmentation: draws from an iteration that is not STEP0 and wraps through 0 inside the run
AUG_RANGES = AU.Ranges(3.0, 20.0, 0.15)
AUG_START = 2 ** 32 - 3
AUG_MIX = AU.seed_mix(SEED, RANK)
AUG_FAULTS = ("aug_iteration_plus_1", "aug_keyed_by_epoch", "aug_other_rank", "conv1_reads_unaugmented",
              "conv1_wgrad_reads_next_warp", "x16_from_fed", "counter_not_advanced")


def _bf(x):
    return x.to(torch.float32).to(BF)           # RNE of the fp32 value, as the kernels store bf16


def _ftz(grads):
    """The kernels run with flush-to-zero: no subnormal gradient reaches the update."""
    return grads.masked_fill_(grads.abs() < A.FLT_MIN, 0.0)


def _update(w, g):
    """fused_sync_sgd on one replica, in place of the engine's aggregation."""
    return lambda t: torch.from_numpy(A.fused_sync_step(A.f32(w), [A.f32(g)], 1, A.step_scale(SCHED, STEP0 + t, 1)))


def _lenet_step(spec, params, x, y, mask, fault, prev, lam=0.0, x_wgrad=None, shadow=None):
    """One LeNet step as the kernels store it.  ``fault``: "dgrad_post_update" runs fc1 dgrad on the updated shadow.
    ``lam``: L2 weight decay (see :func:`_decay`).  ``x_wgrad``: the images conv1 wgrad reads, if not ``x``.  ``shadow``:
    the fp32 weights the bf16 shadow was made from, if not ``params``."""
    B = x.shape[0]
    p, pb = spec.views(params), spec.views((params if shadow is None else shadow).to(BF))
    f1 = R.pool_fwd(R.conv5x5(x.to(BF)[..., None], p["conv1_weights"].to(BF)), p["conv1_biases"])
    a1, code1 = _bf(f1["out"]), f1["code"]
    f2 = R.pool_fwd(R.conv5x5(a1, pb["conv2_weights"]), p["conv2_biases"])
    a2, code2 = _bf(f2["out"]).reshape(B, 3136), f2["code"].reshape(B, 3136)
    w1 = pb["fc1_weights"].double()
    ks = [64 * (49 * z // 7) for z in range(8)]
    h_part = torch.stack([(a2[:, ks[z]:ks[z + 1]].double() @ w1[ks[z]:ks[z + 1]]).float() for z in range(7)])
    ref = R.fc2_fwd_bwd(a2.double() @ w1, p["fc1_biases"], p["fc2_weights"], p["fc2_biases"], y, mask, KEEP)
    dh, h_act, dlogits = _bf(ref["dh"]), ref["h"].float(), ref["dl"].float()
    grads = torch.zeros(spec.arena_numel)
    g = spec.views(grads)
    gw2, gb2, gb1 = R.fc2_wgrad(h_act, dlogits, dh)
    g["fc2_weights"].copy_(gw2), g["fc2_biases"].copy_(gb2), g["fc1_biases"].copy_(gb1)
    g["fc1_weights"].copy_(a2.double().t() @ dh.double())
    w1_dgrad = pb["fc1_weights"]
    if fault == "dgrad_post_update":
        w1_dgrad = spec.views(_update(params, grads)(prev["t"]).to(BF))["fc1_weights"]
    dy, gbc2 = R.fc1_dgrad_unpool(dh, w1_dgrad, code2)
    dy2 = _bf(dy)
    g["conv2_biases"].copy_(gbc2)
    dx1 = _bf(R.conv5x5_dgrad(dy2, pb["conv2_weights"]))
    g["conv2_weights"].copy_(R.conv5x5_wgrad(a1, dy2))
    gw1, gbc1 = R.conv1_wgrad((x if x_wgrad is None else x_wgrad).to(BF), dx1, code1)
    g["conv1_weights"].copy_(gw1.reshape(5, 5, 1, 32)), g["conv1_biases"].copy_(gbc1)
    la = torch.tensor([float(ref["loss"]), float(ref["acc"])], dtype=torch.float32)
    r = dict(a1=a1, code1=code1, a2=a2, code2=code2, h_part=h_part, dh=dh, h_act=h_act, dlogits=dlogits, dy2=dy2,
             dx1=dx1, grads=grads, loss_acc=la)
    if lam:
        _decay(spec, params, r, lam, fault, prev)
    _ftz(grads)
    return r


def _decay(spec, params, r, lam, fault, prev):
    """L2 weight decay as the kernels apply it: lambda v added to the four fc gradients, R of the weights the step read
    into the workspace's last slot, fp32(lambda R) added to the loss word.  ``fault``: one of DECAY_FAULTS."""
    lam = float(np.float32(lam))
    p, g = spec.views(params), spec.views(r["grads"])
    for name in W.LENET_DECAYED:
        if fault == "decay_no_fc1_biases" and name == "fc1_biases":
            continue
        v = p[name]
        if fault == "decay_post_update" and name == "fc1_weights":
            v = spec.views(_update(params, _ftz(r["grads"].clone()))(prev["t"]))[name]   # after the early bucket's update
        g[name].copy_(g[name].double() + (2 if fault == "decay_twice" else 1) * lam * v.double())
    if fault == "decay_conv2_biases":
        g["conv2_biases"].copy_(g["conv2_biases"].double() + lam * p["conv2_biases"].double())
    rr = R.weight_decay_terms(spec, prev["params"] if fault == "decay_R_previous_step" else params, lam)[0]
    r["decay_ws"] = torch.tensor([float(rr)], dtype=torch.float64)
    if fault != "loss_without_decay":
        r["loss_acc"][0] = r["loss_acc"][0] + np.float32(lam * float(rr))


def _mlp_step(spec, params, x, y, fault, prev, shadow=None):
    """One MLP step as the kernels store it.  ``fault``: "bias_not_cleared" adds the previous step's atomically
    accumulated output-layer bias gradient.  ``shadow``: as for :func:`_lenet_step`."""
    L = len(spec.params) // 2
    B = x.shape[0]
    p, pb = spec.views(params), spec.views((params if shadow is None else shadow).to(BF))
    x16 = _bf(x.reshape(B, 784))
    hs, src = [], x16
    for i in range(1, L):
        src = _bf(R.mlp_hidden(src, pb["fc%d_weights" % i], p["fc%d_biases" % i])[0])
        hs.append(src)
    out = R.dense10_xent(src, p["fc%d_weights" % L], p["fc%d_biases" % L], y)
    dl_pad = torch.zeros(B, 64, dtype=BF)
    dl_pad[:, :10] = _bf(out["dl"])
    dhs = [None] * (L - 1)
    dhs[-1] = _bf(out["dh"])
    grads = torch.zeros(spec.arena_numel)
    g = spec.views(grads)
    g["fc%d_weights" % L].copy_(src.double().t() @ dl_pad[:, :10].double())
    g["fc%d_biases" % L].copy_(out["dl"].sum(0))
    if fault == "bias_not_cleared" and prev["t"] > 0:
        g["fc%d_biases" % L].add_(spec.views(prev["grads"])["fc%d_biases" % L])
    for i in range(L - 1, 0, -1):
        below = hs[i - 2] if i > 1 else x16
        g["fc%d_biases" % i].copy_(dhs[i - 1].double().sum(0))
        g["fc%d_weights" % i].copy_(below.double().t() @ dhs[i - 1].double())
        if i > 1:
            dhs[i - 2] = _bf(R.mlp_dgrad(dhs[i - 1], pb["fc%d_weights" % i], hs[i - 2])[0])
    la = torch.tensor([float(out["loss_terms"].mean()), float(out["hits"].double().mean())], dtype=torch.float32)
    return dict(x16=x16, h=hs, dh=dhs, dl_pad=dl_pad, grads=_ftz(grads), loss_acc=la)


def _counter(it):
    """The augmentation counter words [iteration, ticket] as the engine stores them (int32)."""
    return torch.from_numpy(np.array([it & 0xFFFFFFFF, 0], dtype=np.uint32).view(np.int32))


def _augment(x, t, steps, batches, fault):
    """The images augment_affine writes for step t, and those conv1 forward, conv1 wgrad and mlp x16 read: all the
    same buffer unless ``fault`` (one of AUG_FAULTS) says otherwise."""
    it, mix = AUG_START + t, AUG_MIX
    if fault == "aug_iteration_plus_1":              # as if the graph capture's warm-up had consumed an iteration
        it += 1
    if fault == "aug_keyed_by_epoch":
        it = STEP0 + t
    if fault == "aug_other_rank":
        mix = AU.seed_mix(SEED, RANK + 1)
    xa = torch.from_numpy(AU.augment_batch(x.numpy(), mix, it, AUG_RANGES))
    read = dict(fwd=xa, wgrad=xa, x16=xa)
    if fault == "conv1_reads_unaugmented":
        read["fwd"] = x
    if fault == "conv1_wgrad_reads_next_warp" and t + 1 < steps:
        read["wgrad"] = torch.from_numpy(AU.augment_batch(batches[t + 1][0].numpy(), mix, it + 1, AUG_RANGES))
    if fault == "x16_from_fed":
        read["x16"] = x
    return xa, read


def _run(model, fault=None, steps=4, B=8, lam=0.0, aug=False):
    """(spec, init, records, batches fed, update) of an emulated run with at most one seeded fault; ``lam``: L2 weight
    decay (LeNet); ``aug``: random affine augmentation from iteration AUG_START (on with any of AUG_FAULTS)."""
    aug = aug or fault in AUG_FAULTS
    spec = get_model(model, 64)[0]
    gen = torch.Generator().manual_seed(11)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(steps)]
    params = spec.init_flat(SEED)
    init = dict(params=params.clone(), shadow=params.to(BF))
    if aug:
        init["aug_counter"] = _counter(AUG_START)
    records, prev = [], dict(t=0, grads=None, params=params.clone())
    for t in range(steps):
        x, y = batches[t]
        if fault == "batch_t_plus_2" and t == 1:
            x, y = batches[t + 2]
        if fault == "slot1_reads_slot0" and t % 2 == 1:
            x, y = batches[t - 1]
        xa, read = _augment(x, t, steps, batches, fault) if aug else (None, dict(fwd=x, wgrad=x, x16=x))
        prev["t"] = t
        if model == "lenet":
            e = STEP0 + t - (1 if fault == "mask_previous_epoch" and t > 0 else 0)
            mask = dropout_keep_mask(dropout_seed_mix(SEED, e, RANK), B, 512, KEEP)
            r = _lenet_step(spec, params, read["fwd"], y, mask, fault, prev, lam, x_wgrad=read["wgrad"])
        else:
            r = _mlp_step(spec, params, read["x16"], y, fault, prev)
        g = prev["grads"] if fault == "stale_gradient" and t > 0 else r["grads"]
        params = _update(params, g)(t)
        r.update(params=params.clone(), shadow=params.to(BF))
        if aug:
            r.update(aug_images=xa.reshape(B, 784), aug_counter=_counter(AUG_START + t + (fault != "counter_not_advanced")))
        records.append(r)
        prev["grads"] = r["grads"]
        prev["params"] = (init["params"] if t == 0 else records[t - 1]["params"]).clone()   # what step t read
    upd = dict(mode="fused", sched=SCHED, step0=STEP0, k=1, early=(spec.param("fc1_weights").offset,) * 2, late_bf16=False,
               aug=(AUG_RANGES, AUG_MIX) if aug else None, aug_start=AUG_START if aug else 0)
    return spec, init, records, batches, upd


def _results(model, fault=None, lam=0.0, aug=False):
    spec, init, records, batches, upd = _run(model, fault, lam=lam, aug=aug)
    if model == "lenet":
        return T.lenet_trajectory_results("lenet", spec, init, records, batches, upd, SEED, RANK, KEEP, lam)
    return T.mlp_trajectory_results("mlp3", spec, init, records, batches, upd)


@pytest.mark.parametrize("model", ["lenet", "mlp3"])
def test_emulated_trajectory_passes(model):
    res = _results(model)
    assert not T.failures(res), T.failures(res)
    assert sum(1 for n, _, _ in res if ".step3." in n) > 10
    worst = T.worst_by_stage(model, res)
    assert "update_bits_differ" in worst and all(0 <= v <= 1 for v in worst.values()), worst


@pytest.mark.parametrize("model,fault,stage", [
    ("lenet", "dgrad_post_update", "fc1_dgrad_unpool"),
    ("lenet", "mask_previous_epoch", "fc2_fwd_bwd"),
    ("lenet", "batch_t_plus_2", "step1.conv1_fwd"),
    ("mlp3", "bias_not_cleared", "dense10_xent.g_b"),
    ("lenet", "slot1_reads_slot0", "step1.conv1_fwd"),
    ("mlp3", "slot1_reads_slot0", "step1.x16"),
    ("lenet", "stale_gradient", "update_bits_differ"),
    ("mlp3", "stale_gradient", "update_bits_differ"),
])
def test_seeded_fault_fails(model, fault, stage):
    bad = T.failures(_results(model, fault))
    assert any(stage in n for n, _, _ in bad), (fault, bad[:10])


def test_kgtn_update_commits_every_k_th_iteration_and_the_next_adoption_refreshes_the_shadow():
    """K > N: the weights stay put for k - 1 iterations, then take the accumulated k gradients at the commit's step size.
    The commit leaves the bf16 shadow alone; the next iteration's adoption refreshes it, so after iteration t it is RNE
    of the weights recorded after iteration t - 1."""
    spec = get_model("mlp2", 64)[0]
    gen = torch.Generator().manual_seed(3)
    w = spec.init_flat(SEED)
    init = dict(params=w.clone(), shadow=w.to(BF))
    gs = [torch.randn(spec.arena_numel, generator=gen) * 1e-2 * spec.valid_mask() for _ in range(4)]
    c1 = torch.from_numpy(A.sgd(A.f32(w), A.interval_accumulate([A.f32(g) for g in gs[:2]]), A.step_scale(SCHED, STEP0, 2)))
    c2 = torch.from_numpy(A.sgd(A.f32(c1), A.interval_accumulate([A.f32(g) for g in gs[2:]]), A.step_scale(SCHED, STEP0 + 1, 2)))
    upd = dict(mode="kgtn", sched=SCHED, step0=STEP0, k=2, early=(0, 0), late_bf16=False)
    # the shadow is refreshed by the adoption at the start of the iteration after a commit
    recs = [dict(grads=g, params=p, shadow=s.to(BF)) for g, p, s in zip(gs, (w, c1, c1, c2), (w, w, c1, c1))]
    assert not T.failures(T.update_results("kgtn", init, recs, upd))
    assert [T.epoch_of(upd, t) for t in range(4)] == [STEP0, STEP0, STEP0 + 1, STEP0 + 1]
    bad = dict(recs[2], shadow=w.to(BF))               # the adoption did not refresh the shadow
    assert [n for n, _, _ in T.failures(T.update_results("kgtn", init, recs[:2] + [bad] + recs[3:], upd))] == \
        ["kgtn.step2.shadow_bits_differ"]
    recs[1] = dict(recs[1], params=w)                  # the commit not applied
    assert T.failures(T.update_results("kgtn", init, recs, upd))


# ---- L2 weight decay ----------------------------------------------------------------------------------------------------
# 2^-6: with the step size above, one update moves the weights by a visible fraction of lambda W
DECAY_LAM = 2.0 ** -6


@pytest.mark.parametrize("lam", [5e-4, DECAY_LAM])
def test_emulated_decayed_trajectory_passes(lam):
    res = _results("lenet", lam=lam)
    assert not T.failures(res), T.failures(res)
    worst = T.worst_by_stage("lenet", res)
    for stage in ("decay_R[err/bound]", "fc2_wgrad.g_b1[err/bound]", "fc1_wgrad[err/bound]", "fc2_fwd_bwd.loss(CE + lambda R)"):
        assert stage in worst, (stage, sorted(worst))
    assert all(0 <= v <= 1 for v in worst.values()), worst


@pytest.mark.parametrize("fault,stage", [
    ("decay_no_fc1_biases", "fc2_wgrad.g_b1"),
    ("decay_conv2_biases", "fc1_dgrad_unpool.g_bias"),
    ("decay_twice", "fc1_wgrad"),
    ("decay_post_update", "fc1_wgrad"),
    ("decay_R_previous_step", "decay_R"),
    ("loss_without_decay", "fc2_fwd_bwd.loss"),
])
def test_seeded_decay_fault_fails(fault, stage):
    bad = T.failures(_results("lenet", fault, lam=DECAY_LAM))
    assert any(stage in n for n, _, _ in bad), (fault, bad[:10])


def test_decayed_update_with_drop_connect_and_cuts():
    """The update check with drop-connect (the fused kernel's mask of the step's global step, over the decayed gradient)
    and a schedule with cuts inside the run; the same records fail without the mask or without the cuts."""
    spec = get_model("lenet", 64)[0]
    gen = torch.Generator().manual_seed(4)
    w = spec.init_flat(SEED)
    init = dict(params=w.clone(), shadow=w.to(BF))
    sched = LearningRateSchedule(4.0, 1, 0.999, factor=0.5, cuts=[STEP0 + 1, STEP0 + 3])
    seed, keep = 0x2545F491, 0.8
    recs, cur = [], w
    for t in range(4):
        g = torch.randn(spec.arena_numel, generator=gen) * 1e-2 * spec.valid_mask()
        g = g + DECAY_LAM * cur * spec.valid_mask()
        cur = torch.from_numpy(A.fused_sync_step(A.f32(cur), [A.f32(g)], 1, A.step_scale(sched, STEP0 + t, 1),
                                                 drop=(seed, STEP0 + t, keep)))
        recs.append(dict(grads=g, params=cur, shadow=cur.to(BF)))
    upd = dict(mode="fused", sched=sched, step0=STEP0, k=1, early=(0, 0), late_bf16=False, drop=(seed, keep))
    assert not T.failures(T.update_results("drop", init, recs, upd))
    assert T.failures(T.update_results("drop", init, recs, dict(upd, drop=None)))
    assert T.failures(T.update_results("drop", init, recs, dict(upd, sched=SCHED)))


# ---- random affine augmentation ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["lenet", "mlp3"])
def test_emulated_augmented_trajectory_passes(model):
    """Augmented from iteration 2^32 - 3, so the counter wraps through 0 within the 4 steps: the augment stage, the
    counter words and every stage that reads the images (conv1 forward and wgrad, mlp3's x16) against the recorded
    augmented buffer pass, and each premise holds."""
    res = _results(model, aug=True)
    assert not T.failures(res), T.failures(res)
    worst = T.worst_by_stage(model, res)
    for stage in ("augment[err/bound]", "aug_counter_differs", "init.aug_counter_differs",
                  "augment.premise.iteration_plus_1_detectable", "augment.premise.centre_14_detectable"):
        assert stage in worst, (stage, sorted(worst))
    assert all(0 <= v <= 1 for v in worst.values()), worst
    assert sum(1 for n, _, _ in res if ".step3.augment" in n) == 5


@pytest.mark.parametrize("model,fault,stage", [
    ("lenet", "aug_iteration_plus_1", "step0.augment[err/bound]"),
    ("lenet", "aug_keyed_by_epoch", "step0.augment[err/bound]"),
    ("lenet", "aug_other_rank", "step0.augment[err/bound]"),
    ("mlp3", "aug_iteration_plus_1", "step0.augment[err/bound]"),
    ("lenet", "conv1_reads_unaugmented", "step0.conv1_fwd"),
    ("lenet", "conv1_wgrad_reads_next_warp", "step0.conv1_wgrad"),
    ("mlp3", "x16_from_fed", "step0.x16"),
    ("lenet", "counter_not_advanced", "step0.aug_counter_differs"),
])
def test_seeded_augment_fault_fails(model, fault, stage):
    """Each fault fails at its own stage, and only the stages it touches fail."""
    bad = T.failures(_results(model, fault))
    assert any(stage in n for n, _, _ in bad), (fault, bad[:10])
    family = stage.split(".")[1].split("[")[0]
    assert all(family in n for n, _, _ in bad), (fault, bad[:10])


# ---- interval mode ------------------------------------------------------------------------------------------------------
# The control block of one replica in host memory, laid out by an offset table of its own (the checker reads the words
# through the offsets it is given), and an emulated clock in nanoseconds.  Every step takes 10 ns: the adoption (and
# t_start) at its start, the gate (t_arrive) at +6, the close at +8.  The host paces the ticks: before the last step of
# each tick it waits until the deadline has passed, so that step's close commits the tick.
CTRL_OFF = dict(epoch=0, error=4, accepted_steps=8, dropped_steps=12, last_count=16, iv_ticks_committed=20, iv_state=24,
                iv_deadline=32, t_start=40, t_arrive=40 + 8 * T.TIMING_RING)
CTRL_BYTES = 40 + 16 * T.TIMING_RING
TICKS = (1, 3, 2, 4)
INTERVAL_NS = 10_000
IV_FAULTS = ("divisor_1", "divisor_t_minus_1", "accumulator_overwritten", "adoption_late", "k_eq_n_updates",
             "mask_step0_plus_t", "shadow_not_refreshed", "commit_before_deadline", "deadline_rearmed_without_adoption",
             "count_word_off", "epoch_without_commit")


class _Ctrl:
    """The words of the control block the interval kernels write, at CTRL_OFF."""

    def __init__(self):
        self.b = np.zeros(CTRL_BYTES, dtype=np.uint8)

    def _view(self, f):
        n = 8 if f in T.CTRL_U64 else 4
        return self.b[CTRL_OFF[f]:CTRL_OFF[f] + n].view("<u%d" % n)

    def __getitem__(self, f):
        return int(self._view(f)[0])

    def __setitem__(self, f, v):
        self._view(f)[0] = v

    def stamp(self, ring, ns):
        """t_start / t_arrive of the current epoch word."""
        o = CTRL_OFF[ring] + 8 * (self["epoch"] % T.TIMING_RING)
        self.b[o:o + 8].view("<u8")[0] = ns

    def snapshot(self):
        return torch.from_numpy(self.b.copy())


def _run_interval(model, fault=None):
    """(spec, init, records, batches fed, update) of an emulated one-replica interval run with ticks of TICKS gradients
    and at most one seeded fault (one of IV_FAULTS)."""
    spec = get_model(model, 64)[0]
    steps, B = sum(TICKS), 8
    last_of_tick = set(np.cumsum(TICKS) - 1)
    gen = torch.Generator().manual_seed(12)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(steps)]
    params = spec.init_flat(SEED)
    c, now = _Ctrl(), 10 ** 9
    c["epoch"] = STEP0                                   # set_global_step, then the clock is armed
    c["iv_state"], c["iv_deadline"] = (STEP0 + 1) << 32, now + INTERVAL_NS
    init = dict(params=params.clone(), shadow=params.to(BF), ctrl=c.snapshot())
    records, gs, shadow, committed, before = [], [], params.clone(), None, None
    for t in range(steps):
        x, y = batches[t]
        if t in last_of_tick and fault != "commit_before_deadline":
            now = max(now, c["iv_deadline"] + 100)       # the host slept past the deadline
        # iv_adopt + iv_shadow
        if committed is not None:
            c["epoch"] = c["epoch"] + 1
            c["iv_deadline"], c["last_count"], c["iv_state"] = now + INTERVAL_NS, committed, (c["epoch"] + 1) << 32
            if fault != "shadow_not_refreshed":
                shadow = params.clone()
        if fault == "epoch_without_commit" and t == 2:
            c["epoch"] = c["epoch"] + 1
        if fault == "deadline_rearmed_without_adoption" and t == 2:
            c["iv_deadline"] = now + INTERVAL_NS
        c.stamp("t_start", now)
        w_fp32, w_bf16 = params, shadow
        if fault == "adoption_late" and committed is not None:
            w_fp32 = w_bf16 = before                     # computes on the weights from before the commit it should adopt
        committed = None
        if model == "lenet":
            e = STEP0 + t if fault == "mask_step0_plus_t" else c["epoch"]
            mask = dropout_keep_mask(dropout_seed_mix(SEED, e, RANK), B, 512, KEEP)
            r = _lenet_step(spec, w_fp32, x, y, mask, None, dict(t=t), shadow=w_bf16)
        else:
            r = _mlp_step(spec, w_fp32, x, y, None, dict(t=t), shadow=w_bf16)
        # iv_gate, iv_accumulate, iv_close (+ commit), iv_apply
        c.stamp("t_arrive", now + 6)
        gs.append(r["grads"])
        c["iv_state"] = c["iv_state"] + 1 + (fault == "count_word_off" and t == 1)
        c["accepted_steps"] = c["accepted_steps"] + 1
        if t in last_of_tick:
            n = len(gs)
            div = {"divisor_1": 1, "divisor_t_minus_1": max(n - 1, 1)}.get(fault, n)
            acc = A.f32(gs[-1]) if fault == "accumulator_overwritten" else A.interval_accumulate([A.f32(g) for g in gs])
            before = params
            params = torch.from_numpy(A.fused_sync_step(A.f32(params), [acc], 1, A.step_scale(SCHED, c["epoch"], div)))
            c["iv_ticks_committed"] = c["iv_ticks_committed"] + 1
            committed, gs = n, []
        elif fault == "k_eq_n_updates":
            params = torch.from_numpy(A.fused_sync_step(A.f32(params), [A.f32(r["grads"])], 1,
                                                        A.step_scale(SCHED, c["epoch"], 1)))
        now += 10
        r.update(params=params.clone(), shadow=shadow.to(BF), ctrl=c.snapshot())
        records.append(r)
    upd = dict(mode="interval", sched=SCHED, step0=STEP0, k=1, early=(spec.param("fc1_weights").offset,) * 2,
               late_bf16=False, aug=None, aug_start=0, interval_ns=INTERVAL_NS, ctrl_off=CTRL_OFF)
    return spec, init, records, batches, upd


def _interval_results(model, fault=None, mode="interval"):
    spec, init, records, batches, upd = _run_interval(model, fault)
    upd["mode"] = mode
    if model == "lenet":
        return T.lenet_trajectory_results("lenet", spec, init, records, batches, upd, SEED, RANK, KEEP)
    return T.mlp_trajectory_results("mlp3", spec, init, records, batches, upd)


@pytest.mark.parametrize("model", ["lenet", "mlp3"])
def test_emulated_interval_trajectory_passes(model):
    """Ticks of 1, 3, 2 and 4 gradients: every stage on the weights and epoch word of the commit the step adopted, the
    weights unchanged by steps that did not commit, each commit bit for bit, and the control block's words and stamps."""
    spec, init, records, batches, upd = _run_interval(model)
    tr = T.interval_trace(upd, init, records)
    assert tr["commit"] == [t in set(np.cumsum(TICKS) - 1) for t in range(sum(TICKS))]
    assert [n for n, cm in zip(tr["count"], tr["commit"]) if cm] == list(TICKS)
    assert tr["epoch"] == [STEP0, STEP0 + 1, STEP0 + 1, STEP0 + 1, STEP0 + 2, STEP0 + 2] + [STEP0 + 3] * 4
    res = _interval_results(model)
    assert not T.failures(res), T.failures(res)
    worst = T.worst_by_stage(model, res)
    for stage in ("update_bits_differ", "shadow_bits_differ", "init.clock_armed_before_global_step", "count_differs",
                  "epoch_differs", "last_count_differs", "stamps_out_of_order", "open_tick_past_deadline",
                  "commit_before_deadline", "deadline_moved_without_commit", "deadline_not_rearmed_at_adoption"):
        assert stage in worst, (stage, sorted(worst))
    assert all(0 <= v <= 1 for v in worst.values()), worst


def test_emulated_interval_trajectory_fails_under_the_k_eq_n_model():
    """The premise of the GPU runs' check: the K = N model (an update and a new epoch word every step) tells an
    interval run apart."""
    bad = T.failures(_interval_results("lenet", mode="fused"))
    assert any("step1.update_bits_differ" in n for n, _, _ in bad), bad[:10]


@pytest.mark.parametrize("model,fault,stage", [
    ("lenet", "divisor_1", "step3.update_bits_differ"),
    ("mlp3", "divisor_t_minus_1", "step3.update_bits_differ"),
    ("lenet", "accumulator_overwritten", "step3.update_bits_differ"),
    ("mlp3", "accumulator_overwritten", "step3.update_bits_differ"),
    ("lenet", "adoption_late", "step1.conv1_fwd"),
    ("mlp3", "adoption_late", "step1.h1"),
    ("lenet", "k_eq_n_updates", "step1.update_bits_differ"),
    ("mlp3", "k_eq_n_updates", "step1.update_bits_differ"),
    ("lenet", "mask_step0_plus_t", "step2.fc2_fwd_bwd"),
    ("lenet", "shadow_not_refreshed", "step1.shadow_bits_differ"),
    ("mlp3", "shadow_not_refreshed", "step1.shadow_bits_differ"),
    ("lenet", "commit_before_deadline", "step0.commit_before_deadline"),
    ("lenet", "deadline_rearmed_without_adoption", "step2.deadline_moved_without_commit"),
    ("lenet", "count_word_off", "step1.count_differs"),
    ("lenet", "epoch_without_commit", "step2.epoch_differs"),
])
def test_seeded_interval_fault_fails(model, fault, stage):
    bad = T.failures(_interval_results(model, fault))
    assert any(stage in n for n, _, _ in bad), (fault, bad[:10])


def test_interval_clock_armed_before_the_global_step_fails():
    """The clock armed at epoch 0 and the global step set afterwards: the step half of iv_state is 1, not STEP0 + 1."""
    spec, init, records, batches, upd = _run_interval("mlp3")
    c = _Ctrl()
    c.b[:] = init["ctrl"].numpy()
    c["iv_state"] = 1 << 32
    bad = T.failures(T.control_results("mlp3", dict(init, ctrl=c.snapshot()), records, upd))
    assert [n for n, _, _ in bad] == ["mlp3.init.clock_armed_before_global_step"]


def test_stamps_of_a_k_eq_n_run():
    """cdf mode: the stamps of step t sit at its global step; a step whose start was never stamped fails."""
    spec, init, records, batches, upd = _run("mlp3")
    c = _Ctrl()
    init = dict(init, ctrl=c.snapshot())
    for t, r in enumerate(records):
        c["epoch"] = STEP0 + t
        c.stamp("t_start", 100 * t + 1)
        c.stamp("t_arrive", 100 * t + 50)
        c["epoch"] = STEP0 + t + 1
        r["ctrl"] = c.snapshot()
    upd = dict(upd, ctrl_off=CTRL_OFF)
    res = T.control_results("mlp3", init, records, upd)
    assert len(res) == len(records) and not T.failures(res), res
    c.b[CTRL_OFF["t_start"]:CTRL_OFF["t_arrive"]] = 0        # t_start never stamped
    records[-1]["ctrl"] = c.snapshot()
    bad = T.failures(T.control_results("mlp3", init, records, upd))
    assert [n for n, _, _ in bad] == ["mlp3.step3.stamps_out_of_order"]
