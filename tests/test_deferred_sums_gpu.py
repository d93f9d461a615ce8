"""The training step's reproducible sums that run off its data-gradient chain, bit for bit against the sums the kernels
make themselves.

fc2_fwd_bwd's per-row (loss, hit) terms: ``dm_fc2_fwd_bwd_rows`` stores them and ``dm_fc2_loss_sum`` adds them up; the
loss words must be those of ``dm_fc2_fwd_bwd``, whose last CTA adds them, and both must be the one-warp order (lane l
adds rows l, l + 32, ... in fp32, then the xor butterfly).  fc1_dgrad's conv2 bias-gradient slots:
``dm_fc1_dgrad_unpool_slots`` stores one per CTA and ``dm_conv2_wgrad_bias``'s reduction adds them in slot order; the
bias gradient must equal that of ``dm_fc1_dgrad_unpool`` and an fp32 sum of the slots in slot order, and the conv2 weight
gradient that of ``dm_conv2_wgrad``.  Then a graph-replayed training step, with and without weight decay, reports the
loss word that ``dm_fc2_fwd_bwd`` computes from the step's own fc1 partials and pre-step weights."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BATCHES = [1, 37, 256, 1024, 10624]
BF = torch.bfloat16


def _bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().cpu().contiguous()
    return t.view(torch.int16 if t.dtype == BF else torch.int32).numpy()


def _assert_same(what, got, want):
    g, w = _bits(got), _bits(want)
    bad = np.flatnonzero(g.reshape(-1) != w.reshape(-1))
    assert bad.size == 0, "%s: %d of %d differ, first at %d" % (what, bad.size, g.size, bad[0])


def _warp_order_sum(terms: np.ndarray) -> np.ndarray:
    """fc2_loss_sum in fp32: lane l adds rows l, l + 32, ... in row order, then the xor butterfly 16, 8, 4, 2, 1."""
    lanes = np.zeros((32, terms.shape[1]), np.float32)
    for r in range(terms.shape[0]):
        lanes[r % 32] += terms[r]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return lanes[0]


def _slot_order_sum(slots: np.ndarray) -> np.ndarray:
    s = np.zeros(slots.shape[1], np.float32)
    for k in range(slots.shape[0]):
        s += slots[k]
    return s


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_loss_sum_matches_the_last_cta(B):
    from distributedmnist_b200.ops import selfcheck as S
    from distributedmnist_b200.ops.lib import load, stream_ptr
    lib = load()
    g = torch.Generator().manual_seed(700 + B)
    parts = (torch.randn(7, B, 512, generator=g) * 0.3).cuda()
    b1, w2, b2 = ((torch.randn(*s, generator=g) * 0.1).cuda() for s in ((512,), (512, 10), (10,)))
    labels = torch.randint(0, 10, (B,), generator=g).cuda()
    for train in (True, False):
        want = S.run_fc2_fwd_bwd(parts, b1, w2, b2, labels, train, 0x1234, 9)
        o = dict(dh=torch.zeros(B, 512, dtype=BF, device="cuda"), h=torch.zeros(B, 512, device="cuda"),
                 dl=torch.zeros(B, 12, device="cuda"), logits=torch.zeros(B, 10, device="cuda"))
        rows = torch.full((B, 2), float("nan"), device="cuda")
        la = torch.zeros(2, device="cuda")
        st = torch.tensor([9], dtype=torch.int32, device="cuda")
        lib.dm_fc2_fwd_bwd_rows(parts, parts.stride(0), 7, b1, w2, b2, labels, o["dh"], o["h"], o["dl"], rows, o["logits"],
                                B, int(train), 0x1234, st, 0.5, stream_ptr())
        lib.dm_fc2_loss_sum(rows, B, la, stream_ptr())
        torch.cuda.synchronize()
        for k in ("dh", "h", "dl", "logits"):
            _assert_same("%s train=%d" % (k, train), o[k], want[k])
        _assert_same("loss words train=%d" % train, la, want["la"])
        assert _warp_order_sum(rows.cpu().numpy()).tobytes() == want["la"].cpu().numpy().tobytes()


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_bias_sum_in_the_reduction_matches_fc1_dgrad_unpool(B):
    from distributedmnist_b200.ops import selfcheck as S
    from distributedmnist_b200.ops.lib import load, stream_ptr
    lib = load()
    g = torch.Generator().manual_seed(800 + B)
    dh = (torch.randn(B, 512, generator=g) * 0.01).to(BF).cuda()
    w1 = (torch.randn(3136, 512, generator=g) * 0.05).to(BF).cuda()
    code2 = S._codes(g, (B, 3136)).cuda()
    a1 = torch.rand(B, 14, 14, 32, generator=g).to(BF).cuda()
    dy_want, gb_want = S.run_fc1_dgrad_unpool(dh, w1, code2)

    n = int(lib.dm_unpool_bias_slots(B))
    assert n == (B + 127) // 128 * 49
    slots = torch.full((n, 64), float("nan"), device="cuda")
    dy = torch.full((B, 14, 14, 64), 7.0, dtype=BF, device="cuda")
    lib.dm_fc1_dgrad_unpool_slots(dh, w1, code2, dy, slots, B, stream_ptr())
    gw, gb = torch.zeros(25 * 32 * 64, device="cuda"), torch.zeros(64, device="cuda")
    lib.dm_conv2_wgrad_bias(a1, dy, gw, slots, n, gb, B, stream_ptr())
    gw_want = torch.zeros(25 * 32 * 64, device="cuda")
    lib.dm_conv2_wgrad(a1, dy_want, gw_want, B, stream_ptr())
    torch.cuda.synchronize()
    _assert_same("dy2", dy, dy_want)
    _assert_same("conv2 bias gradient", gb, gb_want)
    assert _slot_order_sum(slots.cpu().numpy()).tobytes() == gb_want.cpu().numpy().tobytes()
    _assert_same("conv2 weight gradient", gw, gw_want)


@pytest.mark.parametrize("lam", [0.0, 5e-4])
@pytest.mark.parametrize("B", BATCHES)
def test_graph_replayed_step_reports_the_kernels_loss_word(B, lam):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.ops import selfcheck as S
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(B, be, seed=11, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 4, 0.7), 1, 1))
    lam = float(np.float32(lam))
    if lam:
        eng.arm_weight_decay(lam)
    g = torch.Generator().manual_seed(900 + B)
    eng.load_batch(torch.rand(B, 28, 28, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g))
    w = eng.params.clone()
    epoch = be.read_status()["epoch"]
    eng.train_step()
    loss, acc = eng.loss_acc()
    v = eng.spec.views(w)
    want = S.run_fc2_fwd_bwd(eng.h_part, v["fc1_biases"], v["fc2_weights"], v["fc2_biases"], eng.labels[eng._slot], True,
                             eng._seed_mix0, epoch, eng.keep_prob)["la"].cpu().numpy()
    if lam:
        want[0] = want[0] + np.float32(lam * eng.weight_decay_r())
    assert np.float32(loss).tobytes() == want[0].tobytes() and np.float32(acc).tobytes() == want[1].tobytes()
    be.check_error()
