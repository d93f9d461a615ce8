"""The LeNet kernels and training step against their float64 references at batches above 1024, up to the largest batch
the engine accepts (``dm_lenet_max_batch()``, 10 624 rows), and the refusal of the next one.

Several kernels change behaviour as the batch grows: fc1_dgrad_unpool's last CTA sums the conv2 bias-gradient slots
(49 per 128-row tile) in shared-memory chunks of 384; the conv2 weight gradient walks ever more images per CTA, so its
TMA ring wraps hundreds of times; conv1's weight gradient keeps its capped grid and grows only the tiles per CTA; the
conv2 forward and data-gradient tiles run many rounds per SM over one stack of 14 B image rows.  The batches:

* 2048, the evaluation chunk: 784 bias-gradient slots, chunks of 384 + 384 + 16;
* 4133, a multiple of neither 32 nor 128: the last conv2 forward / data-gradient tile and the last GEMM row tile are
  partial;
* 6016: 47 row tiles, 2303 slots, five full chunks and one of 383;
* 10 624, the limit: 4067 slots, 11 chunks.

The checks are those of test_kernel_refs_gpu.py (grid data bitwise, continuous data within the precision bounds), with
the references evaluated a chunk of rows at a time (``selfcheck.REF_ROWS``); weight-gradient references still sum the
whole batch in float64.  fc1_dgrad_unpool's grid weights are narrower above 8192 rows so that the exact conv2
bias-gradient sums stay below 2^24 grid units.  conv2_fwd, conv2_dgrad and fc1_dgrad_unpool write into poisoned
outputs with a poisoned tail, so they also show every output element written and nothing written past the batch."""
import pytest
import torch

pytestmark = pytest.mark.gpu

LIMIT = 10624
BATCHES = [2048, 4133, 6016, LIMIT]
GUARD = 3 * 14 * 14 * 64          # three batch rows of dy2 (and more than a row of every conv2 output) past the end


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def _stale(B):
    """a batch of another size, run first so the workspace holds stale partial sums: the limit (more slots than this
    launch reads) or, at the limit, the evaluation chunk"""
    return LIMIT if B < LIMIT else 2048


def test_declared_limit_is_fc1_dgrad_unpools():
    """dm_lenet_max_batch() is the largest batch fc1_dgrad_unpool runs: one row more and it refuses before launching."""
    from distributedmnist_b200.ops.lib import KernelLibraryError, load, stream_ptr
    lib = load()
    assert lib.dm_lenet_max_batch() == LIMIT
    B = LIMIT + 1
    dh = torch.zeros(B, 512, dtype=torch.bfloat16, device="cuda")
    w1 = torch.zeros(3136, 512, dtype=torch.bfloat16, device="cuda")
    code = torch.zeros(B, 3136, dtype=torch.uint8, device="cuda")
    dy = torch.full((B, 14, 14, 64), 7.0, dtype=torch.bfloat16, device="cuda")
    gb = torch.zeros(64, device="cuda")
    with pytest.raises(KernelLibraryError, match="code -6"):
        lib.dm_fc1_dgrad_unpool(dh, w1, code, dy, gb, B, stream_ptr())
    torch.cuda.synchronize()
    assert bool((dy == 7.0).all()) and not bool(gb.any()), "the refused launch wrote its outputs"


@pytest.mark.parametrize("B", BATCHES)
def test_conv1_fwd_tc(B):
    _run("check_conv1_fwd_tc", B=B, seed=100 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_conv1_wgrad_tc(B):
    _run("check_conv1_wgrad", B=B, seed=200 + B, stale_B=_stale(B))


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_fwd_writes_exactly_its_outputs(B):
    _run("check_conv2_fwd", B=B, seed=300 + B, guard=GUARD)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_dgrad_writes_exactly_its_output(B):
    _run("check_conv2_dgrad", B=B, seed=400 + B, guard=GUARD)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_wgrad(B):
    _run("check_conv2_wgrad", B=B, seed=500 + B, stale_B=_stale(B))


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("B", BATCHES)
def test_fc1_fwd_split_k_then_fc2_fwd_bwd(B, train):
    _run("check_fc1_fwd", B=B, seed=600 + B, train=train)


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_fwd_bwd_after_stale_launch(B):
    _run("check_fc2_loss", B=B, seed=660 + B, stale_B=_stale(B))


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_wgrad(B):
    _run("check_fc2_wgrad", B=B, seed=700 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_wgrad_f32_and_bf16(B):
    _run("check_fc1_wgrad", B=B, seed=800 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_dgrad_unpool_writes_exactly_its_output(B):
    _run("check_fc1_dgrad_unpool", B=B, seed=900 + B, stale_B=_stale(B), guard=GUARD)


# The continuous-data bound of a decayed gradient grows as B^2 (B terms, each sum of |terms| ~ B), so the smaller
# lambdas of selfcheck.DECAY_LAMS fall below it here and their premise check (decay_term_detectable) fails: these
# batches use the largest one and a larger one, on grid data bit for bit as everywhere.
LARGE_BATCH_LAMS = (2.0 ** -4, 0.25)


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_wgrad_decay(B):
    _run("check_fc1_wgrad_decay", B=B, seed=1000 + B, lams=LARGE_BATCH_LAMS)


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_wgrad_decay(B):
    _run("check_fc2_wgrad_decay", B=B, seed=1100 + B, lams=LARGE_BATCH_LAMS)


@pytest.mark.parametrize("ctas", [8, 27])
def test_weight_gradient_split_structure(ctas):
    """8 CTAs: conv2_wgrad runs one split walking all 4133 images (its 3-stage ring wraps 1377 times, its accumulator is
    folded 64 times) and conv1_wgrad 8 slices in groups of 3; 27: three conv2 splits of 1377 or 1378 images and 27 conv1
    slices in groups of 6.  Before conv2_wgrad folded its accumulator every WG_FOLD images, one split of 4133 images
    missed the continuous-data bound (a normwise error of 9.1e-4, three splits 3.1e-4, against 2^-12)."""
    from distributedmnist_b200.ops.lib import load
    lib = load()
    if lib.dm_num_sms() < ctas:
        pytest.skip("device has fewer than %d SMs" % ctas)
    prev = lib.dm_get_max_ctas()
    try:
        assert lib.dm_set_max_ctas(ctas) == ctas
        _run("check_conv2_wgrad", B=4133, seed=1200 + ctas, stale_B=2048)
        _run("check_conv1_wgrad", B=4133, seed=1300 + ctas, stale_B=2048)
    finally:
        lib.dm_set_max_ctas(prev)              # whatever was in force before (0: the default)


@pytest.mark.parametrize("B", [2048, LIMIT])
def test_lenet_bucketed_trajectory(B, monkeypatch):
    """Three graph-replayed steps: the two slot graphs' captures and one replay."""
    from test_step_trajectory_gpu import _batches, _check, _feed, _lenet
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(B)
    batches = _batches(eng, 3, seed=B)
    _feed(eng, rec, batches)
    _check("lenet.B%d.bucket2" % B, eng, be, rec, batches)


def test_lenet_decayed_keep_08_trajectory(monkeypatch):
    from test_step_trajectory_gpu import LAM, _batches, _check, _feed, _lenet
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(4133, keep_prob=0.8, lam=LAM)
    batches = _batches(eng, 3, seed=4133)
    _feed(eng, rec, batches)
    _check("lenet.B4133.keep0.8.decay", eng, be, rec, batches, LAM)


def test_engine_refuses_a_batch_past_the_limit_and_runs_the_limit():
    """One row past dm_lenet_max_batch() is refused by the engine, naming the flag and the limit, before it allocates
    anything, and by train.py's flag validation; the limit itself builds and trains."""
    from types import SimpleNamespace

    from distributedmnist_b200 import train
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.schedule import LearningRateSchedule
    from test_step_trajectory_gpu import _backend
    be = _backend()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match=r"--batch_size=10625 .*--batch_size <= 10624"):
        CudaLeNetEngine(LIMIT + 1, be, use_graph=False)
    assert torch.cuda.memory_allocated() == before
    ctx = SimpleNamespace(on_gpu=True)
    flags = SimpleNamespace(backend="auto", model="lenet", batch_size=LIMIT + 1)
    with pytest.raises(ValueError, match="10624"):
        train.check_batch_flags(flags, ctx)
    train.check_batch_flags(SimpleNamespace(backend="auto", model="lenet", batch_size=LIMIT), ctx)
    train.check_batch_flags(SimpleNamespace(backend="auto", model="mlp2", batch_size=LIMIT + 1), ctx)

    eng = CudaLeNetEngine(LIMIT, be, use_graph=False)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 100, 1.0), 1, 1))
    g = torch.Generator().manual_seed(5)
    before = eng.params.clone()
    eng.load_batch((torch.rand(LIMIT, 28, 28, 1, generator=g) - 0.5).numpy(), torch.randint(0, 10, (LIMIT,), generator=g).numpy())
    eng.train_step()
    loss, _ = eng.loss_acc()
    torch.cuda.synchronize()
    be.check_error()
    assert loss == loss and loss > 0
    assert not torch.equal(before, eng.params)
