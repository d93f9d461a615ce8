"""The LeNet training step is bit-reproducible on one GPU: every cross-CTA sum goes through per-CTA workspace slots added
up in slot order.  (The MLP path still accumulates with fp32 atomics and is not covered here.)"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _engine(B, seed, use_graph):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    return CudaLeNetEngine(B, be, seed=seed, use_graph=use_graph), be


def _batches(n, B, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(B, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)) for _ in range(n)]


def test_forward_backward_twice_is_bitwise_equal():
    eng, _ = _engine(256, 3, use_graph=False)
    (x, y), = _batches(1, 256, 4)
    runs = []
    for _ in range(2):
        eng.load_batch(x.numpy(), y.numpy())
        eng.forward_backward(0)
        torch.cuda.synchronize()
        runs.append((eng.grads.clone(), eng.loss_acc()))
    assert torch.equal(runs[0][0], runs[1][0]), "gradient arena differs between two identical passes"
    assert runs[0][1] == runs[1][1]


def test_train_steps_bitwise_equal_through_native_runner():
    """Same seed, same batches: load_batch + train_step on one engine, pack_batch + step_packed (bench.py's path) on the
    other; five graph-replayed steps each."""
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.schedule import LearningRateSchedule
    batches = _batches(5, 256, 5)
    out = []
    for packed in (False, True):
        eng, be = _engine(256, 11, use_graph=True)
        eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 2, 0.5), 1, 1))
        losses = []
        bufs = [eng.pack_batch(x, y) for x, y in batches] if packed else None
        for s, (x, y) in enumerate(batches):
            if packed:
                ev, buf, _ = eng.step_packed(bufs[s])
                ev.synchronize()
                losses.append((float(buf[0]), float(buf[1])))
            else:
                eng.load_batch(x.numpy(), y.numpy())
                eng.train_step()
                losses.append(eng.loss_acc())
        torch.cuda.synchronize()
        be.check_error()
        out.append((eng.params.clone(), eng.shadow.clone(), losses, eng.step_info().global_step))
        eng._leave_native_runner()
    (p0, s0, l0, g0), (p1, s1, l1, g1) = out
    assert g0 == g1 == 5
    assert l0 == l1
    assert torch.equal(p0, p1) and torch.equal(s0, s1)


def _slot_reduced_results(B, seed):
    from distributedmnist_b200.ops import selfcheck as S
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, 28, 28, generator=g) - 0.5).cuda()
    dp = (torch.randn(B, 14, 14, 32, generator=g) * 0.1).to(torch.bfloat16).cuda()
    c1 = S._codes(g, (B, 14, 14, 32)).cuda()
    a1 = torch.rand(B, 14, 14, 32, generator=g).to(torch.bfloat16).cuda()
    dy = (torch.randn(B, 14, 14, 64, generator=g) * 0.1).to(torch.bfloat16).cuda()
    dh = (torch.randn(B, 512, generator=g) * 0.1).to(torch.bfloat16).cuda()
    w1 = (torch.randn(3136, 512, generator=g) * 0.05).to(torch.bfloat16).cuda()
    c2 = S._codes(g, (B, 3136)).cuda()
    parts = torch.randn(7, B, 512, generator=g).cuda()
    b1, w2, b2 = torch.randn(512, generator=g).cuda(), torch.randn(512, 10, generator=g).cuda(), torch.randn(10, generator=g).cuda()
    lab = torch.randint(0, 10, (B,), generator=g).cuda()
    res = {"conv1_wgrad_tc": S.run_conv1_wgrad(x, dp, c1, tc=True), "conv2_wgrad": S.run_conv2_wgrad(a1, dy),
           "fc1_dgrad_unpool.g_bias": S.run_fc1_dgrad_unpool(dh, w1, c2)[1],
           "fc2_fwd_bwd.loss_acc": S.run_fc2_fwd_bwd(parts, b1, w2, b2, lab)["la"]}
    torch.cuda.synchronize()
    return res


def test_slot_reduced_kernels_repeat_bitwise_after_a_larger_launch():
    first = _slot_reduced_results(256, 6)
    _slot_reduced_results(1024, 7)            # other CTA counts: more slots written, tickets reset by a larger grid
    again = _slot_reduced_results(256, 6)
    for k in first:
        a, b = first[k], again[k]
        for ta, tb in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
            assert torch.equal(ta, tb), k
