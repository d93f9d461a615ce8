"""Helper process: the aggregation kernels driven directly on N replicas, each step checked bit for bit against the exact
emulation of ops/aggrefs.py.  Every rank all-gathers every replica's gradients (and bf16 fc1 gradients) before the step and
emulates the step itself from its own weights, so a wrong contributor order, a doubled or missing contributor, a shard
boundary off by one, the wrong drop mask or a stale shadow shows on the rank where it happens.

argv: <out json with RANK placeholder> <comma-separated cases>
cases: p2p (K = N, peer loads), kofn (K = N - 1, last rank delayed on the device), drop (drop-connect), nvls (K = N,
multimem), bucket1 (csrc/fused_sync.cu bucketed kernels), v2_ll_bf16 / v2_ll_fp32 / v2_flags (csrc/fused_bucket.cu, LeNet
layout), v2_mlp (MLP layout, phases 3 / 4, fp32 late kernel), interval (csrc/fused_interval.cu, last rank delayed)."""
import hashlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributedmnist_b200.models import lenet_spec, mlp_spec  # noqa: E402
from distributedmnist_b200.ops import aggrefs as A  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402
from distributedmnist_b200.schedule import LearningRateSchedule  # noqa: E402

SCHED = LearningRateSchedule(0.05, 1, 0.999)       # p = step: the step size changes every step
STEPS = 4
RAGGED = 4 * (65536 * 3 + 5)                        # numel4 divisible by none of 2 .. 8


def fp(t):
    return hashlib.sha1(t.detach().cpu().numpy().tobytes()).hexdigest()


def _param(spec, name):
    q = [p for p in spec.params if p.name == name][0]
    return q.offset, q.offset + q.numel


def _grad(seed, n):
    """Magnitudes spread over 2^-6 .. 2^6: the order of the adds changes the rounded sums."""
    rng = np.random.default_rng(seed)
    return torch.from_numpy((rng.standard_normal(n) * 2.0 ** rng.integers(-6, 7, n)).astype(np.float32))


class Case:
    def __init__(self, ctx, name, nvls=False):
        self.ctx, self.name = ctx, name
        self.n, self.r = ctx.world_size, ctx.rank
        self.be = FusedBackend(ctx, timeout_ms=10000.0, use_nvls=nvls)
        self.res = {"case": name, "bad_w": 0, "bad_sh": 0, "masks": [], "counts": [], "steps": [], "bound_excess": 0.0}

    def gather(self, t):
        if self.n == 1:
            return [A.f32(t.float())]
        out = [torch.empty_like(t) for _ in range(self.n)]
        dist.all_gather(out, t)
        return [A.f32(x.float()) for x in out]

    def check(self, params, want):
        torch.cuda.synchronize()
        self.res["bad_w"] += int((A.bits(params) != A.bits(want)).sum())
        sh = self.be.shadow.view(torch.int16).cpu().numpy().view(np.uint16)
        self.res["bad_sh"] += int((sh != A.bf16_bits(want)).sum())

    def arena(self, numel):
        params, grads = self.be.allocate(numel), self.be.allocate(numel)
        params.copy_((torch.randn(numel, generator=torch.Generator().manual_seed(5)) * 0.05).to(self.ctx.device))
        self.be.attach_shadow(params)
        self.be.set_global_step(5000)
        return params, grads

    def finish(self, params):
        self.be.check_error()
        self.res["fp"] = fp(params)
        self.res["nvls"] = bool(self.be.nvls_active)
        self.be.close()
        return self.res


def run_sync(ctx, name):
    """fused_sync_sgd_kernel: K = N (p2p, drop, nvls) or K = N - 1 with the last rank delayed (kofn)."""
    c = Case(ctx, name, nvls=name == "nvls")
    be, n, r = c.be, c.n, c.r
    params, grads = c.arena(RAGGED)
    if name == "drop":
        be.drop_connect_(grads, 0.9, 0)
    k = n - 1 if name == "kofn" else n
    for s in range(STEPS):
        grads.copy_(_grad(1000 * s + r, RAGGED).to(ctx.device))
        allg = c.gather(grads)
        w, step = A.f32(params), be.device_epoch
        torch.cuda.synchronize()
        be.barrier()
        if name == "kofn" and r == n - 1:
            be.enqueue_straggler_delay(1.0, 20000.0)
        be.enqueue(params, grads, k, SCHED.initial_learning_rate, SCHED.decay_rate, SCHED.decay_steps)
        torch.cuda.synchronize()
        be.barrier()                  # the late rank returns before the pushes it waits for are all observed by the others
        info = be.last_step_info(check=True)
        count = bin(info.mask).count("1")
        c.res["masks"].append(info.mask)
        c.res["counts"].append(info.count)
        c.res["steps"].append(info.global_step)
        scale = A.step_scale(SCHED, step, count)
        drop = (be.drop_seed, step, be.drop_keep) if name == "drop" else None
        if name == "nvls" and n >= 3 and be.nvls_active:
            # the switch adds in an unspecified order: bound |w' - (w - scale * sum)| by the fp32 sum and fma roundings
            g64 = np.stack([g.astype(np.float64) for g in allg])
            exact = w.astype(np.float64) - float(scale) * g64.sum(0)
            bound = float(scale) * (n - 1) * 2.0 ** -23 * np.abs(g64).sum(0) + 2.0 ** -23 * np.abs(exact)
            got = A.f32(params).astype(np.float64)
            c.res["bound_excess"] = max(c.res["bound_excess"], float((np.abs(got - exact) - bound).max()))
            sh = be.shadow.view(torch.int16).cpu().numpy().view(np.uint16)
            c.res["bad_sh"] += int((sh != A.bf16_bits(A.f32(params))).sum())
        else:
            c.check(params, A.fused_sync_step(w, allg, info.mask, scale, drop))
    return c.finish(params)


def run_bucket1(ctx, name):
    """csrc/fused_sync.cu bucketed path (DMNIST_BUCKET=1): fp32 two-shot early bucket + one-shot late bucket, rank order."""
    c = Case(ctx, name)
    be, r = c.be, c.r
    spec = lenet_spec()
    e0, e1 = _param(spec, "fc1_weights")
    params, grads = c.arena(spec.arena_numel)
    for s in range(STEPS):
        grads.copy_(_grad(1000 * s + r, spec.arena_numel).to(ctx.device))
        allg = c.gather(grads)
        w, step = A.f32(params), be.device_epoch
        torch.cuda.synchronize()
        be.barrier()
        lr = (SCHED.initial_learning_rate, SCHED.decay_rate, SCHED.decay_steps)
        be.enqueue_bucket(params, grads, 1, e0, e1, e0, e1, *lr)
        be.enqueue_bucket(params, grads, 2, 0, spec.arena_numel, e0, e1, *lr)
        torch.cuda.synchronize()
        be.barrier()
        c.res["steps"].append(be.device_epoch)
        c.check(params, A.fused_sync_step(w, allg, (1 << c.n) - 1, A.step_scale(SCHED, step, c.n)))
    return c.finish(params)


def run_v2(ctx, name):
    """csrc/fused_bucket.cu on the LeNet layout (early = fc1, phases 1 + 2) or the MLP layout (early = fc2, phases 3, 4, 2)."""
    c = Case(ctx, name)
    be, n, r = c.be, c.n, c.r
    mlp = name == "v2_mlp"
    spec = mlp_spec(3, 1024) if mlp else lenet_spec()
    e0, e1 = _param(spec, "fc2_weights" if mlp else "fc1_weights")
    be.late_ll, be.late_bf16 = name != "v2_flags", name != "v2_ll_fp32"
    numel = spec.arena_numel
    params, grads = c.arena(numel)
    g16 = be.allocate_buffer((e1 - e0) * 2)
    inbox = be.allocate_buffer(2 * n * (numel - (e1 - e0)) * 8) if n > 1 else None
    g16v = g16.view(torch.bfloat16, 0, e1 - e0)
    rounds = A.late_bucket_rounds_bf16(numel, e1 - e0, be.late_ll, be.late_bf16)
    c.res["late_bf16"] = rounds
    for s in range(STEPS):
        grads.copy_(_grad(1000 * s + r, numel).to(ctx.device))
        g16v.copy_(_grad(777 * s + r, e1 - e0).to(torch.bfloat16).to(ctx.device))
        allg, allg16 = c.gather(grads), c.gather(g16v)      # before the step: the early reduce works in place
        w, step = A.f32(params), be.device_epoch
        torch.cuda.synchronize()
        be.barrier()
        for phase in ((3, 4, 2) if mlp else (1, 2)):
            be.enqueue_bucket_v2(params, grads, g16, inbox, phase, e0, e1, SCHED.initial_learning_rate, SCHED.decay_rate,
                                 SCHED.decay_steps)
        torch.cuda.synchronize()
        be.barrier()
        c.res["steps"].append(be.device_epoch)
        c.check(params, A.bucket_step(w, allg, allg16, (e0, e1), A.step_scale(SCHED, step, n), rounds))
    return c.finish(params)


def run_interval(ctx, name, interval_ms=2.0, iters=120, delay_us=6000.0):
    """Device interval mode, last rank delayed so that it misses ticks.  Rank q's gradient is the same tensor g_q on every
    iteration, so a tick's accumulator on q is the sequential sum of c_q copies, c_q = the iterations q had accepted for that
    step.  Every tick is rebuilt from the committed mask and divisor (as published by a replica that adopted it alone) and
    from every rank's per-iteration record; the weights after the last tick must match bit for bit on every rank."""
    c = Case(ctx, name)
    be, n, r = c.be, c.n, c.r
    numel = 1 << 18
    params, grads = c.arena(numel)
    w0 = A.f32(params)
    acc = be.allocate(numel)
    grads.copy_(_grad(31 + r, numel).to(ctx.device))
    allg = c.gather(grads)
    slow = n > 1 and r == n - 1
    if slow:
        iters = max(4, int(iters * 250.0 / delay_us))
    be.interval_arm(interval_ms)
    rows = []
    for _ in range(iters):
        be.enqueue_interval_begin(params)
        be.enqueue_straggler_delay(1.0, delay_us if slow else 200.0)
        be.enqueue_interval_end(params, grads, acc, SCHED.initial_learning_rate, SCHED.decay_rate, SCHED.decay_steps)
        st = be.read_status()
        rows.append((st["epoch"], st["last_late"], st["last_mask"], st["last_count"]))
    torch.cuda.synchronize()
    be.check_error()
    be.barrier()
    time.sleep(0.05)
    be.enqueue_interval_begin(params)            # adopt whatever was committed last
    torch.cuda.synchronize()
    be.barrier()
    last = be.device_epoch
    all_rows = be.all_gather_object(rows)
    first = 5000
    w = w0
    unknown = 0
    for e in range(first, last):
        cnt = [sum(1 for (ep, late, _, _) in all_rows[q] if ep == e and not late) for q in range(n)]
        mask, total = None, None
        for q in range(n):                       # a replica whose epoch moved from e to e + 1 in one iteration
            rq = all_rows[q]
            for i in range(1, len(rq)):
                if rq[i - 1][0] == e and rq[i][0] == e + 1:
                    mask, total = rq[i][2], rq[i][3]
                    break
            if mask is not None:
                break
        if mask is None:
            unknown += 1
            mask = sum(1 << q for q in range(n) if cnt[q])
            total = sum(cnt)
        c.res["masks"].append(mask)
        c.res["counts"].append(total)
        if sum(cnt[q] for q in range(n) if (mask >> q) & 1) != total:
            c.res["bad_w"] += numel            # the records do not explain the committed divisor
            continue
        accs = [A.interval_accumulate([allg[q]] * cnt[q]) if (mask >> q) & 1 else None for q in range(n)]
        w = A.fused_sync_step(w, accs, mask, A.step_scale(SCHED, e, total))
    c.res["steps"] = [first, last]
    c.res["unknown_ticks"] = unknown
    c.res["dropped"] = be.read_status()["dropped_steps"]
    c.check(params, w)
    return c.finish(params)


RUNNERS = {"p2p": run_sync, "kofn": run_sync, "drop": run_sync, "nvls": run_sync, "bucket1": run_bucket1,
           "v2_ll_bf16": run_v2, "v2_ll_fp32": run_v2, "v2_flags": run_v2, "v2_mlp": run_v2, "interval": run_interval}


def main():
    out_json = sys.argv[1].replace("RANK", os.environ.get("RANK", "0"))
    ctx = init_context(None, want_gpu=True)
    out = {"rank": ctx.rank, "n": ctx.world_size, "cases": {}}
    for name in sys.argv[2].split(","):
        out["cases"][name] = RUNNERS[name](ctx, name)
    with open(out_json, "w") as f:
        json.dump(out, f)
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
