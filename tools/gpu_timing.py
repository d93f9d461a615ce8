"""The harness the GPU measurement scripts under tools/ share: the card query, a one-replica engine on synthetic packed
batches, CUDA-event windows of training steps, alternation between configurations, child processes and JSON output.

A script imports it as ``import gpu_timing``: ``python tools/<script>.py`` puts tools/ on ``sys.path``, and this module
puts the repository root there too, so the script can import the package after it.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine  # noqa: E402
from distributedmnist_b200.parallel.context import ReplicaContext  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402


def card() -> dict:
    """The name, power limit and max SM clock of GPU 0, as nvidia-smi reads them; "?" in each field when the query fails."""
    query = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"]
    try:
        r = subprocess.run(query, capture_output=True, text=True)
        fields = [v.strip() for v in r.stdout.strip().split(",")] if r.returncode == 0 else []
    except OSError:
        fields = []
    if len(fields) != 3:
        fields = ["?"] * 3
    return dict(zip(("gpu", "power_limit", "max_sm_clock"), fields))


def _engine(ctx, model, batch, hidden, optimizer):
    be = FusedBackend(ctx)
    eng = CudaLeNetEngine(batch, be, use_graph=True) if model == "lenet" else \
        CudaMlpEngine(model, batch, be, hidden=hidden, use_graph=True)
    eng.attach_optimizer(optimizer(be))
    return eng


def one_replica_engine(model, batch, hidden, optimizer):
    """A graph-replaying engine of `model` (``hidden`` is ignored for lenet) on its own backend, one replica on cuda:0,
    with ``optimizer(backend)`` attached."""
    torch.cuda.set_device(0)
    return _engine(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"), model, batch, hidden, optimizer)


def packed_batches(eng, n, seed, on_device):
    """`n` packed batches of uniform images in [-0.5, 0.5) and random labels: pinned host buffers, or device-resident."""
    g = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    out = []
    for _ in range(n):
        p = eng.pack_batch(torch.rand(B, 784, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g),
                           pin=not on_device)
        out.append(p.cuda() if on_device else p)
    return out


def timed_steps(eng, bufs, steps) -> float:
    """Microseconds per step of `steps` back-to-back ``step_packed`` calls cycling through `bufs`: CUDA events around the
    calls, then a synchronise."""
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
        eng.step_packed(bufs[i % len(bufs)])
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / max(steps, 1)


def timed_launches(fn, n, warmup) -> float:
    """Microseconds per call of `n` back-to-back calls of `fn` after `warmup` calls: CUDA events around them."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / n


def alternate(configs, steps, warmup, rounds, before_block=None) -> dict:
    """`configs` maps a name to (engine, packed batches).  Every configuration runs one block of `warmup` steps, then
    `rounds` rounds run one timed block of `steps` steps per configuration, in the dict's order, so that a drift of the
    clocks spreads over all of them.  ``before_block(engine)`` runs ahead of every block.  Returns {name: [microseconds
    per step of each round]}."""
    def block(name, k):
        eng, bufs = configs[name]
        if before_block is not None:
            before_block(eng)
        return timed_steps(eng, bufs, k)

    for name in configs:
        block(name, warmup)
    us = {name: [] for name in configs}
    for _ in range(rounds):
        for name in configs:
            us[name].append(block(name, steps))
    return us


def _last_json(text):
    return json.loads([ln for ln in text.splitlines() if ln.startswith("{")][-1])


def child_json(argv, env=None) -> dict:
    """Runs ``python argv...`` with `env` added to this process's environment; returns the last JSON line it printed."""
    r = subprocess.run([sys.executable] + list(argv), capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    if r.returncode != 0:
        raise RuntimeError(r.stdout[-2000:] + r.stderr[-4000:])
    return _last_json(r.stdout)


def replicas_json(argv, gpus) -> dict:
    """Runs ``python argv...`` as `gpus` replicas, one process per GPU (a single child when `gpus` is 1); returns the last
    JSON line rank 0 printed."""
    if gpus == 1:
        return child_json(argv)
    from distributedmnist_b200.parallel.launcher import run_replicas
    with tempfile.TemporaryDirectory() as d:
        codes = run_replicas(argv, gpus, timeout=1800, out_dir=d)
        text = open(os.path.join(d, sorted(os.listdir(d))[0])).read()
    if codes != [0] * gpus:
        raise SystemExit("a replica failed: %s" % codes)
    return _last_json(text)


def emit(result, out_path) -> None:
    """Prints `result` as one JSON line and, given a path, writes that line to it."""
    line = json.dumps(result)
    print(line, flush=True)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


def _modes_worker(modes, steps, warmup, repeats):
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.schedule import LearningRateSchedule
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        FLAGS.parse([])
        ctx = init_context(FLAGS, want_gpu=True)
    else:
        torch.cuda.set_device(0)
        ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    n = ctx.world_size
    sched = LearningRateSchedule(0.01, 1000, 0.95)
    # one engine per mode, each with its own arenas and control block, so the modes can alternate without re-capturing
    configs = {}
    for mode, make in modes.items():
        eng = _engine(ctx, "lenet", 256, 0, lambda be: make(be, sched, n))
        configs[mode] = (eng, packed_batches(eng, 4, 1 + ctx.rank, on_device=False))
    us = alternate(configs, steps, warmup, repeats, before_block=lambda eng: eng.backend.device_barrier())
    for eng, _bufs in configs.values():
        torch.cuda.synchronize()
        eng.backend.check_error()
    return dict(replicas=n, us_per_step=us, launches_per_step={m: e.launches_per_step for m, (e, _b) in configs.items()})


def compare_modes(modes) -> None:
    """Main of a script that times LeNet steps at B = 256 under several aggregation modes on ``--gpus`` replicas, one
    process per replica, and prints rank 0's times.  `modes` maps a mode's name to ``make(backend, schedule, replicas)``,
    which builds the mode's optimizer."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        res = _modes_worker(modes, a.steps, a.warmup, a.repeats)
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps(res), flush=True)
        return
    res = replicas_json([os.path.abspath(sys.argv[0]), "--worker", "--steps", str(a.steps), "--warmup", str(a.warmup),
                         "--repeats", str(a.repeats)], a.gpus)
    out = dict(card(), model="lenet", batch=256, **res)
    out["median_us_per_step"] = {m: sorted(v)[len(v) // 2] for m, v in res["us_per_step"].items()}
    emit(out, a.out)
