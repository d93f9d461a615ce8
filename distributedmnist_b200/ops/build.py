"""In-tree build of the sm_90a kernel library (``distributedmnist_b200/lib/libdmnist_b200.so``).

``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` per ``csrc/*.cu`` (in
parallel), then one link.  No torch headers are involved: the library exposes a
plain C ABI that takes raw device pointers and a stream handle, and Python calls
it through ``ctypes`` -- so each translation unit compiles in seconds and the
``.so`` has no ABI coupling to the installed PyTorch.  The CUDA runtime is linked
statically and driver symbols are resolved at run time, so the library loads on a
CPU-only box too (build check) and travels to the GPU box with the snapshot.
"""
from __future__ import annotations

import hashlib
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from typing import List

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "csrc")
LIB_DIR = os.path.join(ROOT, "distributedmnist_b200", "lib")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(LIB_DIR, "libdmnist_b200.so")
STAMP = os.path.join(LIB_DIR, "libdmnist_b200.stamp")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
              "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def sources() -> List[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, f), "rb") as fh:
                h.update(f.encode() + b"\0" + fh.read())
    h.update(" ".join(ARCH_FLAGS + NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    try:
        with open(STAMP) as f:
            return os.path.exists(LIB_PATH) and f.read().strip() == _digest()
    except OSError:
        return False


_SERIALIZED_WGMMA = re.compile(r"\(C7511\).*wgmma\.mma_async instructions are serialized.*in the function '(\S+?)'")


def serialized_wgmma_kernels(ptxas_log: str) -> List[str]:
    """Kernels whose wgmmas ptxas serialized (warning C7511): it then waits for every wgmma to complete before the next
    is issued, which typically costs a wgmma kernel a large part of its tensor-core throughput."""
    return [m.group(1) for m in _SERIALIZED_WGMMA.finditer(ptxas_log)]


def _compile(src: str) -> str:
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
    cmd = [NVCC] + ARCH_FLAGS + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = obj[:-2] + ".log"
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (src, (r.stdout + r.stderr)[-6000:]))
    serialized = serialized_wgmma_kernels(r.stdout + r.stderr)
    if serialized:
        raise RuntimeError("ptxas serialized the wgmma pipeline (C7511) of %s in %s; see %s"
                           % (", ".join(serialized), src, log))
    return obj


def build(force: bool = False, verbose: bool = True) -> str:
    if not force and is_fresh():
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    srcs = sources()
    if verbose:
        print("[dmnist build] nvcc sm_90a: %d sources" % len(srcs), file=sys.stderr)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    cmd = [NVCC] + ARCH_FLAGS + ["-shared", "-o", LIB_PATH] + objs + ["-cudart", "static", "-lrt", "-lpthread", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s" % (r.stdout + r.stderr)[-4000:])
    with open(STAMP, "w") as f:
        f.write(_digest())
    if verbose:
        print("[dmnist build] wrote %s" % LIB_PATH, file=sys.stderr)
    return LIB_PATH


PROBE_DIR = os.path.join(CSRC, "probes")
PROBE_LIB_PATH = os.path.join(LIB_DIR, "libdmnist_probes.so")


def build_probes() -> str:
    """Bring-up probes (csrc/probes/*.cu: SM co-residency probe) as their OWN library --
    they are measurement tools, not part of the product ``libdmnist_b200.so``."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    srcs = sorted(os.path.join(PROBE_DIR, f) for f in os.listdir(PROBE_DIR) if f.endswith(".cu"))
    srcs.append(os.path.join(CSRC, "host_utils.cu"))
    cmd = [NVCC] + ARCH_FLAGS + [f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")] + ["-I", CSRC, "-shared", "-o", PROBE_LIB_PATH] \
        + srcs + ["-cudart", "static", "-lrt", "-lpthread", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("probe build failed:\n%s" % (r.stdout + r.stderr)[-4000:])
    return PROBE_LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    if "--probes" in sys.argv:
        print(build_probes())
