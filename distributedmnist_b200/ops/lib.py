"""ctypes loader for the sm_90a kernel library.

The library is built in-tree by ``ops/build.py``.  On a box with a GPU a missing
or unloadable library is a hard error -- the CUDA path never silently falls back
to PyTorch ops.

Every entry point is declared once, in ``_SIGNATURES``: ctypes then converts and
checks each argument against the C declaration, and a launcher's nonzero return
raises :class:`KernelLibraryError`.  Callers pass tensors, ``None``, ints and
floats directly.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from . import build as _build

_lib: Optional[ctypes.CDLL] = None


class KernelLibraryError(RuntimeError):
    pass


class VoidPtr(ctypes.c_void_p):
    """``void*`` / ``const void*`` parameter: a tensor passes its ``data_ptr()``, ``None`` passes NULL, and an int address
    or anything ``c_void_p`` accepts (ctypes pointers, arrays, ``byref``) passes as it is."""

    @classmethod
    def from_param(cls, obj):
        if isinstance(obj, torch.Tensor):
            return ctypes.c_void_p(obj.data_ptr())
        return ctypes.c_void_p.from_param(obj)


STATUS, VALUE = True, False      # the return value: 0 or an error code (raised), or a result returned as it is


def _signatures() -> dict:
    """``name: (kind, restype, argtypes)`` of every entry point, in the order of the C declarations."""
    P = VoidPtr                                       # void*, const void*
    PP = ctypes.POINTER(ctypes.c_void_p)              # void* const* (peer tables), void**
    PULL = ctypes.POINTER(ctypes.c_ulonglong)         # unsigned long long*
    PI = ctypes.POINTER(ctypes.c_int)                 # int*
    i, u, ll, ull = ctypes.c_int, ctypes.c_uint, ctypes.c_longlong, ctypes.c_ulonglong
    f, d, s = ctypes.c_float, ctypes.c_double, ctypes.c_char_p
    S, V = STATUS, VALUE
    return {
        # augment.cu
        "dm_augment_affine": (S, i, [P, P, i, P, u, d, d, d, P, P]),
        # augment_elastic.cu
        "dm_augment_elastic": (S, i, [P, P, i, P, u, d, d, d, d, P, i, P, P, P]),
        # batch_gather.cu
        "dm_gather_batch": (S, i, [P, P, P, i, P, P]),
        # conv1_tc.cu, conv2_tc.cu
        "dm_conv1_fwd_tc": (S, i, [P, P, P, P, P, i, P, i, P, i, P, i, P]),
        "dm_conv1_wgrad_tc": (S, i, [P, P, P, P, P, i, P]),
        "dm_conv2_fwd": (S, i, [P, P, P, P, P, i, P]),
        "dm_conv2_dgrad": (S, i, [P, P, P, i, P]),
        "dm_conv2_wgrad": (S, i, [P, P, P, i, P]),
        # eval_best.cu
        "dm_best_state_bytes": (V, i, []),
        "dm_eval_best_decide": (S, i, [P, P, P, u, P, P, P]),
        "dm_eval_best_copy": (S, i, [P, P, P, ll, P]),
        # eval_head.cu
        "dm_eval_state_bytes": (V, i, []),
        "dm_eval_max_rows": (V, i, []),
        "dm_eval_stamp": (S, i, [P, P]),
        "dm_eval_head": (S, i, [P, ll, i, P, P, P, P, P, P, P, P, P, i, P, i, i, P]),
        # eval_patience.cu
        "dm_patience_state_bytes": (V, i, []),
        "dm_eval_patience": (S, i, [P, P, P, u, u, u, u, P, PP, i, i, P]),
        # eval_plateau.cu
        "dm_plateau_state_bytes": (V, i, []),
        "dm_eval_plateau": (S, i, [P, P, P, u, u, u, u, P, PP, i, P]),
        # eval_snapshot.cu
        "dm_snap_state_bytes": (V, i, []),
        "dm_snap_select": (S, i, [P, P, i, i, d, P]),
        "dm_snap_copy": (S, i, [P, P, P, P, ll, ll, ll, ll, ll, P]),
        "dm_snap_validate": (S, i, [P, P, i, i, P]),
        "dm_snap_keep": (S, i, [P, P, P, ll, P]),
        "dm_snap_test_emulate": (S, i, [P, P, ll, u, i, i, i, P]),
        "dm_snap_test_writer": (S, i, [P, P, ll, u, i, d, i, P, P]),
        # eval_target.cu
        "dm_tta_stamp": (S, i, [P, P]),
        "dm_eval_target": (S, i, [P, P, P, u, u, u, PP, i, i, P]),
        "dm_stop_publish": (S, i, [P, P, P]),
        # fused_async.cu
        "dm_async_stats_bytes": (V, i, []),
        "dm_async_begin": (S, i, [PP, i, P, P, P, ll, i, P]),
        "dm_async_end": (S, i, [PP, PP, P, P, i, i, ll, d, d, i, i, P, P]),
        "dm_ssp_stats_bytes": (V, i, []),
        "dm_ssp_wait": (S, i, [P, P, P, i, i, u, d, P]),
        "dm_ssp_publish": (S, i, [PP, P, i, i, i, P]),
        # fused_gossip.cu
        "dm_gossip_stats_bytes": (V, i, []),
        "dm_gossip_apply": (S, i, [PP, i, P, P, P, ll, d, d, i, i, P]),
        "dm_gossip_exchange": (S, i, [PP, PP, P, P, P, i, i, ll, d, i, P]),
        # fused_local.cu
        "dm_local_stats_bytes": (V, i, []),
        "dm_local_apply": (S, i, [PP, i, P, P, P, ll, u, d, d, i, i, P, P]),
        "dm_local_average": (S, i, [PP, PP, P, P, i, i, ll, u, i, d, i, P, P]),
        "dm_local_average_shard": (S, i, [P, PP, i, i, ll, u, i, P, P]),
        # fused_bucket.cu, fused_interval.cu
        "dm_bucket_sync": (S, i, [PP, PP, PP, PP, PP, i, i, i, ll, ll, ll, d, d, i, d, P, i, P, P, P, i, i]),
        "dm_interval_arm": (S, i, [P, d, P]),
        "dm_interval_begin": (S, i, [P, P, P, ll, P]),
        "dm_interval_end": (S, i, [PP, PP, PP, PP, i, i, ll, d, d, i, d, i, P, P]),
        "dm_kgtn_begin": (S, i, [P, i, P, P, ll, P]),
        "dm_kgtn_end": (S, i, [PP, PP, PP, PP, i, i, i, ll, d, d, i, d, i, P, P, P]),
        # fused_sync.cu
        "dm_sync_ctrl_bytes": (V, i, []),
        "dm_sync_ctrl_offset": (V, i, [s]),
        "dm_fused_sync_sgd": (S, i, [PP, PP, PP, i, i, i, ll, d, d, i, f, u, d, P, i, P, P, P]),
        "dm_fused_sync_bucket": (S, i, [PP, PP, PP, i, i, i, ll, ll, ll, ll, d, d, i, d, P, i, P, P, P]),
        "dm_sync_set_host_mirror": (S, i, [P, P]),
        "dm_sync_set_lr_cuts": (S, i, [P, P, d]),
        "dm_sync_set_lr_schedule": (S, i, [P, u, d, u, d]),
        "dm_f32_to_bf16": (S, i, [P, P, ll, P]),
        "dm_straggler_delay": (S, i, [P, f, u, u, P]),
        "dm_straggler_state_bytes": (V, i, []),
        "dm_straggler_sample": (S, i, [P, P, u, P]),
        "dm_device_barrier": (S, i, [PP, i, i, d, P]),
        "dm_stamp_arrive": (S, i, [P, P]),
        "dm_stamp_start": (S, i, [P, P]),
        # gemm_tc.cu
        "dm_gemm_bf16": (S, i, [P, P, P, i, i, i, i, i, i, i, i, i, i, i, ll, P, P]),
        "dm_gemm_decay_ctas": (V, i, [i, i]),
        "dm_gemm_bf16_decay": (S, i, [P, P, P, i, i, i, i, i, i, i, P, f, P, P]),
        "dm_fc1_dgrad_unpool": (S, i, [P, P, P, P, P, i, P]),
        # host_utils.cu
        "dm_version": (V, i, []),
        "dm_set_max_ctas": (V, i, [i]),
        "dm_get_max_ctas": (V, i, []),
        "dm_num_sms": (V, i, []),
        "dm_lenet_max_batch": (V, i, []),
        "dm_set_pdl": (V, i, [i]),
        "dm_device_cc": (V, i, [i]),
        # lenet_simt.cu, mlp_simt.cu, moving_average.cu
        "dm_fc2_fwd_bwd": (S, i, [P, ll, i, P, P, P, P, P, P, P, P, P, i, i, u, P, f, P]),
        "dm_fc2_wgrad": (S, i, [P, P, P, P, P, P, i, P]),
        "dm_fc2_wgrad_decay_ctas": (V, i, []),
        "dm_fc2_wgrad_decay": (S, i, [P, P, P, P, P, P, i, P, P, P, f, P, P]),
        "dm_dense10_xent": (S, i, [P, P, P, P, P, P, P, P, P, i, i, i, P]),
        "dm_relu_bwd_colsum": (S, i, [P, P, P, P, i, i, P]),
        "dm_moving_average": (S, i, [P, P, ll, P, d, P, P, ll, ll, ll, ll, P]),
        # litmus.cu
        "dm_litmus_mp": (S, i, [i, P, P, P, P, P, P, i, i, d, P]),
        # step_runner.cu
        "dm_runner_create": (V, ctypes.c_void_p, [P, P, P, P, P, P, ull, i]),
        "dm_runner_step": (V, i, [P, P]),
        "dm_runner_arm_gather": (S, i, [P, P, P, P, P, i]),
        "dm_runner_step_indices": (V, i, [P, P]),
        "dm_runner_wait": (S, i, [P, i]),
        "dm_runner_wait_copy": (S, i, [P, i]),
        "dm_runner_query": (V, i, [P, i]),
        "dm_runner_destroy": (V, None, [P]),
        # symm_mem.cu.  The VMM and multicast calls return their codes: VmmBuffer votes on them across the ranks.
        "dm_set_device": (S, i, [i]),
        "dm_symm_alloc": (S, i, [ull, PP]),
        "dm_symm_ipc_handle": (S, i, [P, P]),
        "dm_symm_ipc_open": (S, i, [P, PP]),
        "dm_symm_ipc_close": (V, i, [P]),
        "dm_memset_async": (S, i, [P, i, ull, P]),
        "dm_vmm_multicast_supported": (V, i, [i]),
        "dm_vmm_round_size": (V, ll, [ull, i, i]),
        "dm_vmm_create": (V, i, [ull, i, PULL, PI, PP]),
        "dm_vmm_import": (V, i, [i, PULL]),
        "dm_vmm_map": (V, i, [ull, ull, i, PP]),
        "dm_close_fd": (V, i, [i]),
        "dm_mc_create": (V, i, [ull, i, PULL, PI]),
        "dm_mc_add_device": (V, i, [ull, i]),
        "dm_mc_bind": (V, i, [ull, ull, ull]),
        # weight_decay.cu
        "dm_weight_decay_loss": (S, i, [P, i, f, P, P]),
    }


_SIGNATURES = _signatures()


def _raise_on_error(rc, func, args):
    if rc != 0:
        raise KernelLibraryError("%s failed with code %d" % (func.__name__, rc))
    return rc


def declare(fn, kind: bool, restype, argtypes):
    """Give the foreign function ``fn`` its C signature; a STATUS function raises on a nonzero return."""
    fn.restype, fn.argtypes = restype, argtypes
    if kind is STATUS:
        fn.errcheck = _raise_on_error
    return fn


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not os.path.exists(path):
        if not build_if_missing:
            raise KernelLibraryError("kernel library %s is missing; run `python -m distributedmnist_b200.ops.build`" % path)
        _build.build()
    try:
        lib = ctypes.CDLL(path)
    except OSError as e:
        raise KernelLibraryError("cannot load %s: %s" % (path, e))
    for name, sig in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise KernelLibraryError("kernel library %s has no %s: it is out of date, rebuild it with "
                                     "`python -m distributedmnist_b200.ops.build`" % (path, name)) from None
        declare(fn, *sig)
    _lib = lib
    return _lib


# For foreign functions called without a declared signature (the probe library, csrc/probes/): the caller builds the
# arguments and checks the return code itself.  Calls into the kernel library need neither.
def check(rc: int, what: str) -> None:
    if rc != 0:
        raise KernelLibraryError("%s failed with code %d" % (what, rc))


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream_ptr(stream: Optional[torch.cuda.Stream] = None) -> ctypes.c_void_p:
    s = torch.cuda.current_stream() if stream is None else stream
    return ctypes.c_void_p(s.cuda_stream)


def require_hopper(device: torch.device) -> None:
    """The library holds sm_90a code only (wgmma, TMA): it loads on nothing but a compute capability 9.0 device."""
    cc = load().dm_device_cc(device.index or 0)
    if cc != 90:
        raise KernelLibraryError("device %s has compute capability %d; this library is sm_90a-only" % (device, cc))
