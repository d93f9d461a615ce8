"""Symmetric memory: identical buffers on every rank, each mapped into every peer.

Three allocators, same interface (``local_ptr``, ``peer_ptrs``, ``multicast_ptr``, ``view``, ``ptr_table``):

* :class:`VmmBuffer` -- the product path on NVSwitch systems: CUDA virtual-memory-management allocations bound to an
  **NVLS multicast object**, set up by the kernel library itself (``csrc/symm_mem.cu``: ``cuMemCreate`` /
  ``cuMulticastCreate`` / ``cuMulticastBindMem``); POSIX file descriptors are passed between the processes over AF_UNIX
  sockets (``SCM_RIGHTS``) by :class:`_FdChannel`.  Besides the peer addresses it yields ``multicast_ptr``: one virtual
  address whose loads are reduced *inside the switch* (``multimem.ld_reduce``) and whose stores are replicated to every
  rank (``multimem.st``) -- what the aggregation kernels use when every replica contributes (SURVEY §5.8).
* :class:`MulticastBuffer` -- the same memory model obtained through ``torch.distributed._symmetric_memory``
  (fallback / A-B reference, ``DMNIST_SYMM=torch``).
* :class:`SymmetricBuffer` -- ``cudaMalloc`` + CUDA IPC, handles exchanged over the process group.  Always available;
  peer (P2P) addresses only.  The control block always lives here.

All are exposed as ordinary ``torch`` tensors (zero-copy) plus the table of peer device pointers the kernels take.
"""
from __future__ import annotations

import ctypes
import os
import socket
import struct
import sys
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from ..ops.lib import load

_TYPESTR = {torch.float32: "<f4", torch.uint8: "|u1", torch.int32: "<i4", torch.bfloat16: None, torch.int64: "<i8",
            torch.uint16: "<u2"}


class _CudaArray:
    """Minimal ``__cuda_array_interface__`` carrier."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}
        self._owner = owner


class SymmetricBuffer:
    """One symmetric allocation of ``nbytes`` (zero-initialised) on every rank."""

    def __init__(self, nbytes: int, rank: int, world_size: int, device: torch.device, group=None):
        self.lib = load()
        self.nbytes = (nbytes + 255) // 256 * 256
        self.rank, self.world_size, self.device = rank, world_size, device
        p = ctypes.c_void_p()
        self.lib.dm_symm_alloc(self.nbytes, ctypes.byref(p))
        self.local_ptr = int(p.value)
        self.peer_ptrs: List[int] = [0] * world_size
        self.peer_ptrs[rank] = self.local_ptr
        self._opened: List[int] = []
        if world_size > 1:
            h = ctypes.create_string_buffer(64)
            self.lib.dm_symm_ipc_handle(ctypes.c_void_p(self.local_ptr), h)
            handles: List[Optional[bytes]] = [None] * world_size
            dist.all_gather_object(handles, bytes(h.raw), group=group)
            for r, hb in enumerate(handles):
                if r == rank:
                    continue
                q = ctypes.c_void_p()
                self.lib.dm_symm_ipc_open(ctypes.create_string_buffer(hb, 64), ctypes.byref(q))
                self.peer_ptrs[r] = int(q.value)
                self._opened.append(int(q.value))
        self.multicast_ptr = 0
        self._bytes = torch.as_tensor(_CudaArray(self.local_ptr, self.nbytes, self), device=device)

    def view(self, dtype: torch.dtype, offset_bytes: int = 0, numel: Optional[int] = None) -> torch.Tensor:
        item = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - offset_bytes) // item
        return self._bytes[offset_bytes:offset_bytes + numel * item].view(dtype)

    def ptr_table(self, offset_bytes: int = 0):
        """``(c_void_p * world)`` of peer addresses (index = rank) for the kernel launchers."""
        arr = (ctypes.c_void_p * self.world_size)()
        for r, p in enumerate(self.peer_ptrs):
            arr[r] = p + offset_bytes
        return arr

    def close(self) -> None:
        for p in self._opened:
            self.lib.dm_symm_ipc_close(ctypes.c_void_p(p))
        self._opened = []


class MulticastBuffer:
    """Symmetric allocation with an NVLS multicast mapping (``multicast_ptr`` is 0 when the fabric has none)."""

    def __init__(self, nbytes: int, rank: int, world_size: int, device: torch.device, group=None):
        import warnings

        import torch.distributed._symmetric_memory as tsm
        self.nbytes = (nbytes + 255) // 256 * 256
        self.rank, self.world_size, self.device = rank, world_size, device
        group = group if group is not None else dist.group.WORLD
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                tsm.enable_symm_mem_for_group(group.group_name)       # no-op on current PyTorch
            except Exception:  # noqa: BLE001
                pass
        self._t = tsm.empty(self.nbytes, dtype=torch.uint8, device=device)
        self._t.zero_()
        torch.cuda.synchronize(device)
        self._hdl = tsm.rendezvous(self._t, group)
        self.local_ptr = int(self._t.data_ptr())
        self.peer_ptrs: List[int] = [int(p) for p in self._hdl.buffer_ptrs]
        assert self.peer_ptrs[rank] == self.local_ptr, "symmetric memory: local pointer mismatch"
        mc = int(getattr(self._hdl, "multicast_ptr", 0) or 0)
        self.multicast_ptr = mc
        self._bytes = self._t

    view = SymmetricBuffer.view
    ptr_table = SymmetricBuffer.ptr_table

    def close(self) -> None:
        self._hdl = None


class _FdChannel:
    """Pass POSIX file descriptors between the ranks of one box: one AF_UNIX datagram socket per process (abstract
    namespace, so nothing touches the file system), ``SCM_RIGHTS`` ancillary data.  Messages carry (tag, sender) so
    exchanges belonging to different buffers cannot be confused."""

    _instance: Optional["_FdChannel"] = None

    def __init__(self, rank: int, world_size: int, group=None):
        self.rank, self.world = rank, world_size
        tokens: List[Optional[int]] = [None] * world_size
        dist.all_gather_object(tokens, os.getpid(), group=group)
        self._base = "dmnist-fd-%d" % tokens[0]
        self.sock = socket.socket(socket.AF_UNIX, socket.SOCK_DGRAM)
        self.sock.bind(self._addr(rank))
        self.sock.settimeout(60.0)
        self._pending: Dict[Tuple[int, int], int] = {}
        self._tag = 0
        dist.barrier(group=group)                 # every socket is bound before anybody sends

    @classmethod
    def get(cls, rank: int, world_size: int) -> "_FdChannel":
        if cls._instance is None or cls._instance.world != world_size:
            cls._instance = cls(rank, world_size)
        return cls._instance

    def _addr(self, r: int) -> str:
        return "\0%s-%d" % (self._base, r)

    def next_tag(self) -> int:
        self._tag += 1
        return self._tag

    def send(self, fd: int, to: int, tag: int) -> None:
        # (socket.send_fds() drops its `address` argument in CPython <= 3.12, so the ancillary message is built here)
        import array
        self.sock.sendmsg([struct.pack("ii", tag, self.rank)],
                          [(socket.SOL_SOCKET, socket.SCM_RIGHTS, array.array("i", [fd]))], 0, self._addr(to))

    def recv(self, frm: int, tag: int) -> int:
        while (tag, frm) not in self._pending:
            data, fds, _flags, _addr = socket.recv_fds(self.sock, 16, 4)
            t, r = struct.unpack("ii", data[:8])
            self._pending[(t, r)] = fds[0]
        return self._pending.pop((tag, frm))

    def all_to_all(self, fd: int) -> List[int]:
        """Every rank contributes one fd; returns the N fds indexed by rank (own entry = ``fd``)."""
        tag = self.next_tag()
        for r in range(self.world):
            if r != self.rank:
                self.send(fd, r, tag)
        return [fd if r == self.rank else self.recv(r, tag) for r in range(self.world)]

    def broadcast(self, fd: Optional[int], src: int = 0) -> int:
        tag = self.next_tag()
        if self.rank == src:
            for r in range(self.world):
                if r != src:
                    self.send(fd, r, tag)
            return fd
        return self.recv(src, tag)


def _all_ok(ok: bool, group=None) -> bool:
    """Collective AND: every rank takes the same branch after a step that may fail locally."""
    flags: List[Optional[bool]] = [None] * dist.get_world_size(group)
    dist.all_gather_object(flags, bool(ok), group=group)
    return all(flags)


class VmmBuffer:
    """Symmetric allocation from the kernel library's own VMM + NVLS multicast set-up (``csrc/symm_mem.cu``)."""

    def __init__(self, nbytes: int, rank: int, world_size: int, device: torch.device, want_multicast: bool = True, group=None):
        self.lib = load()
        lib, dev = self.lib, device.index or 0
        self.rank, self.world_size, self.device = rank, world_size, device
        size = int(lib.dm_vmm_round_size(ctypes.c_ulonglong(max(nbytes, 256)), dev, world_size))
        if not _all_ok(size > 0, group):
            raise RuntimeError("VMM allocation granularity query failed (rc %d)" % size)
        self.nbytes = self._alloc_bytes = size
        chan = _FdChannel.get(rank, world_size)
        h, fd, p = ctypes.c_ulonglong(), ctypes.c_int(-1), ctypes.c_void_p()
        rc = lib.dm_vmm_create(ctypes.c_ulonglong(size), dev, ctypes.byref(h), ctypes.byref(fd), ctypes.byref(p))
        if not _all_ok(rc == 0, group):
            raise RuntimeError("dm_vmm_create failed (rc %d)" % rc)
        self._handle, self.local_ptr = int(h.value), int(p.value)
        fds = chan.all_to_all(int(fd.value))
        self.peer_ptrs: List[int] = [0] * world_size
        self._mapped: List[int] = []
        self._handles: List[int] = []
        ok = True
        for r, f in enumerate(fds):
            if r == rank:
                self.peer_ptrs[r] = self.local_ptr
                continue
            hr, pr = ctypes.c_ulonglong(), ctypes.c_void_p()
            rc = lib.dm_vmm_import(int(f), ctypes.byref(hr))
            if rc == 0:
                rc = lib.dm_vmm_map(hr, ctypes.c_ulonglong(size), dev, ctypes.byref(pr))
            lib.dm_close_fd(int(f))
            if rc != 0:
                ok = False
                continue
            self._handles.append(int(hr.value))
            self._mapped.append(int(pr.value))
            self.peer_ptrs[r] = int(pr.value)
        if not _all_ok(ok, group):
            raise RuntimeError("mapping the peers' VMM allocations failed")
        # ---- NVLS multicast object over the N physical allocations --------------------------------------------
        self.multicast_ptr = 0
        self._mc_handle = 0
        mc_ok = want_multicast and world_size > 1 and int(lib.dm_vmm_multicast_supported(dev)) == 1
        if _all_ok(mc_ok, group):
            mch, mcfd = ctypes.c_ulonglong(), ctypes.c_int(-1)
            rc = 0
            if rank == 0:
                rc = lib.dm_mc_create(ctypes.c_ulonglong(size), world_size, ctypes.byref(mch), ctypes.byref(mcfd))
            if _all_ok(rc == 0, group):
                f = chan.broadcast(int(mcfd.value) if rank == 0 else None, 0)
                if rank != 0:
                    rc = lib.dm_vmm_import(int(f), ctypes.byref(mch))
                    lib.dm_close_fd(int(f))
                if rc == 0:
                    rc = lib.dm_mc_add_device(mch, dev)
                if _all_ok(rc == 0, group):                    # (collective: every device is added before anyone binds)
                    rc = lib.dm_mc_bind(mch, ctypes.c_ulonglong(self._handle), ctypes.c_ulonglong(size))
                    if _all_ok(rc == 0, group):
                        mp = ctypes.c_void_p()
                        rc = lib.dm_vmm_map(mch, ctypes.c_ulonglong(size), dev, ctypes.byref(mp))
                        if _all_ok(rc == 0, group):
                            self.multicast_ptr, self._mc_handle = int(mp.value), int(mch.value)
                if rank == 0 and int(mcfd.value) >= 0:
                    lib.dm_close_fd(int(mcfd.value))
        lib.dm_close_fd(int(fd.value))
        self._bytes = torch.as_tensor(_CudaArray(self.local_ptr, self.nbytes, self), device=device)

    def close(self) -> None:
        pass     # mappings live until process exit (the driver reclaims VMM ranges; unmapping under live tensors is unsafe)


VmmBuffer.view = SymmetricBuffer.view
VmmBuffer.ptr_table = SymmetricBuffer.ptr_table


def allocate_symmetric(nbytes: int, rank: int, world_size: int, device: torch.device, want_multicast: bool):
    """Arena allocator used by the fused backend: NVLS-capable when asked for and available, IPC otherwise.

    ``DMNIST_SYMM`` = ``own`` (default: csrc/symm_mem.cu VMM + multicast) | ``torch`` (torch's symmetric memory) | ``ipc``."""
    mode = os.environ.get("DMNIST_SYMM", "own")
    if want_multicast and world_size > 1 and mode != "ipc":
        if mode == "own":
            try:
                return VmmBuffer(nbytes, rank, world_size, device)
            except Exception as e:  # noqa: BLE001
                print("[dmnist] own VMM/NVLS allocator unavailable (%s: %s); trying torch symmetric memory"
                      % (type(e).__name__, str(e).splitlines()[0][:200]), file=sys.stderr)
        try:
            return MulticastBuffer(nbytes, rank, world_size, device)
        except Exception as e:  # noqa: BLE001 -- no NVSwitch / VMM: P2P still works
            print("[dmnist] multicast symmetric memory unavailable (%s: %s); using CUDA-IPC peer mappings"
                  % (type(e).__name__, str(e).splitlines()[0][:200]), file=sys.stderr)
    return SymmetricBuffer(nbytes, rank, world_size, device)
