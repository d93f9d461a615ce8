"""The ctypes declarations of the kernel library (ops/lib.py) against its C definitions, and what the binding does with
the arguments and return codes -- all without a GPU."""
import ctypes
import glob
import os
import re
import shutil
import subprocess

import pytest
import torch

from distributedmnist_b200.ops import build
from distributedmnist_b200.ops import lib as L

# C parameter / return type -> the ctypes type the table must declare for it
_PARAM = {
    "void*": L.VoidPtr, "const void*": L.VoidPtr,
    "void* const*": ctypes.POINTER(ctypes.c_void_p), "void**": ctypes.POINTER(ctypes.c_void_p),
    "unsigned long long*": ctypes.POINTER(ctypes.c_ulonglong), "int*": ctypes.POINTER(ctypes.c_int),
    "const char*": ctypes.c_char_p,
    "int": ctypes.c_int, "unsigned int": ctypes.c_uint, "long long": ctypes.c_longlong,
    "unsigned long long": ctypes.c_ulonglong, "float": ctypes.c_float, "double": ctypes.c_double,
}
_RETURN = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "void*": ctypes.c_void_p, "void": None}

_DEFINITION = re.compile(r'^(?:extern\s+"C"\s+)?([A-Za-z_][\w \t*]*?)\s*\b(dm_\w+)\s*\(([^)]*)\)\s*\{', re.M)


def _c_type(decl: str) -> str:
    """``const void* src`` -> ``const void*`` (the parameter name dropped, spacing normalised)."""
    t = re.sub(r"\s*\b\w+$", "", decl.strip())
    return re.sub(r"\s*\*", "*", re.sub(r"\s+", " ", t))


def _c_definitions() -> dict:
    """``name: (return type, [parameter types])`` of every top-level ``dm_*`` function defined in csrc/*.cu."""
    out = {}
    for path in sorted(glob.glob(os.path.join(build.CSRC, "*.cu"))):
        with open(path) as f:
            src = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S))
        for m in _DEFINITION.finditer(src):
            params = [p for p in m.group(3).split(",") if p.strip() not in ("", "void")]
            assert m.group(2) not in out, "%s defined twice" % m.group(2)
            out[m.group(2)] = (_c_type(m.group(1) + " x"), [_c_type(p) for p in params])
    return out


def test_table_declares_exactly_the_c_entry_points():
    defs = _c_definitions()
    assert len(defs) > 50
    assert sorted(L._SIGNATURES) == sorted(defs)
    for name, (ret, params) in defs.items():
        _kind, restype, argtypes = L._SIGNATURES[name]
        assert restype is _RETURN[ret], name
        assert argtypes == [_PARAM[p] for p in params], name


def _stub(name, result=0):
    """A C-callable stand-in for entry point ``name`` with the table's signature: records the arguments the C side
    receives and returns ``result``."""
    kind, restype, argtypes = L._SIGNATURES[name]
    seen = []

    def body(*args):
        seen.append([getattr(a, "value", a) for a in args])     # VoidPtr arrives as an instance, scalars as ints / floats
        return result

    fn = ctypes.CFUNCTYPE(restype, *argtypes)(body)
    fn.__name__ = name
    return L.declare(fn, kind, restype, argtypes), seen


def test_tensor_passes_its_address_and_none_passes_null():
    fn, seen = _stub("dm_eval_best_copy")
    src, dst = torch.arange(8, dtype=torch.float32), torch.zeros(8)
    fn(None, src, dst, dst.numel(), ctypes.c_void_p(0x1230))
    assert seen == [[None, src.data_ptr(), dst.data_ptr(), 8, 0x1230]]
    fn(0x40, ctypes.byref(ctypes.c_int()), ctypes.create_string_buffer(16), 1, None)    # int addresses and ctypes objects
    assert seen[-1][0] == 0x40 and seen[-1][1] and seen[-1][2]


def test_scalars_keep_their_c_type():
    fn, seen = _stub("dm_fused_sync_sgd")
    table = (ctypes.c_void_p * 2)(1, 2)
    fn(table, table, table, 0, 2, 2, 2 ** 40, 0.01, 0.95, 1000, 0.5, 2 ** 32 - 1, 30000, None, 132, None, None, None)
    args = seen[-1]
    assert args[6] == 2 ** 40                                        # long long: no 32-bit truncation
    assert args[7] == 0.01 and args[12] == 30000.0                   # double, also from an int
    assert args[10] == 0.5 and args[11] == 2 ** 32 - 1               # float, unsigned int


def test_mistyped_arguments_are_refused_at_the_call():
    fn, seen = _stub("dm_eval_best_copy")
    t = torch.zeros(4)
    with pytest.raises(ctypes.ArgumentError):
        fn(t, t, t, 4.0, None)                                       # float in a long long slot
    with pytest.raises(ctypes.ArgumentError):
        fn(t, t, t, t, None)                                         # tensor in a scalar slot
    with pytest.raises(ctypes.ArgumentError):
        _stub("dm_conv2_dgrad")[0](t, t, t, 2.0, None)               # float in an int slot
    with pytest.raises(ctypes.ArgumentError):
        fn(1.5, t, t, 4, None)                                       # float in a pointer slot
    with pytest.raises(TypeError):
        fn(t, t, t, 4)                                               # an argument short
    assert seen == []


def test_status_entry_raises_and_value_entry_returns():
    fn, _ = _stub("dm_conv2_dgrad", result=-3)
    with pytest.raises(L.KernelLibraryError, match=r"^dm_conv2_dgrad failed with code -3$"):
        fn(None, None, None, 1, None)
    ok, _ = _stub("dm_conv2_dgrad", result=0)
    assert ok(None, None, None, 1, None) == 0
    for name in ("dm_runner_step", "dm_vmm_map"):
        fn, _ = _stub(name, result=-3)
        args = [None, None] if name == "dm_runner_step" else [1, 2, 0, None]
        assert fn(*args) == -3


def test_vmm_and_multicast_entries_never_raise():
    """VmmBuffer votes on these codes across the ranks: a local exception would leave the other ranks in the vote."""
    for name in ("dm_vmm_round_size", "dm_vmm_create", "dm_vmm_import", "dm_vmm_map", "dm_vmm_multicast_supported",
                 "dm_mc_create", "dm_mc_add_device", "dm_mc_bind", "dm_close_fd"):
        assert L._SIGNATURES[name][0] is L.VALUE, name


_built = pytest.mark.skipif(not os.path.exists(build.LIB_PATH), reason="kernel library not built")


@_built
def test_load_binds_every_entry():
    lib = L.load(build_if_missing=False)
    for name, (kind, restype, argtypes) in L._SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and fn.argtypes == argtypes, name
        assert (fn.errcheck is not None) == (kind is L.STATUS), name


@_built
def test_library_exports_nothing_undeclared():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    out = subprocess.run([nm, "-D", "--defined-only", build.LIB_PATH], check=True, capture_output=True, text=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if ln.split() and ln.split()[-1].startswith("dm_")}
    assert exported == set(L._SIGNATURES)


@_built
def test_missing_symbol_names_it_and_asks_for_a_rebuild(monkeypatch):
    monkeypatch.setattr(L, "_lib", None)
    monkeypatch.setitem(L._SIGNATURES, "dm_not_in_the_library", (L.STATUS, ctypes.c_int, []))
    with pytest.raises(L.KernelLibraryError, match=r"dm_not_in_the_library.*rebuild"):
        L.load(build_if_missing=False)
    assert L._lib is None
