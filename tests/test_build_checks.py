"""The in-tree build refuses kernels whose wgmma pipeline ptxas serialized (warning C7511)."""
import pytest

from distributedmnist_b200.ops import build


def test_serialized_wgmma_warning_names_the_kernel():
    log = (
        "ptxas info    : (C7519) warpgroup.arrive is injected in around line 9395 by compiler to allow use of registers "
        "in GMMA in function '_ZN2dm18conv2_wgrad_kernelILi4EEEv14CUtensorMap_stS1_Pfii'\n"
        "ptxas info    : (C7511) Potential Performance Loss: wgmma.mma_async instructions are serialized due to "
        "insufficient register resources for the wgmma pipeline in the function "
        "'_ZN2dm18conv2_wgrad_kernelILi4EEEv14CUtensorMap_stS1_Pfii'\n"
        "ptxas info    : Compiling entry function '_ZN2dm16conv2_fwd_kernelE14CUtensorMap_stS0_PKfP13__nv_bfloat16Phi' "
        "for 'sm_90a'\n"
        "ptxas info    : Used 126 registers, used 2 barriers\n")
    assert build.serialized_wgmma_kernels(log) == ["_ZN2dm18conv2_wgrad_kernelILi4EEEv14CUtensorMap_stS1_Pfii"]


def test_clean_ptxas_log_passes():
    log = ("ptxas info    : Compiling entry function '_ZN2dm6kernelEv' for 'sm_90a'\n"
           "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
           "ptxas info    : Used 40 registers\n")
    assert build.serialized_wgmma_kernels(log) == []


def test_compile_fails_on_serialized_wgmma(tmp_path, monkeypatch):
    class Done:
        returncode = 0
        stdout = ""
        stderr = ("ptxas info    : (C7511) Potential Performance Loss: wgmma.mma_async instructions are serialized due "
                  "to insufficient register resources for the wgmma pipeline in the function '_ZN2dm1kEv'\n")

    monkeypatch.setattr(build, "OBJ_DIR", str(tmp_path))
    monkeypatch.setattr(build.subprocess, "run", lambda *a, **k: Done())
    with pytest.raises(RuntimeError, match=r"_ZN2dm1kEv"):
        build._compile(str(tmp_path / "k.cu"))
