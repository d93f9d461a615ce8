"""The GPU measurement scripts under tools/ and their shared harness, tools/gpu_timing.py, on the CPU: every script that
uses the harness imports and parses its arguments, the card query lives in the harness alone, and it degrades to "?"
without nvidia-smi."""
import glob
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _tools():
    return sorted(glob.glob(os.path.join(ROOT, "tools", "*.py")))


def test_every_harness_script_imports_and_parses_help(tmp_path):
    """A broken import or argument parser in a script shows here, not in a GPU run."""
    scripts = [p for p in _tools() if "\nimport gpu_timing\n" in open(p).read()]
    assert len(scripts) >= 19
    procs = {p: subprocess.Popen([sys.executable, p, "--help"], cwd=tmp_path, stdout=subprocess.PIPE,
                                 stderr=subprocess.STDOUT, text=True) for p in scripts}
    failed = {}
    for p, proc in procs.items():
        out = proc.communicate(timeout=300)[0]
        if proc.returncode != 0 or "usage:" not in out:
            failed[os.path.basename(p)] = out[-2000:]
    assert not failed, failed


def test_only_the_harness_queries_the_card():
    for p in _tools():
        if os.path.basename(p) == "gpu_timing.py":
            continue
        src = open(p).read()
        assert "nvidia-smi" not in src and "def gpu_info" not in src, p


def test_card_without_nvidia_smi(monkeypatch, tmp_path):
    import gpu_timing
    monkeypatch.setenv("PATH", str(tmp_path))
    assert gpu_timing.card() == {"gpu": "?", "power_limit": "?", "max_sm_clock": "?"}
