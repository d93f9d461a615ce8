"""Tooling parity on CPU: Cfg interpolation, role templating/launch, log scraping, figures
(reference tools/tf_ec2.py:17-25,445-615 and tools/benchmark.py)."""
import os
import struct
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def test_cfg_self_interpolation():
    from cluster import Cfg
    c = Cfg({"name": "x", "nfs": "/mnt", "base_out_dir": "%(nfs)s/%(name)s", "n": 3,
             "cmds": ["rm -rf %(base_out_dir)s", 5]})
    assert c["base_out_dir"] == "/mnt/x"
    assert c["cmds"] == ["rm -rf /mnt/x", 5] and c["n"] == 3


def test_every_shipped_cfg_loads_and_templates():
    import glob

    from benchmark import load_cfg_from_file
    files = [f for f in glob.glob(os.path.join(ROOT, "cfg", "*", "*"))]
    assert len(files) >= 17
    for f in files:
        c = load_cfg_from_file(f)
        cmd = c["train_commands"][0]
        assert "--num_replicas_to_aggregate=%s" % c["num_replicas_to_aggregate"] in cmd
        assert "WORKER_HOSTS" in cmd and "ROLE_ID" in cmd and c["name"] in c["base_out_dir"]
    ks = sorted(int(load_cfg_from_file(f)["num_replicas_to_aggregate"])
                for f in files if f.endswith("_aggregate_sync"))
    assert ks == [1, 2, 4, 6, 7, 8]


def test_log_scrapers_and_stats(tmp_path):
    import benchmark as bm
    ev = tmp_path / "run_out_evaluator"
    ev.write_text("Succesfully loaded model from model.ckpt-10 at step=10.\n"
                  "Num examples: 10000  Precision @ 1: 0.912300 Loss: 0.301000 Time: 3.500000\n"
                  "Succesfully loaded model from model.ckpt-20 at step=20.\n"
                  "Num examples: 10000  Precision @ 1: 0.950000 Loss: 0.200000 Time: 5.000000\n")
    t, l, p, s = bm.extract_times_losses_precision(str(ev))
    assert (t, l, p, s) == ([3.5, 5.0], [0.301, 0.2], [0.9123, 0.95], [10, 20])
    ms = tmp_path / "run_out_master"
    ms.write_text("INFO:dmnist:Worker 0: 2026: step 7, loss = 1.0, train_acc = 0.5, test_acc = 0.0(1.0 examples/sec; 0.1  sec/batch)\n"
                  "INFO:dmnist:ELAPSED TIMES [(0.01, 0, 11), (0.02, 1, 11), (0.03, 0, 12), (0.05, 1, 12)]\n"
                  "INFO:dmnist:ITERATION TIMES [0.1, 0.2]\n")
    assert bm.current_iteration(str(ms)) == 7
    ct = bm.extract_compute_times(str(ms))
    assert ct[3] == (0.05, 1, 12) and bm.extract_iteration_times(str(ms)) == [0.1, 0.2]
    st = bm.worker_time_stats(ct)
    assert st["max"] == 0.05 and st["mean_iter_p100"] == pytest.approx(0.035)
    pngs = [bm.plot_time_loss(str(tmp_path), str(tmp_path)), bm.plot_time_cdfs(str(tmp_path), str(tmp_path))]
    for png in pngs:
        data = open(png, "rb").read()
        assert data[:8] == b"\x89PNG\r\n\x1a\n" and struct.unpack(">II", data[16:24]) == (800, 520)


def test_end_to_end_cpu_experiment(tmp_path):
    """benchmark -> cluster.run_tf -> 2 gloo workers + evaluator -> logs -> figures (SURVEY §3.4)."""
    import benchmark as bm
    cfg = bm.load_cfg_from_file(os.path.join(ROOT, "cfg", "cpu_plumbing", "2_workers_gloo_mlp2"))
    cfg["base_out_dir"] = str(tmp_path / "runs" / "%(name)s")
    cfg["max_steps"] = "40"
    out = str(tmp_path / "result_dir")
    figs = bm.plot_figs([cfg], n_iters=30, outdir=out, dest=str(tmp_path / "figs"))
    master = open(os.path.join(out, "2_workers_gloo_mlp2_out_master")).read()
    assert bm.current_iteration(os.path.join(out, "2_workers_gloo_mlp2_out_master")) >= 30, master[-2000:]
    evaluator = open(os.path.join(out, "2_workers_gloo_mlp2_out_evaluator")).read()
    t, l, p, s = bm.extract_times_losses_precision(os.path.join(out, "2_workers_gloo_mlp2_out_evaluator"))
    assert len(t) >= 1 and 0.0 <= p[-1] <= 1.0, evaluator[-2000:]
    assert all(os.path.getsize(f) > 500 for f in figs)
    assert os.path.exists(tmp_path / "runs" / "2_workers_gloo_mlp2" / "results.txt")


def test_ps_role_exits_cleanly():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=ps",
                        "--task_id=0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "no parameter server" in (r.stdout + r.stderr)


def test_no_undefined_names_in_gpu_only_code_paths():
    """The CUDA engine / bench / multi-GPU workers cannot execute on the CPU box: a static undefined-name check keeps a
    typo there from surfacing only inside a GPU run."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "lint_names.py")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]


def test_transfer_client_put_get_recursive(tmp_path):
    """tools/transfer.py: the one-box counterpart of the reference's vendored SCP client (tools/scp.py put :122 / get :158)."""
    from transfer import TransferClient, TransferError
    src = tmp_path / "run" / "train_dir"
    os.makedirs(src / "sub")
    (src / "checkpoint").write_text('model_checkpoint_path: "model.ckpt-7"\n')
    (src / "sub" / "out_master").write_bytes(b"x" * 300000)
    seen = []
    c = TransferClient(progress=lambda name, size, sent: seen.append((name, size, sent)), buff_size=1 << 16)
    c.get(str(src), str(tmp_path / "dl"), recursive=True)
    assert (tmp_path / "dl" / "checkpoint").read_text().startswith("model_checkpoint_path")
    assert (tmp_path / "dl" / "sub" / "out_master").stat().st_size == 300000
    assert seen and seen[-1][1] == seen[-1][2]                      # progress callback reaches 100 %
    c.put([str(src / "checkpoint")], str(tmp_path / "up.txt"))
    assert (tmp_path / "up.txt").exists()
    with pytest.raises(TransferError):
        c.get(str(src), str(tmp_path / "nope"))                     # directory without recursive=True
    with pytest.raises(TransferError):
        c.get(str(tmp_path / "missing"), str(tmp_path / "x"))


def test_benchmark_scrapers_match_the_reference_log_formats(tmp_path):
    import benchmark
    log = tmp_path / "out_master"
    log.write_text(
        "Worker 0: 2026-09-21 08:00:00.000000: step 7, loss = 2.301234, train_acc = 0.125000, test_acc = 0.000000(1234.5 examples/sec; 0.104  sec/batch)\n"
        "INFO ELAPSED TIMES [(0.011, 0, 10), (0.012, 1, 10), (0.031, 2, 10), (0.010, 0, 11)]\n"
        "INFO ITERATION TIMES [0.05, 0.06]\n"
        "Worker 0: 2026-09-21 08:00:01.000000: step 12, loss = 2.100000, train_acc = 0.250000, test_acc = 0.000000(1300.0 examples/sec; 0.098  sec/batch)\n")
    assert benchmark.current_iteration(str(log)) == 12
    ct = benchmark.extract_compute_times(str(log))
    assert len(ct) == 4 and ct[2] == (0.031, 2, 10)
    assert [w for _, w, _ in benchmark.extract_compute_times_no_master(str(log))] == [1, 2]
    assert benchmark.extract_iteration_times(str(log)) == [0.05, 0.06]
    stats = benchmark.worker_time_stats(ct)
    assert stats and abs(stats["max"] - 0.031) < 1e-9


def test_summary_writer_emits_a_tensorboard_event_file(tmp_path):
    """reference: tf.summary.FileWriter(eval_dir) + the two evaluator scalars (src/nn_eval.py:107-110,133-134).  The writer
    produces a real TFRecord/Event file (both CRC-32C checks verified by the reader) next to the JSON-lines mirror."""
    from distributedmnist_b200.utils.summary import SummaryWriter, crc32c, read_events, read_tfevents
    assert crc32c(b"123456789") == 0xE3069283                      # the CRC-32C check value
    w = SummaryWriter(str(tmp_path))
    w.add_scalars({"Validation Accuracy": 0.9871, "Validation Loss": 0.0421}, 301)
    w.add_scalars({"Validation Accuracy": 0.9912, "Validation Loss": 0.0307}, 602)
    w.close()
    assert os.path.basename(w.tfevents_path).startswith("events.out.tfevents.")
    ev = read_tfevents(w.tfevents_path)
    assert ev[0]["file_version"] == "brain.Event:2" and [e["step"] for e in ev] == [0, 301, 602]
    assert abs(ev[2]["scalars"]["Validation Accuracy"] - 0.9912) < 1e-6 and abs(ev[1]["scalars"]["Validation Loss"] - 0.0421) < 1e-6
    js = read_events(w.path)
    assert [e["step"] for e in js] == [301, 602] and js[0]["scalars"]["Validation Loss"] == 0.0421
    # a flipped payload byte must be detected
    raw = bytearray(open(w.tfevents_path, "rb").read())
    raw[-6] ^= 0x40
    bad = tmp_path / "corrupt"
    bad.write_bytes(bytes(raw))
    with pytest.raises(ValueError):
        read_tfevents(str(bad))


def test_shipped_cfg_matrix_is_what_the_generator_writes(tmp_path, monkeypatch):
    """cfg/** is generated (tools/make_cfgs.py); a hand edit of either side must not go unnoticed."""
    import filecmp
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_cfgs", os.path.join(ROOT, "tools", "make_cfgs.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    monkeypatch.setattr(mod, "ROOT", str(tmp_path))
    mod.main()
    generated = sorted(os.path.relpath(os.path.join(d, f), str(tmp_path)) for d, _s, fs in os.walk(str(tmp_path)) for f in fs)
    assert len(generated) >= 17
    for rel in generated:
        assert filecmp.cmp(os.path.join(str(tmp_path), rel), os.path.join(ROOT, rel), shallow=False), rel


def test_ptxas_report_parses_resource_lines(tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(ROOT, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    log = tmp_path / "k.log"
    log.write_text(
        "nvcc ...\n"
        "ptxas info    : Compiling entry function '_ZN2dm6kernelEv' for 'sm_90a'\n"
        "ptxas info    : Function properties for _ZN2dm6kernelEv\n"
        "    24 bytes stack frame, 44 bytes spill stores, 48 bytes spill loads\n"
        "ptxas info    : Used 128 registers, used 1 barriers, 16 bytes smem\n"
        "ptxas info    : Compiling entry function '_ZN2dm5otherEv' for 'sm_90a'\n"
        "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n"
        "ptxas info    : Used 40 registers\n")
    rows = mod.parse(str(log))
    assert [(r["regs"], r["smem"], r["stack"], r["spill_st"], r["spill_ld"], r["barriers"]) for r in rows] == \
        [(128, 16, 24, 44, 48, 1), (40, 0, 0, 0, 0, 0)]
    assert mod.demangle(["_ZN2dm6kernelEv"])[0].startswith("dm::kernel")
