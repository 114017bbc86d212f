"""bench.py's reference arm (`--impl reference`) runs on host cores only, so its side of the
driver contract is checked here without a GPU: one JSON line on stdout with the agreed keys, and
under torchrun rank 0 alone prints while the other ranks exit 0 without work."""
import json
import os
import subprocess
import sys

from emulated import ROOT, bench_dry_run, dry_run_script

REQUIRED = {"impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
            "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"}


def _check_line(out, n_gpus):
    lines = [l for l in out.splitlines() if l.strip()]
    assert len(lines) == 1, out
    d = json.loads(lines[0])
    assert REQUIRED <= set(d), REQUIRED - set(d)
    assert d["impl"] == "reference" and d["n_gpus"] == n_gpus and d["steps"] == 2 and d["warmup"] == 1
    assert d["metric"] == "groth16_prove_constraints_per_sec" and d["unit"] == "constraints/s"
    assert d["higher_is_better"] is True and d["vs_baseline"] is None and d["value"] > 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "model" not in d["config"]


def test_reference_arm_single_process():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1",
                          "--log-size", "10"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    _check_line(res.stdout, 1)


def test_reference_arm_under_torchrun_world2():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "2",
           "--warmup", "1", "--log-size", "10"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    _check_line(res.stdout, 2)


ARGV = ["--log-size", "8", "--steps", "2", "--warmup", "1", "--cpu-sample-log", "8", "--autotune-reps", "1", "--autotune", "2"]


def test_own_arm_dry_run_on_the_emulated_device(tmp_path, emu_lib):
    """bench.py's default workload (prove: value leg, e2e leg, roofline, timeline, cpu_baseline) end
    to end with the CUDA library replaced by the host-fiber build of the same sources and torch.cuda
    stubbed: checks the script and the JSON contract, not the numbers."""
    d = bench_dry_run(emu_lib, tmp_path, "bench.py", ARGV)
    need = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline", "timeline"}
    assert need <= set(d), need - set(d)
    assert d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1 and d["gpu_launches"] > 100
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"]) and d["e2e"]["h2d_bytes_per_step"] > 0
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(d["roofline"])
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"]) and d["cpu_baseline"]["kind"] == "port"
    assert len(d["timeline"]["device_ms_since_prove_start"]) == 8
    assert d["roofline"]["pairs_per_step"] > 0 and d["roofline"]["bucket_entries_per_step"] > d["roofline"]["pairs_per_step"]
    assert "workload" in d["config"] and "model" not in d["config"]
    at = d["autotune"]                                  # the MSM form was measured before the warm-up; every form eligible here
    assert len(at["ms"]) == len(at["forms"]) >= 2 and all(t > 0 for t in at["ms"]) and at["ms"][at["chosen"]] == min(at["ms"])


def test_tuner_child_mode_and_parent_fallback(tmp_path, emu_lib):
    """bench.py's sandboxed tuner: (1) child mode (--tune-child) builds the key and witness, tunes and prints its report --
    run here on the emulated device; (2) a parent whose child cannot run (the real library finds no CUDA device in this
    container) records the error and measures the default form."""
    # (the unsharded tuner itself runs in the dry run above; here) the child of rank 1 of 2 -- the gate in front of the
    # collective tuner: that rank's key shard, no process group
    env = dict(os.environ, WORLD_SIZE="2", RANK="1", LOCAL_RANK="0")
    rep = bench_dry_run(emu_lib, tmp_path, "bench.py", ARGV + ["--tune-child", "--shard-index", "1", "--shard-count", "2"],
                        env=env)["tune_child"]
    assert all(t > 0 for t in rep["ms"]) and rep["name"]
    d = bench_dry_run(emu_lib, tmp_path, "bench.py", ARGV + ["--autotune", "1", "--no-cpu-baseline"])
    at = d["autotune"]
    assert at["error"] and at["chosen"] == 0 and at["where"] == "child process" and "tuner process failed" in d["config"]["msm_form"]
    assert d["value"] > 0 and d["gpu_launches"] > 100


def test_own_arm_dry_run_two_ranks(tmp_path, emu_lib):
    """bench.py --gpus 2 under torchrun with gloo and the emulated device: the sharded step, the max over ranks, the gate in
    front of the collective tuner (the per-rank tuner children cannot run here -- no CUDA device -- so both ranks must stay on
    the default form and say why), the sharded proof == single-GPU proof check, one JSON line from rank 0."""
    script = dry_run_script(emu_lib, tmp_path, "bench.py", ARGV + ["--gpus", "2", "--autotune", "1", "--no-cpu-baseline"])
    env = dict(os.environ, BB_BENCH_DIST_BACKEND="gloo")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip().startswith("{")]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["n_gpus"] == 2 and d["scaling"] == "strong" and d["value"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0
    assert "sharded proof == single-GPU proof" in d["proof_check"] and len(d["proof_sha256"]) == 64
    at = d["autotune"]
    assert at["chosen"] == 0 and at["error"] and "tuner process failed" in d["config"]["msm_form"]
    assert set(d["sharded_host_ms_per_step"]) >= {"queue_witness_msms", "all_gather"}


def test_msm_microbench_dry_run_on_the_emulated_device(tmp_path, emu_lib):
    """bench.py --workload msm (BASELINE configs[2] shape, here 2^10 points): both MSM forms are measured, the result
    is asserted against [sum k_i e_i]G inside the script"""
    d = bench_dry_run(emu_lib, tmp_path, "bench.py", ARGV + ["--workload", "msm", "--log-size", "10"])
    assert d["metric"] == "g1_msm_mpt_per_sec" and d["config"]["result_check"].endswith("equal")
    assert len(d["autotune"]["ms"]) == 2 and all(t > 0 for t in d["autotune"]["ms"])


def test_reference_arm_sizes_its_pool_to_the_cpu_quota(monkeypatch):
    """host_cpu_info(): threads = min(affinity, ceil(cgroup quota)) -- the 1-GPU lease of round 1 reported 128
    cores under a 16-CPU quota (cpu.max = "1600000 100000"), and a 128-thread pool ran 3x slower than 16."""
    import builtins
    import importlib.util
    import io
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    real_open = builtins.open

    def fake_open(path, *a, **k):
        if path == "/sys/fs/cgroup/cpu.max":
            return io.StringIO(fake_open.content)
        return real_open(path, *a, **k)

    monkeypatch.setattr(builtins, "open", fake_open)
    monkeypatch.setattr(os, "sched_getaffinity", lambda pid: set(range(128)), raising=False)
    monkeypatch.delenv("BB_ORACLE_THREADS", raising=False)
    fake_open.content = "1600000 100000\n"
    info = bench.host_cpu_info()
    assert info["threads"] == 16 and info["cgroup_quota_cpus"] == 16.0 and info["affinity"] == 128
    fake_open.content = "max 100000\n"
    assert bench.host_cpu_info()["threads"] == 128
    fake_open.content = "250000 100000\n"
    assert bench.host_cpu_info()["threads"] == 3
    monkeypatch.setenv("BB_ORACLE_THREADS", "5")
    assert bench.host_cpu_info()["threads"] == 5
