"""Parameters::read / VerifyingKey::read on the device -- bb_params_read and bb_vk_read, csrc/decode.cu -- executed on
host threads (tests/native/) and compared with params_io.read_parameters and with the restatement of the reference's
reader.  The test bodies are those of test_gpu_params_read.py at small sizes."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_params_read as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_params_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with verify.cu, decode.cu and r1cs.cu compiled in"""
    spec = importlib.util.spec_from_file_location("build_emu_params", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "decode.cu", "r1cs.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_params")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_params_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_params_lib, None        # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_round_trip_small_keys(worker):
    G.test_round_trip_small_keys(worker)


def test_emulated_round_trip_mimc_and_generated(worker):
    G.test_round_trip_mimc_and_generated(worker, rounds=30)


def test_emulated_proofs(worker):
    G.test_proofs(worker, rounds=30)


def test_emulated_every_rejection_class(worker):
    G.test_every_rejection_class(worker)


def test_emulated_precedence(worker):
    G.test_precedence(worker)


def test_emulated_argument_errors(worker):
    G.test_argument_errors(worker)


def test_emulated_profile_and_bytes(worker):
    G.test_profile_and_bytes(worker)


DRY_RUN = """
import importlib.util, sys
sys.path.insert(0, ROOT)
import torch
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
spec = importlib.util.spec_from_file_location("bench_params_read", ROOT + "/bench_params_read.py")
bp = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bp)
sys.argv = ["bench_params_read.py", "--steps", "1", "--warmup", "0", "--log-size", "4"]
bp.main()
"""


def test_emulated_bench_params_read_dry_run(tmp_path, emu_params_lib):
    """bench_params_read.py at 2^4 constraints on the emulated library: one JSON line, both modes and both sources, old and
    new path, and every check passing"""
    script = tmp_path / "dry_params_read.py"
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_params_lib!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "params_read_ms" and d["config"]["log_size"] == 4 and d["config"]["file_bytes"] > 0
    for mode in ("checked", "unchecked"):
        m = d[mode]
        assert {"pinned", "hbm", "old", "stages_ms"} <= set(m)
        for leg in ("pinned", "hbm", "old"):
            assert set(m[leg]) == {"ms", "gb_per_s"} and m[leg]["ms"] >= 0
        assert set(m["stages_ms"]) == {"params.upload", "params.g1", "params.g2"}
    assert d["checks"] == {"vectors": "equal", "proofs": "equal", "corrupt_b_g2_middle": "reported"}
    assert {"name", "power_limit_w", "sm_max_mhz", "sm_mhz"} <= set(d["gpu"])
