"""Groth16 parameter generation and parameter-file writing on the device -- bb_groth16_generate (csrc/generate.cu) and
bb_params_write (csrc/decode.cu) -- executed on host threads (tests/native/) and compared with the host generator and
params_io.write_parameters.  The test bodies are those of test_gpu_generate.py at small sizes."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_generate as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_generate_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with verify.cu, decode.cu, r1cs.cu and generate.cu compiled in"""
    spec = importlib.util.spec_from_file_location("build_emu_generate", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "decode.cu", "r1cs.cu", "generate.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_generate")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_generate_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_generate_lib, None      # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_parity_small_circuits(worker):
    G.test_parity_small_circuits(worker)


def test_emulated_parity_xor_demo_oracle0(worker):
    G.test_parity_xor_demo_oracle0(worker)


def test_emulated_parity_mimc(worker):
    G.test_parity_mimc(worker, rounds=30)


def test_emulated_parity_random(worker):
    G.test_parity_random(worker, big=False)


def test_emulated_edge_toxic(worker):
    G.test_edge_toxic(worker)


def test_emulated_errors(worker):
    G.test_errors(worker)


def test_emulated_random_keys(worker):
    G.test_random_keys(worker, rounds=10)


def test_emulated_write(worker):
    G.test_write(worker, rounds=10)


def test_emulated_write_identity_h(worker):
    G.test_write_identity_h(worker)


def test_emulated_profile_stages(worker):
    G.test_profile_stages(worker)


DRY_RUN = """
import importlib.util, sys
sys.path.insert(0, ROOT)
import torch
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
spec = importlib.util.spec_from_file_location("bench_generate", ROOT + "/bench_generate.py")
bg = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bg)
sys.argv = ["bench_generate.py", "--log-size", "4", "--old-log-size", "4", "--oracle-log-size", "4", "--steps", "1"]
bg.main()
"""


def test_emulated_bench_generate_dry_run(tmp_path, emu_generate_lib):
    """bench_generate.py at 2^4 constraints on the emulated library: one JSON line, every check passing"""
    script = tmp_path / "dry_generate.py"
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_generate_lib!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "generate_ms" and d["config"]["log_size"] == 4
    assert {"seeded", "random", "write", "old", "oracle1", "gpu", "checks"} <= set(d)
    assert set(d["seeded"]["stages_ms"]) == {"generate.transpose", "generate.lagrange", "generate.qap", "generate.g1", "generate.g2"}
    assert set(d["write"]) == {"pinned", "hbm"}
    assert d["checks"] == {"proof": "equal", "verifies": "yes", "write_read": "equal"}
