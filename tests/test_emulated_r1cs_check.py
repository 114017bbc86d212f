"""Checking witnesses against the constraint system -- bb_r1cs_check and bb_r1cs_check_batch in csrc/r1cs.cu -- executed
on host threads (tests/native/) and compared with a Python-integer evaluation of every row.  The test bodies are those of
test_gpu_r1cs_check.py; the GPU file adds rows of more than 2048 terms and 2^20 constraints."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_r1cs_check as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_r1cs_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with r1cs.cu (and verify.cu, which it links against) compiled in"""
    spec = importlib.util.spec_from_file_location("build_emu_r1cs_check", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "r1cs.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_r1cs_check")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_r1cs_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_r1cs_lib, None        # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_check_xor_demo(worker):
    G.test_check_xor_demo(worker)


def test_emulated_check_zero_coeffs(worker):
    G.test_check_zero_coeffs(worker)


def test_emulated_check_mimc322_circuit(worker):
    G.test_check_mimc322_circuit(worker)


def test_emulated_check_mimc322_oracle(worker):
    G.test_check_mimc322_oracle(worker)


def test_emulated_check_random(worker):
    G.test_check_random(worker, big=False)


def test_emulated_check_batch(worker):
    G.test_check_batch(worker, lengths=(1, 40))


def test_emulated_check_errors(worker):
    G.test_check_errors(worker)


def test_emulated_check_mimc(worker):
    """the synthetic MiMC witness and its single corruptions at 2^6 constraints"""
    G.check_mimc(worker, 6)


DRY_RUN = """
import importlib.util, sys
sys.path.insert(0, ROOT)
import torch
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
spec = importlib.util.spec_from_file_location("bench_r1cs_check", ROOT + "/bench_r1cs_check.py")
br = importlib.util.module_from_spec(spec)
spec.loader.exec_module(br)
sys.argv = ["bench_r1cs_check.py", "--steps", "1", "--warmup", "1", "--log-size", "6", "--batch", "3"]
br.main()
"""


def test_emulated_bench_r1cs_check_dry_run(tmp_path, emu_r1cs_lib):
    """bench_r1cs_check.py at 2^6 constraints and a batch of 3 on the emulated library: one JSON line with the check's
    stages, the batch legs, the eval and prove references and the equality checks"""
    script = tmp_path / "dry_r1cs_check.py"
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_r1cs_lib!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "r1cs_check_ms" and d["config"]["constraints"] == 64 and d["value"] >= 0   # emulated events read 0 ms
    assert {"eval_ms", "compare_ms", "compare_bytes", "roofline", "batch_hbm", "batch_host", "r1cs_eval_ms", "prove_ms",
            "share_of_prove", "checks", "gpu"} <= set(d)
    assert d["compare_bytes"] == 3 * 64 * 32
    for leg in ("batch_hbm", "batch_host"):
        assert d[leg]["items"] == 3 and d[leg]["launches_per_item"] == 2
    assert d["checks"] == {"satisfied": "equal", "corrupted": "equal", "batch": "equal"}
