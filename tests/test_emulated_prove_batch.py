"""The batch prover -- bb_groth16_prove_batch and bb_groth16_prove_r1cs_batch -- executed on host threads (tests/native/)
and compared item by item with create_proof.  The test bodies are those of test_gpu_prove_batch.py at the sizes a host
reaches; the GPU file adds 2^17 and 2^20 constraints."""
import importlib.util
import os

import pytest

import bellman_b200 as bb

import test_gpu_prove_batch as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_batch_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with r1cs.cu and verify.cu compiled in"""
    spec = importlib.util.spec_from_file_location("build_emu_batch", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "r1cs.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_batch")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_batch_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_batch_lib, None        # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_bytes_mimc(worker):
    G.test_bytes_mimc322(worker, rounds=30, sizes=(1, 2, 5, 9))


def test_emulated_bytes_xor_demo(worker):
    G.test_bytes_xor_demo(worker)


def test_emulated_generated_key_verifies(worker):
    G.test_generated_key_verifies(worker, rounds=10, count=3)


def test_emulated_status_per_item(worker):
    G.test_status_per_item(worker, rounds=20)


def test_emulated_argument_errors(worker):
    G.test_argument_errors(worker)


def test_emulated_r1cs_batch(worker):
    G.test_r1cs_batch(worker, rounds=30, count=4)


DRY_RUN = """
import importlib.util, sys
sys.path.insert(0, ROOT)
import torch
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
spec = importlib.util.spec_from_file_location("bench_prove_batch", ROOT + "/bench_prove_batch.py")
bp = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bp)
sys.argv = ["bench_prove_batch.py", "--steps", "1", "--warmup", "1", "--log-size", "6", "--batch", "3"]
bp.main()
"""


def test_emulated_bench_prove_batch_dry_run(tmp_path, emu_batch_lib):
    """bench_prove_batch.py at 2^6 constraints on the emulated library: one JSON line with the three legs, launches per
    proof, the host tail, the sub-batches and the equality check"""
    import json
    import subprocess
    import sys
    script = tmp_path / "dry_prove_batch.py"
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_batch_lib!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "prove_batch_proofs_per_s" and d["config"]["constraints"] == 64 and d["config"]["batch"] == 3
    assert {"batch_hbm", "batch_host", "loop_hbm", "launches_per_proof", "host_tail_ms", "sub_batches", "checks", "gpu"} <= set(d)
    for leg in ("batch_hbm", "batch_host", "loop_hbm"):
        assert set(d[leg]) == {"ms_per_batch", "proofs_per_s"}
    assert d["checks"] == {"proofs": "equal"} and d["sub_batches"] == 1
    assert d["launches_per_proof"]["batch"] < d["launches_per_proof"]["loop"]
    assert {"name", "power_limit_w", "sm_max_mhz", "sm_mhz"} <= set(d["gpu"])
