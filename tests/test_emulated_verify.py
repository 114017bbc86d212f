"""Groth16 verification -- the pairing tower, the Miller loop, the final exponentiation and the batch verifier of
csrc/verify.cu -- executed on host threads (tests/native/) and compared with the oracle's Python pairing and
verifier.  The test bodies are those of test_gpu_verify.py at the same sizes; the GPU file adds the sizes only a
device reaches."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_verify as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_verify_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with verify.cu compiled in beside its sources"""
    spec = importlib.util.spec_from_file_location("build_emu_verify", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu",) if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_verify")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_verify_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_verify_lib, None      # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_tower_operations(worker):
    G.test_tower_operations(worker)


def test_emulated_gt_convention(worker):
    G.test_gt_convention(worker)


def test_emulated_gt_matches_oracle(worker):
    G.test_gt_matches_oracle(worker)


def test_emulated_batch_verifies_mimc_proofs(worker):
    G.test_batch_verifies_mimc_proofs(worker)


def test_emulated_batch_edge_cases(worker):
    G.test_batch_edge_cases(worker)


def test_emulated_synthetic_batch_generator(worker):
    G.test_synthetic_batch_generator(worker)


DRY_RUN = """
import importlib.util, sys
sys.path.insert(0, ROOT)
import torch
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
spec = importlib.util.spec_from_file_location("bench_verify", ROOT + "/bench_verify.py")
bv = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bv)
sys.argv = ["bench_verify.py", "--steps", "2", "--warmup", "1"] + EXTRA
bv.main()
"""


def test_emulated_bench_verify_dry_run(tmp_path, emu_verify_lib):
    """bench_verify.py at 2^3 proofs on the emulated library: one JSON line with the agreed keys; the script itself
    asserts that the timed batch is accepted and a batch with one C replaced is rejected"""
    script = tmp_path / "dry_verify.py"
    out = tmp_path / "dump"
    extra = ["--log-size", "3", "--inputs", "2", "--dump-outputs", str(out)]
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_verify_lib!r}\nEXTRA = {extra!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    need = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "cpu_baseline", "stages_ms_per_step", "fp_mul"}
    assert need <= set(d), need - set(d)
    assert d["metric"] == "groth16_batch_verify_proofs_per_sec" and d["unit"] == "proofs/s" and d["value"] > 0
    assert d["steps"] == 2 and d["warmup"] == 1 and d["n_gpus"] == 1
    assert d["config"]["proofs"] == 8 and d["config"]["inputs_per_proof"] == 2
    assert d["cpu_baseline"] is None and d["cpu_baseline_reason"]
    assert {"value", "unit", "h2d_bytes_per_step"} <= set(d["e2e"]) and d["e2e"]["h2d_bytes_per_step"] > 0
    assert {"scalar_mul", "msms", "miller", "product", "final_exp"} <= set(d["stages_ms_per_step"])
    assert d["fp_mul"]["per_pair_miller"] > 7000 and d["fp_mul"]["peak"] == 27.3
    assert d["config"]["checks"] == {"timed_batch": "accepted", "one_c_replaced": "rejected"}
    assert sorted(os.listdir(out)) == ["gt_tampered.npy", "verdicts.npy"]
