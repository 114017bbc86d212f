"""Groth16 verification -- the pairing tower, the Miller loop, the final exponentiation and the batch verifier of
csrc/verify.cu -- executed on host threads (tests/native/) and compared with the oracle's Python pairing and
verifier.  The test bodies are those of test_gpu_verify.py at the same sizes; the GPU file adds the sizes only a
device reaches."""
import os

import test_gpu_verify as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


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


def test_emulated_bench_verify_dry_run(tmp_path, emu_lib):
    """bench_verify.py at 2^3 proofs on the emulated library: one JSON line with the agreed keys; the script itself
    asserts that the timed batch is accepted and a batch with one C replaced is rejected"""
    out = tmp_path / "dump"
    d = bench_dry_run(emu_lib, tmp_path, "bench_verify.py",
                      ["--steps", "2", "--warmup", "1", "--log-size", "3", "--inputs", "2", "--dump-outputs", str(out)])
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
