"""Checking witnesses against the constraint system -- bb_r1cs_check and bb_r1cs_check_batch in csrc/r1cs.cu -- executed
on host threads (tests/native/) and compared with a Python-integer evaluation of every row.  The test bodies are those of
test_gpu_r1cs_check.py; the GPU file adds rows of more than 2048 terms and 2^20 constraints."""
import test_gpu_r1cs_check as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


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


def test_emulated_bench_r1cs_check_dry_run(tmp_path, emu_lib):
    """bench_r1cs_check.py at 2^6 constraints and a batch of 3 on the emulated library: one JSON line with the check's
    stages, the batch legs, the eval and prove references and the equality checks"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_r1cs_check.py",
                      ["--steps", "1", "--warmup", "1", "--log-size", "6", "--batch", "3"])
    assert d["metric"] == "r1cs_check_ms" and d["config"]["constraints"] == 64 and d["value"] >= 0   # emulated events read 0 ms
    assert {"eval_ms", "compare_ms", "compare_bytes", "roofline", "batch_hbm", "batch_host", "r1cs_eval_ms", "prove_ms",
            "share_of_prove", "checks", "gpu"} <= set(d)
    assert d["compare_bytes"] == 3 * 64 * 32
    for leg in ("batch_hbm", "batch_host"):
        assert d[leg]["items"] == 3 and d[leg]["launches_per_item"] == 2
    assert d["checks"] == {"satisfied": "equal", "corrupted": "equal", "batch": "equal"}
