"""The batch prover -- bb_groth16_prove_batch and bb_groth16_prove_r1cs_batch -- executed on host threads (tests/native/)
and compared item by item with create_proof.  The test bodies are those of test_gpu_prove_batch.py at the sizes a host
reaches; the GPU file adds 2^17 and 2^20 constraints."""
import test_gpu_prove_batch as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


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


def test_emulated_bench_prove_batch_dry_run(tmp_path, emu_lib):
    """bench_prove_batch.py at 2^6 constraints on the emulated library: one JSON line with the three legs, launches per
    proof, the host tail, the sub-batches and the equality check"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_prove_batch.py",
                      ["--steps", "1", "--warmup", "1", "--log-size", "6", "--batch", "3"])
    assert d["metric"] == "prove_batch_proofs_per_s" and d["config"]["constraints"] == 64 and d["config"]["batch"] == 3
    assert {"batch_hbm", "batch_host", "loop_hbm", "launches_per_proof", "host_tail_ms", "sub_batches", "checks", "gpu"} <= set(d)
    for leg in ("batch_hbm", "batch_host", "loop_hbm"):
        assert set(d[leg]) == {"ms_per_batch", "proofs_per_s"}
    assert d["checks"] == {"proofs": "equal"} and d["sub_batches"] == 1
    assert d["launches_per_proof"]["batch"] < d["launches_per_proof"]["loop"]
    assert {"name", "power_limit_w", "sm_max_mhz", "sm_mhz"} <= set(d["gpu"])
