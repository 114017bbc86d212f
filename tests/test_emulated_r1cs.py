"""The constraint system on the device -- bb_r1cs_* and bb_groth16_prove_r1cs in csrc/r1cs.cu -- executed on host threads
(tests/native/) and compared with oracle-0's ProvingAssignment and with create_proof on the host-evaluated assignment.
The test bodies are those of test_gpu_r1cs.py; the GPU file adds the sizes only a device reaches (a row of 2^16 terms,
2^20 constraints)."""
import pytest

import test_gpu_r1cs as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


def test_emulated_eval_xor_demo(worker):
    G.test_eval_xor_demo(worker)


def test_emulated_eval_zero_coeffs(worker):
    G.test_eval_zero_coeffs(worker)


def test_emulated_eval_mimc322(worker):
    G.test_eval_mimc322(worker)


def test_emulated_eval_random(worker):
    G.test_eval_random(worker, big=False)


def test_emulated_prove_mimc322(worker):
    G.test_prove_mimc322(worker)


def test_emulated_prove_generated_key_verifies(worker):
    G.test_prove_generated_key_verifies(worker, rounds=10)


def test_emulated_errors(worker):
    G.test_errors(worker)


def test_emulated_synth_mimc(worker):
    """bb_synth_mimc_r1cs against bb_synth_mimc_witness and the two prove paths, at 2^6 constraints"""
    G.check_synth(worker, 6)


@pytest.mark.parametrize("workload", ["mimc", "long-rows"])
def test_emulated_bench_r1cs_dry_run(tmp_path, emu_lib, workload):
    """bench_r1cs.py at 2^6 constraints on the emulated library: one JSON line with the eval, the two prove legs from HBM
    and from host buffers, the bytes copied per proof and the equality checks"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_r1cs.py",
                      ["--steps", "1", "--warmup", "1", "--log-size", "6", "--workload", workload])
    assert d["metric"] == "r1cs_eval_ms" and d["config"]["constraints"] == 64 and d["value"] >= 0   # emulated events read 0 ms
    assert {"nnz", "bytes", "fr_products", "roofline", "prove_hbm", "prove_host", "h2d_bytes_per_proof", "checks", "gpu"} <= set(d)
    assert d["nnz"] == {"a": 3 * 31 + 2, "b": 4 * 31, "c": 3 * 31} and d["fr_products"] == 4 * 31   # ci in A, twice in B, -1 in C
    assert set(d["prove_hbm"]) == set(d["prove_host"]) == {"from_witness_ms", "from_abc_ms"}
    h2d = d["h2d_bytes_per_proof"]
    assert h2d["from_abc"] - h2d["from_witness"] == 3 * 64 * 32 and h2d["from_witness"] >= 65 * 32    # a, b, c stay off the bus
    assert d["checks"] == {"a_b_c": "equal", "densities": "equal", "proof": "equal"}
    if workload == "long-rows":
        assert d["long_rows"]["value"] >= 0 and d["long_rows"]["checks"] == "equal"
