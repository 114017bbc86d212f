"""Groth16 parameter generation and parameter-file writing on the device -- bb_groth16_generate (csrc/generate.cu) and
bb_params_write (csrc/decode.cu) -- executed on host threads (tests/native/) and compared with the host generator and
params_io.write_parameters.  The test bodies are those of test_gpu_generate.py at small sizes."""
import test_gpu_generate as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


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


def test_emulated_bench_generate_dry_run(tmp_path, emu_lib):
    """bench_generate.py at 2^4 constraints on the emulated library: one JSON line, every check passing"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_generate.py",
                      ["--log-size", "4", "--old-log-size", "4", "--oracle-log-size", "4", "--steps", "1"])
    assert d["metric"] == "generate_ms" and d["config"]["log_size"] == 4
    assert {"seeded", "random", "write", "old", "oracle1", "gpu", "checks"} <= set(d)
    assert set(d["seeded"]["stages_ms"]) == {"generate.transpose", "generate.lagrange", "generate.qap", "generate.g1", "generate.g2"}
    assert set(d["write"]) == {"pinned", "hbm"}
    assert d["checks"] == {"proof": "equal", "verifies": "yes", "write_read": "equal"}
