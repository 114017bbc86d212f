"""Parameters::read / VerifyingKey::read on the device -- bb_params_read and bb_vk_read, csrc/decode.cu -- executed on
host threads (tests/native/) and compared with params_io.read_parameters and with the restatement of the reference's
reader.  The test bodies are those of test_gpu_params_read.py at small sizes."""
import test_gpu_params_read as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


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


def test_emulated_bench_params_read_dry_run(tmp_path, emu_lib):
    """bench_params_read.py at 2^4 constraints on the emulated library: one JSON line, both modes and both sources, old and
    new path, and every check passing"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_params_read.py", ["--steps", "1", "--warmup", "0", "--log-size", "4"])
    assert d["metric"] == "params_read_ms" and d["config"]["log_size"] == 4 and d["config"]["file_bytes"] > 0
    for mode in ("checked", "unchecked"):
        m = d[mode]
        assert {"pinned", "hbm", "old", "stages_ms"} <= set(m)
        for leg in ("pinned", "hbm", "old"):
            assert set(m[leg]) == {"ms", "gb_per_s"} and m[leg]["ms"] >= 0
        assert set(m["stages_ms"]) == {"params.upload", "params.g1", "params.g2"}
    assert d["checks"] == {"vectors": "equal", "proofs": "equal", "corrupt_b_g2_middle": "reported"}
    assert {"name", "power_limit_w", "sm_max_mhz", "sm_mhz"} <= set(d["gpu"])
