"""Proving from the witness on a sharded key -- bb_groth16_prove_r1cs_begin in csrc/r1cs.cu -- executed on host threads
(tests/native/).  The test bodies are those of test_gpu_r1cs_shard.py at the sizes a host reaches; the GPU file adds the
MiMC-322 key in up to eight shards and the 2^16 bench key."""
import test_gpu_r1cs_shard as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


def test_emulated_owner_mimc(worker):
    G.test_owner_mimc322(worker, rounds=20)


def test_emulated_owner_from_assembly(worker):
    G.test_owner_from_assembly(worker, rounds=10)


def test_emulated_owner_random(worker):
    G.test_owner_random(worker, log_rows=6)


def test_emulated_sharded_mimc(worker):
    G.test_sharded_mimc(worker, rounds=20, counts=(1, 2, 3))


def test_emulated_sharded_synth(worker):
    G.check_synth_sharded(worker, 6, 2)


def test_emulated_counters(worker):
    G.test_counters(worker, rounds=20)


def test_emulated_errors(worker):
    G.test_errors(worker)


def test_emulated_bench_r1cs_shard_dry_run(tmp_path, emu_lib):
    """bench_r1cs_shard.py at 2^6 constraints on the emulated library: one JSON line with the owner stage per polynomial
    against bb_r1cs_eval + bb_h_coset_evals, the one-rank proof legs and the bytes per rank, every check equal"""
    d = bench_dry_run(emu_lib, tmp_path, "bench_r1cs_shard.py", ["--steps", "1", "--warmup", "1", "--log-size", "6"])
    assert d["metric"] == "r1cs_owner_stage_ms" and d["config"]["constraints"] == 64 and d["value"] >= 0
    assert set(d["owner"]) == {"a", "b", "c"}
    for leg in d["owner"].values():
        assert 0 < leg["launches"] == leg["in_proof_launches"] <= leg["today_launches"] and leg["vectors"] == "equal"
        assert {"device_ms", "stages_ms", "today_device_ms", "today_stages_ms", "with_msms_stages_ms"} <= set(leg)
    assert set(d["one_rank"]) == {"split_ms", "replicated_ms", "prove_r1cs_ms"}
    assert d["checks"] == {"vectors": "equal", "proof": "equal", "launches": "equal"}
    h2d = d["h2d_bytes_per_rank_per_proof"]
    assert h2d["today"] - h2d["from_witness"] == 64 * 32 and h2d["from_witness"] >= (2 + 63) * 32     # b stays off the bus
    assert d["multi_gpu"] == "not measured"
