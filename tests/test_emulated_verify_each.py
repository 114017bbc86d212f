"""verify_proof for every proof of a batch -- bb_groth16_verify_each in csrc/verify.cu -- executed on host threads
(tests/native/) and compared with the oracle's Python pairing and verifier and with the batch-of-one path.  The test
bodies are those of test_gpu_verify_each.py at the same sizes; the GPU file adds the sizes only a device reaches."""
import os

import test_gpu_verify_each as G
from emulated import bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


def test_emulated_each_gt_matches_oracle(worker):
    G.test_each_gt_matches_oracle(worker)


def test_emulated_each_verdicts_mimc(worker):
    G.test_each_verdicts_mimc(worker)


def test_emulated_each_identities(worker):
    G.test_each_identities(worker)


def test_emulated_each_errors(worker):
    G.test_each_errors(worker)


def test_emulated_bench_verify_each_dry_run(tmp_path, emu_lib):
    """bench_verify.py --each at 2^3 proofs on the emulated library: one JSON line with the `each` object, its check
    flagging exactly the first, middle and last proof, and verdicts_each.npy among the dumped outputs"""
    out = tmp_path / "dump"
    d = bench_dry_run(emu_lib, tmp_path, "bench_verify.py",
                      ["--steps", "1", "--warmup", "1", "--log-size", "3", "--inputs", "2", "--each", "--dump-outputs", str(out)])
    assert d["metric"] == "groth16_batch_verify_proofs_per_sec" and d["config"]["proofs"] == 8
    e = d["each"]
    assert {"value", "unit", "ms_per_step", "e2e", "stages_ms_per_step", "fp_mul_per_proof", "checks"} <= set(e)
    assert e["unit"] == "proofs/s" and e["value"] > 0 and e["e2e"]["value"] > 0
    assert set(e["stages_ms_per_step"]) == {"upload", "psi", "miller", "final_exp", "download"}
    assert e["checks"] == {"flagged": "first, middle, last", "n_invalid": 3}
    assert sorted(os.listdir(out)) == ["gt_tampered.npy", "verdicts.npy", "verdicts_each.npy"]
