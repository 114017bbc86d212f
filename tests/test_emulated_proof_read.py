"""Proof::read / Proof::write over a batch -- csrc/decode.cu -- executed on host threads (tests/native/) and compared with
the oracle's restatement of Proof::read.  The test bodies are those of test_gpu_proof_read.py at the same sizes; the GPU
file adds the sizes only a device reaches."""
import importlib.util
import os
import subprocess

import test_gpu_proof_read as G
from emulated import ROOT, bench_dry_run, worker  # noqa: F401  (the emulated-library fixture)


def test_emulated_round_trip(worker):
    G.test_round_trip(worker)


def test_emulated_sign_choice(worker):
    G.test_sign_choice(worker)


def test_emulated_every_rejection_class(worker):
    G.test_every_rejection_class(worker)


def test_emulated_priority(worker):
    G.test_priority(worker)


def test_emulated_fast_subgroup_check_matches_rP(worker):
    G.test_fast_subgroup_check_matches_rP(worker)


def test_emulated_mixed_batch(worker):
    G.test_mixed_batch(worker)


def test_emulated_verifier_from_bytes(worker):
    G.test_verifier_from_bytes(worker)


def test_emulated_library_sources_are_the_makefiles():
    """the emulated library compiles the translation units libbellman_b200.so links, in the Makefile's order (as make
    itself reads SRCS); and nothing outside decode.cu calls into it"""
    spec = importlib.util.spec_from_file_location("build_emu_default", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    srcs = subprocess.run(["make", "-s", "--no-print-directory", "-C", os.path.join(ROOT, "bellman_b200", "csrc"),
                           "--eval", "print-srcs: ; @echo $(SRCS)", "print-srcs"], capture_output=True, text=True, check=True)
    assert mod.SOURCES == srcs.stdout.split()
    for name in os.listdir(os.path.join(ROOT, "bellman_b200", "csrc")):
        if name != "decode.cu" and name.endswith((".cu", ".cuh")):
            text = open(os.path.join(ROOT, "bellman_b200", "csrc", name)).read()
            assert "bb_proofs_" not in text and "bb_diag_points_decompress" not in text, name


def test_emulated_bench_verify_from_bytes_dry_run(tmp_path, emu_lib):
    """bench_verify.py --from-bytes at 2^3 proofs on the emulated library: one JSON line with the from_bytes leg, both of
    its checks passing, and the dump file set of the run without the flag"""
    out = tmp_path / "dump"
    d = bench_dry_run(emu_lib, tmp_path, "bench_verify.py",
                      ["--steps", "2", "--warmup", "1", "--log-size", "3", "--inputs", "2", "--from-bytes", "--dump-outputs", str(out)])
    assert d["metric"] == "groth16_batch_verify_proofs_per_sec" and d["config"]["proofs"] == 8
    fb = d["from_bytes"]
    assert {"value", "unit", "ms_per_step", "decode_ms", "h2d_bytes_per_step", "checks"} <= set(fb)
    assert fb["unit"] == "proofs/s" and fb["value"] > 0 and fb["h2d_bytes_per_step"] >= 8 * 192
    assert fb["checks"] == {"decoded_points": "equal", "corrupted_b_at_middle": "reported"}
    assert fb["corrupted"]["index"] == 4 and fb["corrupted"]["status"] in (0x23, 0x24)
    assert set(fb["decode_stages_ms"]) == {"upload", "g1", "g2", "status", "download"}
    assert sorted(os.listdir(out)) == ["gt_tampered.npy", "verdicts.npy"]
