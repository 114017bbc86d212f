"""Proof::read / Proof::write over a batch -- csrc/decode.cu -- executed on host threads (tests/native/) and compared with
the oracle's restatement of Proof::read.  The test bodies are those of test_gpu_proof_read.py at the same sizes; the GPU
file adds the sizes only a device reaches."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_proof_read as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_read_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with verify.cu and decode.cu compiled in beside its sources"""
    spec = importlib.util.spec_from_file_location("build_emu_read", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "decode.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_read")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_read_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_read_lib, None        # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


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


def test_default_emulated_library_does_not_need_decode():
    """nothing outside decode.cu calls into it: the default source list of build_emu.py stays without it"""
    spec = importlib.util.spec_from_file_location("build_emu_default", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert "decode.cu" not in mod.SOURCES
    for name in os.listdir(os.path.join(ROOT, "bellman_b200", "csrc")):
        if name != "decode.cu" and name.endswith((".cu", ".cuh")):
            text = open(os.path.join(ROOT, "bellman_b200", "csrc", name)).read()
            assert "bb_proofs_" not in text and "bb_diag_points_decompress" not in text, name


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


def test_emulated_bench_verify_from_bytes_dry_run(tmp_path, emu_read_lib):
    """bench_verify.py --from-bytes at 2^3 proofs on the emulated library: one JSON line with the from_bytes leg, both of
    its checks passing, and the dump file set of the run without the flag"""
    script = tmp_path / "dry_read.py"
    out = tmp_path / "dump"
    extra = ["--log-size", "3", "--inputs", "2", "--from-bytes", "--dump-outputs", str(out)]
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_read_lib!r}\nEXTRA = {extra!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "groth16_batch_verify_proofs_per_sec" and d["config"]["proofs"] == 8
    fb = d["from_bytes"]
    assert {"value", "unit", "ms_per_step", "decode_ms", "h2d_bytes_per_step", "checks"} <= set(fb)
    assert fb["unit"] == "proofs/s" and fb["value"] > 0 and fb["h2d_bytes_per_step"] >= 8 * 192
    assert fb["checks"] == {"decoded_points": "equal", "corrupted_b_at_middle": "reported"}
    assert fb["corrupted"]["index"] == 4 and fb["corrupted"]["status"] in (0x23, 0x24)
    assert set(fb["decode_stages_ms"]) == {"upload", "g1", "g2", "status", "download"}
    assert sorted(os.listdir(out)) == ["gt_tampered.npy", "verdicts.npy"]
