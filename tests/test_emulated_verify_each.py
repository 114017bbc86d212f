"""verify_proof for every proof of a batch -- bb_groth16_verify_each in csrc/verify.cu -- executed on host threads
(tests/native/) and compared with the oracle's Python pairing and verifier and with the batch-of-one path.  The test
bodies are those of test_gpu_verify_each.py at the same sizes; the GPU file adds the sizes only a device reaches."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

import test_gpu_verify_each as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_each_lib(tmp_path_factory):
    """the emulated library of tests/native/build_emu.py with verify.cu and decode.cu compiled in beside its sources"""
    spec = importlib.util.spec_from_file_location("build_emu_each", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.SOURCES = list(mod.SOURCES) + [s for s in ("verify.cu", "decode.cu") if s not in mod.SOURCES]
    lib, _ = mod.build(str(tmp_path_factory.mktemp("bb_emu_each")))
    return lib


@pytest.fixture(scope="module")
def worker(emu_each_lib):
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = emu_each_lib, None        # this module only: the mirror talks to the emulated library
    try:
        w = bb.Worker(0)
        yield w
        w.close()
    finally:
        bb.LIB_PATH, bb._lib = saved


def test_emulated_each_gt_matches_oracle(worker):
    G.test_each_gt_matches_oracle(worker)


def test_emulated_each_verdicts_mimc(worker):
    G.test_each_verdicts_mimc(worker)


def test_emulated_each_identities(worker):
    G.test_each_identities(worker)


def test_emulated_each_errors(worker):
    G.test_each_errors(worker)


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
sys.argv = ["bench_verify.py", "--steps", "1", "--warmup", "1"] + EXTRA
bv.main()
"""


def test_emulated_bench_verify_each_dry_run(tmp_path, emu_each_lib):
    """bench_verify.py --each at 2^3 proofs on the emulated library: one JSON line with the `each` object, its check
    flagging exactly the first, middle and last proof, and verdicts_each.npy among the dumped outputs"""
    script = tmp_path / "dry_each.py"
    out = tmp_path / "dump"
    extra = ["--log-size", "3", "--inputs", "2", "--each", "--dump-outputs", str(out)]
    script.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {emu_each_lib!r}\nEXTRA = {extra!r}\n" + DRY_RUN)
    res = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    d = json.loads(lines[0])
    assert d["metric"] == "groth16_batch_verify_proofs_per_sec" and d["config"]["proofs"] == 8
    e = d["each"]
    assert {"value", "unit", "ms_per_step", "e2e", "stages_ms_per_step", "fp_mul_per_proof", "checks"} <= set(e)
    assert e["unit"] == "proofs/s" and e["value"] > 0 and e["e2e"]["value"] > 0
    assert set(e["stages_ms_per_step"]) == {"upload", "psi", "miller", "final_exp", "download"}
    assert e["checks"] == {"flagged": "first, middle, last", "n_invalid": 3}
    assert sorted(os.listdir(out)) == ["gt_tampered.npy", "verdicts.npy", "verdicts_each.npy"]
