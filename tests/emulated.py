"""What the emulated-library tests share: the Python mirror pointed at the host-fiber build of the product sources
(tests/native/, the session fixture `emu_lib`), and the bench scripts run end to end on it.  A helper module, not a
test module: a test module imports `worker` as its fixture."""
import contextlib
import json
import os
import subprocess
import sys

import pytest

import bellman_b200 as bb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def use_library(lib):
    """the mirror talks to `lib` inside the block and to the library it had before after it"""
    saved = (bb.LIB_PATH, bb._lib)
    bb.LIB_PATH, bb._lib = lib, None
    try:
        yield
    finally:
        bb.LIB_PATH, bb._lib = saved


@pytest.fixture(scope="module")
def worker(emu_lib):
    with use_library(emu_lib):                       # this module only: the mirror talks to the emulated library
        w = bb.Worker(0)
        yield w
        w.close()


DRY_RUN = """
import importlib.util, os, sys
sys.path.insert(0, ROOT)
import torch
torch.cuda.set_device = lambda *a, **k: None
torch.cuda.synchronize = lambda *a, **k: None
_to = torch.Tensor.to
torch.Tensor.to = lambda self, *a, **k: self if (a and isinstance(a[0], str) and a[0].startswith("cuda")) else _to(self, *a, **k)
torch.Tensor.pin_memory = lambda self, *a, **k: self
import bellman_b200 as bb
bb.LIB_PATH, bb._lib = EMU_LIB, None          # the product sources on host fibers (tests/native)
os.environ["LOCAL_RANK"] = "0"                # the emulation has one device: under torchrun every rank uses it
spec = importlib.util.spec_from_file_location(SCRIPT[:-3], os.path.join(ROOT, SCRIPT))
bench = importlib.util.module_from_spec(spec)
spec.loader.exec_module(bench)
sys.argv = [SCRIPT] + ARGV
bench.main()
"""


def dry_run_script(lib, tmp_path, script, argv):
    """a Python file that runs the bench script `script` (a file name at the repository root) with `argv` on the library
    `lib`, with torch.cuda stubbed and pinned memory left pageable"""
    path = tmp_path / ("dry_" + script)
    path.write_text(f"ROOT = {ROOT!r}\nEMU_LIB = {lib!r}\nSCRIPT = {script!r}\nARGV = {list(argv)!r}\n" + DRY_RUN)
    return path


def bench_dry_run(lib, tmp_path, script, argv, env=None):
    """runs dry_run_script(...) and returns the one JSON line it must print"""
    res = subprocess.run([sys.executable, str(dry_run_script(lib, tmp_path, script, argv))], capture_output=True, text=True,
                         timeout=900, cwd=ROOT, env=env)
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    return json.loads(lines[0])
