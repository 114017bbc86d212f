"""create_proof_r1cs_sharded on CPU: gloo ranks under torch.distributed.run, each running the product sources on host fibers
(tests/native) over its (base range x window) shard, proving from the witness alone -- split by polynomial (the owners
evaluate their matrix straight into the buffer they broadcast) and replicated, from host and from "device" witnesses."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = textwrap.dedent('''
    import os, sys, random
    import numpy as np
    import torch.distributed as dist
    sys.path.insert(0, os.environ["BB_ROOT"]); sys.path.insert(0, os.path.join(os.environ["BB_ROOT"], "tests"))
    import bellman_b200 as bb
    bb.LIB_PATH, bb._lib = os.environ["BB_EMU_LIB"], None            # host-fiber execution of the product sources
    from bellman_b200 import r1cs as RC
    from bellman_b200.distributed import create_proof_r1cs_sharded, create_proof_sharded
    from oracle import o1

    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    R = o1.FR_MODULUS
    rng = random.Random(6)
    mc = o1.Mimc(40, seed=9)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    w = mc.witness()
    worker = bb.Worker(0)
    r1cs = RC.R1CS.synth_mimc(worker, 40, 9)
    mine = bb.Parameters(worker, mc.export_params(), shard_index=rank, shard_count=world)
    r, s = rng.randrange(R), rng.randrange(R)
    want = mc.expected_proof(r, s)
    assert create_proof_sharded(r1cs.assignment(w["inputs"], w["aux"]), mine, mine, r, s) == (want if rank == 0 else None)
    dev = {}
    for name in ("inputs", "aux"):                  # the emulated device reads host memory: "device" witness arrays
        dev[name] = worker.device_alloc(w[name].nbytes)
        worker.upload(dev[name], w[name])
    for split_h in (True, False):
        for device_ptrs in (None, dev):
            proof = create_proof_r1cs_sharded(r1cs, mine, mine, w["inputs"], w["aux"], r, s, device_ptrs=device_ptrs, split_h=split_h)
            assert proof == (want if rank == 0 else None), (split_h, device_ptrs is not None)
    # an identity base on one rank's shard: every rank raises UnexpectedIdentity
    bad = mc.export_params()
    if rank == world - 1:
        bad["l"] = np.array(bad["l"], copy=True); bad["l"].reshape(-1, 12)[-1] = 0
    broken = bb.Parameters(worker, bad, shard_index=rank, shard_count=world)
    for split_h in (True, False):
        try:
            create_proof_r1cs_sharded(r1cs, broken, broken, w["inputs"], w["aux"], r, s, split_h=split_h)
            raise SystemExit("expected UnexpectedIdentity")
        except bb.UnexpectedIdentity:
            pass
    # a witness of the wrong length on one rank: every rank raises, the failing rank's own text included
    aux = w["aux"][:-1] if rank == 1 else w["aux"]
    for split_h in (True, False):
        try:
            create_proof_r1cs_sharded(r1cs, mine, mine, w["inputs"], aux, r, s, split_h=split_h)
            raise SystemExit("expected an argument error")
        except bb.BackendError as e:
            assert "rank 1" in str(e) and "witness has" in str(e), str(e)
    for p in dev.values():
        worker.device_free(p)
    worker.close()
    dist.destroy_process_group()
    open(os.path.join(os.path.dirname(os.path.abspath(__file__)), f"ok.{rank}"), "w").write("ok")
''')


@pytest.mark.parametrize("world", [2, 3])
def test_r1cs_sharded_prove_gloo_emulated_device(tmp_path, emu_lib, world):
    """Two ranks split the H pipeline a, c | b; three a | b | c.  Rank 0 gets mc.expected_proof(r, s), as from
    create_proof_sharded on the host-evaluated assignment; other ranks None; errors on one rank raise everywhere."""
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, BB_ROOT=ROOT, BB_EMU_LIB=emu_lib)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29551 + world), str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout + res.stderr
    assert all((tmp_path / f"ok.{r}").exists() for r in range(world)), res.stdout + res.stderr
