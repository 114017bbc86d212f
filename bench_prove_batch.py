"""Batch proving benchmark: B distinct witnesses of the MiMC shape (bb_synth_mimc_witness seeds) against one synthetic key
(bb_synth_crs) at 2^--log-size constraints, proved three ways:
  batch_hbm    bb_groth16_prove_batch with every witness resident in HBM
  batch_host   bb_groth16_prove_batch from page-locked host buffers
  loop_hbm     bb_groth16_prove once per item, witnesses in HBM
JSON fields: per leg proofs_per_s and ms_per_batch (mean over --steps after --warmup); launches_per_proof of the batch and
of the loop; host_tail_ms (per sub-batch: host time from the last MSM result to the proof bytes, profile mode, one extra
call); sub_batches; checks.proofs = "equal" when the batch's bytes equal the loop's; gpu (card name, power limit, maximum SM
clock and the SM clock sampled after the timed legs, read in the same run).
--sweep prints one such line per (log size, B) in {10, 14, 17, 20} x {1, 16, 64}, skipping cells that do not fit.
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bellman_b200 as bb  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--log-size", type=int, default=14, help="log2 of the constraints")
    ap.add_argument("--batch", type=int, default=64, help="witnesses per call")
    ap.add_argument("--sweep", action="store_true", help="log sizes {10, 14, 17, 20} x batches {1, 16, 64}")
    return ap.parse_args()


def gpu_info():
    """card name, power limit, maximum and current SM clock, read in the run they describe"""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2]), "sm_mhz": float(out[3])}
    except Exception:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None, "sm_mhz": None}


def timed(worker, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    worker.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        out = fn()
    worker.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps, out


def cell(worker, log_size, batch, steps, warmup):
    rounds = (1 << (log_size - 1)) - 1
    items = []
    for k in range(batch):
        asg, shape = bb.synth_mimc(rounds, seed=100 + k, pinned=True)
        items.append(asg)
    params = bb.Parameters.synthetic(worker, 7, shape)
    rs = [0x1234567 + 3 * k for k in range(batch)]
    ss = [0x7654321 + 5 * k for k in range(batch)]
    dev, held = [], []
    for asg in items:
        d = {}
        for key, arr in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
            p = worker.device_alloc(max(arr.nbytes, 32))
            worker.upload(p, arr)
            d[key] = bb._addr(p)
            held.append(p)
        dev.append(d)

    def batch_hbm():
        return bb.create_proof_batch(items, params, rs, ss, dev)

    def batch_host():
        return bb.create_proof_batch(items, params, rs, ss)

    def loop_hbm():
        return [bb.create_proof(a, params, r, s, d) for a, r, s, d in zip(items, rs, ss, dev)]

    res = {"metric": "prove_batch_proofs_per_s", "config": {"log_size": log_size, "constraints": 1 << log_size, "batch": batch,
                                                            "steps": steps, "warmup": warmup}}
    outs = {}
    for name, fn in (("batch_hbm", batch_hbm), ("batch_host", batch_host), ("loop_hbm", loop_hbm)):
        ms, outs[name] = timed(worker, fn, steps, warmup)
        res[name] = {"ms_per_batch": ms, "proofs_per_s": batch / (ms * 1e-3) if ms > 0 else None}
    res["value"] = res["batch_hbm"]["proofs_per_s"]
    l0 = worker.kernel_launches
    batch_hbm()
    lb = worker.kernel_launches - l0
    l0 = worker.kernel_launches
    loop_hbm()
    ll = worker.kernel_launches - l0
    res["launches_per_proof"] = {"batch": lb / batch, "loop": ll / batch}
    worker.set_option("profile", 1)
    worker.profile_reset()
    batch_hbm()
    tail_ms, subs, _ = worker.profile_read("prove_batch.host_tail")
    worker.set_option("profile", 0)
    res["host_tail_ms"] = tail_ms / subs if subs else None
    res["sub_batches"] = subs
    same = all(isinstance(p, bytes) for p in outs["batch_hbm"]) and outs["batch_hbm"] == outs["loop_hbm"] == outs["batch_host"]
    res["checks"] = {"proofs": "equal" if same else "DIFFERENT"}
    for p in held:
        worker.device_free(p)
    params.free()
    return res


def main():
    args = parse()
    sys.stdout.flush()
    real = os.dup(1)                # exactly one JSON line per cell on stdout; library chatter goes to stderr
    os.dup2(2, 1)
    worker = bb.Worker(0)
    cells = [(l, b) for l in (10, 14, 17, 20) for b in (1, 16, 64)] if args.sweep else [(args.log_size, args.batch)]
    for log_size, batch in cells:
        try:
            res = cell(worker, log_size, batch, args.steps, args.warmup)
        except (bb.BackendError, MemoryError) as e:
            if not args.sweep:
                raise
            res = {"metric": "prove_batch_proofs_per_s", "config": {"log_size": log_size, "batch": batch}, "skipped": str(e)[:200]}
        res["gpu"] = gpu_info()
        os.write(real, (json.dumps(res) + "\n").encode())
    worker.close()


if __name__ == "__main__":
    main()
