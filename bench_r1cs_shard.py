#!/usr/bin/env python
"""bench_r1cs_shard.py -- proving from the witness on a sharded key (bb_groth16_prove_r1cs_begin) on ONE device.

    python bench_r1cs_shard.py --steps K --warmup W [--log-size 20]

The key, witness and constraint system are bench_r1cs.py's: bb_synth_mimc_witness(rounds, 20), Parameters.synthetic(worker,
21, shape) and bb_synth_mimc_r1cs(rounds, 20), 2^log-size constraints, default MSM form.  The line holds
  owner         per polynomial a, b, c, the owner stage of a rank that owns it, witness in HBM, N = m:
                  device_ms / stages_ms: the stage alone, with no MSM in flight (bb_diag_r1cs_owner_stage: matrix i
                    evaluated straight into the transform buffer, ifft + coset_fft there): CUDA events of the profile
                    mode (r1cs_owner.eval, r1cs_owner.transforms), mean over K steps;
                  today_device_ms / today_stages_ms: what an owner does without this call, the same way -- bb_r1cs_eval of
                    all three polynomials into HBM (r1cs.eval), then bb_h_coset_evals of its polynomial from HBM
                    (h_coset_evals: copy, padding, transforms) -- alternated step by step with the new stage;
                  with_msms_stages_ms: the same stages inside begin(own = that polynomial) / wait / end, with the seven
                    witness MSMs the call queues running alongside;
                  launches / today_launches: kernel launches of the stage alone and of today's two calls;
                    in_proof_launches: those of a begin / wait / end pair with own = that polynomial minus one with
                    own = 0, both ending on the same vectors (asserted equal to `launches`);
                  vectors: the stage's vector, alone and inside a proof, against today's, byte for byte (asserted);
  value         device_ms of a;
  one_rank      shard 0 of 1: median ms of begin (split, own = 7) / wait / end / finalize, of begin (replicated) / end /
                finalize, and of bb_groth16_prove_r1cs, alternated step by step; their proof bytes compared (asserted);
  h2d_bytes_per_rank_per_proof   host witness, a rank owning one polynomial: bb_ctx_bytes_copied of the new path and of
                create_proof_sharded's path (bb_h_coset_evals_async of its polynomial from the host + bb_groth16_prove_begin);
  multi_gpu     "not measured": one device cannot time N ranks;
  gpu, clocks   card name, power limit and maximum SM clock (nvidia-smi), SM clock sampled during the timed legs.
Prints one JSON line on stdout; writes nothing else.
"""
import argparse
import ctypes as C
import importlib.util
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(_spec)             # the clock sampler, emit / log of bench.py
_spec.loader.exec_module(bench)
_spec = importlib.util.spec_from_file_location("bench_r1cs", os.path.join(ROOT, "bench_r1cs.py"))
bench_r1cs = importlib.util.module_from_spec(_spec)        # gpu_info
_spec.loader.exec_module(bench_r1cs)

FR_MODULUS = bench.FR_MODULUS


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints (bench.py's MiMC workload)")
    return ap.parse_args()


def run(args):
    import bellman_b200 as bb
    from bellman_b200 import r1cs as RC
    log_n = args.log_size
    rounds = (1 << (log_n - 1)) - 1
    worker = bb.Worker(0)
    bench.log("synthesising the MiMC-chain witness and its constraint system (CPU, product-side generator)")
    asg, shape = bb.synth_mimc(rounds, seed=20, pinned=True)
    n = shape["num_constraints"]
    m = n                                                   # 2^log-size constraints: N = m
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    assert r1cs.n_constraints == n == 1 << log_n
    params = bb.Parameters.synthetic(worker, 21, shape)
    r, s = 0x1234567 % FR_MODULUS, 0x7654321 % FR_MODULUS
    dev = {}
    for name, arr in (("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
        dev[name] = worker.device_alloc(arr.nbytes)
        worker.upload(dev[name], arr)
    evals = [worker.device_alloc(m * 32) for _ in range(3)]
    abc = {k: worker.device_alloc(n * 32) for k in "abc"}
    today_out = worker.device_alloc(m * 32)

    def get(p):
        h = np.zeros((m, 4), np.uint64)
        worker.download(p, h)
        return h

    def owner_new(own):
        state = RC.prove_r1cs_begin(r1cs, params, None, None, own, evals, device_ptrs=dev)
        bb.h_coset_evals_wait(worker)
        return state

    src, _ = r1cs._witness_args(dev["inputs"], dev["aux"], True)

    def owner_alone(i):
        """the owner stage of polynomial i with no MSM in flight (bb_diag_r1cs_owner_stage)"""
        bb._check(bb.load_library().bb_diag_r1cs_owner_stage(worker._h, r1cs._h, *src, C.c_int(i), C.c_void_p(bb._addr(evals[i]))))

    def owner_today(i):
        r1cs.eval(dev["inputs"], dev["aux"], on_device=True, out=abc)
        bb.h_coset_evals(worker, abc["abc"[i]], n, today_out, on_device=True)

    def launches(fn):
        l0 = worker.kernel_launches
        fn()
        worker.synchronize()
        return worker.kernel_launches - l0

    def device_ms(stages):
        return sum(worker.profile_read(st)[0] for st in stages) / args.steps

    want = []                                               # today's three vectors
    for i in range(3):
        owner_today(i)
        want.append(get(today_out))

    zeros = np.zeros((m, 4), np.uint64)

    def in_proof(own):
        """begin / wait / end with own; an unowned buffer holds the vector its owner gives (as after a broadcast), an owned
        one zeros until the owner writes it, so that the last transform and the h MSM (whose launches depend on their
        scalars) run on the same vectors whatever `own` is"""
        for i in range(3):
            worker.upload(evals[i], zeros if own >> i & 1 else want[i])
        state = owner_new(own)
        got = [get(evals[i]) for i in range(3) if own >> i & 1]
        bb.prove_end(state, evals)
        return got

    sampler = bench.ClockSampler(0)
    sampler.start()
    owner, vectors_equal = {}, True
    for i, name in enumerate("abc"):
        for _ in range(args.warmup):
            owner_alone(i)
            owner_today(i)
            in_proof(1 << i)
            in_proof(0)
        worker.set_option("profile", 1)
        worker.profile_reset()
        for _ in range(args.steps):                         # alternated step by step, each ending in a device synchronise
            owner_alone(i)
            owner_today(i)
        new_ms = {st: round(device_ms(["r1cs_owner." + st]), 4) for st in ("eval", "transforms")}
        today_ms = {"r1cs_eval": round(device_ms(["r1cs.eval"]), 4), "h_coset_evals": round(device_ms(["h_coset_evals"]), 4)}
        worker.profile_reset()
        for _ in range(args.steps):
            in_proof(1 << i)
        with_msms = {st: round(device_ms(["r1cs_owner." + st]), 4) for st in ("eval", "transforms")}
        worker.set_option("profile", 0)
        worker.profile_reset()
        worker.upload(evals[i], zeros)
        owner_alone(i)
        same = np.array_equal(get(evals[i]), want[i]) and np.array_equal(in_proof(1 << i)[0], want[i])
        vectors_equal &= same
        owner[name] = {"terms": r1cs.nnz[i], "device_ms": round(sum(new_ms.values()), 4), "stages_ms": new_ms,
                       "launches": launches(lambda: owner_alone(i)),
                       "in_proof_launches": launches(lambda: in_proof(1 << i)) - launches(lambda: in_proof(0)),
                       "today_device_ms": round(sum(today_ms.values()), 4), "today_stages_ms": today_ms,
                       "today_launches": launches(lambda: owner_today(i)),
                       "with_msms_stages_ms": with_msms, "vectors": "equal" if same else "DIFFERENT"}

    # one rank: split with every polynomial owned, replicated, and bb_groth16_prove_r1cs, alternated
    def split():
        state = owner_new(7)
        return bb.finalize(params, [bb.prove_end(state, evals)], r, s)

    def replicated():
        return bb.finalize(params, [bb.prove_end(RC.prove_r1cs_begin(r1cs, params, None, None, device_ptrs=dev))], r, s)

    def whole():
        return RC.create_proof_r1cs(r1cs, params, None, None, r, s, device_ptrs=dev)

    legs = {"split_ms": split, "replicated_ms": replicated, "prove_r1cs_ms": whole}
    for fn in legs.values():
        for _ in range(args.warmup):
            fn()
    times, proofs = {k: [] for k in legs}, set()
    for _ in range(args.steps):
        for k, fn in legs.items():
            t0 = time.perf_counter()
            proofs.add(fn())
            times[k].append(1e3 * (time.perf_counter() - t0))
    clocks = sampler.stop()
    one_rank = {k: round(float(np.median(v)), 3) for k, v in times.items()}

    # host->device bytes of one proof of a rank owning b, host witness: the new path against create_proof_sharded's
    def h2d(fn):
        h0, _ = worker.bytes_copied()
        fn()
        worker.synchronize()
        return worker.bytes_copied()[0] - h0

    def new_rank():
        state = RC.prove_r1cs_begin(r1cs, params, asg.input_assignment, asg.aux_assignment, 2, evals)
        bb.h_coset_evals_wait(worker)
        bb.prove_end(state, evals)

    def today_rank():
        bb.h_coset_evals_async(worker, asg.b, n, evals[1])
        state = bb.prove_begin(asg, params)
        bb.h_coset_evals_wait(worker)
        bb.prove_end(state, evals)

    bytes_rank = {"from_witness": h2d(new_rank), "today": h2d(today_rank)}

    checks = {"vectors": "equal" if vectors_equal else "DIFFERENT", "proof": "equal" if len(proofs) == 1 else "DIFFERENT",
              "launches": "equal" if all(o["launches"] == o["in_proof_launches"] for o in owner.values()) else "DIFFERENT"}
    line = {"metric": "r1cs_owner_stage_ms", "value": owner["a"]["device_ms"], "unit": "ms", "lower_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup,
            "config": {"workload": f"mimc-2^{log_n}", "constraints": n, "rounds": rounds,
                       "witness": "bb_synth_mimc_witness(rounds, 20) in HBM; constraint system bb_synth_mimc_r1cs(rounds, 20)",
                       "key": "Parameters.synthetic(worker, 21, shape), one shard; default MSM form",
                       "timing": "owner: device ms from CUDA events (profile mode), mean over K steps, the new stage alone "
                                 "and today's calls alternated step by step; one_rank: host wall clock around blocking calls, "
                                 "median over K steps, the three legs alternated"},
            "owner": owner, "one_rank": one_rank, "h2d_bytes_per_rank_per_proof": bytes_rank,
            "multi_gpu": "not measured", "checks": checks, "gpu": bench_r1cs.gpu_info(), "clocks": clocks}
    bench.emit(line)
    assert checks == {"vectors": "equal", "proof": "equal", "launches": "equal"}, checks
    for p in list(dev.values()) + evals + list(abc.values()) + [today_out]:
        worker.device_free(p)
    r1cs.free()
    params.free()
    worker.close()


def main():
    args = parse()
    # stdout carries exactly ONE JSON line: whatever libraries print goes to stderr until the result is ready
    sys.stdout.flush()
    bench._REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    run(args)


if __name__ == "__main__":
    main()
