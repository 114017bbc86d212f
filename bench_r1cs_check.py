#!/usr/bin/env python
"""bench_r1cs_check.py -- checking witnesses against the constraint system on the device (bb_r1cs_check,
bb_r1cs_check_batch): TestConstraintSystem::which_is_unsatisfied over the resident matrices, against the evaluation and
the proof it would precede.

    python bench_r1cs_check.py --steps K --warmup W [--log-size 20] [--batch 64]

The workload is bench.py's: the MiMC chain of bb_synth_mimc_witness(rounds, seed=20) with 2^log-size constraints, its
constraint system bb_synth_mimc_r1cs(rounds, 20) and Parameters.synthetic(worker, 21, shape).

The line holds
  value           device ms of one check with the witness in HBM (CUDA events of the profile mode, mean over K steps):
                  eval_ms (the a, b, c evaluation, csr_eval_queue) + compare_ms (k_r1cs_check);
  check_wall_ms   median host wall clock of one blocking check from HBM;
  compare_bytes, roofline   the bytes the compare must read (a, b, c: 3 n Fr) over compare_ms, against the HBM bandwidth;
  batch_hbm, batch_host     --batch B items (every fourth corrupted) from HBM and from pinned host memory: median wall ms
                  of the blocking batch call over K steps, per item, kernel launches and host-to-device bytes per item;
  r1cs_eval_ms    device ms of bb_r1cs_eval (witness and results in HBM), prove_ms the median wall ms of one
                  bb_groth16_prove_r1cs from HBM, and share_of_prove: the check, its compare pass alone and one batch
                  item as fractions of that proof;
  checks          a satisfied witness reports none; a witness corrupted at the first, middle and last aux index reports the
                  first failing row and the count of an evaluation of every row those variables touch in Python integers;
                  each batch item equals its single call (all asserted);
  gpu, clocks     card name, power limit and maximum SM clock (nvidia-smi), SM clock sampled during the timed legs.
Prints one JSON line on stdout; writes nothing else.
"""
import argparse
import importlib.util
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("bench_r1cs", os.path.join(ROOT, "bench_r1cs.py"))
br = importlib.util.module_from_spec(_spec)                 # gpu_info, roofline and time_eval of bench_r1cs.py
_spec.loader.exec_module(br)
bench = br.bench                                           # the clock sampler, emit / log and the HBM peak of bench.py

FR_MODULUS = bench.FR_MODULUS
R_INV = pow(1 << 256, -1, FR_MODULUS)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints (bench.py's MiMC workload)")
    ap.add_argument("--batch", type=int, default=64, help="items of the batch legs")
    return ap.parse_args()


def to_int(limbs):
    """Montgomery limbs -> the canonical integer"""
    return (int(limbs[0]) | int(limbs[1]) << 64 | int(limbs[2]) << 128 | int(limbs[3]) << 192) * R_INV % FR_MODULUS


def to_mont(v):
    m = v * (1 << 256) % FR_MODULUS
    return np.array([(m >> (64 * j)) & ((1 << 64) - 1) for j in range(4)], np.uint64)


def expected_unsat(mats, n_inputs, inputs, aux, changed_vars):
    """(first, count) for a witness that differs from a satisfying one only at `changed_vars`: the rows reading them,
    evaluated in Python integers"""
    rows = set()
    for off, var, _ in mats:
        for v in changed_vars:
            rows.update((np.searchsorted(off, np.nonzero(var == v)[0], side="right") - 1).tolist())
    z = lambda v: to_int(inputs[v] if v < n_inputs else aux[v - n_inputs])
    bad = []
    for k in sorted(rows):
        a, b, c = (sum(to_int(cf[t]) * z(int(var[t])) for t in range(int(off[k]), int(off[k + 1]))) % FR_MODULUS for off, var, cf in mats)
        if a * b % FR_MODULUS != c:
            bad.append(k)
    return (bad[0] if bad else None, len(bad))


def pinned(shape):
    import torch
    return torch.zeros(shape, dtype=torch.int64).pin_memory()


def median_ms(fn, args):
    for _ in range(args.warmup):
        fn()
    ts = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def run(args):
    import bellman_b200 as bb
    from bellman_b200 import r1cs as RC
    log_n, B = args.log_size, args.batch
    rounds = (1 << (log_n - 1)) - 1
    worker = bb.Worker(0)
    bench.log("synthesising the MiMC-chain witness and its constraint system (CPU, product-side generator)")
    asg, shape = bb.synth_mimc(rounds, seed=20, pinned=True)
    n = shape["num_constraints"]
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    assert r1cs.n_constraints == n == 1 << log_n
    ni, na = r1cs.n_inputs, r1cs.n_aux
    params = bb.Parameters.synthetic(worker, 21, shape)
    inp, aux = asg.input_assignment, asg.aux_assignment
    dev = {"inputs": worker.device_alloc(inp.nbytes), "aux": worker.device_alloc(aux.nbytes)}
    worker.upload(dev["inputs"], inp)
    worker.upload(dev["aux"], aux)
    peak_gbs, peak_src = bench.peaks()

    # the checks: satisfied, then corrupted at the first, middle and last aux index
    mats = RC.synth_mimc_matrices(rounds, 20)
    first, count, bits = r1cs.unsatisfied(dev["inputs"], dev["aux"], on_device=True, bits=True)
    satisfied_ok = (first, count, bool(bits.any())) == (None, 0, False) and r1cs.unsatisfied(inp, aux) == (None, 0)
    idx = (0, na // 2, na - 1)
    bad = aux.copy()
    for j in idx:
        bad[j] = to_mont((to_int(aux[j]) + 1) % FR_MODULUS)
    want_bad = expected_unsat(mats, ni, inp, bad, [ni + j for j in idx])
    d_bad = worker.device_alloc(bad.nbytes)
    worker.upload(d_bad, bad)
    corrupted_ok = (want_bad[1] > 0 and r1cs.unsatisfied(inp, bad) == want_bad
                    and r1cs.unsatisfied(dev["inputs"], d_bad, on_device=True) == want_bad)
    worker.device_free(d_bad)

    # one check from HBM: device stages (profile mode), then wall clock
    for _ in range(args.warmup):
        r1cs.unsatisfied(dev["inputs"], dev["aux"], on_device=True)
    worker.set_option("profile", 1)
    worker.profile_reset()
    for _ in range(args.steps):
        r1cs.unsatisfied(dev["inputs"], dev["aux"], on_device=True)
    eval_ms = worker.profile_read("r1cs_check.eval")[0] / args.steps
    compare_ms = worker.profile_read("r1cs_check.compare")[0] / args.steps
    worker.set_option("profile", 0)
    sampler = bench.ClockSampler(0)
    sampler.start()
    check_wall = median_ms(lambda: r1cs.unsatisfied(dev["inputs"], dev["aux"], on_device=True), args)

    # the batch legs: B items, every fourth one corrupted at an aux index of its own
    bench.log(f"batch legs: {B} items of {(ni + na) * 32 / 2**20:.1f} MB")
    t_in, t_aux = pinned((B, ni, 4)), pinned((B, na, 4))
    b_in, b_aux = t_in.numpy().view(np.uint64), t_aux.numpy().view(np.uint64)
    b_in[:] = inp
    b_aux[:] = aux
    for i in range(1, B, 4):
        j = (i * 7919) % na
        b_aux[i, j] = to_mont((to_int(aux[j]) + 1) % FR_MODULUS)
    bdev = {"inputs": worker.device_alloc(b_in.nbytes), "aux": worker.device_alloc(b_aux.nbytes)}
    worker.upload(bdev["inputs"], b_in)
    worker.upload(bdev["aux"], b_aux)
    singles = [r1cs.unsatisfied(b_in[i], b_aux[i]) for i in range(B)]
    legs = {"hbm": lambda: RC.check_r1cs_batch(r1cs, None, None, count=B, device_ptrs=bdev),
            "host": lambda: RC.check_r1cs_batch(r1cs, b_in, b_aux)}
    batch, batch_ok = {}, sum(f is not None for f, _ in singles) == len(range(1, B, 4))
    for leg, fn in legs.items():
        l0, (h0, _) = worker.kernel_launches, worker.bytes_copied()
        batch_ok &= fn() == singles
        launches, h2d = worker.kernel_launches - l0, worker.bytes_copied()[0] - h0
        ms = median_ms(fn, args)
        batch[leg] = {"items": B, "ms": ms, "ms_per_item": ms / B, "launches_per_item": launches / B, "h2d_bytes_per_item": h2d // B}

    # the references in the same run: bb_r1cs_eval alone, and one proof from the witness in HBM
    outs = {k: worker.device_alloc(n * 32) for k in "abc"}
    r1cs_eval_ms = br.time_eval(args, worker, r1cs, dev["inputs"], dev["aux"], outs)
    r, s = 0x1234567, 0x7654321
    prove_ms = median_ms(lambda: RC.create_proof_r1cs(r1cs, params, None, None, r, s, device_ptrs=dev), args)
    clocks = sampler.stop()

    check_ms = eval_ms + compare_ms
    compare_bytes = 3 * n * 32
    checks = {"satisfied": "equal" if satisfied_ok else "DIFFERENT", "corrupted": "equal" if corrupted_ok else "DIFFERENT",
              "batch": "equal" if batch_ok else "DIFFERENT"}
    share = lambda ms: ms / prove_ms if prove_ms > 0 else None
    line = {"metric": "r1cs_check_ms", "value": check_ms, "unit": "ms", "lower_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup,
            "config": {"workload": f"mimc-2^{log_n}", "constraints": n, "rounds": rounds, "batch": B,
                       "witness": "bb_synth_mimc_witness(rounds, 20); constraint system bb_synth_mimc_r1cs(rounds, 20)",
                       "key": "Parameters.synthetic(worker, 21, shape); default MSM form",
                       "timing": "value, eval_ms, compare_ms, r1cs_eval_ms: CUDA events (profile mode), mean over K steps; "
                                 "*_wall / batch / prove: host wall clock around blocking calls, median over K steps"},
            "eval_ms": eval_ms, "compare_ms": compare_ms, "check_wall_ms": check_wall,
            "compare_bytes": compare_bytes, "compare_bytes_model": "a, b, c read once: 3 n x 32 B (no atomics when satisfied)",
            "roofline": dict(br.roofline(compare_bytes, compare_ms, peak_gbs), peak_source=peak_src),
            "batch_hbm": batch["hbm"], "batch_host": batch["host"],
            "r1cs_eval_ms": r1cs_eval_ms, "prove_ms": prove_ms,
            "share_of_prove": {"check": share(check_ms), "compare_pass": share(compare_ms),
                               "batch_hbm_item": share(batch["hbm"]["ms_per_item"])},
            "corrupted": {"aux_indices": list(idx), "first": want_bad[0], "count": want_bad[1]},
            "checks": checks, "gpu": br.gpu_info(), "clocks": clocks}
    bench.emit(line)
    assert checks == {"satisfied": "equal", "corrupted": "equal", "batch": "equal"}, checks
    for p in (*outs.values(), *dev.values(), *bdev.values()):
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
