#!/usr/bin/env python
"""bench_r1cs.py -- proving from the witness alone: the constraint system on the device (bb_r1cs_eval,
bb_groth16_prove_r1cs) against bb_groth16_prove from a, b, c.

    python bench_r1cs.py --steps K --warmup W [--log-size 20] [--workload mimc|long-rows]

The key and witness are bench.py's: the MiMC chain of bb_synth_mimc_witness(rounds, seed=20) with 2^log-size constraints
and Parameters.synthetic(worker, 21, shape); the constraint system is bb_synth_mimc_r1cs(rounds, 20), the same circuit.
The MSM runs its default form in both paths (no per-key tuning), so the two legs differ only in where a, b, c come from.

The line holds
  value         r1cs.eval: device milliseconds of the evaluation (CUDA events of the profile mode), witness and
                results in HBM, mean over K steps;
  nnz, bytes, fr_products, roofline   the terms per matrix, the bytes the evaluation must move (the matrices once,
                z once, a, b, c written) and its Fr products (terms with a coefficient other than one), over the HBM
                bandwidth: the share of the HBM roofline;
  prove_hbm     median ms of a prove from the witness in HBM and of bb_groth16_prove from a, b, c and the witness in
                HBM, the two alternated step by step in one run;
  prove_host    the same pair from pinned host buffers;
  h2d_bytes_per_proof   bytes each host leg copies to the device per proof (bb_ctx_bytes_copied);
  checks        a, b, c, the densities and the 192 proof bytes of the two paths, compared (and asserted);
  gpu, clocks   card name, power limit and maximum SM clock (nvidia-smi), SM clock sampled during the timed legs.
--workload long-rows adds `long_rows`: an R1CS whose rows have 2^10 - 2^14 terms over the same witness, its eval time,
terms and roofline share, and a check of five rows (one of each length) against Python integers.
Prints one JSON line on stdout; writes nothing else.
"""
import argparse
import importlib.util
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(_spec)             # the clock sampler, emit / log and the HBM peak of bench.py
_spec.loader.exec_module(bench)

FR_MODULUS = bench.FR_MODULUS


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints (bench.py's MiMC workload)")
    ap.add_argument("--workload", choices=["mimc", "long-rows"], default="mimc",
                    help="long-rows: also time an R1CS of rows with 2^10 - 2^14 terms (adds `long_rows`)")
    return ap.parse_args()


def gpu_info():
    """card name, power limit and maximum SM clock, read in the run they describe"""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception:
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def eval_bytes(r1cs):
    """bytes one evaluation must move: per term its uint32 index and, unless the coefficient is one, its 32-byte
    coefficient; z read once; per row (3 n) a uint32 offset and row id, and the 32-byte result"""
    terms, unit = sum(r1cs.nnz), sum(r1cs.unit)
    return 4 * terms + 32 * (terms - unit) + 32 * (r1cs.n_inputs + r1cs.n_aux) + 3 * r1cs.n_constraints * (4 + 4 + 32)


def time_eval(args, worker, r1cs, d_in, d_aux, outs):
    """mean device ms of r1cs.eval over K steps after W warm-ups"""
    for _ in range(args.warmup):
        r1cs.eval(d_in, d_aux, on_device=True, out=outs)
    worker.set_option("profile", 1)
    worker.profile_reset()
    for _ in range(args.steps):
        r1cs.eval(d_in, d_aux, on_device=True, out=outs)
    ms = worker.profile_read("r1cs.eval")[0] / args.steps
    worker.set_option("profile", 0)
    return ms


def roofline(nbytes, ms, peak_gbs):
    achieved = nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None
    return {"bound": "hbm", "achieved_gbs": achieved, "peak_gbs": peak_gbs,
            "fraction": (achieved / peak_gbs) if achieved else None}


def long_rows_leg(args, worker, RC, z_in, z_aux, d_in, d_aux, peak_gbs):
    """rows of 2^10 .. 2^14 terms (cycling) over the MiMC witness: the one-warp and one-CTA kernels"""
    rng = np.random.default_rng(7)
    ni, na = z_in.shape[0], z_aux.shape[0]
    n_rows = max(5, 1 << max(0, args.log_size - 10))
    lengths = [1 << (10 + (i % 5)) for i in range(n_rows)]
    off = np.zeros(n_rows + 1, np.uint64)
    off[1:] = np.cumsum(lengths)
    terms = int(off[-1])
    var = rng.integers(0, ni + na, terms, dtype=np.uint32)
    coef = rng.integers(0, 1 << 63, (terms, 4), dtype=np.uint64)
    coef[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)                             # below r (its top limb is 0x73ed...)
    empty = (np.zeros(n_rows + 1, np.uint64), np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64))
    r1cs = RC.R1CS(worker, ni, na, (off, var, coef), empty, empty)
    n = r1cs.n_constraints
    outs = {k: worker.device_alloc(n * 32) for k in "abc"}
    ms = time_eval(args, worker, r1cs, d_in, d_aux, outs)
    a = np.zeros((n, 4), np.uint64)
    worker.download(outs["a"], a)
    for p in outs.values():
        worker.device_free(p)
    # five rows, one of each length, against Python integers (Montgomery: a = sum coef z R^-1)
    to_int = lambda row: int(row[0]) | int(row[1]) << 64 | int(row[2]) << 128 | int(row[3]) << 192
    z = np.concatenate([z_in, z_aux])
    r_inv = pow(1 << 256, -1, FR_MODULUS)
    ok = True
    for k in range(5):
        lo, hi = int(off[k]), int(off[k + 1])
        want = sum(to_int(coef[t]) * to_int(z[var[t]]) for t in range(lo, hi)) * r_inv % FR_MODULUS
        ok &= to_int(a[k]) == want
    nbytes = eval_bytes(r1cs)
    line = {"value": ms, "unit": "ms", "rows": n_rows, "row_terms": "2^10 .. 2^14, cycling", "terms": terms, "bytes": nbytes,
            "fr_products": terms, "roofline": roofline(nbytes, ms, peak_gbs), "checks": "equal" if ok else "DIFFERENT"}
    r1cs.free()
    return line


def run(args):
    import bellman_b200 as bb
    from bellman_b200 import r1cs as RC
    log_n = args.log_size
    rounds = (1 << (log_n - 1)) - 1
    worker = bb.Worker(0)
    bench.log("synthesising the MiMC-chain witness and its constraint system (CPU, product-side generator)")
    asg, shape = bb.synth_mimc(rounds, seed=20, pinned=True)
    n = shape["num_constraints"]
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    assert r1cs.n_constraints == n == 1 << log_n
    params = bb.Parameters.synthetic(worker, 21, shape)
    r, s = 0x1234567 % FR_MODULUS, 0x7654321 % FR_MODULUS
    dev = {}                                                # inputs resident in HBM for the `prove_hbm` leg
    for name, arr in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
        dev[name] = worker.device_alloc(arr.nbytes)
        worker.upload(dev[name], arr)
    peak_gbs, peak_src = bench.peaks()

    # the evaluation alone, witness and results in HBM
    outs = {k: worker.device_alloc(n * 32) for k in "abc"}
    eval_ms = time_eval(args, worker, r1cs, dev["inputs"], dev["aux"], outs)
    got = []
    for k in "abc":
        h = np.zeros((n, 4), np.uint64)
        worker.download(outs[k], h)
        got.append(h)
    for p in outs.values():
        worker.device_free(p)
    same_abc = all(np.array_equal(g, getattr(asg, k)) for g, k in zip(got, "abc"))
    same_dens = all(np.array_equal(g, getattr(asg, k)) for g, k in
                    zip(r1cs.density_words(), ("a_aux_density", "b_input_density", "b_aux_density")))

    # the two prove paths, alternated step by step: in HBM, then from pinned host buffers
    legs = {
        "hbm": (lambda: RC.create_proof_r1cs(r1cs, params, None, None, r, s, device_ptrs=dev),
                lambda: bb.create_proof(asg, params, r, s, dev)),
        "host": (lambda: RC.create_proof_r1cs(r1cs, params, asg.input_assignment, asg.aux_assignment, r, s),
                 lambda: bb.create_proof(asg, params, r, s)),
    }
    sampler = bench.ClockSampler(0)
    sampler.start()
    times, proofs, h2d = {}, {}, {}
    for leg, fns in legs.items():
        for fn in fns:
            for _ in range(args.warmup):
                fn()
        ts = ([], [])
        h = [0, 0]
        for _ in range(args.steps):
            for j, fn in enumerate(fns):
                h0, _ = worker.bytes_copied()
                t0 = time.perf_counter()
                proof = fn()
                ts[j].append(1e3 * (time.perf_counter() - t0))
                h[j] += worker.bytes_copied()[0] - h0
                proofs[(leg, j)] = proof
        times[leg] = {"from_witness_ms": float(np.median(ts[0])), "from_abc_ms": float(np.median(ts[1]))}
        h2d[leg] = (h[0] // args.steps, h[1] // args.steps)
    clocks = sampler.stop()
    same_proof = len(set(proofs.values())) == 1
    long_rows = (long_rows_leg(args, worker, RC, asg.input_assignment, asg.aux_assignment, dev["inputs"], dev["aux"], peak_gbs)
                 if args.workload == "long-rows" else None)

    nbytes = eval_bytes(r1cs)
    checks = {"a_b_c": "equal" if same_abc else "DIFFERENT", "densities": "equal" if same_dens else "DIFFERENT",
              "proof": "equal" if same_proof else "DIFFERENT"}
    line = {"metric": "r1cs_eval_ms", "value": eval_ms, "unit": "ms", "lower_is_better": True, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup,
            "config": {"workload": f"mimc-2^{log_n}" + (" + long-rows" if long_rows else ""), "constraints": n, "rounds": rounds,
                       "witness": "bb_synth_mimc_witness(rounds, 20); constraint system bb_synth_mimc_r1cs(rounds, 20)",
                       "key": "Parameters.synthetic(worker, 21, shape); default MSM form",
                       "timing": "value: CUDA events around the evaluation kernels (profile mode), mean over K steps; prove legs: host "
                                 "wall clock around each blocking prove, median over K steps, the two paths alternated"},
            "nnz": dict(zip("abc", r1cs.nnz)), "unit_coefficients": dict(zip("abc", r1cs.unit)),
            "bytes": nbytes, "bytes_model": "4 per term + 32 per coefficient other than one + 32 per witness value (z read once) "
                                             "+ 40 per row of the three matrices (offset, row id, result)",
            "fr_products": sum(r1cs.nnz) - sum(r1cs.unit),
            "roofline": dict(roofline(nbytes, eval_ms, peak_gbs), peak_source=peak_src),
            "prove_hbm": times["hbm"], "prove_host": times["host"],
            "h2d_bytes_per_proof": {"from_witness": int(h2d["host"][0]), "from_abc": int(h2d["host"][1]),
                                    "hbm_legs": [int(h2d["hbm"][0]), int(h2d["hbm"][1])]},
            "checks": checks, "proof_sha256_prefix": __import__("hashlib").sha256(proofs[("hbm", 0)]).hexdigest()[:16],
            "gpu": gpu_info(), "clocks": clocks}
    if long_rows is not None:
        line["long_rows"] = long_rows
    bench.emit(line)
    assert checks == {"a_b_c": "equal", "densities": "equal", "proof": "equal"}, checks
    assert long_rows is None or long_rows["checks"] == "equal", long_rows
    r1cs.free()
    params.free()
    for p in dev.values():
        worker.device_free(p)
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
