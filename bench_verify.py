#!/usr/bin/env python
"""bench_verify.py -- Groth16 batch verification throughput on H100 (batch::Verifier::verify,
groth16/src/verifier/batch.rs:100-173, through bb_groth16_verify_batch).

    python bench_verify.py --steps K --warmup W [--log-size 12] [--inputs 7] [--dump-outputs DIR]

A step verifies one batch of 2^log-size synthetic proofs with --inputs public inputs each.  The proofs come from
bb_synth_proof_batch (trapdoor scalars, fixed-base multiplications on the device) before the timed region, and the
random z_i from a seeded generator, so every run sees the same batch.  `value` is proofs/s with the batch resident in
HBM, `e2e` the same batch from pinned host buffers.  Outside the timed regions the script asserts that the batch is
accepted and that the same batch with C_0 replaced by C_1 is rejected.  The line carries the per-stage device
milliseconds (CUDA events of the library's profile mode) and the Fp-multiplication rate of the Miller loops.

--from-bytes adds a `from_bytes` object: proofs/s of decode + verify with the batch as 192-byte Proof::write encodings
in pinned host memory (bb_proofs_read into HBM, then the batch verifier), the decode.* stage milliseconds and the bytes
copied to the device per step.  Without it the line is exactly the one above.

--each adds an `each` object: proofs/s of bb_groth16_verify_each (verify_proof for every proof, one device call; the
fallback that finds the bad proofs of a rejected batch) on the same batch, in HBM and from the pinned host buffers, its
verify_each.* stage milliseconds (from a profiled pass of their own), the Fp multiplications per proof of its kernels, the milliseconds of the key's first
call (which builds the prepared lines and ic tables), and a check outside the timed regions: with C replaced at the first,
middle and last index exactly those three proofs are flagged.

--dump-outputs DIR writes the two verdicts and the G_T value of the rejected batch (deterministic under the seeded z)
as float64 .npy files, the format of bench.py --dump-outputs; with --each also verdicts_each, the per-proof verdicts of
that leg's check.  Prints one JSON line on stdout; writes nothing else.
"""
import argparse
import importlib.util
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

_spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(_spec)             # the clock sampler, emit / log and the dump format of bench.py
_spec.loader.exec_module(bench)

FR_MODULUS = bench.FR_MODULUS
DEFAULT_LOG = 12        # 4096 proofs: about the Sapling spend proofs of one full 2 MB Zcash block (384-byte spend descriptions)
DEFAULT_INPUTS = 7      # public inputs of a Sapling spend proof (rk, cv, anchor, nullifier as Fr elements)
FP_MUL_PEAK = 27.3      # G Fp-mul/s: tools/ubench.cu k_fmul<Fp>, best launch shape, H100 SXM 80 GB at a 700 W power limit


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device (multi-GPU verification is not implemented)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--log-size", type=int, default=DEFAULT_LOG, help="log2 of the proofs per batch")
    ap.add_argument("--inputs", type=int, default=DEFAULT_INPUTS, help="public inputs per proof")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write the verdicts and the rejected batch's G_T value as DIR/<name>.npy")
    ap.add_argument("--from-bytes", action="store_true",
                    help="also time decode + verify of the batch as 192-byte Proof::write encodings in pinned host memory (adds `from_bytes`)")
    ap.add_argument("--each", action="store_true",
                    help="also time verify_proof for every proof of the batch in one call, bb_groth16_verify_each (adds `each`)")
    return ap.parse_args()


def miller_fp_muls_per_pair():
    """Fp multiplications of one pair's Miller loop in csrc/tower.cuh, from its step counts: an Fp2 product costs 3 Fp
    products, an Fp2 squaring or an Fp2 x Fp product 2."""
    fp12_sqr = 2 * 6 * 3                                    # two Fp6 products of 6 Fp2 products
    mul_line = 15 * 3                                       # fp12_mul_line: 15 Fp2 products
    dbl = 5 * 2 + 3 * 2 + 4 * 3                             # miller_dbl_step: 5 Fp2 squarings, 3 Fp2 x Fp, 4 Fp2 products
    add = 11 * 3 + 3 * 2 + 2 * 2                            # miller_add_step: 11 Fp2 products, 3 Fp2 x Fp, 2 Fp2 squarings
    return 63 * (fp12_sqr + dbl + mul_line) + 5 * (add + mul_line)


def each_fp_muls_per_proof(n_inputs):
    """Fp multiplications of one proof in bb_groth16_verify_each, counted as miller_fp_muls_per_pair counts them (an Fp2
    product 3, an Fp2 squaring or Fp2 x Fp product 2; inversions by fp_inv_gcd not counted)"""
    fp12_sqr, mul_line, dbl, add = 36, 45, 28, 43
    stored_line = 3 * 2 + mul_line                          # a stored line at P: 3 Fp2 x Fp products, then the sparse product
    psi = n_inputs * 32 * 10 + 3                            # k_each_psi: mixed XYZZ additions (8 products, 2 squarings), G1Eval
    miller = 63 * (fp12_sqr + dbl + mul_line + 2 * stored_line) + 5 * (add + mul_line + 2 * stored_line)
    fp12_mul, cyc_sqr, frob1, frob2, inv = 54, 18, 15, 30, 109
    exp_x = 63 * cyc_sqr + 5 * fp12_mul
    final_exp = (inv + fp12_mul + frob2 + fp12_mul                                  # easy part
                 + 5 * exp_x + 2 * fp12_mul + fp12_mul + frob1                        # five x-powers; (x - 1)^2; x + p
                 + 2 * fp12_mul + frob2 + 2 * fp12_mul + cyc_sqr                      # x^2 + p^2 - 1; t^3
                 + 24)                                                                # the canonical comparison
    return {"psi": psi, "miller": miller, "final_exp": final_exp, "total": psi + miller + final_exp}


EACH_STAGES = ("upload", "psi", "miller", "final_exp", "download")


def each_leg(args, worker, pvk, d, host, timed):
    """--each: bb_groth16_verify_each on the timed batch, from HBM and from the pinned host buffers.  Outside the timed
    regions: the key's first call (it builds the prepared lines and ic tables), and C replaced at the first, middle and
    last index, which must flag exactly those three."""
    from bellman_b200 import verifier as V
    n, L = host["a"].shape[0], args.inputs
    t0 = time.perf_counter()
    first = V.verify_each_arrays(pvk, d["a"], d["b"], d["c"], d["x"], on_device=True, n=n, n_inputs=L)
    first_ms = 1e3 * (time.perf_counter() - t0)

    def step_value():
        V.verify_each_arrays(pvk, d["a"], d["b"], d["c"], d["x"], on_device=True, n=n, n_inputs=L)

    def step_e2e():
        V.verify_each_arrays(pvk, host["a"], host["b"], host["c"], host["x"], n_inputs=L)

    dt, launches, _ = timed(step_value)
    dt_e2e, _, h2d = timed(step_e2e)
    worker.set_option("profile", 1)                         # the stages in a run of their own: the timings above are unprofiled
    timed(step_value)
    stages = {s: worker.profile_read("verify_each." + s)[0] / args.steps for s in EACH_STAGES}
    worker.set_option("profile", 0)
    bad = sorted({0, n // 2, n - 1})
    c_bad = host["c"].copy()
    for pos in bad:
        c_bad[pos] = host["c"][(pos + 1) % n]
    verdicts = V.verify_each_arrays(pvk, host["a"], host["b"], c_bad, host["x"], n_inputs=L)     # n_invalid is checked there
    flagged = np.flatnonzero(verdicts).tolist()
    checks = {"flagged": "first, middle, last" if flagged == bad and not first.any() else f"{flagged} (timed batch: {np.flatnonzero(first).tolist()})",
              "n_invalid": int(np.count_nonzero(verdicts))}
    return {"value": n * args.steps / dt, "unit": "proofs/s", "ms_per_step": 1e3 * dt / args.steps, "gpu_launches": int(launches),
            "e2e": {"value": n * args.steps / dt_e2e, "unit": "proofs/s", "ms_per_step": 1e3 * dt_e2e / args.steps, "h2d_bytes_per_step": int(h2d)},
            "stages_ms_per_step": {k: round(v, 3) for k, v in stages.items()},
            "fp_mul_per_proof": each_fp_muls_per_proof(L), "first_call_ms": round(first_ms, 3),
            "source": "the timed batch; step = bb_groth16_verify_each (verdicts for every proof, no z)",
            "checks": checks}, verdicts


DECODE_STAGES = ("decode.upload", "decode.g1", "decode.g2", "decode.status", "decode.download")


def from_bytes_leg(args, worker, pvk, d, host, z, timed):
    """--from-bytes: the batch as n x 192 bytes (bb_proofs_write on the device) in pinned host memory; a step is one
    bb_proofs_read into device buffers plus the batch verification of the decoded points.  Outside the timed region: the
    decoded points equal the synthetic batch, and one flipped x byte of B at the middle proof is reported there."""
    import torch

    from bellman_b200 import verifier as V
    n, L = host["a"].shape[0], args.inputs
    d_bytes = worker.device_alloc(n * 192)
    V.write_proofs_device(worker, d["a"], d["b"], d["c"], n, d_bytes)
    keep = torch.zeros(n * 192, dtype=torch.uint8).pin_memory()
    data = keep.numpy()
    worker.download(d_bytes, data)
    worker.device_free(d_bytes)
    out = {k: worker.device_alloc(n * w * 8) for k, w in (("a", 12), ("b", 24), ("c", 12))}
    dev = (out["a"], out["b"], out["c"])

    def step_bytes():
        _, _, _, status = V.read_proofs(worker, data, n=n, out_device=dev)
        if status.any():
            raise AssertionError(f"{int((status != 0).sum())} proofs of the timed batch do not read")
        V.verify_batch_arrays(pvk, *dev, d["x"], z=z, on_device=True, n=n, n_inputs=L)

    worker.set_option("profile", 1)
    dt, _, h2d = timed(step_bytes)
    decode = {s.split(".")[1]: worker.profile_read(s)[0] / args.steps for s in DECODE_STAGES}
    worker.set_option("profile", 0)
    same = True
    for key, w in (("a", 12), ("b", 24), ("c", 12)):
        got = np.zeros((n, w), np.uint64)
        worker.download(out[key], got)
        same = same and np.array_equal(got, host[key])
    mid = n // 2
    bad = data.copy()
    bad[192 * mid + 48 + 95] ^= 1                               # the last byte of x.c0 of B
    _, _, _, status = V.read_proofs(worker, bad, n=n)
    flagged = np.flatnonzero(status)
    reported = flagged.tolist() == [mid] and int(status[mid]) >> 4 == 2
    for p in out.values():
        worker.device_free(p)
    return {"value": n * args.steps / dt, "unit": "proofs/s", "ms_per_step": 1e3 * dt / args.steps,
            "decode_ms": round(sum(decode.values()), 3), "decode_stages_ms": {k: round(v, 3) for k, v in decode.items()},
            "h2d_bytes_per_step": int(h2d),
            "source": "the timed batch as Proof::write bytes (bb_proofs_write on the device) in pinned host memory; "
                      "step = bb_proofs_read into HBM + bb_groth16_verify_batch on the decoded points",
            "checks": {"decoded_points": "equal" if same else "DIFFERENT", "corrupted_b_at_middle": "reported" if reported else "MISSED"},
            "corrupted": {"index": mid, "status": int(status[mid])}}


def run(args):
    import torch

    import bellman_b200 as bb
    from bellman_b200 import verifier as V
    log_n, L = args.log_size, args.inputs
    if L < 0:
        raise SystemExit("--inputs must be >= 0")
    n = 1 << log_n
    worker = bb.Worker(0)
    bench.log(f"generating {n} synthetic proofs with {L} public inputs on the device")
    d = {"a": worker.device_alloc(n * 96), "b": worker.device_alloc(n * 192), "c": worker.device_alloc(n * 96),
         "x": worker.device_alloc(max(1, n * L) * 32)}
    vk = V.synth_proof_batch(worker, 51, n, L, d["a"], d["b"], d["c"], d["x"])
    pvk = bb.prepare_verifying_key(worker, vk)

    keep, host = [], {}                                     # the same batch in page-locked host memory (e2e leg)
    for key, shape in (("a", (n, 12)), ("b", (n, 24)), ("c", (n, 12)), ("x", (n, L, 4))):
        t = torch.zeros(shape, dtype=torch.int64).pin_memory()
        keep.append(t)
        arr = t.numpy().view(np.uint64)
        if arr.size:
            worker.download(d[key], arr)
        host[key] = arr
    rng = random.Random(52)
    z = [rng.randrange(1, FR_MODULUS) for _ in range(n)]

    def step_value():
        V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=z, on_device=True, n=n, n_inputs=L)

    def step_e2e():
        V.verify_batch_arrays(pvk, host["a"], host["b"], host["c"], host["x"], z=z, n_inputs=L)

    def timed(step):
        for _ in range(args.warmup):
            step()
        worker.synchronize()
        worker.profile_reset()
        l0 = worker.kernel_launches
        h0, _ = worker.bytes_copied()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step()
        worker.synchronize()
        dt = time.perf_counter() - t0
        h1, _ = worker.bytes_copied()
        return dt, worker.kernel_launches - l0, (h1 - h0) / args.steps

    bench.log("timed region: batch resident in HBM")
    sampler = bench.ClockSampler(0)
    sampler.start()
    worker.set_option("profile", 1)
    dt_val, launches, _ = timed(step_value)
    clocks = sampler.stop()
    stage = lambda *names: sum(worker.profile_read(nm)[0] for nm in names) / args.steps
    stages = {"accumulators": stage("verify.accumulators"), "scalar_mul": stage("verify.scalar_mul"),
              "msms": stage("msm_total_g1"), "msm_wait": stage("verify.msm_wait"),
              "miller": stage("verify.miller", "verify.miller_tail"), "product": stage("verify.product"),
              "final_exp": stage("verify.final_exp")}
    worker.set_option("profile", 0)
    bench.log(f"value leg: {1e3 * dt_val / args.steps:.2f} ms/step; timed region: pinned host buffers (e2e)")
    dt_e2e, _, h2d = timed(step_e2e)
    # outside the timed regions: the timed batch is accepted, and the same batch with C_0 replaced by C_1 is rejected
    ok, _ = V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=z, on_device=True, n=n, n_inputs=L, gt=True)
    c_bad = host["c"].copy()
    c_bad[0] = host["c"][1 % n]
    ok_bad, gt_bad = V.verify_batch_arrays(pvk, host["a"], host["b"], c_bad, host["x"], z=z, n_inputs=L, gt=True)
    checks = {"timed_batch": "accepted" if ok else "REJECTED", "one_c_replaced": "rejected" if not ok_bad else "ACCEPTED"}
    from_bytes = from_bytes_leg(args, worker, pvk, d, host, z, timed) if args.from_bytes else None
    each, verdicts_each = each_leg(args, worker, pvk, d, host, timed) if args.each else (None, None)
    per_pair = miller_fp_muls_per_pair()
    miller_ms = stages["miller"]
    line = {"metric": "groth16_batch_verify_proofs_per_sec", "value": n * args.steps / dt_val, "unit": "proofs/s", "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * dt_val / args.steps, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "u32 limbs (381-bit Fp / 255-bit Fr Montgomery integers)", "data": "synthetic",
            "config": {"workload": f"groth16-batch-verify-2^{log_n}", "proofs": n, "inputs_per_proof": L, "pairs": n + 3,
                       "proofs_source": "bb_synth_proof_batch: [a]G1, [b]G2, [c]G1 from trapdoor scalars, made on the device before the timed region",
                       "z": "seeded (random.Random(52)), canonical, uploaded each step",
                       "timing": "host wall clock over K steps bracketed by device synchronize; stages by CUDA events on the main stream "
                                 "(msms: the two MSM jobs on their own streams, summed)",
                       "checks": checks},
            "e2e": {"value": n * args.steps / dt_e2e, "unit": "proofs/s", "h2d_bytes_per_step": int(h2d), "ms_per_step": 1e3 * dt_e2e / args.steps},
            "gpu_launches": int(launches), "clocks": clocks,
            "stages_ms_per_step": {k: round(v, 3) for k, v in stages.items()},
            "fp_mul": {"per_pair_miller": per_pair, "unit": "G Fp-mul/s",
                       "miller_rate": (per_pair * (n + 3) / (miller_ms * 1e-3) / 1e9) if miller_ms > 0 else None,
                       "peak": FP_MUL_PEAK, "peak_source": "tools/ubench.cu k_fmul<Fp>, best launch shape, on an H100 SXM (80 GB HBM3, 700 W power limit)",
                       "model": "miller_fp_muls_per_pair(): 63 doubling and 5 addition steps of csrc/tower.cuh counted in Fp products"},
            "cpu_baseline": None,
            "cpu_baseline_reason": "oracle-1 has no CPU pairing; the Python pairing of oracle-0 is a correctness reference, not a timed baseline"}
    if from_bytes is not None:
        line["from_bytes"] = from_bytes
    if each is not None:
        line["each"] = each
    dumps = {"verdicts": np.array([int(ok), int(ok_bad)], np.uint32), "gt_tampered": gt_bad}
    if each is not None:
        dumps["verdicts_each"] = verdicts_each
    bench.dump_outputs(args.dump_outputs, dumps)
    bench.emit(line)
    assert ok and not ok_bad, checks
    if from_bytes is not None:
        assert from_bytes["checks"] == {"decoded_points": "equal", "corrupted_b_at_middle": "reported"}, from_bytes["checks"]
    if each is not None:
        assert each["checks"] == {"flagged": "first, middle, last", "n_invalid": 3}, each["checks"]
    pvk.free()
    for p in d.values():
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
