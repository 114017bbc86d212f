#!/usr/bin/env python
"""Device time per kernel of the flagship prove (bench.py's 2^20-constraint MiMC chain on one GPU).

Builds the same synthetic key and witness as bench.py (seeds 20 and 21, r and s as there), selects the MSM form -- by
the per-key tuner in this process (default), by index (--form, see bellman_b200.tuning_names()) or by msm_precompute
(--precompute) -- proves --warm times, then records --proofs proofs under torch.profiler with CUDA activities.
Prints the device time per proof of every kernel (template arguments shortened to the field) and of the stages the
kernels belong to, and writes the Chrome trace and the tables under --out.

The kernels of one prove run on several streams at once, so the sum of their device times exceeds the wall time of a
proof; the table says where the device's time goes, not what is on the critical path.

    python tools/prove_kernel_profile.py --out bench_out/profile
"""
import argparse
import collections
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = [                                   # (stage, kernel-name pattern), first match wins
    ("halving rounds: phase 1", r"^k_aff_phase1"),
    ("halving rounds: phase 3", r"^k_aff_phase3"),
    ("halving rounds: batch inversion", r"^k_binv_"),
    ("digits / sort / scan", r"^k_(msm_digits|scan_|size_|dense_offsets|msm_classify)"),
    ("XYZZ accumulation", r"^k_msm_(accumulate|merge_big|sum_list)"),
    ("bucket reduction", r"^k_(bucket_fold|msm_reduce|msm_level_sums|point_tree_sum|msm_fold_slots)"),
    ("NTT and H pipeline", r"^k_ntt"),
]


def short_name(name):
    """'void bb::k_aff_phase3<bb::Fe<bb::FpCfg>, true>(...)' -> 'k_aff_phase3<Fp, true>'"""
    m = re.search(r"(k_\w+)(<[^()]*>)?\(", name)
    if not m:
        return name[:80]
    targs = (m.group(2) or "").replace("bb::Fe<bb::FpCfg>", "Fp").replace("bb::Fe<bb::FrCfg>", "Fr").replace("bb::", "")
    return m.group(1) + targs


def stage_of(kernel):
    for stage, pat in STAGES:
        if re.search(pat, kernel):
            return stage
    return "other"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints (bench.py: 20)")
    ap.add_argument("--form", type=int, default=None, help="MSM form index to apply instead of running the tuner")
    ap.add_argument("--precompute", type=int, default=None, help="msm_precompute option instead of running the tuner")
    ap.add_argument("--warm", type=int, default=3, help="proofs before the profiled ones")
    ap.add_argument("--proofs", type=int, default=3, help="profiled proofs")
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "prove_kernel_profile"))
    args = ap.parse_args()
    if args.warm < 1 or args.proofs < 1:
        ap.error("--warm and --proofs must be at least 1")

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bellman_b200 as bb

    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    worker = bb.Worker(0)
    if args.precompute is not None:
        worker.set_option("msm_precompute", args.precompute)
    rounds = (1 << (args.log_size - 1)) - 1
    asg, shape = bb.synth_mimc(rounds, seed=20, pinned=True)
    params = bb.Parameters.synthetic(worker, 21, shape)
    r, s = 0x1234567, 0x7654321
    keep, dev = [], {}
    for name, arr in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
        t = torch.from_numpy(arr.view(np.int64)).to("cuda:0")
        keep.append(t)
        dev[name] = t.data_ptr()
    torch.cuda.synchronize()

    form = None
    if args.form is not None:
        params.apply_tuning(args.form)
        form = {"chosen": args.form, "name": bb.tuning_names()[args.form]}
    elif args.precompute is None:
        form = params.autotune(asg, reps=1, device_ptrs=dev)
    print(f"MSM form: {form if form else 'msm_precompute=%d' % args.precompute}", flush=True)

    for _ in range(args.warm):
        proof = bb.create_proof(asg, params, r, s, dev)
    worker.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.warm):
        bb.create_proof(asg, params, r, s, dev)
    worker.synchronize()
    wall_ms = 1e3 * (time.perf_counter() - t0) / args.warm

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.proofs):
            assert bb.create_proof(asg, params, r, s, dev) == proof
        worker.synchronize()
        torch.cuda.synchronize()
    trace = os.path.join(args.out, "prove.pt.trace.json")
    prof.export_chrome_trace(trace)

    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    per_kernel = collections.defaultdict(lambda: [0.0, 0])
    for e in events:
        if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset"):
            key = short_name(e["name"]) if e["cat"] == "kernel" else e["cat"]
            per_kernel[key][0] += e.get("dur", 0.0) / 1e3 / args.proofs
            per_kernel[key][1] += 1
    total = sum(v[0] for v in per_kernel.values())
    per_stage = collections.defaultdict(float)
    for k, (ms, _) in per_kernel.items():
        per_stage[stage_of(k) if k.startswith("k_") else "copies / memsets"] += ms

    dev_name = torch.cuda.get_device_name(0)
    lines = [f"device: {dev_name}; form: {form['name'] if form else 'msm_precompute=%d' % args.precompute}; "
             f"{wall_ms:.2f} ms per proof without the profiler (mean of {args.warm}); {args.proofs} proofs profiled",
             f"device time per proof, summed over streams: {total:.2f} ms", "",
             f"{'stage':<36} {'ms/proof':>9} {'share':>7}"]
    for stage, ms in sorted(per_stage.items(), key=lambda kv: -kv[1]):
        lines.append(f"{stage:<36} {ms:9.3f} {100 * ms / total:6.1f}%")
    lines += ["", f"{'kernel':<48} {'ms/proof':>9} {'launches':>9} {'share':>7}"]
    for k, (ms, n) in sorted(per_kernel.items(), key=lambda kv: -kv[1][0]):
        lines.append(f"{k:<48} {ms:9.3f} {n // args.proofs:9d} {100 * ms / total:6.1f}%")
    text = "\n".join(lines)
    print(text)
    with open(os.path.join(args.out, "kernels.txt"), "w") as f:
        f.write(text + "\n")
    with open(os.path.join(args.out, "kernels.json"), "w") as f:
        json.dump({"device": dev_name, "form": form, "wall_ms_per_proof": wall_ms, "device_ms_per_proof": total,
                   "stages": per_stage, "kernels": {k: {"ms_per_proof": v[0], "launches": v[1] // args.proofs} for k, v in per_kernel.items()}},
                  f, indent=1)
    worker.close()


if __name__ == "__main__":
    main()
