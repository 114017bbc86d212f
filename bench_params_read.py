"""Key loading benchmark: Parameters::read of a key file on the device (params_io.read_parameters_device, bb_params_read)
against the host reader feeding an upload (Parameters(worker, params_io.read_parameters(data, checked))).

The key has the shape bench.py proves (bb_synth_mimc_shape at 2^--log-size constraints); its points are [k_i]G for
seeded k_i (bb_fixed_base_mul), written with params_io.write_parameters outside the timed region.
JSON fields, per mode (checked, unchecked): pinned / pageable / hbm (the new reader from page-locked host memory, pageable
host memory and HBM) and old (the host reader + upload), each {ms, gb_per_s of file}, mean over --steps after --warmup,
the legs alternated within each step (the old path runs --old-steps times); stages_ms: params.upload / params.g1 /
params.g2 of one profiled read from pinned memory.  checks: vectors (every resident vector and vk point of the new key
equals the old key's, through bb_diag_crs_download), proofs (one proof from each key, same bytes), corrupt_b_g2_middle (a
point outside the subgroup in the middle of b_g2 is reported at that section and index).  gpu: card name, power limit,
maximum and current SM clock, read in the same run.  Writes nothing to the tree."""
import argparse
import ctypes as C
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bellman_b200 as bb  # noqa: E402
from bellman_b200 import params_io as PIO  # noqa: E402

P = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--old-steps", type=int, default=1, help="runs of the host reader per mode")
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints")
    return ap.parse_args()


def key_shape(log_size):
    rounds = (1 << (log_size - 1)) - 1
    shape = np.zeros(7, np.uint64)
    bb._check(bb.load_library().bb_synth_mimc_shape(C.c_size_t(rounds), bb._ptr(shape)))
    ni, na = int(shape[0]), int(shape[1])
    return rounds, dict(ic=ni, h=int(shape[3]) - 1, l=na, a=ni + int(shape[4]), b=int(shape[5]) + int(shape[6]))


def make_key_file(worker, log_size, seed=1):
    """the bytes of a Parameters file of bench.py's shape: seeded [k_i]G points (not a trapdoor key)"""
    _, n = key_shape(log_size)
    rng = np.random.default_rng(seed)

    def pts(group, count):
        k = rng.integers(0, 2**63, size=(count, 4), dtype=np.uint64)
        k[:, 3] &= np.uint64((1 << 62) - 1)                    # below r
        k[:, 0] |= np.uint64(1)                                # not zero
        return bb.fixed_base_mul(worker, group, k, bb.FORM_CANONICAL) if count else np.zeros((0, 12 if group == bb.G1 else 24), np.uint64)

    p = dict(vk_g1=pts(bb.G1, 3), vk_g2=pts(bb.G2, 3), ic=pts(bb.G1, n["ic"]), h=pts(bb.G1, n["h"]), l=pts(bb.G1, n["l"]),
             a=pts(bb.G1, n["a"]), b_g1=pts(bb.G1, n["b"]), b_g2=pts(bb.G2, n["b"]))
    return PIO.write_parameters(p)


# a point of E'(Fp2) outside the order-r subgroup: a random x whose x^3 + 4(u + 1) is a square (the cofactor is ~2^254)
def _f2mul(a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P)


def _f2pow(a, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = _f2mul(r, a)
        a = _f2mul(a, a)
        e >>= 1
    return r


def off_subgroup_g2_bytes(seed=3):
    rng = random.Random(seed)
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        a = _f2mul(_f2mul(x, x), x)
        a = ((a[0] + 4) % P, (a[1] + 4) % P)
        a1 = _f2pow(a, (P - 3) // 4)                          # eprint 2012/685, Algorithm 9
        alpha = _f2mul(_f2mul(a1, a1), a)
        x0 = _f2mul(a1, a)
        y = (-x0[1] % P, x0[0]) if alpha == (P - 1, 0) else _f2mul(_f2pow(((1 + alpha[0]) % P, alpha[1]), (P - 1) // 2), x0)
        if _f2mul(y, y) == a:
            return b"".join(v.to_bytes(48, "big") for v in (x[1], x[0], y[1], y[0]))


def b_g2_middle(data):
    """offset and index of the middle point of b_g2"""
    off = 864
    for k in range(6):                                        # ic, h, l, a, b_g1, b_g2
        n = int.from_bytes(data[off:off + 4], "big")
        start = off + 4
        size = 192 if k == 5 else 96
        off = start + n * size
    return start + (n // 2) * 192, n // 2


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    args = parse()
    sys.stdout.flush()
    real = os.dup(1)                # exactly one JSON line on stdout; library chatter goes to stderr
    os.dup2(2, 1)
    import torch
    from bench_prove_batch import gpu_info
    worker = bb.Worker(0)
    rounds, _ = key_shape(args.log_size)
    data = make_key_file(worker, args.log_size)
    nbytes = len(data)
    pin_t = torch.frombuffer(bytearray(data), dtype=torch.uint8).pin_memory()
    pinned = pin_t.numpy()
    pageable = np.frombuffer(data, np.uint8)
    d_file = worker.device_alloc(nbytes)
    worker.upload(d_file, pageable)
    legs = {"pinned": pinned, "pageable": pageable, "hbm": (d_file, nbytes)}
    res = {"metric": "params_read_ms", "config": {"log_size": args.log_size, "constraints": 1 << args.log_size, "file_bytes": nbytes,
                                                  "steps": args.steps, "warmup": args.warmup, "old_steps": args.old_steps}}
    gbps = lambda ms: nbytes / (ms * 1e-3) / 1e9 if ms > 0 else None
    for mode, checked in (("checked", True), ("unchecked", False)):
        times = {k: [] for k in (*legs, "old")}
        for step in range(args.warmup + args.steps):
            for leg, src in legs.items():
                ms, params = timed(lambda: PIO.read_parameters_device(worker, src, checked=checked))
                params.free()
                if step >= args.warmup:
                    times[leg].append(ms)
            if step >= args.warmup and len(times["old"]) < args.old_steps:
                ms, params = timed(lambda: bb.Parameters(worker, PIO.read_parameters(data, checked=checked, worker=worker)))
                params.free()
                times["old"].append(ms)
        m = {leg: {"ms": float(np.mean(v)), "gb_per_s": gbps(float(np.mean(v)))} for leg, v in times.items()}
        worker.set_option("profile", 1)
        worker.profile_reset()
        PIO.read_parameters_device(worker, pinned, checked=checked).free()
        m["stages_ms"] = {s: worker.profile_read(s)[0] for s in ("params.upload", "params.g1", "params.g2")}
        worker.set_option("profile", 0)
        res[mode] = m
    res["value"] = res["checked"]["pinned"]["ms"]

    # checks: the resident points, one proof from each key, a corrupted b_g2
    new = PIO.read_parameters_device(worker, pinned, checked=True)
    old = bb.Parameters(worker, PIO.read_parameters(data, checked=False, worker=worker))
    a, b = PIO.download_parameters(new), PIO.download_parameters(old)
    same = new.lens == old.lens and all(np.array_equal(a[k], b[k]) for k in a)
    asg, _ = bb.synth_mimc(rounds, seed=11)
    r, s = 0x1234567, 0x7654321
    proofs_same = bb.create_proof(asg, new, r, s) == bb.create_proof(asg, old, r, s)
    new.free()
    old.free()
    off, idx = b_g2_middle(data)
    bad = data[:off] + off_subgroup_g2_bytes() + data[off + 192:]
    try:
        PIO.read_parameters_device(worker, bad, checked=True).free()
        reported = None
    except PIO.InvalidData as e:
        reported = (e.section, e.index, e.why)
    res["checks"] = {"vectors": "equal" if same else "DIFFERENT", "proofs": "equal" if proofs_same else "DIFFERENT",
                     "corrupt_b_g2_middle": "reported" if reported == ("b_g2", idx, 4) else f"NOT REPORTED: {reported}"}
    worker.device_free(d_file)
    res["gpu"] = gpu_info()
    os.write(real, (json.dumps(res) + "\n").encode())
    worker.close()


if __name__ == "__main__":
    main()
