"""Key generation benchmark: generate_parameters on the device (generator.generate_parameters_device, bb_groth16_generate)
for the constraint system bench.py proves (bb_synth_mimc_r1cs at 2^--log-size constraints), and Parameters::write of the
resident key (params_io.write_parameters_device, bb_params_write).

JSON fields: seeded / random: {ms} mean over --steps after --warmup of a generation with fixed toxic waste and of
generate_random_parameters_device; seeded.stages_ms: generate.transpose / .lagrange / .qap / .g1 / .g2 of one profiled
generation.  write: pinned / hbm {ms, gb_per_s} of bb_params_write into page-locked host memory and into HBM.  old: the host
generator (generator.generate_parameters over Python integers) plus the upload Parameters(worker, dict), at 2^--old-log-size
constraints.  oracle1: the CPU oracle's generator (o1.Mimc.generate) at 2^--oracle-log-size constraints.  checks: proof (a
proof from the generated key equals the trapdoor-expected bytes of the oracle), verifies (it verifies under the generated
verifying key), write_read (the written file read back with bb_params_read holds the same vectors).  gpu: card name, power
limit, maximum and current SM clock, read in the same run.  Writes nothing to the tree."""
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
from bellman_b200 import generator as GEN  # noqa: E402
from bellman_b200 import params_io as PIO  # noqa: E402
from bellman_b200 import r1cs as RC  # noqa: E402

R = GEN.FR_MODULUS
SEED = 20
STAGES = ("generate.transpose", "generate.lagrange", "generate.qap", "generate.g1", "generate.g2")


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, choices=[1], help="one device")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--log-size", type=int, default=20, help="log2 of the constraints")
    ap.add_argument("--old-log-size", type=int, default=12, help="log2 of the constraints for the host generator")
    ap.add_argument("--oracle-log-size", type=int, default=16, help="log2 of the constraints for the CPU oracle's generator")
    return ap.parse_args()


def rounds_of(log_size):
    return (1 << (log_size - 1)) - 1


def mimc_assembly(rounds):
    """the KeypairAssembly of bb_synth_mimc_r1cs(rounds, SEED): the host generator's input"""
    mats = []
    for terms in (3 * rounds, 4 * rounds, 3 * rounds):
        mats.append((np.zeros(2 * rounds + 1, np.uint64), np.zeros(terms, np.uint32), np.zeros((terms, 4), np.uint64)))
    bb._check(bb.load_library().bb_synth_mimc_r1cs(C.c_size_t(rounds), C.c_uint64(SEED), *[bb._ptr(x) for m in mats for x in m]))
    asm = GEN.KeypairAssembly()
    for _ in range(2):
        asm.alloc_input()
    for _ in range(2 * rounds + 1):
        asm.alloc()
    n = 2 * rounds
    lcs = [[[] for _ in range(n)] for _ in range(3)]
    for m, (off, var, cf) in enumerate(mats):
        vals = GEN._mont_to_ints(cf)
        for k in range(n):
            for t in range(int(off[k]), int(off[k + 1])):
                v = int(var[t])
                lcs[m][k].append((("input", v) if v < 2 else ("aux", v - 2), vals[t]))
    for k in range(n):
        asm.enforce(lcs[0][k], lcs[1][k], lcs[2][k])
    return asm


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sum(ts) / len(ts)


def main():
    args = parse()
    from oracle import o1
    from oracle.oracle0 import pairing as PR
    from bench_prove_batch import gpu_info
    import torch
    rng = random.Random(7)
    tox = [rng.randrange(1, R) for _ in range(5)]
    worker = bb.Worker(0)
    rounds = rounds_of(args.log_size)
    r1cs = RC.R1CS.synth_mimc(worker, rounds, SEED)

    def seeded():
        p, v = GEN.generate_parameters_device(worker, r1cs, *tox)
        p.free()
        v.free()

    def rand():
        p, v = GEN.generate_random_parameters_device(worker, r1cs)
        p.free()
        v.free()

    res = {"metric": "generate_ms", "config": {"log_size": args.log_size, "constraints": r1cs.n_constraints, "rounds": rounds,
                                               "circuit": f"bb_synth_mimc_r1cs({rounds}, {SEED})", "steps": args.steps, "warmup": args.warmup}}
    res["seeded"] = {"ms": round(timed(seeded, args.steps, args.warmup), 3)}
    res["random"] = {"ms": round(timed(rand, args.steps, args.warmup), 3)}
    worker.set_option("profile", 1)
    worker.profile_reset()
    params, pvk = GEN.generate_parameters_device(worker, r1cs, *tox)
    res["seeded"]["stages_ms"] = {s: round(worker.profile_read(s)[0], 3) for s in STAGES}
    worker.set_option("profile", 0)

    # bb_params_write into page-locked host memory and into HBM
    n = len(PIO.write_parameters_device(params, pvk))
    host = torch.empty(n, dtype=torch.uint8).pin_memory()
    dev = worker.device_alloc(n)
    lib = bb.load_library()
    got = C.c_size_t()

    def write(ptr, on_device):
        bb._check(lib.bb_params_write(worker._h, params._h, pvk._h, C.c_int(0), C.c_void_p(ptr), C.c_size_t(n), C.c_int(on_device), C.byref(got)))

    res["write"] = {}
    for leg, ptr, on_dev in (("pinned", host.data_ptr(), 0), ("hbm", bb._addr(dev), 1)):
        ms = timed(lambda: write(ptr, on_dev), args.steps, args.warmup)
        res["write"][leg] = {"ms": round(ms, 3), "gb_per_s": round(n / ms / 1e6, 3)}
    res["config"]["file_bytes"] = n
    worker.device_free(dev)

    # checks: the trapdoor-expected proof, verification, write -> read
    mc = o1.Mimc(rounds, seed=SEED)
    mc.set_toxic(tox)
    wit = mc.witness()
    r, s = rng.randrange(R), rng.randrange(R)
    proof = RC.create_proof_r1cs(r1cs, params, wit["inputs"], wit["aux"], r, s)
    checks = {"proof": "equal" if proof == mc.expected_proof(r, s) else "DIFFERENT"}
    a, b, c = PR.proof_read(proof)
    try:
        bb.verify_proof(pvk, (o1.g1_from_affine_ints([a])[0], o1.g2_from_affine_ints([b])[0], o1.g1_from_affine_ints([c])[0]),
                        o1.fr_to_ints(wit["inputs"][1:]))
        checks["verifies"] = "yes"
    except bb.InvalidProof:
        checks["verifies"] = "NO"
    back = PIO.read_parameters_device(worker, host.numpy())
    d1, d2 = PIO.download_parameters(params), PIO.download_parameters(back)
    checks["write_read"] = "equal" if all(np.array_equal(d1[k], d2[k]) for k in d1) else "DIFFERENT"
    back.free()
    params.free()
    pvk.free()
    r1cs.free()

    # the old path at a smaller size: the host generator and the upload
    old_rounds = rounds_of(args.old_log_size)
    asm = mimc_assembly(old_rounds)

    def old():
        p = GEN.generate_parameters(worker, asm, *tox)
        bb.Parameters(worker, p).free()

    res["old"] = {"log_size": args.old_log_size, "ms": round(timed(old, 1, 0), 3)}
    old_r1cs = RC.R1CS.synth_mimc(worker, old_rounds, SEED)
    res["old"]["device_ms_same_size"] = round(timed(lambda: [x.free() for x in GEN.generate_parameters_device(worker, old_r1cs, *tox)], 3, 1), 3)
    old_r1cs.free()
    # the CPU oracle's generator (oracle-1, multi-threaded C++)
    o_rounds = rounds_of(args.oracle_log_size)
    omc = o1.Mimc(o_rounds, seed=SEED)
    omc.set_toxic(tox)
    t0 = time.perf_counter()
    omc.generate()
    res["oracle1"] = {"log_size": args.oracle_log_size, "ms": round((time.perf_counter() - t0) * 1e3, 3), "threads": o1.num_threads()}
    res["checks"] = checks
    res["gpu"] = gpu_info()
    worker.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
