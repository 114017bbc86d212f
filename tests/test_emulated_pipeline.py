"""The product's own sources -- host orchestration and every kernel of the MSM / NTT / prover
pipeline -- executed on host threads (tests/native/cuda_emu/cuda_runtime.h, built by
tests/native/build_emu.py from the unmodified bellman_b200/csrc/*.cu) and compared with the CPU
oracle at small sizes.

What this covers without a GPU: the launch sequences, buffer sizes, index arithmetic, counting
sort, bucket scheduling, task splitting, multi-level bucket reduction, NTT tiling, the prover's job
graph, shard policy and error semantics -- through the same C ABI and the same Python mirror the
GPU tests use (the test bodies are the ones in test_gpu_parity.py wherever their sizes allow).
What it does not cover: anything nvcc/ptxas/the hardware does.  The emulated library is test
infrastructure: it is built into a temporary directory and never loaded by the product.
"""
import os
import random

import numpy as np
import pytest

import bellman_b200 as bb
from oracle import o1

import test_gpu_parity as G
from emulated import ROOT, use_library, worker  # noqa: F401  (the emulated-library fixture)

R = o1.FR_MODULUS


def test_emulated_field_and_point_kernels(worker):
    G.test_field_arithmetic(worker)
    G.test_fp_inversion_both_ways(worker)
    G.test_point_arithmetic(worker)
    G.test_bucket_reduction_kernels(worker)


@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 8, 9, 10, 11, 12, 13])
def test_emulated_ntt(worker, log_n):
    G.test_ntt_matches_oracle(worker, log_n)


def test_emulated_ntt_variants(worker):
    G.test_ntt_tile_shapes_do_not_change_results(worker)
    G.test_ntt_padding_and_degree_limit(worker)
    G.test_ntt_canonical_form_is_also_exact(worker)
    G.test_domain_methods_compose_like_the_reference(worker)
    G.test_h_poly_matches_oracle(worker)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 1000])
def test_emulated_multiexp_g1(worker, n):
    G.test_multiexp_g1_matches_oracle(worker, n)


@pytest.mark.parametrize("n", [0, 3, 40, 300])
def test_emulated_multiexp_g2(worker, n):
    G.test_multiexp_g2_matches_oracle(worker, n)


@pytest.mark.parametrize("n,rounds,batch", [(1, 3, 16), (2, 1, 16), (33, 2, 4), (1000, 3, 16), (1000, 1, 1), (3000, 4, 7),
                                            (5000, 3, 1)])
def test_emulated_affine_rounds_g1(worker, n, rounds, batch):
    force = _force_affine(worker)
    try:
        G.test_affine_rounds_g1_match_oracle(worker, force, n, rounds, batch)
    finally:
        force(-1)


@pytest.mark.parametrize("n,rounds", [(3, 2), (40, 3), (300, 3)])
def test_emulated_affine_rounds_g2(worker, n, rounds):
    force = _force_affine(worker)
    try:
        G.test_affine_rounds_g2_match_oracle(worker, force, n, rounds)
    finally:
        force(-1)


def test_emulated_affine_rounds_special(worker):
    force = _force_affine(worker)
    try:
        G.test_affine_rounds_special_pairs(worker, force)
        G.test_affine_rounds_error_semantics(worker, force)
    finally:
        force(-1)


def _force_affine(worker):
    def force(rounds, batch=16):
        worker.set_option("msm_affine_rounds", rounds)
        worker.set_option("msm_affine_batch", batch)
    return force


def test_emulated_fr_dot(worker):
    G.test_fr_dot_diagnostic(worker)


def test_emulated_multiexp_windows(worker):
    n = 700
    bases = o1.g1_fixed_mul(o1.fr_random(41, n))
    ex = o1.fr_random(42, n)
    rc, want = o1.multiexp(1, bases, 0, None, ex)
    try:
        for c in (2, 3, 5, 8, 13, 15, 16):
            worker.set_option("msm_window_bits", c)
            assert np.array_equal(G._gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want), c
    finally:
        worker.set_option("msm_window_bits", 0)


def test_emulated_multiexp_density_fast_paths_and_skew(worker):
    rng = np.random.default_rng(5)
    n = 1200
    dens = rng.random(n) < 0.5
    k, off = int(dens.sum()), 7
    bases = o1.g1_fixed_mul(o1.fr_random(51, off + k + 3))
    ex = o1.fr_random(52, n)
    kind = rng.integers(0, 4, n)
    ex[kind == 0] = 0                                   # Exponent::Zero / One fast paths
    ex[kind == 1] = o1.fr_from_ints([1])[0]
    rc, want = o1.multiexp(1, bases, off, dens.astype(np.uint8), ex)
    assert rc == 0
    assert np.array_equal(G._gpu_multiexp(worker, bb.G1, bases, off, dens, ex), want)
    # skewed scalars: the oversized-bucket (task) path
    m = 1500
    b2 = o1.g1_fixed_mul(o1.fr_random(81, m))
    cases = {
        "all twos": o1.fr_from_ints([2] * m),
        "bytes+big": o1.fr_from_ints([int(x) for x in rng.integers(0, 256, m - 5)] + [R - 1, R - 2, 3, 1 << 200, 7]),
        "same value": np.repeat(o1.fr_random(82, 1), m, axis=0),
    }
    for name, e in cases.items():
        rc, want = o1.multiexp(1, b2, 0, None, e)
        assert rc == 0 and np.array_equal(G._gpu_multiexp(worker, bb.G1, b2, 0, None, e), want), name
    try:                                                # every bucket above 3 entries is cut into tasks
        worker.set_option("msm_big_cap", 3)
        e = o1.fr_random(83, m)
        rc, want = o1.multiexp(1, b2, 0, None, e)
        assert np.array_equal(G._gpu_multiexp(worker, bb.G1, b2, 0, None, e), want)
    finally:
        worker.set_option("msm_big_cap", 0)


def test_emulated_multiexp_error_semantics(worker):
    G.test_multiexp_error_semantics(worker)


def test_emulated_prove_mimc322_and_shards(worker):
    """BASELINE.json configs[0] through the whole prover, plus the (base range x window) shards"""
    rng = random.Random(71)
    mc = o1.Mimc(322, seed=3)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    asg = G._assignment(mc.witness())
    r, s = rng.randrange(R), rng.randrange(R)
    proof = bb.create_proof(asg, params, r, s)
    assert len(proof) == 192 and proof == mc.prove(r, s) == mc.expected_proof(r, s)
    for count in (2, 8):                                 # 2 window shards; 2 base ranges x 4 window shards
        parts = []
        for k in range(count):
            pk = bb.Parameters(worker, mc.export_params(), shard_index=k, shard_count=count)
            parts.append(bb.prove_partials(asg, pk))
            pk.free()
        assert bb.finalize(params, parts, r, s) == proof, count
        assert bb.finalize(params, parts, r, s, static=bb.finalize_static(params, r, s)) == proof



def test_emulated_prover_error_precedence(worker):
    G.test_prove_error_precedence(worker)


def test_emulated_generate_parameters(worker):
    G.test_generate_parameters_matches_oracle(worker)


def test_emulated_multiexp_fuzz(worker):
    """Random small MSMs -- group, size, density, offset, missing bases, identity bases, 0/1/small/
    negative scalars, window size, task splitting, scalar form -- against the oracle, including which
    SynthesisError comes back.  (1320 seeds of this generator ran clean at the end of round 1.)"""
    errs = {2: bb.UnexpectedIdentity, 3: bb.IoError}
    pool1 = o1.g1_fixed_mul(o1.fr_random(7, 400))
    pool2 = o1.g2_fixed_mul(o1.fr_random(8, 120))
    try:
        for case in range(70):
            rng = random.Random(case)
            group = 1 if rng.random() < 0.75 else 2
            pool = pool1 if group == 1 else pool2
            n = rng.choice([0, 1, 2, 3, 5, 17, 31, 32, 33, 64, 65, 100, 150]) if group == 1 else rng.choice([0, 1, 2, 7, 33, 60])
            dens = None
            if rng.random() < 0.6:
                p_set = rng.choice([0.1, 0.5, 0.9, 1.0])
                dens = np.array([rng.random() < p_set for _ in range(n)], dtype=bool)
            k = n if dens is None else int(dens.sum())
            off = rng.choice([0, 0, 1, 5, 20])
            nb = max(0, off + k + rng.choice([0, 0, 0, 3, -1, -2]))          # negative slack: the source runs dry
            bases = pool[[rng.randrange(pool.shape[0]) for _ in range(nb)]].copy().reshape(nb, pool.shape[1])
            for j in range(nb):
                if rng.random() < 0.04:
                    bases[j] = 0                                              # identity base
            vals = [rng.choice([rng.randrange(R), rng.randrange(R), 0, 1, rng.randrange(300), R - 1, (1 << 254) + rng.randrange(1 << 20)]) % R
                    for _ in range(n)]
            ex = o1.fr_from_ints(vals) if n else np.zeros((0, 4), np.uint64)
            worker.set_option("msm_window_bits", rng.choice([0, 0, 2, 3, 4, 7, 8, 11, 13]))
            worker.set_option("msm_big_cap", rng.choice([0, 0, 2, 5]))
            rc, want = o1.multiexp(group, bases, off, None if dens is None else dens.astype(np.uint8), ex)
            form = rng.choice([bb.FORM_MONTGOMERY, bb.FORM_CANONICAL])
            sc = ex if form == bb.FORM_MONTGOMERY else o1.fr_to_canonical(ex)
            dm = bb.FullDensity if dens is None else bb.DensityTracker(dens)
            try:
                got = bb.multiexp(worker, (bb.Bases(worker, bb.G1 if group == 1 else bb.G2, bases), off), dm, sc, form).wait()
                assert rc == 0 and np.array_equal(got, want), case
            except bb.SynthesisError as e:
                assert rc in errs and isinstance(e, errs[rc]), (case, rc, e)
    finally:
        worker.set_option("msm_window_bits", 0)
        worker.set_option("msm_big_cap", 0)


def test_emulated_bench_paths(worker):
    """What bench.py times: the synthetic MiMC-chain witness, the device-generated synthetic CRS, a
    witness already resident in device memory (`value` leg) against host buffers (`e2e` leg), and
    the N-way synthetic shards of `--gpus N` -- all must give one and the same proof."""
    asg, shape = bb.synth_mimc(60, seed=20)
    assert shape["num_constraints"] == 122 and shape["m"] == 128
    params = bb.Parameters.synthetic(worker, 21, shape)
    r, s = 0x1234567, 0x7654321
    p_host = bb.create_proof(asg, params, r, s)
    assert len(p_host) == 192 and bb.create_proof(asg, params, r, s) == p_host
    dev, bufs = {}, []
    for name, arr in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
        d = worker.device_alloc(arr.nbytes)
        worker.upload(d, arr)
        dev[name] = d.value
        bufs.append(d)
    assert bb.create_proof(asg, params, r, s, dev) == p_host
    for count in (2, 4, 8):
        parts = []
        for k in range(count):
            pk = bb.Parameters.synthetic(worker, 21, shape, shard_index=k, shard_count=count)
            parts.append(bb.prove_partials(asg, pk, dev))
            pk.free()
        assert bb.finalize(params, parts, r, s) == p_host, count
    for d in bufs:
        worker.device_free(d)


def test_emulated_profile_timeline(worker):
    """profile mode: the per-job device timeline and the host milestones of bb_groth16_prove that
    bench.py reports (`timeline`); in the emulation the times are zeros, the plumbing is what is checked"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    asg, shape = bb.synth_mimc(20, seed=3)
    params = bb.Parameters.synthetic(worker, 5, shape)
    worker.set_option("profile", 1)
    worker.profile_reset()
    try:
        for _ in range(2):
            bb.create_proof(asg, params, 11, 13)
        tl = bench.read_timeline(worker)
    finally:
        worker.set_option("profile", 0)
    assert set(tl["device_ms_since_prove_start"]) == {"h", "l", "a_inputs", "a_aux", "b_g1_inputs", "b_g1_aux", "b_g2_inputs", "b_g2_aux"}
    assert all(set(v) == {"queued", "accumulate_start", "accumulate_end", "done"} for v in tl["device_ms_since_prove_start"].values())
    host = tl["host_ms_since_prove_start"]
    assert 0 <= host["queued"] <= host["static_done"] <= host["msms_done"] <= host["proof_done"]
    assert worker.profile_read("host.proof_done")[1] == 2


def test_emulated_pipeline_over_the_host_arithmetic_path(tmp_path):
    """The same kernels compiled over mp.cuh's host arithmetic (64-bit CIOS, used by the product for
    window folds, scalar multiplications and encodings) instead of the modelled PTX chains: both
    implementations of the field must drive the pipeline to the same points and proofs."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(ROOT, "tests", "native", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    lib, _ = be.build(str(tmp_path / "emu_host"), emulate_ptx=False)
    with use_library(lib):
        w = bb.Worker(0)
        G.test_field_arithmetic(w)
        G.test_point_arithmetic(w)
        G.test_ntt_matches_oracle(w, 9)
        G.test_multiexp_g1_matches_oracle(w, 1000)
        G.test_multiexp_g2_matches_oracle(w, 40)
        rng = random.Random(3)
        mc = o1.Mimc(30, seed=2)
        mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
        mc.generate()
        r, s = rng.randrange(R), rng.randrange(R)
        assert bb.create_proof(G._assignment(mc.witness()), bb.Parameters(w, mc.export_params()), r, s) == mc.prove(r, s)
        w.close()


def test_emulated_prove_begin_end(worker):
    G.test_prove_begin_end_with_coset_evaluations(worker)
