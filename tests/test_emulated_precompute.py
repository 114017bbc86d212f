"""MSMs over resident window multiples (bb_bases_precompute / option msm_precompute) in the host-thread
emulation of the product sources (see test_emulated_pipeline.py): same points, same proofs, same
error semantics as the per-window path."""
import numpy as np
import pytest

import bellman_b200 as bb
from oracle import o1

import test_gpu_parity as G
import test_emulated_pipeline as E
from emulated import worker  # noqa: F401  (the emulated-library fixture)


@pytest.fixture()
def precompute(worker):
    worker.set_option("msm_precompute", 1)
    yield worker
    worker.set_option("msm_precompute", 0)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 33, 1000])
def test_emulated_precompute_g1(precompute, n):
    G.test_multiexp_g1_matches_oracle(precompute, n)


@pytest.mark.parametrize("n", [3, 40, 300])
def test_emulated_precompute_g2(precompute, n):
    G.test_multiexp_g2_matches_oracle(precompute, n)


def test_emulated_precompute_variants(precompute):
    E.test_emulated_multiexp_windows(precompute)
    E.test_emulated_multiexp_density_fast_paths_and_skew(precompute)
    G.test_multiexp_error_semantics(precompute)
    # explicit table construction, then queries of different densities / offsets over the same bases
    n = 600
    pts = o1.g1_fixed_mul(o1.fr_random(91, n))
    bases = bb.Bases(precompute, bb.G1, pts).precompute()
    rng = np.random.default_rng(9)
    for off, m in ((0, n), (5, 200), (599, 1)):
        dens = rng.random(m + 50) < 0.8
        dens[np.cumsum(dens) > n - off] = False              # never run past the end
        ex = o1.fr_random(92 + off, m + 50)
        rc, want = o1.multiexp(1, pts, off, dens.astype(np.uint8), ex)
        assert rc == 0
        got = bb.multiexp(precompute, (bases, off), bb.DensityTracker(dens), ex).wait()
        assert np.array_equal(got, want)


def test_emulated_precompute_prove_and_shards(precompute):
    """a 2^7-constraint MiMC proof and its 2-way shards over per-window-slot tables (the 322-round proof and the 8-way
    shards run under the one-bucket-set form below)"""
    import random
    rng = random.Random(72)
    mc = o1.Mimc(60, seed=4)
    mc.set_toxic([rng.randrange(1, o1.FR_MODULUS) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(precompute, mc.export_params())
    asg = G._assignment(mc.witness())
    r, s = rng.randrange(o1.FR_MODULUS), rng.randrange(o1.FR_MODULUS)
    proof = bb.create_proof(asg, params, r, s)
    assert proof == mc.prove(r, s) == mc.expected_proof(r, s)
    parts = []
    for k in range(2):
        pk = bb.Parameters(precompute, mc.export_params(), shard_index=k, shard_count=2)
        parts.append(bb.prove_partials(asg, pk))
        pk.free()
    assert bb.finalize(params, parts, r, s) == proof


@pytest.mark.parametrize("variant", [33])
def test_emulated_accumulate_variants(worker, variant):
    """The retired options -- msm_acc_variant (round 1's launch-bound / prefetch variants of the accumulate kernel),
    msm_affine_tma (bulk-copy staged halving rounds), msm_reduce_2d (bucket reduction without row / column sums) and
    ntt_radix8 (register radix-8 NTT passes) -- selected second implementations that were measured (no gain) and removed;
    each key, set away from its old default, is still accepted and changes nothing"""
    retired = {"msm_acc_variant": (variant, 0), "msm_affine_tma": (1, 0), "msm_reduce_2d": (0, 1), "ntt_radix8": (1, 0)}
    for key, (value, default) in retired.items():
        worker.set_option(key, value)
        try:
            for pre in (0, 1):
                worker.set_option("msm_precompute", pre)
                G.test_multiexp_g1_matches_oracle(worker, 1000)
                G.test_multiexp_g2_matches_oracle(worker, 40)
                G.test_multiexp_error_semantics(worker)
        finally:
            worker.set_option(key, default)
            worker.set_option("msm_precompute", 0)


# ---- msm_precompute = 2: one bucket set for all windows ------------------------------------------------
@pytest.fixture()
def unified(worker):
    worker.set_option("msm_precompute", 2)
    yield worker
    worker.set_option("msm_precompute", 0)
    worker.set_option("msm_unified_rows_log", 3)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 33, 1000])
def test_emulated_unified_g1(unified, n):
    G.test_multiexp_g1_matches_oracle(unified, n)


@pytest.mark.parametrize("n", [3, 40, 300])
def test_emulated_unified_g2(unified, n):
    G.test_multiexp_g2_matches_oracle(unified, n)


@pytest.mark.parametrize("rounds", [1, 2, 4, 6])
def test_emulated_unified_forced_rounds(unified, rounds):
    unified.set_option("msm_affine_rounds", rounds)
    try:
        G.test_multiexp_g1_matches_oracle(unified, 1000)
        G.test_multiexp_g2_matches_oracle(unified, 40)
        G.test_multiexp_error_semantics(unified)
    finally:
        unified.set_option("msm_affine_rounds", -1)


def test_emulated_unified_variants(unified):
    E.test_emulated_multiexp_windows(unified)
    E.test_emulated_multiexp_density_fast_paths_and_skew(unified)
    G.test_multiexp_error_semantics(unified)


def test_emulated_tables_come_and_go(worker):
    """bb_bases_precompute / bb_bases_drop_table / the option: whichever way the table of a base vector appears or
    disappears between two MSMs, the point is the same"""
    n = 300
    pts = o1.g1_fixed_mul(o1.fr_random(95, n))
    ex = o1.fr_random(96, n)
    rc, want = o1.multiexp(1, pts, 0, None, ex)
    bases = bb.Bases(worker, bb.G1, pts)
    try:
        for prepare in (lambda: None, bases.precompute, bases.drop_table,
                        lambda: worker.set_option("msm_precompute", 2), bases.drop_table,           # rebuilt on first use
                        lambda: worker.set_option("msm_precompute_groups", 2),                       # G2 only: this G1 table is left alone
                        bases.drop_table, lambda: worker.set_option("msm_precompute", 1), bases.drop_table):
            prepare()
            assert np.array_equal(bb.multiexp(worker, (bases, 0), bb.FullDensity, ex).wait(), want)
    finally:
        worker.set_option("msm_precompute", 0)
        worker.set_option("msm_precompute_groups", 3)
        bases.free()


def test_emulated_unified_deep_rounds(unified):
    G.unified_deep_rounds_case(unified, 1 << 13)            # the rounds chosen by the fill: 8 of them


def test_emulated_unified_prove_and_shards(unified):
    E.test_emulated_prove_mimc322_and_shards(unified)
    G.test_prove_begin_end_with_coset_evaluations(unified)


def test_emulated_autotune(worker):
    G.autotune_case(worker, 60, reps=1)
    assert bb.load_library().bb_tuning_name(99) is None
    # one shard of a window-sharded key: its partial sums depend on the form (the forms cut the scalars into windows of
    # different sizes), so the single-process tuner only measures it and leaves the default form active
    asg, shape = bb.synth_mimc(63, seed=20)
    whole = bb.Parameters.synthetic(worker, 21, shape)
    proof = bb.create_proof(asg, whole, 5, 7)
    shards = [bb.Parameters.synthetic(worker, 21, shape, shard_index=k, shard_count=2) for k in range(2)]
    default_parts = [bb.prove_partials(asg, p) for p in shards]
    rep = shards[1].autotune(asg, reps=1)
    assert all(t > 0 for t in rep["ms"])
    assert bb.prove_partials(asg, shards[1]) == default_parts[1]                  # still the default form
    for index in (1, 5):                                                           # the SAME form on all shards: same proof
        for p in shards:
            p.apply_tuning(index)
        assert bb.finalize(whole, [bb.prove_partials(asg, p) for p in shards], 5, 7) == proof, index
    for p in shards + [whole]:
        p.apply_tuning(0)
        p.free()


def test_emulated_table_forms_fuzz(worker):
    """Random small MSMs under the table forms -- form 1 / 2, group mask, forced or fill-chosen rounds, pairs per thread,
    stop of the rounds, window size, task splitting, density, offset, missing and identity bases, 0 / 1 / small / negative
    scalars, scalar form -- against the oracle, including which SynthesisError comes back.  (1200 seeds of this generator
    ran clean when the one-bucket-set form was written.)"""
    import random
    R = o1.FR_MODULUS
    errs = {2: bb.UnexpectedIdentity, 3: bb.IoError}
    pool1 = o1.g1_fixed_mul(o1.fr_random(7, 400))
    pool2 = o1.g2_fixed_mul(o1.fr_random(8, 120))
    keys = ("msm_window_bits", "msm_big_cap", "msm_precompute", "msm_affine_rounds")
    try:
        for case in range(45):
            rng = random.Random(case)
            group = 1 if rng.random() < 0.75 else 2
            pool = pool1 if group == 1 else pool2
            n = rng.choice([0, 1, 2, 3, 5, 17, 31, 32, 33, 64, 65, 100, 150, 400]) if group == 1 else rng.choice([0, 1, 2, 7, 33, 60])
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
            worker.set_option("msm_precompute", rng.choice([2, 2, 2, 1]))
            worker.set_option("msm_precompute_groups", rng.choice([3, 3, 1, 2]))
            worker.set_option("msm_affine_rounds", rng.choice([-1, -1, 0, 1, 2, 3, 5, 8]))
            worker.set_option("msm_affine_batch", rng.choice([16, 16, 1, 3, 7]))
            worker.set_option("msm_unified_rows_log", rng.choice([3, 0, 2, 5]))
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
        for key in keys:
            worker.set_option(key, -1 if key == "msm_affine_rounds" else 0)
        worker.set_option("msm_precompute_groups", 3)
        worker.set_option("msm_affine_batch", 16)
        worker.set_option("msm_unified_rows_log", 3)
