"""The MSM's exceptional additions -- an identity operand, P = Q (a doubling) and P = -Q (a cancellation to the
identity) -- at every stage that adds points, on keys whose points are known multiples of the generator.

Every base is [k_i]G for a Python integer k_i, so an MSM over scalars e_i is [sum k_i e_i mod r]G and a proof is three
points whose exponents follow prover.rs:320-360 exactly:
    A = alpha + sum a + r delta,   B = beta + sum b2 + s delta,   C = H + L + s (alpha + sum a) + r (beta + sum b1) + r s delta
The k_i come from families that make points collide: every base G, bases in {+-G, +-2G, +-3G}, +-G alternating, bytes
and random (the control).  The scalars come from families that put many digits into one bucket (all zero, one, r - 1,
one value), into few buckets (nibbles), one per window (powers of two), into a -1 in every window so that the carry runs
to the top window, and k next to -k.  So every stage -- the halving rounds, the bucket accumulation and its task split,
the bucket reductions, the slot and window folds, the ones list, the host fold and finalisation -- meets equal and
opposite operands, in G1 and in G2, in the single job, in sharded keys and in batches whose items fill their bucket
segments very differently.  Proofs whose points or partial sums are the identity are built by solving for one aux value.
tests/test_emulated_exceptional_sums.py runs the same bodies on the emulated device (tests/native/) at smaller sizes.
"""
import contextlib
import random

import numpy as np
import pytest

import bellman_b200 as bb
from oracle import o1

pytestmark = pytest.mark.gpu

R = o1.FR_MODULUS


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# points from exponents
# --------------------------------------------------------------------------------------------
WIDTH = {bb.G1: 12, bb.G2: 24}


def mul_g(group, ks, worker=None):
    """[k]G for Python integers k (mod r), one row each (k = 0: the all-zero identity row).  Equal k are multiplied once;
    many distinct k go through the device's fixed-base multiplication when a worker is given (the suite checks it
    against the oracle in test_gpu_parity.test_point_arithmetic)."""
    ks = [int(k) % R for k in ks]
    if not ks:
        return np.zeros((0, WIDTH[group]), np.uint64)
    uniq = sorted(set(ks))
    fr = o1.fr_from_ints(uniq)
    if worker is not None and len(uniq) > 4096:
        pts = bb.fixed_base_mul(worker, group, fr)
    else:
        pts = o1.g1_fixed_mul(fr) if group == bb.G1 else o1.g2_fixed_mul(fr)
    row = {k: i for i, k in enumerate(uniq)}
    return np.ascontiguousarray(pts[[row[k] for k in ks]])


def compressed(group, e):
    p = mul_g(group, [e])
    return bytes((o1.g1_compress(p) if group == bb.G1 else o1.g2_compress(p))[0])


def proof_bytes(eA, eB, eC):
    """Proof::write of ([eA]G1, [eB]G2, [eC]G1): the identity is the compressed point at infinity"""
    return compressed(bb.G1, eA) + compressed(bb.G2, eB) + compressed(bb.G1, eC)


# --------------------------------------------------------------------------------------------
# families
# --------------------------------------------------------------------------------------------
KEY_FAMILIES = ("ones", "small", "alternating", "bytes", "random")


def key_family(name, n, rng):
    """discrete logs of n bases"""
    if name == "ones":
        return [1] * n
    if name == "small":
        return [rng.choice((1, 2, 3, -1, -2, -3)) for _ in range(n)]
    if name == "alternating":
        return [1 if i % 2 == 0 else -1 for i in range(n)]
    if name == "bytes":
        return [rng.randrange(1, 256) for _ in range(n)]
    assert name == "random"
    return [rng.randrange(1, R) for _ in range(n)]


SCALAR_FAMILIES = ("zero", "one", "minus_one", "same", "nibbles", "powers_of_two", "carry", "plus_minus", "random")


def window_bits(n, forced=0):
    """the window an MSM of n terms takes (msm.cu choose_window), or the forced one"""
    if 2 <= forced <= 24:
        return forced
    return 4 if n < 32 else 8 if n < (1 << 13) else 15 if n < (1 << 19) else 16 if n < (1 << 23) else 17


def carry_scalar(c):
    """the scalar whose signed c-bit digits are -1 in windows 0 .. W' - 1 and +1 in window W' = floor(254 / c): the
    carry runs through every window up to the top"""
    top = 254 // c
    return (1 << (c * top)) - sum(1 << (c * w) for w in range(top))


def scalar_family(name, n, rng, c):
    if name == "zero":
        return [0] * n
    if name == "one":
        return [1] * n
    if name == "minus_one":
        return [R - 1] * n
    if name == "same":
        return [rng.randrange(R)] * n
    if name == "nibbles":
        return [rng.randrange(16) for _ in range(n)]
    if name == "powers_of_two":
        return [1 << (i % 255) for i in range(n)]
    if name == "carry":
        return [carry_scalar(c)] * n
    if name == "plus_minus":                        # k and -k on neighbouring bases
        out = []
        for i in range(n):
            out.append(rng.randrange(1, R) if i % 2 == 0 else R - out[-1])
        return out
    assert name == "random"
    return [rng.randrange(R) for _ in range(n)]


def fr(ints):
    return o1.fr_from_ints([int(v) % R for v in ints]) if len(ints) else np.zeros((0, 4), np.uint64)


def canonical(ints):
    return o1.ints_to_limbs([int(v) % R for v in ints], 4) if len(ints) else np.zeros((0, 4), np.uint64)


# --------------------------------------------------------------------------------------------
# worker options
# --------------------------------------------------------------------------------------------
# The option values a fresh context starts with: the initialisers of bb_ctx's opt_* members in csrc/bb_internal.cuh.  The
# C ABI has no call that reads an option back, so options() restores these rather than the previous values; they must
# follow the header when a default changes there.
DEFAULTS = dict(msm_window_bits=0, msm_affine_rounds=-1, msm_affine_batch=16, msm_big_cap=0, msm_precompute=0,
                msm_precompute_groups=3, msm_unified_rows_log=3, msm_reduce_k=4, msm_reduce_k1=4, prove_batch_max=0,
                shard_windows=4)


@contextlib.contextmanager
def options(worker, **kv):
    try:
        for k, v in kv.items():
            worker.set_option(k, v)
        yield
    finally:
        for k in DEFAULTS:
            worker.set_option(k, DEFAULTS[k])


def expected_msm(ks, es, offset=0, density=None, lo=0, hi=None):
    """sum e_i k_(offset + rank_i) mod r over the scalars the density map selects (multiexp.rs:242-243), counting only
    the bases with global index in [lo, hi)"""
    hi = len(ks) if hi is None else hi
    tot, rank = 0, 0
    for i, e in enumerate(es):
        if density is not None and not density[i]:
            continue
        g = offset + rank
        rank += 1
        if lo <= g < hi:
            tot += e * ks[g]
    return tot % R


# --------------------------------------------------------------------------------------------
# 1. single MSM jobs
# --------------------------------------------------------------------------------------------
# Each configuration drives the job through other stages: small windows make deep buckets, forced halving rounds
# pair equal and opposite points in k_aff_phase1 / k_aff_phase3, a small big-bucket cap sends every bucket through the
# task sums and k_msm_merge_big, 11-bit windows through the two-dimensional reduction (k_bucket_fold), form 1 through
# k_msm_fold_slots, form 2 through one bucket set; "density" adds a density map and an offset, "device" device scalars
# (Exponent::Bits), "ranges" splits the bases into three global ranges (bb.Bases(..., global_offset, global_len)).
MSM_CONFIGS = {
    "default": dict(),
    "w3": dict(msm_window_bits=3),
    "w4_rounds3_b5": dict(msm_window_bits=4, msm_affine_rounds=3, msm_affine_batch=5),
    "w5_rounds5_b1_cap4": dict(msm_window_bits=5, msm_affine_rounds=5, msm_affine_batch=1, msm_big_cap=4),
    "w11_rounds1": dict(msm_window_bits=11, msm_affine_rounds=1, msm_affine_batch=16),
    "form1_w4_cap3": dict(form=1, msm_window_bits=4, msm_big_cap=3),
    "form2_w5_rounds4_b5": dict(form=2, msm_window_bits=5, msm_affine_rounds=4, msm_affine_batch=5, msm_unified_rows_log=0),
    "form2_w11_rounds2": dict(form=2, msm_window_bits=11, msm_affine_rounds=2, msm_unified_rows_log=1),
    "density_w4_rounds2_cap3": dict(density=True, msm_window_bits=4, msm_affine_rounds=2, msm_big_cap=3),
    "device_w3_rounds2_b16": dict(device=True, msm_window_bits=3, msm_affine_rounds=2),
    "ranges_w4_rounds3": dict(ranges=3, msm_window_bits=4, msm_affine_rounds=3, msm_affine_batch=5),
}


def run_msm(worker, group, ks, es, cfg, rng, check_oracle=True):
    """one MSM job over bases [k_i]G and scalars es under the configuration cfg; compared with [expected]G and, for a
    whole base vector from the host, with the oracle's multiexp (which also returns its error code)"""
    cfg = dict(cfg)
    form = cfg.pop("form", 0)
    use_density, device, ranges = cfg.pop("density", False), cfg.pop("device", False), cfg.pop("ranges", 0)
    n = len(es)
    offset, dens = 0, None
    if use_density:
        dens = [rng.random() < 0.6 for _ in range(n)]
        offset = 5
        need = offset + sum(dens) + 3                                  # 3 trailing bases are never read
        ks = (ks * (need // max(len(ks), 1) + 1))[:need]
    pts = mul_g(group, ks, worker)
    with options(worker, msm_precompute=form, **cfg):
        results = []
        bounds = [(0, len(ks))] if not ranges else [(len(ks) * j // ranges, len(ks) * (j + 1) // ranges) for j in range(ranges)]
        for lo, hi in bounds:
            bases = bb.Bases(worker, group, pts[lo:hi], global_offset=lo, global_len=len(ks))
            if form:
                bases.precompute()
            if device:
                d = worker.device_alloc(max(32 * n, 32))
                try:
                    if n:
                        worker.upload(d, canonical(es))
                    got = bb.multiexp_device(worker, (bases, offset), d, n, bb.FORM_CANONICAL).wait()
                finally:
                    worker.device_free(d)
            else:
                dm = bb.FullDensity if dens is None else bb.DensityTracker(dens)
                got = bb.multiexp(worker, (bases, offset), dm, fr(es)).wait()
            bases.free()
            results.append((got, expected_msm(ks, es, offset, dens, lo, hi)))
    for got, e in results:
        assert np.array_equal(got, mul_g(group, [e])), e
    if check_oracle and not ranges:
        rc, want = o1.multiexp(group, pts, offset, None if dens is None else np.array(dens, np.uint8), fr(es))
        assert rc == 0 and np.array_equal(results[0][0], want)


def identity_under_zero(ks, es):
    """bases whose scalar is zero become the identity: they must be skipped (multiexp.rs:245), not reported"""
    return [0 if e == 0 else k for k, e in zip(ks, es)]


@pytest.mark.parametrize("config", list(MSM_CONFIGS))
@pytest.mark.parametrize("group", [bb.G1, bb.G2], ids=["G1", "G2"])
def test_msm_special_sums(worker, group, config, n_g1=1500, n_g2=400, combos=None):
    """every key family under every scalar family (or the (key, scalar) pairs `combos` lists) in one configuration"""
    cfg = MSM_CONFIGS[config]
    n = n_g1 if group == bb.G1 else n_g2
    rng = random.Random(100 * group + list(MSM_CONFIGS).index(config))
    c = window_bits(n, cfg.get("msm_window_bits", 0))
    pairs = combos if combos is not None else [(kf, sf) for kf in KEY_FAMILIES for sf in SCALAR_FAMILIES]
    for kf, sf in pairs:
        ks = key_family(kf, n, rng)
        es = scalar_family(sf, n, rng, c)
        if sf == "nibbles" and not cfg.get("density"):
            ks = identity_under_zero(ks, es)
        try:
            run_msm(worker, group, ks, es, cfg, rng)
        except AssertionError as e:
            raise AssertionError(f"{config}: keys {kf}, scalars {sf}: {e}") from None


def test_msm_cancels_with_nonzero_scalars(worker, n=64):
    """G and -G under scalar 1 (the ones list), under 2 (one bucket) and k, -k on one base: the identity from nonzero
    scalars, in both groups, with and without halving rounds"""
    for group in (bb.G1, bb.G2):
        for cfg in (dict(), dict(msm_affine_rounds=2, msm_window_bits=4), dict(form=2, msm_affine_rounds=1, msm_window_bits=4)):
            for es, ks in (([1] * n, [1, -1] * (n // 2)), ([2] * n, [1, -1] * (n // 2)), ([5, R - 5] * (n // 2), [3] * n)):
                run_msm(worker, group, ks, es, cfg, random.Random(0))
        # 256 ones: the ones list spans two CTAs of k_msm_sum_list, whose partial sums k_point_tree_sum then doubles
        # (every base G) or cancels (G in the first CTA's half, -G in the second's)
        for ks in ([1] * 256, [1] * 128 + [-1] * 128):
            run_msm(worker, group, ks, [1] * 256, dict(), random.Random(0))


# --------------------------------------------------------------------------------------------
# targeted collisions in the stages after the buckets
# --------------------------------------------------------------------------------------------
def horner_collision(c, sign):
    """keys and scalars of a two-term MSM with window c whose window sums are W_1 = 2G and W_0 = sign 2^(c+1) G: the
    Horner fold's step from window 1 to window 0 adds 2^c W_1 = 2^(c+1) G to W_0, a doubling (sign 1) or a cancellation
    (sign -1).  Form 1 folds bucket 2 (digit 2) over slots 0 and 1, [sign 2^c]G and 2^c G: the same doubling or
    cancellation in k_msm_fold_slots.  Digit 2 rather than 1 keeps the single job's ones list out of it."""
    return [sign * (1 << c), 1], [2, 2 << c]


def test_msm_fold_collisions(worker, c=4):
    """the host Horner fold of a single job (form 0) and k_msm_fold_slots (form 1) double and cancel, in both groups"""
    for group in (bb.G1, bb.G2):
        for sign in (1, -1):
            ks, es = horner_collision(c, sign)
            for form in (0, 1, 2):
                run_msm(worker, group, ks, es, dict(form=form, msm_window_bits=c), random.Random(0))


def test_bucket_reduction_collisions(worker):
    """the two bucket reductions on buckets that are equal or opposite, in both groups.  Scalar d + 1 puts base d into
    bucket d of window 0 (digits up to D are positive), so bucket d holds [k_d]G.
      * 11-bit windows (D = 1024, the two-dimensional form, rows of 32): k_d = -1 where d // 8 is odd.  The row folds of
        k_bucket_fold add buckets 8 apart (opposite: cancellations), the column folds buckets 256 apart (equal: doublings).
      * 10-bit windows (D = 512, the running-sum form) with msm_reduce_k1 = 2: level 0 has 256 runs, two CTAs, whose
        partial sums k_msm_level_sums adds.  Every bucket G makes them equal, -G in the upper half opposite.  Buckets 0
        and 256 stay empty so that the halves match (scalar 1 would take the ones list)."""
    rng = random.Random(5)
    for group in (bb.G1, bb.G2):
        n = 1024
        run_msm(worker, group, [1 if (d // 8) % 2 == 0 else -1 for d in range(n)], [d + 1 for d in range(n)],
                dict(msm_window_bits=11), rng)
        ds = [d for d in range(1, 512) if d != 256]
        for ks in ([1] * len(ds), [1 if d < 256 else -1 for d in ds]):
            run_msm(worker, group, ks, [d + 1 for d in ds], dict(msm_window_bits=10, msm_reduce_k1=2), rng)


# --------------------------------------------------------------------------------------------
# 2. keys and witnesses of a Groth16 circuit whose exponents are known
# --------------------------------------------------------------------------------------------
class Key:
    """the exponents of a Parameters dict: h (m - 1), l (aux), a (inputs + a_aux density), b (b_input + b_aux density,
    G1 and G2), alpha, beta, delta; `params()` the points"""

    def __init__(self, family, rng, n_inputs, n_aux, m, a_aux_density, b_input_density, b_aux_density):
        self.ni, self.na, self.m = n_inputs, n_aux, m
        self.a_aux, self.b_in, self.b_aux = list(a_aux_density), list(b_input_density), list(b_aux_density)
        self.h = key_family(family, m - 1, rng)
        self.l = key_family(family, n_aux, rng)
        self.a = key_family(family, n_inputs + sum(self.a_aux), rng)
        nb = sum(self.b_in) + sum(self.b_aux)
        self.b1 = key_family(family, nb, rng)
        self.b2 = key_family(family, nb, rng)
        first = key_family(family, 3, rng)
        self.alpha, self.beta, self.delta = first[0], first[1], first[2]
        self.gamma = 7

    def params(self, worker=None):
        return dict(vk_g1=mul_g(bb.G1, [self.alpha, self.beta, self.delta]), vk_g2=mul_g(bb.G2, [self.beta, self.gamma, self.delta]),
                    h=mul_g(bb.G1, self.h, worker), l=mul_g(bb.G1, self.l, worker), a=mul_g(bb.G1, self.a, worker),
                    b_g1=mul_g(bb.G1, self.b1, worker), b_g2=mul_g(bb.G2, self.b2, worker))

    def partials(self, w):
        """the eight partial sums' exponents (prover.cu job order h, l, a_inputs, a_aux, b_g1 inputs / aux, b_g2 ...)"""
        nbi = sum(self.b_in)
        return [expected_msm(self.h, w.h),
                expected_msm(self.l, w.aux),
                expected_msm(self.a, w.inputs),
                expected_msm(self.a, w.aux, self.ni, self.a_aux),
                expected_msm(self.b1, w.inputs, 0, self.b_in),
                expected_msm(self.b1, w.aux, nbi, self.b_aux),
                expected_msm(self.b2, w.inputs, 0, self.b_in),
                expected_msm(self.b2, w.aux, nbi, self.b_aux)]

    def proof(self, w, r, s):
        """(A, B, C) exponents, prover.rs:320-360"""
        h, l, a_in, a_aux, b1_in, b1_aux, b2_in, b2_aux = self.partials(w)
        a = (self.alpha + a_in + a_aux) % R
        eA = (a + r * self.delta) % R
        eB = (self.beta + b2_in + b2_aux + s * self.delta) % R
        eC = (h + l + s * a + r * (self.beta + b1_in + b1_aux) + r * s * self.delta) % R
        return eA, eB, eC

    def proof_bytes(self, w, r, s):
        return proof_bytes(*self.proof(w, r, s))


class Witness:
    """inputs, aux and the a, b, c evaluations of one item as Python integers, h = the quotient's coefficients"""

    def __init__(self, key, inputs, aux, a, b, c):
        self.key, self.inputs, self.aux, self.a, self.b, self.c = key, list(inputs), list(aux), list(a), list(b), list(c)
        self.h = o1.fr_to_ints(o1.h_poly(fr(a), fr(b), fr(c)))

    def assignment(self):
        k = self.key
        return bb.ProvingAssignment(fr(self.a), fr(self.b), fr(self.c), fr(self.inputs), fr(self.aux), k.a_aux, k.b_in, k.b_aux)

    def device_ptrs(self, worker):
        asg = self.assignment()
        out = {}
        for name, arr in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment), ("aux", asg.aux_assignment)):
            out[name] = worker.device_alloc(max(arr.nbytes, 32))
            if arr.nbytes:
                worker.upload(out[name], arr)
        return out

    def with_aux(self, j, v):
        aux = list(self.aux)
        aux[j] = v % R
        w = Witness.__new__(Witness)
        w.key, w.inputs, w.aux, w.a, w.b, w.c, w.h = self.key, self.inputs, aux, self.a, self.b, self.c, self.h
        return w


def circuit_shape(rng, n_inputs, n_aux, n_constraints):
    m = 1
    while m < n_constraints:
        m *= 2
    a_aux = [rng.random() < 0.7 for _ in range(n_aux)]
    b_in = [i % 2 == 0 for i in range(n_inputs)]
    b_aux = [rng.random() < 0.6 for _ in range(n_aux)]
    return dict(n_inputs=n_inputs, n_aux=n_aux, m=m, a_aux_density=a_aux, b_input_density=b_in, b_aux_density=b_aux), n_constraints


def witness(key, family, rng, n_constraints, c=8):
    """inputs[0] = 1 and the rest of the inputs and the aux from one scalar family; a, b, c random but for the
    all-zero family"""
    vals = scalar_family(family, key.ni - 1 + key.na, rng, c)
    evals = [[0] * n_constraints for _ in range(3)] if family == "zero" else \
        [[rng.randrange(R) for _ in range(n_constraints)] for _ in range(3)]
    return Witness(key, [1] + vals[:key.ni - 1], vals[key.ni - 1:], *evals)


def solve_aux(w, j, target):
    """the witness with aux[j] chosen so that the exponent target(w) is zero (target is affine in aux[j])"""
    e0, e1 = target(w.with_aux(j, 0)), target(w.with_aux(j, 1))
    assert (e1 - e0) % R, "aux value does not reach this exponent"
    return w.with_aux(j, -e0 * pow(e1 - e0, -1, R))


def split_partials(blob):
    """960 bytes -> six G1 and two G2 affine rows"""
    g1 = np.frombuffer(blob[:576], np.uint64).reshape(6, 12)
    g2 = np.frombuffer(blob[576:], np.uint64).reshape(2, 24)
    return g1, g2


def check_partials(key, w, blob):
    g1, g2 = split_partials(blob)
    e = key.partials(w)
    assert np.array_equal(g1, mul_g(bb.G1, e[:6])), "G1 partial sums"
    assert np.array_equal(g2, mul_g(bb.G2, e[6:])), "G2 partial sums"


FORMS = ("per-window", "form 1", "form 2")


def set_form(worker, params, form):
    """0: per-window bucket sets; 1: a bucket array per window slot over resident multiples; 2: one bucket set"""
    params.apply_tuning(1 if form == 2 else 0)
    if form == 1:
        params.precompute()
        worker.set_option("msm_precompute", 1)


SHAPE = dict(n_inputs=3, n_aux=700, n_constraints=600)
DEEP = dict(msm_window_bits=4, msm_affine_rounds=3, msm_affine_batch=5, msm_big_cap=8)    # deep buckets in small jobs


# --------------------------------------------------------------------------------------------
# 3. proofs: single, sharded, batched
# --------------------------------------------------------------------------------------------
def test_single_proofs(worker, shape=SHAPE, combos=None, opts=None, create_all=True):
    """prove_partials: each of the eight partial sums in its exponent; finalize and create_proof against the formula
    for r, s in {0, 1, 2, r - 1, random} (create_all=False: create_proof for the random pair only).  combos: (key
    family, witness family) pairs, by default every pair"""
    rng = random.Random(61)
    sh, nc = circuit_shape(rng, **shape)
    c = window_bits(sh["n_aux"], (opts or {}).get("msm_window_bits", 0))
    combos = combos if combos is not None else [(kf, wf) for kf in KEY_FAMILIES for wf in SCALAR_FAMILIES]
    with options(worker, **(opts or {})):
        for kf in dict.fromkeys(kf for kf, _ in combos):
            key = Key(kf, rng, **sh)
            params = bb.Parameters(worker, key.params(worker))
            for wf in [wf for k, wf in combos if k == kf]:
                w = witness(key, wf, rng, nc, c)
                asg = w.assignment()
                blob = bb.prove_partials(asg, params)
                check_partials(key, w, blob)
                rs = [(0, 0), (1, 2), (2, R - 1), (R - 1, 1), (rng.randrange(R), rng.randrange(R))]
                for r, s in rs:
                    assert bb.finalize(params, [blob], r, s) == key.proof_bytes(w, r, s), (kf, wf, r, s)
                for r, s in (rs if create_all else rs[-1:]):
                    assert bb.create_proof(asg, params, r, s) == key.proof_bytes(w, r, s), (kf, wf, r, s)
            params.free()


def test_sharded_proofs(worker, shape=SHAPE, counts=(2, 3, 5, 8), key_families=("ones", "alternating", "small"),
                        witness_families=("one", "carry", "nibbles"), by_range=4, opts=None):
    """the partial sums of 2, 3, 5 and 8 shards (window shards first, base ranges second) and of base ranges alone
    (shard_windows = 1) add up to the proof of the formula"""
    rng = random.Random(62)
    sh, nc = circuit_shape(rng, **shape)
    with options(worker, **(opts or {})):
        for kf, wf in zip(key_families, witness_families):
            key = Key(kf, rng, **sh)
            p = key.params(worker)
            params = bb.Parameters(worker, p)
            w = witness(key, wf, rng, nc, window_bits(sh["n_aux"], (opts or {}).get("msm_window_bits", 0)))
            asg = w.assignment()
            r, s = rng.randrange(R), rng.randrange(R)
            want = key.proof_bytes(w, r, s)
            plans = [(cnt, 4) for cnt in counts] + ([(by_range, 1)] if by_range else [])
            for cnt, sw in plans:
                worker.set_option("shard_windows", sw)
                parts = []
                for k in range(cnt):
                    pk = bb.Parameters(worker, p, shard_index=k, shard_count=cnt)
                    parts.append(bb.prove_partials(asg, pk))
                    pk.free()
                assert bb.finalize(params, parts, r, s) == want, (kf, wf, cnt, sw)
            worker.set_option("shard_windows", 4)
            params.free()


def batch_items(key, rng, nc, c):
    """items of one sub-batch whose bucket fills differ by orders of magnitude: every digit in one bucket, all zero,
    random, r - 1 everywhere, the carry through every window, k next to -k"""
    return [witness(key, wf, rng, nc, c) for wf in ("one", "zero", "random", "minus_one", "carry", "plus_minus", "nibbles")]


def run_batch(worker, params, key, items, rng, device=False, rs=None):
    rs = rs or [(rng.randrange(R), rng.randrange(R)) for _ in items]
    ptrs, held = None, []
    if device:
        ptrs = [w.device_ptrs(worker) for w in items]
        held = [p for d in ptrs for p in d.values()]
    try:
        got = bb.create_proof_batch([w.assignment() for w in items], params, [r for r, _ in rs], [s for _, s in rs], ptrs)
    finally:
        for p in held:
            worker.device_free(p)
    for i, (w, (r, s)) in enumerate(zip(items, rs)):
        assert got[i] == key.proof_bytes(w, r, s), (i, got[i])


def test_batches(worker, shape=SHAPE, key_families=("ones", "small", "alternating", "random"), count=7, batch_max=3, opts=None,
                 forms=(0, 1, 2)):
    """create_proof_batch over items of different families in one sub-batch, every item against the formula: whole
    batches and uneven sub-batches (prove_batch_max), each from host and from device witnesses, in the three forms"""
    rng = random.Random(63)
    sh, nc = circuit_shape(rng, **shape)
    for kf in key_families:
        key = Key(kf, rng, **sh)
        params = bb.Parameters(worker, key.params(worker))
        items = batch_items(key, rng, nc, window_bits(sh["n_aux"], (opts or {}).get("msm_window_bits", 0)))[:count]
        with options(worker, **(opts or {})):
            for form in forms:
                set_form(worker, params, form)
                for device in (False, True):
                    try:
                        run_batch(worker, params, key, items, rng, device=device)
                        worker.set_option("prove_batch_max", batch_max)
                        run_batch(worker, params, key, items, rng, device=device)
                        worker.set_option("prove_batch_max", 0)
                    except AssertionError as e:
                        raise AssertionError(f"keys {kf}, {FORMS[form]}, {'device' if device else 'host'} witnesses: {e}") from None
        params.apply_tuning(0)
        params.free()


def identity_items(key, rng, nc):
    """(witness, r, s, what) for proofs with an identity point or partial sum, solved for one aux value each"""
    base = witness(key, "random", rng, nc)
    ja = next(j for j in range(key.na) if key.a_aux[j])
    jb = next(j for j in range(key.na) if key.b_aux[j])
    rnd = rng.randrange(1, R)
    out = []
    w = solve_aux(base, ja, lambda v: key.proof(v, 0, 0)[0])                      # alpha + sum a = 0, r = 0: A = O
    out.append((w, 0, rng.randrange(R), "alpha + sum a = 0, r = 0"))
    w = solve_aux(base, ja, lambda v: key.proof(v, rnd, 0)[0])                    # A = O with a random r
    out.append((w, rnd, rng.randrange(R), "A = O"))
    s = rng.randrange(1, R)
    w = solve_aux(base, jb, lambda v: key.proof(v, 0, s)[1])                      # B = O
    out.append((w, rng.randrange(R), s, "B = O"))
    r, s = rng.randrange(R), rng.randrange(R)
    w = solve_aux(base, ja, lambda v: key.proof(v, r, s)[2])                      # C = O
    out.append((w, r, s, "C = O"))
    return out


def test_identity_results(worker, shape=SHAPE, opts=None, forms=(0, 1, 2), single_forms=(0, 1, 2)):
    """proofs whose A, B or C is the point at infinity, and an L partial sum that is the identity with every scalar one
    (G and -G alternating: the ones list on the single path, bucket 1 of window 0 in a batch) -- each alone and as one
    item among ordinary items of a batch, in the three forms"""
    rng = random.Random(64)
    sh, nc = circuit_shape(rng, **shape)
    sh["n_aux"] += sh["n_aux"] % 2
    sh["a_aux_density"] = (sh["a_aux_density"] + [True])[:sh["n_aux"]]
    sh["b_aux_density"] = (sh["b_aux_density"] + [True])[:sh["n_aux"]]
    key = Key("random", rng, **sh)
    key.l = [1, -1] * (sh["n_aux"] // 2)                                         # L = sum aux_j (+-G)
    params = bb.Parameters(worker, key.params(worker))
    cases = identity_items(key, rng, nc)
    ones = witness(key, "one", rng, nc)
    assert key.partials(ones)[1] == 0
    cases.append((ones, rng.randrange(R), rng.randrange(R), "L = O from scalars one"))
    for w, r, s, what in cases:
        e = key.proof(w, r, s)
        assert 0 in e or what.startswith("L"), what
    ordinary = [witness(key, wf, rng, nc) for wf in ("random", "nibbles")]
    with options(worker, **(opts or {})):
        for form in forms:
            set_form(worker, params, form)
            for w, r, s, what in (cases if form in single_forms else ()):
                asg = w.assignment()
                assert bb.create_proof(asg, params, r, s) == key.proof_bytes(w, r, s), (FORMS[form], what)
                check_partials(key, w, bb.prove_partials(asg, params))
            # one identity case per item, ordinary items around them
            items, rs = [], []
            for w, r, s, _ in cases:
                items += [ordinary[len(items) % 2], w]
                rs += [(rng.randrange(R), rng.randrange(R)), (r, s)]
            run_batch(worker, params, key, items, rng, rs=rs)
    params.apply_tuning(0)
    params.free()


def test_batch_horner_fold(worker, shape=SHAPE, c=4):
    """the device Horner fold of a batched job (k_msm_fold_windows) in both groups: the L vector (G1) and the b_g2 aux
    vector (G2) start with [2^c]G, G, [-2^c]G, and aux values 2 and 2^(c+1) make the step from window 1 to window 0 a
    doubling (aux 0 and 1) or a cancellation (aux 2 and 1), next to an ordinary item"""
    rng = random.Random(65)
    sh, nc = circuit_shape(rng, **shape)
    sh["b_aux_density"][:3] = [True] * 3
    key = Key("random", rng, **sh)
    ks, es = horner_collision(c, 1)
    key.l[:3] = [ks[0], ks[1], -ks[0]]
    nbi = sum(key.b_in)
    key.b2[nbi:nbi + 3] = [ks[0], ks[1], -ks[0]]
    params = bb.Parameters(worker, key.params(worker))

    def item(aux_at):
        aux = [0] * key.na
        for j, v in aux_at.items():
            aux[j] = v
        return Witness(key, [1] + [rng.randrange(R) for _ in range(key.ni - 1)], aux,
                       *[[rng.randrange(R) for _ in range(nc)] for _ in range(3)])

    items = [item({0: es[0], 1: es[1]}), witness(key, "random", rng, nc), item({2: es[0], 1: es[1]})]
    assert key.partials(items[2])[1] == 0 and key.partials(items[2])[7] == 0
    with options(worker, msm_window_bits=c):
        run_batch(worker, params, key, items, rng)
    params.free()
