"""Every G_T value the device computes, checked against Python integers (oracle/oracle0): the Fp2 operations of field.cuh
on many lanes and at edge elements, the Fp12 operations of tower.cuh lane by lane, the multi-pairing at many pairs, and
the values the batch verifier and verify_each take their verdicts from.

With trapdoor scalars on both sides every pairing value is a power of g = e(G1, G2)^k, k = gt_exponent(): e([a]G1, [b]G2)
is g^(ab).  So the expected value of a multi-pairing or of a verifier is g^E for an exponent E computed exactly mod r,
and one fixed-base window table of g turns each E into a G_T value with about 32 Fp12 products, with no Python pairing
per lane.  The batch verifier's exponent (csrc/verify.cu, stages in its header) is
    E = sum_i z_i (-a_i b_i + delta c_i + gamma psi_i + alpha beta),   psi_i = t_0 + sum_j x_ij t_j   (mod r)
for proofs A_i = [a_i], B_i = [b_i], C_i = [c_i] and a key alpha, beta, gamma, delta, ic_j = [t_j]; it is anchored to the
oracle's multi_pairing over the verifier's own pairs by test_batch_exponent_matches_pairs.  verify_each's value i is
g^(a_i b_i - gamma psi_i - delta c_i), its last value g^(alpha beta).
tests/test_emulated_gt.py runs the same bodies on the emulated device (tests/native/) at smaller sizes.
"""
import ctypes as C
import functools
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import verifier as V
from oracle import o1
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

from test_gpu_verify import _fp12_from_mont, _fp12_to_mont, gt_to_oracle
from test_gpu_verify_each import trapdoor_key

pytestmark = pytest.mark.gpu

R = F.FR_MODULUS
P = F.FP_MODULUS
ONE = PR.Fp12.one()
ZERO = PR.Fp12.zero()


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# G_T from exponents
# --------------------------------------------------------------------------------------------
class GtPow:
    """e -> g^e (e mod r) by 8-bit windows: 32 x 256 precomputed powers of g, then at most 32 products"""

    def __init__(self, g):
        self.tab = []
        base = g
        for _ in range(32):
            row = [ONE, base]
            for _ in range(254):
                row.append(row[-1] * base)
            self.tab.append(row)
            base = row[-1] * base

    def __call__(self, e):
        e %= R
        acc = ONE
        for w in range(32):
            d = (e >> (8 * w)) & 255
            if d:
                acc = acc * self.tab[w][d]
        return acc


@functools.lru_cache(maxsize=None)
def gt_pow():
    """the window table of g = e(G1, G2)^k in the device's convention, checked once against a plain power"""
    k = V.gt_exponent() % R
    g = PR.pairing(F.G1_GEN, F.G2_GEN).pow(k)
    t = GtPow(g)
    e = random.Random(1).randrange(R)
    assert t(e) == g.pow(e) and t(R) == ONE and t(1) == g and g != ONE
    return t


# --------------------------------------------------------------------------------------------
# Fp2 (bb_selftest_field, field 2) against (c0, c1) arithmetic mod p
# --------------------------------------------------------------------------------------------
MONT = pow(2, 384, P)
MONT_INV = pow(MONT, -1, P)


def _ints(arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 6)
    return [int.from_bytes(arr[i].tobytes(), "little") for i in range(arr.shape[0])]


def _limbs(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(48, "little") for v in vals), np.uint64).reshape(-1, 6).copy()


def _selftest_fp2(worker, op, a, b):
    out = np.zeros_like(a)
    rc = bb.load_library().bb_selftest_field(worker._h, C.c_int(2), C.c_int(op), a.ctypes.data_as(C.c_void_p),
                                             b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_size_t(a.shape[0]))
    assert rc == 0
    return out


def _fp2_ref(op, x, y):
    (a0, a1), (b0, b1) = x, y
    if op in (0, 5):
        return (a0 * b0 - a1 * b1) % P, (a0 * b1 + a1 * b0) % P
    if op == 1:
        return (a0 + b0) % P, (a1 + b1) % P
    if op == 2:
        return (a0 - b0) % P, (a1 - b1) % P
    if op in (3, 6):
        return (a0 * a0 - a1 * a1) % P, 2 * a0 * a1 % P
    n = (a0 * a0 + a1 * a1) % P                                  # op 4: 1 / (a0 + a1 u) = (a0 - a1 u) / (a0^2 + a1^2)
    if n == 0:
        return 0, 0
    ni = pow(n, -1, P)
    return a0 * ni % P, -a1 * ni % P


def test_fp2_operations(worker, n_random=4000, seed=41):
    """every Fp2 op on every pair of elements whose components come from the Fp edge list of test_field_arithmetic
    (10^4 lanes), on raw Montgomery limb patterns and on random lanes; the inlined mul_inl / sqr_inl equal the
    out-of-line operator* / sqr() bit for bit"""
    rng = random.Random(seed)
    edge = [0, 1, 2, P - 1, P - 2, (1 << 383) % P, (1 << 64) - 1, (1 << 32) - 1, (P - 1) // 2, (P + 1) // 2]
    els = [(c0, c1) for c0 in edge for c1 in edge]
    xs = [x for x in els for _ in els] + [(rng.randrange(P), rng.randrange(P)) for _ in range(n_random)]
    ys = [y for _ in els for y in els] + [(rng.randrange(P), rng.randrange(P)) for _ in range(n_random)]
    mont = lambda els_: _limbs([c * MONT % P for e in els_ for c in e]).reshape(-1, 12)
    a, b = mont(xs), mont(ys)
    # limb patterns taken directly as Montgomery words (all below p): all-ones words, p - 1, alternating words
    raw = [P - 1, (1 << 380) - 1, (1 << 320) - 1, (1 << 64) - 1, sum(((1 << 64) - 1) << (128 * k) for k in range(3))]
    raw_els = [(r0, r1) for r0 in raw for r1 in raw]
    ra = _limbs([c for e in raw_els for _ in raw_els for c in e]).reshape(-1, 12)
    rb = _limbs([c for _ in raw_els for e in raw_els for c in e]).reshape(-1, 12)
    a, b = np.concatenate([a, ra]), np.concatenate([b, rb])
    x_can = [tuple(v * MONT_INV % P for v in pair) for pair in zip(*[iter(_ints(a))] * 2)]
    y_can = [tuple(v * MONT_INV % P for v in pair) for pair in zip(*[iter(_ints(b))] * 2)]
    got = {}
    for op in range(7):
        got[op] = _selftest_fp2(worker, op, a, b)
        want = [c * MONT % P for x, y in zip(x_can, y_can) for c in _fp2_ref(op, x, y)]
        have = _ints(got[op])
        bad = [i // 2 for i, (h, w) in enumerate(zip(have, want)) if h != w]
        assert not bad, (op, len(bad), bad[:8])
    assert np.array_equal(got[5], got[0]) and np.array_equal(got[6], got[3])
    inv = got[4]                                                 # one more check of the inverse: x * (1/x) = 1 on the device
    prod = _selftest_fp2(worker, 0, a, inv)
    nz = [i for i, x in enumerate(x_can) if x != (0, 0)]
    assert all(_ints(prod[i]) == [MONT % P, 0] for i in nz)


# --------------------------------------------------------------------------------------------
# Fp12 (bb_diag_fp12) lane by lane against the oracle's Fp12
# --------------------------------------------------------------------------------------------
def tower(coeffs):
    """up to 12 Fp integers in the device's tower order (c0.c0.c0, c0.c0.c1, ..., c1.c2.c1; the rest zero) -> the oracle's
    Fp12"""
    return gt_to_oracle(o1.ints_to_limbs([x % P for x in coeffs] + [0] * (12 - len(coeffs)), 6))


def fp12_lanes(worker, op, xs, ys):
    a = np.stack([_fp12_to_mont(x) for x in xs])
    b = np.stack([_fp12_to_mont(y) for y in ys])
    out = np.zeros_like(a)
    assert bb.load_library().bb_diag_fp12(worker._h, C.c_int(op), a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                                          out.ctypes.data_as(C.c_void_p), C.c_size_t(len(xs))) == 0
    return [_fp12_from_mont(row) for row in out]


@functools.lru_cache(maxsize=None)
def _frobenius_images(k):
    wk = PR.W.pow(P ** k)
    imgs = [ONE]
    for _ in range(11):
        imgs.append(imgs[-1] * wk)
    return imgs


def frobenius(a, k):
    """a^(p^k): the p^k-power map fixes Fp, so it is the linear map sending w^i to (w^(p^k))^i"""
    acc = ZERO
    for c, img in zip(a.c, _frobenius_images(k)):
        if c:
            acc = acc + img.scale(c)
    return acc


def easy_part(a):
    """a^((p^6 - 1)(p^2 + 1)): in the cyclotomic subgroup, and outside G_T for a random a"""
    t = frobenius(a, 6) * a.inv()
    return frobenius(t, 2) * t


HARD = 3 * (P ** 4 - P ** 2 + 1) // R


def final_exp(a):
    """a^(3 (p^12 - 1) / r), the device's final exponentiation, as the easy part then the hard part"""
    return easy_part(a).pow(HARD)


def edge_elements(rng):
    """zero, one, -1, each tower coefficient alone at 1 and at p - 1, all coefficients p - 1, Fp2 and Fp6 subfield elements
    and pure-w elements (tower c0 = 0)"""
    unit = lambda t, v: tower([v if s == t else 0 for s in range(12)])
    els = [ZERO, ONE, tower([P - 1])]
    els += [unit(t, v) for t in range(12) for v in (1, P - 1)]
    els.append(tower([P - 1] * 12))
    for _ in range(2):
        els.append(tower([rng.randrange(P), rng.randrange(P)]))
        els.append(tower([rng.randrange(P) for _ in range(6)]))
        els.append(tower([0] * 6 + [rng.randrange(P) for _ in range(6)]))
    return els


def in_fp6(a):
    """a lies in the subfield Fp6 (tower c1 = 0)"""
    return not _fp12_to_mont(a).reshape(12, 6)[6:].any()


def lanes_of(rng, n, edges):
    """n different elements: every edge element once (when n allows) among random ones, shuffled"""
    out = list(edges) if n >= len(edges) else []
    out += [tower([rng.randrange(P) for _ in range(12)]) for _ in range(n - len(out))]
    rng.shuffle(out)
    return out


def test_fp12_operations(worker, sizes=(1, 63, 64, 65, 200), n_final_exp=8, seed=43):
    """the eight ops of bb_diag_fp12 at each lane count, a different element on every lane and the edge elements among
    them; ops 0, 1, 4, 5, 7 in value, the inverse by a * (1/a) = 1 and zero -> zero, the cyclotomic squaring on
    cyclotomic-subgroup lanes, the final exponentiation in value on n_final_exp lanes spread over the sizes, one on every
    nonzero Fp6 lane and zero on zero"""
    rng = random.Random(seed)
    edges = edge_elements(rng)
    fe_left = n_final_exp
    for si, n in enumerate(sizes):
        xs, ys = lanes_of(rng, n, edges), lanes_of(rng, n, edges)
        assert len(xs) == n and len(ys) == n
        got = fp12_lanes(worker, 0, xs, ys)
        assert all(got[i] == xs[i] * ys[i] for i in range(n)), (n, [i for i in range(n) if got[i] != xs[i] * ys[i]][:8])
        got = fp12_lanes(worker, 1, xs, ys)
        assert all(got[i] == xs[i] * xs[i] for i in range(n)), n
        got = fp12_lanes(worker, 2, xs, ys)
        for i in range(n):
            assert (got[i] == ZERO) if xs[i].is_zero() else (got[i] * xs[i] == ONE), (n, i)
        for op, k in ((4, 1), (5, 2)):
            got = fp12_lanes(worker, op, xs, ys)
            assert all(got[i] == frobenius(xs[i], k) for i in range(n)), (n, op)
        lines = []                                               # op 7: the sparse line of b's c0.c0, c0.c1 and c1.c1
        for y in ys:
            w = _fp12_to_mont(y).reshape(12, 6).copy()
            w[[4, 5, 6, 7, 10, 11]] = 0
            lines.append(_fp12_from_mont(w.reshape(72)))
        got = fp12_lanes(worker, 7, xs, ys)
        assert all(got[i] == xs[i] * lines[i] for i in range(n)), n
        # cyclotomic squaring: g^k for random k and easy-part images (outside G_T) alternate, one among them
        cyc = [gt_pow()(rng.randrange(R)) if i % 2 else easy_part(tower([rng.randrange(P) for _ in range(12)])) for i in range(n)]
        cyc[rng.randrange(n)] = ONE
        got = fp12_lanes(worker, 3, cyc, ys)
        assert all(got[i] == cyc[i] * cyc[i] for i in range(n)), n
        # final exponentiation: value lanes at the last lane, the CTA's first lanes, the rest checked as a class
        per = fe_left // (len(sizes) - si)
        fe_left -= per
        value_lanes = sorted({n - 1, 0, 64 % n, 63 % n, n // 2}, reverse=True)[:per]
        for i in value_lanes:
            xs[i] = tower([rng.randrange(P) for _ in range(12)])
        got = fp12_lanes(worker, 6, xs, ys)
        for i in range(n):
            if xs[i].is_zero():
                assert got[i] == ZERO, (n, i)
            elif in_fp6(xs[i]):
                assert got[i] == ONE, (n, i)
        for i in value_lanes:
            assert got[i] == final_exp(xs[i]), (n, i)
    assert fe_left == 0


def test_final_exp_decomposition():
    """the exponent final_exp uses is the device's 3 (p^12 - 1) / r"""
    assert (P ** 4 - P ** 2 + 1) % R == 0
    assert (P ** 6 - 1) * (P ** 2 + 1) * HARD == 3 * PR.FINAL_EXP


# --------------------------------------------------------------------------------------------
# bb_diag_multi_pairing at many pairs
# --------------------------------------------------------------------------------------------
def pairing_of_scalars(worker, a, b):
    """the device's prod_i e([a_i] G1, [b_i] G2) (a scalar 0 gives the identity), as the oracle's Fp12"""
    g1 = o1.g1_fixed_mul(o1.fr_from_ints(a)) if a else np.zeros((0, 12), np.uint64)
    g2 = o1.g2_fixed_mul(o1.fr_from_ints(b)) if b else np.zeros((0, 24), np.uint64)
    return gt_to_oracle(V.multi_pairing(worker, g1, g2))


def check_pairing(worker, a, b):
    e = sum(x * y for x, y in zip(a, b)) % R
    got = pairing_of_scalars(worker, a, b)
    assert got == gt_pow()(e), (len(a), e)


def test_multi_pairing_values(worker, sizes=tuple(sorted(set(range(1, 71)) | {129, 1000})), seed=45):
    """the value at every n of `sizes` is g^(sum a_i b_i); identities on either side at the first, a middle and the last
    position; repeated pairs; P and -P against one Q; a large product whose exponent is zero is exactly one"""
    rng = random.Random(seed)
    rnd = lambda: rng.randrange(1, R)
    for n in sizes:
        check_pairing(worker, [rnd() for _ in range(n)], [rnd() for _ in range(n)])
    n = max(sizes)
    for side in (0, 1):                                          # identity A or B at the first, a middle, the last position
        a, b = [rnd() for _ in range(n)], [rnd() for _ in range(n)]
        for pos in (0, n // 2, n - 1):
            (a, b)[side][pos] = 0
        check_pairing(worker, a, b)
    a, b = [rnd() for _ in range(n)], [rnd() for _ in range(n)]  # repeated pairs, P and -P against the same Q
    for i in range(0, n - 1, 3):
        a[i + 1], b[i + 1] = a[i], b[i]
    if n >= 4:
        a[2], b[2] = R - a[3], b[3]
    check_pairing(worker, a, b)
    a, b = [rnd() for _ in range(n)], [rnd() for _ in range(n)]  # sum a_i b_i = 0: exactly one
    b[-1] = -sum(x * y for x, y in zip(a[:-1], b[:-1])) * pow(a[-1], -1, R) % R
    assert b[-1] and sum(x * y for x, y in zip(a, b)) % R == 0
    assert pairing_of_scalars(worker, a, b) == ONE


# --------------------------------------------------------------------------------------------
# the batch verifier's value (bb_diag_verify_batch_gt) and verify_each's values
# --------------------------------------------------------------------------------------------
def psi_of(s, x):
    return (s["t"][0] + sum(xj * tj for xj, tj in zip(x, s["t"][1:]))) % R


def make_proofs(s, rng, n, L, errors, a=None, b=None, x=None):
    """proofs A = [a_i], B = [b_i], C = [c_i] with a_i b_i = alpha beta + gamma psi_i + delta c_i - errors[i]: proof i is
    valid iff errors[i] = 0.  Inputs draw 0, 1 and r - 1 among random values."""
    a = list(a) if a is not None else [rng.randrange(1, R) for _ in range(n)]
    b = list(b) if b is not None else [rng.randrange(1, R) for _ in range(n)]
    pool = [0, 1, R - 1]
    x = x if x is not None else [[pool[(i + j) % 3] if (i + j) % 4 == 0 else rng.randrange(R) for j in range(L)] for i in range(n)]
    dinv = pow(s["delta"], -1, R)
    c = [(a[i] * b[i] - s["alpha"] * s["beta"] - s["gamma"] * psi_of(s, x[i]) + errors[i]) * dinv % R for i in range(n)]
    return {"a": a, "b": b, "c": c, "x": x, "L": L}


def proof_arrays(pr):
    n, L = len(pr["a"]), pr["L"]
    A = o1.g1_fixed_mul(o1.fr_from_ints(pr["a"])) if n else np.zeros((0, 12), np.uint64)
    B = o1.g2_fixed_mul(o1.fr_from_ints(pr["b"])) if n else np.zeros((0, 24), np.uint64)
    Cc = o1.g1_fixed_mul(o1.fr_from_ints(pr["c"])) if n else np.zeros((0, 12), np.uint64)
    flat = [v for row in pr["x"] for v in row]
    X = (o1.fr_from_ints(flat) if flat else np.zeros((0, 4), np.uint64)).reshape(n, L, 4)
    return A, B, Cc, X


def batch_exponent(s, pr, z):
    ab = s["alpha"] * s["beta"]
    return sum(zi * (-ai * bi + s["delta"] * ci + s["gamma"] * psi_of(s, xi) + ab)
               for zi, ai, bi, ci, xi in zip(z, pr["a"], pr["b"], pr["c"], pr["x"])) % R


def check_batch(pvk, s, pr, z, arrays=None):
    """verdict and value of bb_diag_verify_batch_gt against g^E; returns the verdict"""
    ok, out = V.verify_batch_arrays(pvk, *(arrays or proof_arrays(pr)), z=z, gt=True)
    e = batch_exponent(s, pr, z)
    assert gt_to_oracle(out) == gt_pow()(e), (len(z), pr["L"])
    assert ok == (e == 0), (len(z), pr["L"], e)
    return ok


def check_each(pvk, s, pr):
    """verdicts and the n + 1 values of bb_diag_verify_each_gt against g^(a_i b_i - gamma psi_i - delta c_i) and
    g^(alpha beta)"""
    verdicts, gt = V.verify_each_arrays(pvk, *proof_arrays(pr), gt=True)
    ab = s["alpha"] * s["beta"] % R
    assert gt_to_oracle(gt[-1]) == gt_pow()(ab)
    for i, (ai, bi, ci, xi) in enumerate(zip(pr["a"], pr["b"], pr["c"], pr["x"])):
        e = (ai * bi - s["gamma"] * psi_of(s, xi) - s["delta"] * ci) % R
        assert gt_to_oracle(gt[i]) == gt_pow()(e), i
        assert verdicts[i] == (0 if e == ab else 1), i
    return verdicts


# z values that feed mul_bits in k_proof_pairs / k_alpha_pair: 1, 2, r - 1, powers of two and long runs of ones
Z_SPECIAL = [1, 2, R - 1, R - 2, 1 << 63, 1 << 64, 1 << 253, (1 << 254) - 1, (1 << 128) - 1, ((1 << 200) - 1) << 50,
             (1 << 64) - 1, (R - 1) // 2]


def z_values(rng, n):
    """the special values on every third lane, in order (all of them from 36 lanes on), random ones between"""
    return [Z_SPECIAL[(i // 3) % len(Z_SPECIAL)] if i % 3 == 0 else rng.randrange(1, R) for i in range(n)]


def new_key(rng, L, t=None):
    s, vk, _ = trapdoor_key(rng, t if t is not None else [rng.randrange(1, R) for _ in range(L + 1)])
    return s, vk


def test_batch_exponent_matches_pairs(worker, seed=47):
    """the exponent form of the batch value, signs included, against the oracle's multi_pairing over the verifier's own
    pairs ([z_i] A_i, -B_i), (sum z_i C_i, delta), (Psi, gamma), ([sum z_i] alpha, beta) for two invalid proofs"""
    rng = random.Random(seed)
    s, vk = new_key(rng, 2)
    pvk = bb.prepare_verifying_key(worker, vk)
    pr = make_proofs(s, rng, 2, 2, [rng.randrange(1, R) for _ in range(2)])
    z = [rng.randrange(1, R) for _ in range(2)]
    g1 = lambda k: F.G1.mul(F.G1_GEN, k % R) if k % R else None
    g2 = lambda k: F.G2.mul(F.G2_GEN, k % R) if k % R else None
    pairs = [(F.G1.mul(g1(ai), zi), F.G2.neg(g2(bi))) for ai, bi, zi in zip(pr["a"], pr["b"], z)]
    acc_c = None
    for ci, zi in zip(pr["c"], z):
        acc_c = F.G1.add(acc_c, F.G1.mul(g1(ci), zi))
    acc = [sum(z)] + [sum(zi * xi[j] for zi, xi in zip(z, pr["x"])) for j in range(2)]
    psi = None
    for accj, tj in zip(acc, s["t"]):
        psi = F.G1.add(psi, F.G1.mul(g1(tj), accj % R))
    pairs += [(acc_c, g2(s["delta"])), (psi, g2(s["gamma"])), (F.G1.mul(g1(s["alpha"]), sum(z) % R), g2(s["beta"]))]
    want = PR.multi_pairing(pairs).pow(V.gt_exponent() % R)
    ok, out = V.verify_batch_arrays(pvk, *proof_arrays(pr), z=z, gt=True)
    assert not ok and gt_to_oracle(out) == want
    assert want == gt_pow()(batch_exponent(s, pr, z))
    pvk.free()


def test_batch_values(worker, sizes=(1, 2, 63, 64, 65, 255, 256, 257, 513, 4096), inputs=(1, 2, 7), seed=49):
    """every proof invalid by its own amount, so that every lane contributes to E: the value is g^E at each batch size
    (column-sum chunks of 256 rows) and input count; L = 0; the same proofs made valid are accepted with value one"""
    rng = random.Random(seed)
    cases = [(n, inputs[i % len(inputs)]) for i, n in enumerate(sizes)] + [(n, L) for L in inputs for n in sizes if n in (65, 257)]
    cases += [(min(sizes[-1], 65), 0), (1, 0)]
    for n, L in cases:
        s, vk = new_key(rng, L)
        pvk = bb.prepare_verifying_key(worker, vk)
        z = z_values(rng, n)
        pr = make_proofs(s, rng, n, L, [rng.randrange(1, R) for _ in range(n)])
        check_batch(pvk, s, pr, z)
        if n in (sizes[-1], 65, 1):                              # the same a, b, x made valid
            good = make_proofs(s, rng, n, L, [0] * n, a=pr["a"], b=pr["b"], x=pr["x"])
            assert check_batch(pvk, s, good, z)
        pvk.free()


def edge_batches(rng, n, L):
    """the identity edges of the batch verifier, each as (name, key scalars, vk, make(errors) -> (proofs, z)):
    sum z_i = 0 ([acc_y] alpha is the identity), sum z_i c_i = 0, Psi the identity by its sum and by identity ic[j] under
    nonzero inputs, identity A, B and C inside the batch"""
    out = []
    s, vk = new_key(rng, L)

    def last_z(pr, weights):                                     # z_last so that sum z_i w_i = 0
        z = [rng.randrange(1, R) for _ in range(n - 1)]
        zl = -sum(zi * wi for zi, wi in zip(z, weights)) * pow(weights[-1], -1, R) % R
        assert zl
        return z + [zl]

    def sum_z(errors):
        pr = make_proofs(s, rng, n, L, errors)
        return pr, last_z(pr, [1] * n)

    def sum_zc(errors):
        pr = make_proofs(s, rng, n, L, errors)
        return pr, last_z(pr, pr["c"])

    def psi_sum(errors):
        pr = make_proofs(s, rng, n, L, errors)
        return pr, last_z(pr, [psi_of(s, xi) for xi in pr["x"]])

    out += [("sum z = 0", s, vk, sum_z), ("sum z c = 0", s, vk, sum_zc), ("Psi = 0 by its sum", s, vk, psi_sum)]
    t = [rng.randrange(1, R) for _ in range(L + 1)]
    t[L] = 0                                                     # the last ic is the identity
    s2, vk2 = new_key(rng, L, t)

    def ic_ident(errors):
        x = [[rng.randrange(1, R) for _ in range(L)] for _ in range(n)]
        return make_proofs(s2, rng, n, L, errors, x=x), [rng.randrange(1, R) for _ in range(n)]

    out.append(("identity ic[L]", s2, vk2, ic_ident))
    pos = sorted({0, n // 2, n - 1})

    def ident(which):
        def make(errors):
            a = [rng.randrange(1, R) for _ in range(n)]
            b = [rng.randrange(1, R) for _ in range(n)]
            x = [[rng.randrange(R) for _ in range(L)] for _ in range(n)]
            if which == "a":
                for p in pos:
                    a[p] = 0
            elif which == "b":
                for p in pos:
                    b[p] = 0
            pr = make_proofs(s, rng, n, L, errors, a=a, b=b, x=x)
            if which == "c":                                     # b_i so that c_i = 0: a_i b_i = alpha beta + gamma psi_i - e_i
                for p in pos:
                    rest = (s["alpha"] * s["beta"] + s["gamma"] * psi_of(s, x[p]) - errors[p]) % R
                    b[p] = rest * pow(a[p], -1, R) % R
                pr = make_proofs(s, rng, n, L, errors, a=a, b=b, x=x)
                assert all(pr["c"][p] == 0 for p in pos)
            return pr, [rng.randrange(1, R) for _ in range(n)]
        return make

    out += [("identity " + w.upper(), s, vk, ident(w)) for w in ("a", "b", "c")]
    return out


def test_batch_identity_edges(worker, n=300, L=2, seed=51):
    """each identity edge with invalid proofs (value g^E) and with all proofs valid (accepted, value one); with
    verify_each's values and verdicts over the same proofs"""
    rng = random.Random(seed)
    for name, s, vk, make in edge_batches(rng, n, L):
        pvk = bb.prepare_verifying_key(worker, vk)
        pr, z = make([rng.randrange(1, R) for _ in range(n)])
        assert not check_batch(pvk, s, pr, z), name
        assert check_each(pvk, s, pr).all(), name
        pr, z = make([0] * n)
        assert check_batch(pvk, s, pr, z), name
        assert not check_each(pvk, s, pr).any(), name
        pvk.free()


def test_batch_soundness_sweep(worker, n=200, L=2, seed=53):
    """proof k alone invalid, for every k: each batch is rejected and its value is g^(z_k e_k)"""
    rng = random.Random(seed)
    s, vk = new_key(rng, L)
    pvk = bb.prepare_verifying_key(worker, vk)
    good = make_proofs(s, rng, n, L, [0] * n)
    errs = [rng.randrange(1, R) for _ in range(n)]
    bad = make_proofs(s, rng, n, L, errs, a=good["a"], b=good["b"], x=good["x"])
    A, B, Cg, X = proof_arrays(good)
    Cb = o1.g1_fixed_mul(o1.fr_from_ints(bad["c"]))
    z = z_values(rng, n)
    for k in range(n):
        c = Cg.copy()
        c[k] = Cb[k]
        pr = dict(good, c=good["c"][:k] + [bad["c"][k]] + good["c"][k + 1:])
        assert batch_exponent(s, pr, z) == z[k] * errs[k] % R
        assert not check_batch(pvk, s, pr, z, arrays=(A, B, c, X)), k
    pvk.free()


def test_each_values(worker, n=4096, L=2, seed=55):
    """verify_each at n proofs, valid ones and ones invalid by distinct amounts mixed: every value and every verdict"""
    rng = random.Random(seed)
    s, vk = new_key(rng, L)
    pvk = bb.prepare_verifying_key(worker, vk)
    errors = [0 if rng.random() < 0.4 else rng.randrange(1, R) for _ in range(n)]
    errors[0], errors[-1] = 0, 1
    pr = make_proofs(s, rng, n, L, errors)
    verdicts = check_each(pvk, s, pr)
    assert verdicts.tolist() == [0 if e == 0 else 1 for e in errors]
    pvk.free()
