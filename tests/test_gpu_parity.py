"""GPU parity: the CUDA path, called through the C ABI, against the CPU oracle (oracle/o1.py)
on the same seeded inputs.  Bit-exact throughout: this is integer arithmetic.

Mirrors the reference's own tests where it has them: multiexp.rs:334-378 (naive == fast),
domain.rs:376-498 (polynomial_arith, fft_composition, parallel_fft_consistency),
groth16/tests/mimc.rs (prove MiMC-322), groth16/src/lib.rs:559 (192-byte proof).
"""
import ctypes as C
import random

import numpy as np
import pytest

import bellman_b200 as bb
from oracle import o1

pytestmark = pytest.mark.gpu

R = o1.FR_MODULUS
P = o1.FP_MODULUS


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def _selftest_field(worker, field, op, a, b):
    out = np.zeros_like(a)
    rc = bb.load_library().bb_selftest_field(worker._h, C.c_int(field), C.c_int(op), a.ctypes.data_as(C.c_void_p),
                                             b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_size_t(a.shape[0]))
    assert rc == 0
    return out


def _selftest_point(worker, group, op, a, b):
    out = np.zeros_like(a)
    rc = bb.load_library().bb_selftest_point(worker._h, C.c_int(group), C.c_int(op), a.ctypes.data_as(C.c_void_p),
                                             b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_size_t(a.shape[0]))
    assert rc == 0
    return out


# --------------------------------------------------------------------------------------------
# field and curve arithmetic
# --------------------------------------------------------------------------------------------
def test_field_arithmetic(worker):
    rng = random.Random(21)
    for field, q, nl, frm, mul, add, sub in ((0, R, 4, o1.fr_from_ints, o1.fr_mul, o1.fr_add, o1.fr_sub),
                                             (1, P, 6, o1.fp_from_ints, o1.fp_mul, o1.fp_add, o1.fp_sub)):
        edge = [0, 1, 2, q - 1, q - 2, (1 << (64 * nl - 1)) % q, (1 << 64) - 1, (1 << 32) - 1, (q - 1) // 2, (q + 1) // 2]
        xs = [x for x in edge for _ in edge] + [rng.randrange(q) for _ in range(4000)]
        ys = [y for _ in edge for y in edge] + [rng.randrange(q) for _ in range(4000)]
        a, b = frm(xs), frm(ys)
        # edge limb patterns directly in Montgomery form too (all-ones limbs below the modulus)
        raw = o1.ints_to_limbs([(q - 1), (1 << (64 * nl - 2)) - 1, ((1 << (64 * (nl - 1))) - 1)], nl)
        a = np.concatenate([a, raw, raw])
        b = np.concatenate([b, raw, raw[::-1]])
        assert np.array_equal(_selftest_field(worker, field, 0, a, b), mul(a, b))
        assert np.array_equal(_selftest_field(worker, field, 1, a, b), add(a, b))
        assert np.array_equal(_selftest_field(worker, field, 2, a, b), sub(a, b))
        assert np.array_equal(_selftest_field(worker, field, 3, a, b), mul(a, a))


def test_fp_inversion_both_ways(worker):
    """fp_inv_gcd (binary Euclid on the raw limbs, what the batched-affine rounds and to_affine use) and the
    Fermat power a^(p-2) against python's pow()."""
    rng = random.Random(22)
    xs = [1, 2, 3, P - 1, P - 2, (P - 1) // 2, (P + 1) // 2, 1 << 380, (1 << 381) - 1 - ((1 << 381) - 1) // P * 0, (1 << 64) - 1, 1 << 32] + \
         [rng.randrange(1, P) for _ in range(3000)] + [rng.randrange(1, 1 << 40) for _ in range(50)]
    xs = [x % P or 1 for x in xs]
    a = o1.fp_from_ints(xs + [0])
    want = o1.fp_from_ints([pow(x, -1, P) for x in xs] + [0])
    for op in (4, 5):
        assert np.array_equal(_selftest_field(worker, 1, op, a, a), want), op


def test_point_arithmetic(worker):
    ks = o1.fr_random(31, 64)
    ks2 = o1.fr_random(32, 64)
    for group, fixed, add, mul in ((bb.G1, o1.g1_fixed_mul, o1.g1_add, o1.g1_mul), (bb.G2, o1.g2_fixed_mul, o1.g2_add, o1.g2_mul)):
        a, b = fixed(ks), fixed(ks2)
        b[0] = a[0]                 # doubling through the addition formulas
        b[1] = 0                    # b = identity
        a[2] = 0                    # a = identity
        a[3] = 0; b[3] = 0          # both
        neg1 = mul(a[4:5], o1.fr_from_ints([R - 1]))
        b[4] = neg1[0]              # a + (-a) = identity
        assert np.array_equal(_selftest_point(worker, group, 0, a, b), add(a, b))
        two_a = add(a, a)
        assert np.array_equal(_selftest_point(worker, group, 1, a, b), add(two_a, b))
        assert np.array_equal(_selftest_point(worker, group, 2, a, b), add(a, b))
        # device fixed-base multiplication (used to manufacture benchmark-size CRS material)
        assert np.array_equal(bb.fixed_base_mul(worker, group, ks), fixed(ks))
        edge = o1.fr_from_ints([0, 1, 2, R - 1, 255, 256, 1 << 255 - 1])
        assert np.array_equal(bb.fixed_base_mul(worker, group, edge), fixed(edge))
        pts = fixed(ks[:4])
        comp = o1.g1_compress(pts) if group == bb.G1 else o1.g2_compress(pts)
        for i in range(4):
            assert bb.point_compress(group, pts[i:i + 1]) == bytes(comp[i])


def test_bucket_reduction_kernels(worker):
    """sum_d d * B_d (multiexp.rs:271-275) through the multi-level reduction, every level shape."""
    lib = bb.load_library()
    rng = random.Random(33)
    # windows of >= 1024 buckets go through row / column sums first
    for D, K in ((1, 8), (2, 8), (8, 8), (64, 2), (64, 8), (512, 16), (1024, 4), (2048, 16), (4096, 8),
                 (4096, 4), (8192, 4), (32768, 8), (32768, 16)):
        ks = [rng.randrange(R) for _ in range(D)]
        for i in range(0, D, 7):
            ks[i] = 0                                   # empty buckets
        pts = o1.g1_fixed_mul(o1.fr_from_ints(ks))
        out = np.zeros((1, 12), np.uint64)
        rc = lib.bb_selftest_bucket_reduce(worker._h, pts.ctypes.data_as(C.c_void_p), C.c_uint32(D), C.c_uint32(K),
                                           out.ctypes.data_as(C.c_void_p))
        assert rc == 0
        want = o1.g1_fixed_mul(o1.fr_from_ints([sum((i + 1) * k for i, k in enumerate(ks)) % R]))
        assert np.array_equal(out, want), (D, K)


# --------------------------------------------------------------------------------------------
# NTT (src/domain.rs)
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [0, 1, 2, 3, 5, 8, 9, 10, 11, 12, 13, 14, 16])
def test_ntt_matches_oracle(worker, log_n):
    o1.set_threads(8)
    v = o1.fr_random(100 + log_n, 1 << log_n)
    for mode, omode in ((bb.NTT_FFT, o1.FFT), (bb.NTT_IFFT, o1.IFFT), (bb.NTT_COSET_FFT, o1.COSET_FFT), (bb.NTT_ICOSET_FFT, o1.ICOSET_FFT)):
        dom = bb.EvaluationDomain.from_coeffs(worker, v)
        assert dom.exp == log_n
        [dom.fft, dom.ifft, dom.coset_fft, dom.icoset_fft][mode]()
        assert np.array_equal(dom.into_coeffs(), o1.fft(v, omode)), (log_n, mode)


def test_ntt_tile_shapes_do_not_change_results(worker):
    v = o1.fr_random(7, 1 << 14)
    want = o1.fft(v, o1.COSET_FFT)
    try:
        for tile_log, col_bits in ((11, 3), (11, 1), (10, 0), (9, 4), (6, 2), (12, 2)):
            worker.set_option("ntt_tile_log", tile_log)
            worker.set_option("ntt_col_bits", col_bits)
            dom = bb.EvaluationDomain.from_coeffs(worker, v)
            dom.coset_fft()
            assert np.array_equal(dom.into_coeffs(), want), (tile_log, col_bits)
    finally:
        worker.set_option("ntt_tile_log", 11)
        worker.set_option("ntt_col_bits", 3)


def test_ntt_padding_and_degree_limit(worker):
    # from_coeffs pads to the next power of two (domain.rs:49-69)
    v = o1.fr_random(8, 13)
    dom = bb.EvaluationDomain.from_coeffs(worker, v)
    assert dom.exp == 4 and dom.coeffs.shape[0] == 16
    dom.fft()
    padded = np.zeros((16, 4), np.uint64); padded[:13] = v
    assert np.array_equal(dom.into_coeffs(), o1.fft(padded, o1.FFT))
    # exp >= S is PolynomialDegreeTooLarge (domain.rs:57-59)
    buf = np.zeros((4, 4), np.uint64)
    rc = bb.load_library().bb_ntt(worker._h, buf.ctypes.data_as(C.c_void_p), C.c_uint32(32), C.c_int(0), C.c_int(1))
    assert rc == 1


def test_ntt_canonical_form_is_also_exact(worker):
    # the transform is linear: canonical integers in, canonical integers out
    ints = [random.Random(9).randrange(R) for _ in range(64)]
    canon = o1.ints_to_limbs(ints, 4)
    rc = bb.load_library().bb_ntt(worker._h, canon.ctypes.data_as(C.c_void_p), C.c_uint32(6), C.c_int(bb.NTT_ICOSET_FFT), C.c_int(0))
    assert rc == 0
    want = o1.fr_to_canonical(o1.fft(o1.fr_from_ints(ints), o1.ICOSET_FFT))
    assert np.array_equal(canon, want)


def test_ntt_full_size_round_trips(worker):
    """BASELINE.json configs[3] at 2^20 here (2^24 in bench.py): size-independent properties of
    domain.rs:436-457 (fft_composition) on the device, plus oracle equality of one transform."""
    log_n = 20
    v = o1.fr_random(11, 1 << log_n)
    d = worker.device_alloc(v.nbytes)
    try:
        worker.upload(d, v)
        bb.ntt_device(worker, d, log_n, bb.NTT_FFT)
        fwd = np.zeros_like(v); worker.download(d, fwd)
        bb.ntt_device(worker, d, log_n, bb.NTT_IFFT)
        back = np.zeros_like(v); worker.download(d, back)
        assert np.array_equal(back, v)
        bb.ntt_device(worker, d, log_n, bb.NTT_COSET_FFT)
        bb.ntt_device(worker, d, log_n, bb.NTT_ICOSET_FFT)
        worker.download(d, back)
        assert np.array_equal(back, v)
        o1.set_threads(0)
        assert np.array_equal(fwd, o1.fft(v, o1.FFT))
    finally:
        worker.device_free(d)


def test_ntt_2e24_matches_oracle(worker):
    """BASELINE.json configs[3] at its full size: the forward transform of 2^24 points equals the
    oracle's (serial_fft semantics, domain.rs:272-314) element for element, and the inverse returns
    the input (domain.rs:436-457)."""
    log_n = 24
    n = 1 << log_n
    d = worker.device_alloc(n * 32)
    try:
        bb.synth_scalars_device(worker, 41, n, d)           # canonical integers < 2^254: valid Montgomery limbs as well
        v = np.zeros((n, 4), np.uint64); worker.download(d, v)
        bb.ntt_device(worker, d, log_n, bb.NTT_FFT)
        fwd = np.zeros_like(v); worker.download(d, fwd)
        bb.ntt_device(worker, d, log_n, bb.NTT_IFFT)
        back = np.zeros_like(v); worker.download(d, back)
        assert np.array_equal(back, v)
        o1.set_threads(0)
        want = o1.fft(v, o1.FFT)
        assert np.array_equal(fwd, want)
    finally:
        worker.device_free(d)


def test_domain_methods_compose_like_the_reference(worker):
    """The H block of create_proof written out with the individual EvaluationDomain methods
    (prover.rs:222-240) equals the fused bb_h_poly and the oracle; distribute_powers + fft
    equals coset_fft (domain.rs:115-118)."""
    n = 700
    a, b = o1.fr_random(501, n), o1.fr_random(502, n)
    c = o1.fr_mul(a, b)
    doms = [bb.EvaluationDomain.from_coeffs(worker, v) for v in (a, b, c)]
    for d in doms:
        d.ifft()
        d.coset_fft()
    A, B, Cc = doms
    A.mul_assign(B)
    A.sub_assign(Cc)
    A.divide_by_z_on_coset()
    A.icoset_fft()
    want = o1.h_poly(a, b, c)
    assert np.array_equal(A.into_coeffs()[:-1], want)
    assert np.array_equal(o1.fr_to_canonical(want), bb.h_poly(worker, a, b, c))
    v = o1.fr_random(503, 1 << 9)
    d1 = bb.EvaluationDomain.from_coeffs(worker, v)
    d1.distribute_powers(7)
    d1.fft()
    assert np.array_equal(d1.into_coeffs(), o1.fft(v, o1.COSET_FFT))
    tau = 0x123456789abcdef
    assert d1.z(tau) == (pow(tau, 512, R) - 1) % R


def test_h_poly_matches_oracle(worker):
    for n in (1, 2, 5, 646, 5000):
        a, b = o1.fr_random(200 + n, n), o1.fr_random(300 + n, n)
        c = o1.fr_mul(a, b)
        c[n // 2] = o1.fr_random(5, 1)[0]          # need not be satisfied: same arithmetic either way
        want = o1.fr_to_canonical(o1.h_poly(a, b, c)) if n > 1 else np.zeros((0, 4), np.uint64)
        got = bb.h_poly(worker, a, b, c)
        assert got.shape == want.shape and np.array_equal(got, want), n


# --------------------------------------------------------------------------------------------
# MSM (src/multiexp.rs)
# --------------------------------------------------------------------------------------------
def _gpu_multiexp(worker, group, bases_arr, offset, density, scalars, form=bb.FORM_MONTGOMERY):
    bases = bb.Bases(worker, group, bases_arr)
    dm = bb.FullDensity if density is None else bb.DensityTracker(density)
    return bb.multiexp(worker, (bases, offset), dm, scalars, form).wait()


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 1000, 1 << 14])
def test_multiexp_g1_matches_oracle(worker, n):
    ks = o1.fr_random(1000 + n, n)
    bases = o1.g1_fixed_mul(ks)
    ex = o1.fr_random(2000 + n, n)
    if n > 8:
        ex[3] = 0; ex[5] = o1.fr_from_ints([1])[0]; ex[6] = o1.fr_from_ints([R - 1])[0]; ex[7] = o1.fr_from_ints([2])[0]
    rc, want = o1.multiexp(1, bases, 0, None, ex)
    assert rc == 0
    got = _gpu_multiexp(worker, bb.G1, bases, 0, None, ex)
    assert np.array_equal(got, want)
    # Exponent::Bits form (canonical integers) gives the same point
    got2 = _gpu_multiexp(worker, bb.G1, bases, 0, None, o1.fr_to_canonical(ex), bb.FORM_CANONICAL)
    assert np.array_equal(got2, want)


def test_multiexp_window_choice_does_not_change_results(worker):
    n = 3000
    bases = o1.g1_fixed_mul(o1.fr_random(41, n))
    ex = o1.fr_random(42, n)
    rc, want = o1.multiexp(1, bases, 0, None, ex)
    try:
        for c in (2, 3, 5, 8, 13, 15, 16, 17):
            worker.set_option("msm_window_bits", c)
            assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want), c
    finally:
        worker.set_option("msm_window_bits", 0)


@pytest.mark.parametrize("n", [0, 3, 40, 2000])
def test_multiexp_g2_matches_oracle(worker, n):
    bases = o1.g2_fixed_mul(o1.fr_random(3000 + n, n))
    ex = o1.fr_random(4000 + n, n)
    rc, want = o1.multiexp(2, bases, 0, None, ex)
    assert rc == 0
    assert np.array_equal(_gpu_multiexp(worker, bb.G2, bases, 0, None, ex), want)


def test_multiexp_density_offset_and_fast_paths(worker):
    rng = np.random.default_rng(5)
    n = 5000
    dens = rng.random(n) < 0.5
    k = int(dens.sum())
    off = 7
    bases = o1.g1_fixed_mul(o1.fr_random(51, off + k + 3))       # 3 trailing bases are ignored
    ex = o1.fr_random(52, n)
    # boolean-heavy witness: Exponent::Zero / Exponent::One fast paths (multiexp.rs:245-252)
    kind = rng.integers(0, 4, n)
    ex[kind == 0] = 0
    ex[kind == 1] = o1.fr_from_ints([1])[0]
    rc, want = o1.multiexp(1, bases, off, dens.astype(np.uint8), ex)
    assert rc == 0
    assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, off, dens, ex), want)
    # repeated bases: buckets must double / cancel correctly
    rep = np.repeat(bases[:5], 40, axis=0)
    ex2 = np.repeat(ex[10:12], 100, axis=0)
    rc, want2 = o1.multiexp(1, rep, 0, None, ex2)
    assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, rep, 0, None, ex2), want2)
    neg = o1.fr_sub(np.zeros((1, 4), np.uint64), ex[10:11])
    both = np.concatenate([ex[10:11], neg])
    got = _gpu_multiexp(worker, bb.G1, np.concatenate([bases[:1], bases[:1]]), 0, None, both)
    assert not got.any()                                           # P*k + P*(-k) = identity


def test_multiexp_skewed_scalars(worker):
    """Witnesses full of equal / tiny values put most bases into a handful of buckets; the
    oversized-bucket path must give the same point (and not serialise on one thread)."""
    rng = np.random.default_rng(8)
    n = 6000
    bases = o1.g1_fixed_mul(o1.fr_random(81, n))
    cases = {
        "all twos": o1.fr_from_ints([2] * n),
        "nibbles": o1.fr_from_ints([int(x) for x in rng.integers(0, 16, n)]),
        "bytes+big": o1.fr_from_ints([int(x) for x in rng.integers(0, 256, n - 5)] + [R - 1, R - 2, 3, 1 << 200, 7]),
        "same 255-bit value": np.repeat(o1.fr_random(82, 1), n, axis=0),
    }
    for name, ex in cases.items():
        rc, want = o1.multiexp(1, bases, 0, None, ex)
        assert rc == 0
        assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want), name
    # force the task path on ordinary data too: every bucket above 3 entries is cut up
    ex = o1.fr_random(83, n)
    rc, want = o1.multiexp(1, bases, 0, None, ex)
    try:
        worker.set_option("msm_big_cap", 3)
        worker.set_option("msm_window_bits", 8)
        assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want)
        b2 = o1.g2_fixed_mul(o1.fr_random(84, 500))
        rc, want2 = o1.multiexp(2, b2, 0, None, ex[:500])
        assert np.array_equal(_gpu_multiexp(worker, bb.G2, b2, 0, None, ex[:500]), want2)
    finally:
        worker.set_option("msm_big_cap", 0)
        worker.set_option("msm_window_bits", 0)


def test_multiexp_naive_property_full_size(worker):
    """benches/slow.rs shape scaled up (2^18 here; bench.py does 2^24): bases are [k_i]G made on
    the device, so the expected point is [sum k_i e_i]G -- multiexp.rs:334-378's property."""
    n = 1 << 18
    ks, ex = o1.fr_random(61, n), o1.fr_random(62, n)
    bases = bb.fixed_base_mul(worker, bb.G1, ks)
    assert np.array_equal(bases[:64], o1.g1_fixed_mul(ks[:64]))
    got = _gpu_multiexp(worker, bb.G1, bases, 0, None, ex)
    tot = sum(a * b for a, b in zip(o1.fr_to_ints(ks), o1.fr_to_ints(ex))) % R
    assert np.array_equal(got, o1.g1_fixed_mul(o1.fr_from_ints([tot])))


def test_multiexp_large_windows(worker):
    """choose_window's top entry (c = 17: the 2^24 path, its top window the carry alone), c = 20 (D = 2^19 buckets)
    and their neighbours, forced at 2^18 points; expected point by multiexp.rs:334-378's property."""
    n = 1 << 18
    ks, ex = o1.fr_random(63, n), o1.fr_random(64, n)
    bases_arr = bb.fixed_base_mul(worker, bb.G1, ks)
    tot = sum(a * b for a, b in zip(o1.fr_to_ints(ks), o1.fr_to_ints(ex))) % R
    want = o1.g1_fixed_mul(o1.fr_from_ints([tot]))
    bases = bb.Bases(worker, bb.G1, bases_arr)
    try:
        for c in (17, 18, 19, 20, 21, 22):
            worker.set_option("msm_window_bits", c)
            got = bb.multiexp(worker, (bases, 0), bb.FullDensity, ex).wait()
            assert np.array_equal(got, want), c
    finally:
        worker.set_option("msm_window_bits", 0)
        bases.free()


def test_multiexp_g2_2e16_matches_oracle(worker):
    n = 1 << 16
    bases = bb.fixed_base_mul(worker, bb.G2, o1.fr_random(3100, n))
    assert np.array_equal(bases[:16], o1.g2_fixed_mul(o1.fr_random(3100, n)[:16]))
    ex = o1.fr_random(4100, n)
    o1.set_threads(0)
    rc, want = o1.multiexp(2, bases, 0, None, ex)
    assert rc == 0
    assert np.array_equal(_gpu_multiexp(worker, bb.G2, bases, 0, None, ex), want)


def test_fr_dot_diagnostic(worker):
    n = 5000
    a, b = o1.fr_to_canonical(o1.fr_random(71, n)), o1.fr_to_canonical(o1.fr_random(72, n))
    da, db = worker.device_alloc(a.nbytes), worker.device_alloc(b.nbytes)
    try:
        worker.upload(da, a); worker.upload(db, b)
        got = bb.fr_dot_device(worker, da, db, n)
        want = sum(x * y for x, y in zip(o1.limbs_to_ints(a), o1.limbs_to_ints(b))) % R
        assert o1.limbs_to_ints(got.reshape(1, 4))[0] == want
    finally:
        worker.device_free(da); worker.device_free(db)


@pytest.mark.parametrize("log_n,c", [(22, 0), (22, 20)])
def test_multiexp_synthetic_bases_naive_property(worker, log_n, c):
    """What bench.py --workload msm asserts at 2^24, here at 2^22: device-made bases [k_i]G, device-made
    scalars, MSM == [sum k_i e_i]G.  The k_i stream and the fixed-base multiplication are themselves
    checked against the oracle on a prefix."""
    n = 1 << log_n
    bases = bb.Bases.synthetic(worker, bb.G1, 31, n)
    d_k, d_e = worker.device_alloc(n * 32), worker.device_alloc(n * 32)
    try:
        bb.synth_scalars_device(worker, 31, n, d_k)
        bb.synth_scalars_device(worker, 32, n, d_e)
        worker.set_option("msm_window_bits", c)
        got = bb.multiexp_device(worker, (bases, 0), d_e, n, bb.FORM_CANONICAL).wait()
        dot = bb.fr_dot_device(worker, d_k, d_e, n)
        want = o1.g1_fixed_mul(o1.fr_from_ints(o1.limbs_to_ints(dot.reshape(1, 4))))
        assert np.array_equal(np.asarray(got).reshape(-1), want.reshape(-1))
        # independent of the device dot product: a 4096-term prefix against python integers
        m = 4096
        kk = np.zeros((m, 4), np.uint64); ee = np.zeros((m, 4), np.uint64)
        worker.download(d_k, kk); worker.download(d_e, ee)
        dm = bb.fr_dot_device(worker, d_k, d_e, m)
        assert o1.limbs_to_ints(dm.reshape(1, 4))[0] == sum(x * y for x, y in zip(o1.limbs_to_ints(kk), o1.limbs_to_ints(ee))) % R
    finally:
        worker.set_option("msm_window_bits", 0)
        worker.device_free(d_k); worker.device_free(d_e)
        bases.free()


@pytest.fixture()
def affine(worker):
    """forces the batched-affine halving rounds (batch_affine.cuh) at sizes where they are off by default"""
    def force(rounds, batch=16):
        worker.set_option("msm_affine_rounds", rounds)
        worker.set_option("msm_affine_batch", batch)
    yield force
    worker.set_option("msm_affine_rounds", -1)
    worker.set_option("msm_affine_batch", 16)


@pytest.mark.parametrize("n,rounds,batch", [(1, 3, 16), (2, 1, 16), (33, 2, 4), (1000, 3, 16), (1000, 1, 1), (3000, 4, 7), (5000, 3, 1),
                                            (1 << 14, 3, 16)])
def test_affine_rounds_g1_match_oracle(worker, affine, n, rounds, batch):
    affine(rounds, batch)
    ks = o1.fr_random(1000 + n, n)
    bases = o1.g1_fixed_mul(ks)
    ex = o1.fr_random(2000 + n, n)
    if n > 8:
        ex[3] = 0; ex[5] = o1.fr_from_ints([1])[0]; ex[6] = o1.fr_from_ints([R - 1])[0]; ex[7] = o1.fr_from_ints([2])[0]
    rc, want = o1.multiexp(1, bases, 0, None, ex)
    assert rc == 0
    assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want)


@pytest.mark.parametrize("n,rounds", [(3, 2), (40, 3), (700, 3)])
def test_affine_rounds_g2_match_oracle(worker, affine, n, rounds):
    affine(rounds)
    bases = o1.g2_fixed_mul(o1.fr_random(3000 + n, n))
    ex = o1.fr_random(4000 + n, n)
    rc, want = o1.multiexp(2, bases, 0, None, ex)
    assert rc == 0
    assert np.array_equal(_gpu_multiexp(worker, bb.G2, bases, 0, None, ex), want)


def test_affine_rounds_special_pairs(worker, affine):
    """Pairs the affine formulas cannot add directly: equal points (doubling through 2y), opposite points
    (the identity travels on as a null row), identity rows meeting points; plus skewed buckets and every
    window size, density maps and the Exponent::Zero / One paths."""
    rng = np.random.default_rng(9)
    n = 4000
    bases = o1.g1_fixed_mul(o1.fr_random(91, n))
    ex = o1.fr_random(92, n)
    for rounds in (1, 2, 3, 5):
        affine(rounds, 5)
        # the same base many times with the same scalar: every pair of a bucket is a doubling, then again
        rep = np.repeat(bases[:6], 64, axis=0)
        ex2 = np.repeat(ex[10:12], 192, axis=0)
        rc, want = o1.multiexp(1, rep, 0, None, ex2)
        assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, rep, 0, None, ex2), want), rounds
        # k P and (-k) P side by side: cancellation inside the rounds
        neg = o1.fr_sub(np.zeros((1, 4), np.uint64), ex[10:11])
        both = np.concatenate([ex[10:11], neg] * 40)
        pts = np.repeat(bases[:1], 80, axis=0)
        got = _gpu_multiexp(worker, bb.G1, pts, 0, None, both)
        assert not got.any(), rounds
        mixed = np.concatenate([both, ex[20:60]])
        mpts = np.concatenate([pts, bases[20:60]])
        rc, want = o1.multiexp(1, mpts, 0, None, mixed)
        assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, mpts, 0, None, mixed), want), rounds
    affine(3)
    cases = {
        "all twos": o1.fr_from_ints([2] * n),
        "nibbles": o1.fr_from_ints([int(x) for x in rng.integers(0, 16, n)]),
        "same 255-bit value": np.repeat(o1.fr_random(93, 1), n, axis=0),
    }
    for name, e in cases.items():
        rc, want = o1.multiexp(1, bases, 0, None, e)
        assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, e), want), name
    try:
        rc, want = o1.multiexp(1, bases, 0, None, ex)
        for c in (3, 8, 13, 16):
            worker.set_option("msm_window_bits", c)
            assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want), c
        worker.set_option("msm_big_cap", 3)
        assert np.array_equal(_gpu_multiexp(worker, bb.G1, bases, 0, None, ex), want)
    finally:
        worker.set_option("msm_window_bits", 0)
        worker.set_option("msm_big_cap", 0)
    dens = rng.random(n) < 0.5
    k = int(dens.sum())
    b2 = o1.g1_fixed_mul(o1.fr_random(94, 7 + k))
    kind = rng.integers(0, 4, n)
    e = ex.copy()
    e[kind == 0] = 0
    e[kind == 1] = o1.fr_from_ints([1])[0]
    rc, want = o1.multiexp(1, b2, 7, dens.astype(np.uint8), e)
    assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, b2, 7, dens, e), want)


def test_affine_rounds_error_semantics(worker, affine):
    """an identity base under a non-zero digit is still UnexpectedIdentity when the rounds consume it"""
    affine(3)
    n = 500
    bases = o1.g1_fixed_mul(o1.fr_random(95, n))
    ex = o1.fr_random(96, n)
    bad = bases.copy(); bad[77] = 0
    with pytest.raises(bb.UnexpectedIdentity):
        _gpu_multiexp(worker, bb.G1, bad, 0, None, ex)
    ex0 = ex.copy(); ex0[77] = 0                                        # a zero scalar skips its base (multiexp.rs:245)
    rc, want = o1.multiexp(1, bad, 0, None, ex0)
    assert rc == 0 and np.array_equal(_gpu_multiexp(worker, bb.G1, bad, 0, None, ex0), want)


def test_multiexp_error_semantics(worker):
    """SURVEY.md App. C 2-4 (multiexp.rs:53-86,242-265,324-329)."""
    bases = o1.g1_fixed_mul(o1.fr_from_ints([5, 6, 7]))
    bases[0] = 0
    f = o1.fr_from_ints
    got = _gpu_multiexp(worker, bb.G1, bases, 0, None, f([0, 2, 3]))               # zero scalar skips the identity base
    assert np.array_equal(got, o1.g1_fixed_mul(f([6 * 2 + 7 * 3])))
    with pytest.raises(bb.UnexpectedIdentity):
        _gpu_multiexp(worker, bb.G1, bases, 0, None, f([2, 2, 3]))
    with pytest.raises(bb.UnexpectedIdentity):
        _gpu_multiexp(worker, bb.G1, bases, 0, None, f([1, 2, 3]))                 # Exponent::One path
    with pytest.raises(bb.IoError):
        _gpu_multiexp(worker, bb.G1, bases[1:], 0, None, f([4, 2, 3]))
    with pytest.raises(bb.IoError):
        _gpu_multiexp(worker, bb.G1, bases[1:], 0, None, f([4, 2, 0]))             # skip() also checks EOF
    with pytest.raises(bb.DensityMismatch):
        _gpu_multiexp(worker, bb.G1, bases, 0, [True, False], f([4, 2, 3]))
    # both an EOF and an identity: the oracle's precedence (top window's error) must match
    for scal in ([2, 2, 3, 9], [1 << 250, 2, 3, 9], [R - 1, 0, 1, 1]):
        rc, _ = o1.multiexp(1, bases, 0, None, f(scal))
        exc = {2: bb.UnexpectedIdentity, 3: bb.IoError}[rc]
        with pytest.raises(exc):
            _gpu_multiexp(worker, bb.G1, bases, 0, None, f(scal))


# --------------------------------------------------------------------------------------------
# whole prover (groth16/src/prover.rs)
# --------------------------------------------------------------------------------------------
def _assignment(w):
    return bb.ProvingAssignment(w["a"], w["b"], w["c"], w["inputs"], w["aux"], w["a_aux_density"],
                                w["b_input_density"], w["b_aux_density"])


def test_prove_mimc322_matches_oracle(worker):
    """BASELINE.json configs[0] on the GPU: MiMC-322 (groth16/tests/mimc.rs), proof bytes identical
    to the CPU restatement and to the proof computed in the exponent from the toxic waste."""
    rng = random.Random(71)
    mc = o1.Mimc(322, seed=3)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    asg = _assignment(mc.witness())
    for _ in range(3):
        r, s = rng.randrange(R), rng.randrange(R)
        proof = bb.create_proof(asg, params, r, s)
        assert len(proof) == 192                                     # groth16/src/lib.rs:559
        assert proof == mc.prove(r, s)
        assert proof == mc.expected_proof(r, s)
    # create_random_proof (prover.rs:164-179): fresh (r, s) every call, and the proof verifies (below)
    rp1, rp2 = bb.create_random_proof(asg, params), bb.create_random_proof(asg, params)
    assert len(rp1) == 192 and rp1 != rp2
    # a key that went through Parameters::write / Parameters::read (groth16/src/lib.rs:258-398)
    from bellman_b200 import params_io
    reloaded = bb.Parameters(worker, params_io.read_parameters(params_io.write_parameters(mc.export_params()), worker=worker))
    assert bb.create_proof(asg, reloaded, r, s) == proof
    # "the proof verifies under the reference verifier": Proof::read + verify_proof
    # (groth16/src/lib.rs:47-99, verifier.rs:23-58) over the oracle's pairing
    from oracle.oracle0 import pairing as PR
    p = mc.export_params()
    g1, g2 = o1.g1_to_affine_ints(p["vk_g1"]), o1.g2_to_affine_ints(p["vk_g2"])
    vk = dict(alpha_g1=g1[0], beta_g2=g2[0], gamma_g2=g2[1], delta_g2=g2[2], ic=o1.g1_to_affine_ints(p["ic"]))
    image = o1.fr_to_ints(mc.witness()["inputs"])[1]
    assert PR.verify_proof(vk, PR.proof_read(proof), [image])
    assert not PR.verify_proof(vk, PR.proof_read(proof), [image ^ 1])
    assert PR.verify_proof(vk, PR.proof_read(rp1), [image])
    # sharded across "devices": the partial sums of the (base range x window) shards add up to the
    # same proof.  2 and 3 shards split the windows only; 8 = 2 base ranges x 4 window shards;
    # 5 has no divisor <= 4 and splits the bases only; shard_windows=1 forces base ranges alone.
    for count in (2, 3, 5, 8):
        parts = []
        for k in range(count):
            pk = bb.Parameters(worker, mc.export_params(), shard_index=k, shard_count=count)
            parts.append(bb.prove_partials(asg, pk))
            pk.free()
        assert bb.finalize(params, parts, r, s) == proof, count
        assert bb.finalize(params, parts, r, s, static=bb.finalize_static(params, r, s)) == proof
    try:
        worker.set_option("shard_windows", 1)
        parts = []
        for k in range(4):
            pk = bb.Parameters(worker, mc.export_params(), shard_index=k, shard_count=4)
            parts.append(bb.prove_partials(asg, pk))
            pk.free()
        assert bb.finalize(params, parts, r, s) == proof
    finally:
        worker.set_option("shard_windows", 4)


def _manufacture_crs(worker, mc):
    """CRS = [dlog]G for the dlogs the oracle derives from the toxic waste (generator.rs:249-415),
    with the group elements produced by the device's fixed-base kernel (checked against the
    oracle's generator in test_point_arithmetic / below)."""
    ks = mc.crs_scalars()
    ni = mc.num_inputs
    a_nz = np.array([bool(v.any()) for v in ks["a"]])
    b_nz = np.array([bool(v.any()) for v in ks["b"]])
    toxic = mc._toxic
    vk1 = bb.fixed_base_mul(worker, bb.G1, o1.fr_from_ints([toxic[0], toxic[1], toxic[3]]))
    vk2 = bb.fixed_base_mul(worker, bb.G2, o1.fr_from_ints([toxic[1], toxic[2], toxic[3]]))
    return dict(vk_g1=vk1, vk_g2=vk2,
                h=bb.fixed_base_mul(worker, bb.G1, ks["h"]),
                l=bb.fixed_base_mul(worker, bb.G1, ks["ext"][ni:]),
                a=bb.fixed_base_mul(worker, bb.G1, ks["a"][a_nz]),           # identities filtered, generator.rs:491-505
                b_g1=bb.fixed_base_mul(worker, bb.G1, ks["b"][b_nz]),
                b_g2=bb.fixed_base_mul(worker, bb.G2, ks["b"][b_nz]))


@pytest.mark.parametrize("rounds", [8191, 524287])
def test_prove_synthetic_chain_trapdoor(worker, rounds):
    """BASELINE.json configs[1]: the 2^20-constraint MiMC chain (R = 524287; 2^14 as a quicker
    case).  The expected 192 bytes are computed in the exponent from the toxic waste
    (o1_mimc_expected_proof: no MSM, no FFT), the way tests/mod.rs:287-370 checks test_xordemo."""
    o1.set_threads(0)
    rng = random.Random(rounds)
    mc = o1.Mimc(rounds, seed=rounds)
    assert mc.num_constraints == 2 * rounds + 2 == mc.m
    mc._toxic = [rng.randrange(1, R) for _ in range(5)]
    mc.set_toxic(mc._toxic)
    p = _manufacture_crs(worker, mc)
    assert p["h"].shape[0] == mc.m - 1 and p["l"].shape[0] == mc.num_aux
    assert p["a"].shape[0] == mc.a_aux_total + mc.num_inputs and p["b_g1"].shape[0] == mc.b_in_total + mc.b_aux_total
    if rounds < 10000:
        mc.generate()                                   # CPU generator agrees with the manufactured CRS
        q = mc.export_params()
        for k in ("vk_g1", "vk_g2", "h", "l", "a", "b_g1", "b_g2"):
            assert np.array_equal(np.asarray(p[k]).reshape(-1), q[k].reshape(-1)), k
    params = bb.Parameters(worker, p)
    asg = _assignment(mc.witness())
    r, s = rng.randrange(R), rng.randrange(R)
    proof = bb.create_proof(asg, params, r, s)
    assert proof == mc.expected_proof(r, s)
    if rounds < 10000:
        assert proof == mc.prove(r, s)


def test_prove_error_precedence(worker):
    """Which SynthesisError create_proof returns when several apply (groth16/src/prover.rs): the
    delta check (:320-324) precedes every wait; the waits run a_inputs, a_aux, b_g1_inputs,
    b_g1_aux, b_g2_inputs, b_g2_aux, h, l (:339-354), so an identity hit in the A query is
    reported even if the (earlier started) l multiexp ran out of bases."""
    rng = random.Random(72)
    mc = o1.Mimc(20, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    asg = _assignment(mc.witness())
    r, s = rng.randrange(R), rng.randrange(R)
    good = mc.export_params()
    proof = bb.create_proof(asg, bb.Parameters(worker, good), r, s)
    assert proof == mc.prove(r, s)

    def variant(**changes):
        p = {k: np.array(v, copy=True) for k, v in good.items()}
        for k, f in changes.items():
            p[k] = f(p[k])
        return bb.Parameters(worker, p)

    def short(v):                      # drop the last base: Source::next runs out (IoError UnexpectedEof)
        return v.reshape(-1, v.shape[-1])[:-1]

    def ident(row):                    # an identity base that a non-zero scalar hits (UnexpectedIdentity)
        def f(v):
            v = v.reshape(-1, v.shape[-1]).copy()
            v[row] = 0
            return v
        return f

    with pytest.raises(bb.IoError):
        bb.create_proof(asg, variant(l=short), r, s)
    with pytest.raises(bb.UnexpectedIdentity):
        bb.create_proof(asg, variant(a=ident(3)), r, s)
    with pytest.raises(bb.UnexpectedIdentity):                    # a_aux is waited for before l
        bb.create_proof(asg, variant(l=short, a=ident(3)), r, s)
    with pytest.raises(bb.IoError):                               # b_g1_aux (EOF) before h (identity)
        bb.create_proof(asg, variant(b_g1=short, h=ident(2)), r, s)
    with pytest.raises(bb.UnexpectedIdentity):                    # h (identity) before l (EOF)
        bb.create_proof(asg, variant(l=short, h=ident(2)), r, s)

    def zero_delta(v):
        v = v.reshape(3, -1).copy()
        v[2] = 0
        return v
    with pytest.raises(bb.UnexpectedIdentity):                    # delta = identity wins over an EOF
        bb.create_proof(asg, variant(vk_g1=zero_delta, l=short, b_g1=short), r, s)
    with pytest.raises(bb.UnexpectedIdentity):
        bb.create_proof(asg, variant(vk_g2=zero_delta), r, s)
    # sharded flow: the partial-sum call reports the same error
    with pytest.raises(bb.UnexpectedIdentity):
        bb.prove_partials(asg, variant(vk_g1=zero_delta))


# --------------------------------------------------------------------------------------------
# parameter generation on the device (groth16/src/generator.rs; SURVEY section 8f rank 3)
# --------------------------------------------------------------------------------------------
class _AssemblyAdapter:
    """lets an oracle-0 circuit closure synthesise into the product's KeypairAssembly"""

    def __init__(self, asm):
        self.asm = asm

    def alloc(self, f):
        from oracle.oracle0 import bellman as B
        return B.Var(False, self.asm.alloc()[1])

    def alloc_input(self, f):
        from oracle.oracle0 import bellman as B
        return B.Var(True, self.asm.alloc_input()[1])

    def enforce(self, a, b, c):
        conv = lambda lc: [(("input" if v.is_input else "aux", v.idx), k) for v, k in lc.terms]
        self.asm.enforce(conv(a), conv(b), conv(c))


def test_generate_parameters_matches_oracle(worker):
    from bellman_b200 import generator as GEN
    from oracle.oracle0 import bellman as B, fields as F
    rng = random.Random(90)
    fr = B.Bls12.fr
    constants = [rng.randrange(R) for _ in range(5)]
    xl, xr = rng.randrange(R), rng.randrange(R)
    circuit = B.mimc_circuit(fr, xl, xr, constants)
    alpha, beta, gamma, delta, tau = (rng.randrange(1, R) for _ in range(5))
    k1, k2 = rng.randrange(1, R), rng.randrange(1, R)
    g1, g2 = F.G1.mul(F.G1_GEN, k1), F.G2.mul(F.G2_GEN, k2)
    want = B.generate_parameters(B.Bls12, circuit, g1, g2, alpha, beta, gamma, delta, tau)

    asm = GEN.KeypairAssembly()
    asm.alloc_input()                                          # ONE, generator.rs:188
    circuit(_AssemblyAdapter(asm))
    got = GEN.generate_parameters(worker, asm, alpha, beta, gamma, delta, tau, g1_scalar=k1, g2_scalar=k2)
    assert (got["num_inputs"], got["num_aux"], got["m"]) == (want.num_inputs, want.num_aux, want.m)

    def g1_ints(arr):
        return o1.g1_to_affine_ints(np.ascontiguousarray(arr).reshape(-1, 12))

    def g2_ints(arr):
        return o1.g2_to_affine_ints(np.ascontiguousarray(arr).reshape(-1, 24))

    assert g1_ints(got["vk_g1"]) == [want.alpha_g1, want.beta_g1, want.delta_g1]
    assert g2_ints(got["vk_g2"]) == [want.beta_g2, want.gamma_g2, want.delta_g2]
    for name, conv in (("ic", g1_ints), ("h", g1_ints), ("l", g1_ints), ("a", g1_ints), ("b_g1", g1_ints), ("b_g2", g2_ints)):
        assert conv(got[name]) == list(getattr(want, name)), name
    # the generated key proves: same bytes as the oracle's prover on the oracle's key
    from bellman_b200 import params_io
    blob = params_io.write_parameters(got)
    params = bb.Parameters(worker, params_io.read_parameters(blob, worker=worker))
    wit = B.synthesize_witness(B.Bls12, circuit)
    r, s = rng.randrange(R), rng.randrange(R)
    proof = B.proof_bytes(B.create_proof(B.Bls12, circuit, want, r, s))
    asg = bb.ProvingAssignment(o1.fr_from_ints(wit.a), o1.fr_from_ints(wit.b), o1.fr_from_ints(wit.c),
                               o1.fr_from_ints(wit.input_assignment), o1.fr_from_ints(wit.aux_assignment),
                               wit.a_aux_density, wit.b_input_density, wit.b_aux_density)
    assert bb.create_proof(asg, params, r, s) == proof
    # an unconstrained auxiliary variable and a non-invertible delta are errors (generator.rs:228-243,466-470)
    asm2 = GEN.KeypairAssembly()
    asm2.alloc_input()
    circuit(_AssemblyAdapter(asm2))
    asm2.alloc()
    with pytest.raises(GEN.UnconstrainedVariable):
        GEN.generate_parameters(worker, asm2, alpha, beta, gamma, delta, tau)
    asm3 = GEN.KeypairAssembly()
    asm3.alloc_input()
    circuit(_AssemblyAdapter(asm3))
    with pytest.raises(bb.UnexpectedIdentity):
        GEN.generate_parameters(worker, asm3, alpha, beta, gamma, 0, tau)

# resident window multiples (bb_bases_precompute / msm_precompute): same points, one bucket set
# --------------------------------------------------------------------------------------------
@pytest.fixture()
def precompute(worker):
    worker.set_option("msm_precompute", 1)
    yield worker
    worker.set_option("msm_precompute", 0)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 33, 1000, 1 << 14])
def test_precompute_multiexp_g1(precompute, n):
    test_multiexp_g1_matches_oracle(precompute, n)


@pytest.mark.parametrize("n", [3, 40, 2000])
def test_precompute_multiexp_g2(precompute, n):
    test_multiexp_g2_matches_oracle(precompute, n)


def test_precompute_variants(precompute):
    test_multiexp_window_choice_does_not_change_results(precompute)
    test_multiexp_density_offset_and_fast_paths(precompute)
    test_multiexp_skewed_scalars(precompute)
    test_multiexp_error_semantics(precompute)
    test_multiexp_naive_property_full_size(precompute)


def test_precompute_prove(precompute):
    test_prove_mimc322_matches_oracle(precompute)
    test_prove_synthetic_chain_trapdoor(precompute, 8191)
    test_prove_error_precedence(precompute)


# msm_precompute = 2: ONE bucket set for all windows over the same tables, halving rounds by its fill
# --------------------------------------------------------------------------------------------
@pytest.fixture()
def unified(worker):
    worker.set_option("msm_precompute", 2)
    yield worker
    worker.set_option("msm_precompute", 0)
    worker.set_option("msm_unified_rows_log", 3)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 33, 1000, 1 << 14, 1 << 16])
def test_unified_multiexp_g1(unified, n):
    test_multiexp_g1_matches_oracle(unified, n)          # 2^14: fill 18 -> 1 round, 2^16: fill 72 -> 3 rounds


@pytest.mark.parametrize("n", [3, 40, 2000])
def test_unified_multiexp_g2(unified, n):
    test_multiexp_g2_matches_oracle(unified, n)


def test_unified_variants(unified):
    test_multiexp_window_choice_does_not_change_results(unified)
    test_multiexp_density_offset_and_fast_paths(unified)
    test_multiexp_skewed_scalars(unified)
    test_multiexp_error_semantics(unified)
    test_multiexp_naive_property_full_size(unified)      # 2^18, c = 15: fill 288 -> 5 rounds
    test_multiexp_g2_2e16_matches_oracle(unified)        # G2, fill 72 -> 3 rounds


def unified_deep_rounds_case(worker, n=1 << 13):
    """a small window (c = 8: 128 buckets, 32 windows) makes the shared buckets deep: fill 2048 -> the maximum of
    8 halving rounds with the default stop, and every stop from 2^0 to 2^12 rows gives the same point"""
    bases_arr = o1.g1_fixed_mul(o1.fr_random(5100, n))
    ex = o1.fr_random(5101, n)
    ex[3] = 0; ex[5] = o1.fr_from_ints([1])[0]; ex[6] = o1.fr_from_ints([R - 1])[0]
    rc, want = o1.multiexp(1, bases_arr, 0, None, ex)
    assert rc == 0
    try:
        worker.set_option("msm_window_bits", 8)
        bases = bb.Bases(worker, bb.G1, bases_arr)
        for rows_log in (3, 0, 5, 12):
            worker.set_option("msm_unified_rows_log", rows_log)
            assert np.array_equal(bb.multiexp(worker, (bases, 0), bb.FullDensity, ex).wait(), want), rows_log
        bases.free()
    finally:
        worker.set_option("msm_window_bits", 0)
        worker.set_option("msm_unified_rows_log", 3)


def test_unified_deep_rounds(unified):
    unified_deep_rounds_case(unified)


def test_unified_synthetic_bases_naive_property(unified):
    test_multiexp_synthetic_bases_naive_property(unified, 22, 0)     # 2^22, c = 16: fill 2048 -> 8 rounds


def test_unified_prove(unified):
    test_prove_mimc322_matches_oracle(unified)
    test_prove_synthetic_chain_trapdoor(unified, 8191)
    test_prove_error_precedence(unified)
    test_prove_begin_end_with_coset_evaluations(unified)


def test_unified_prove_2e20(unified):
    test_prove_synthetic_chain_trapdoor(unified, 524287)


def autotune_case(worker, rounds, reps=2):
    """bb_groth16_autotune: every MSM form proves the same witness, only forms with the default form's partial sums
    are eligible, the key is left configured for the chosen one and proves to the expected bytes"""
    rng = random.Random(rounds + 1)
    mc = o1.Mimc(rounds, seed=rounds + 2)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    asg = _assignment(mc.witness())
    try:
        rep = params.autotune(asg, reps=reps)
        names = bb.tuning_names()
        assert len(rep["ms"]) == len(names) >= 2 and 0 <= rep["chosen"] < len(names) and rep["name"] == names[rep["chosen"]]
        assert rep["ms"][0] > 0 and rep["ms"][rep["chosen"]] > 0
        assert all(t > 0 for t in rep["ms"]), rep                # every form available, working and byte-identical here
        assert rep["ms"][rep["chosen"]] == min(rep["ms"])
        r, s = rng.randrange(R), rng.randrange(R)
        assert bb.create_proof(asg, params, r, s) == mc.expected_proof(r, s)
        for index in range(len(names)):                           # and by hand: every form, same proof
            params.apply_tuning(index)
            assert bb.create_proof(asg, params, r, s) == mc.expected_proof(r, s), names[index]
    finally:
        params.apply_tuning(0)
        params.free()


def test_autotune(worker):
    autotune_case(worker, 8191)


def test_prove_begin_end_with_coset_evaluations(worker):
    """The two-step prove of the multi-GPU flow on one device: bb_groth16_prove_begin queues the witness MSMs,
    bb_h_coset_evals takes a, b, c through ifft + coset_fft one by one (as three ranks would), and
    bb_groth16_prove_end finishes with the last transform and the h MSM.  Same 960 partial-sum bytes and the same
    proof as the one-call path; also with the H pipeline left to prove_end (no evaluations passed)."""
    rng = random.Random(44)
    mc = o1.Mimc(100, seed=45)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    asg = _assignment(mc.witness())
    r, s = rng.randrange(R), rng.randrange(R)
    want = bb.prove_partials(asg, params)
    n = asg.a.shape[0]
    m = 1
    while m < n:
        m *= 2
    bufs = [worker.device_alloc(m * 32) for _ in range(3)]
    try:
        state = bb.prove_begin(asg, params)
        for poly, d in zip((asg.a, asg.b, asg.c), bufs):
            bb.h_coset_evals(worker, poly, n, d)
        got = bb.prove_end(state, bufs)
        assert got == want
        assert bb.finalize(params, [got], r, s) == mc.prove(r, s) == mc.expected_proof(r, s)
        state = bb.prove_begin(asg, params)
        assert bb.prove_end(state, None) == want
    finally:
        for d in bufs:
            worker.device_free(d)
