"""Every point-validity decision (csrc/encoding.cuh) on points built to reach its edges: torsion points of each prime of
the cofactors, eigenvectors of the endomorphisms the subgroup tests use, points whose square root takes each branch, x = 0,
and coordinates next to p at every limb.  Each family is fed to every path that reads or checks points:

  1  bb_diag_points_decompress, subgroup check on and off       (decode.cu, k_decode_g1 / k_decode_g2)
  2  bb_proofs_read with the point as A, B or C; BatchVerifier.queue_bytes
  3  bb_params_read checked and unchecked, bb_vk_read, and params_io.read_parameters on the same files
  4  bb_points_validate ([r]P on the device), both values of check_subgroup
  5  bb_groth16_generate with such a point as the caller's generator (the host rP_is_identity)
  6  the host helpers bb_point_add, bb_point_mul, bb_point_compress
  7  write-back: points read unchecked come back byte for byte through bb_proofs_write and bb_params_write

Expected values come from Python integers twice over: the oracle's restatements of from_compressed / from_uncompressed
(test_gpu_proof_read.classify_point, test_gpu_params_read.classify / restate) and the exact order of each point, computed
here with a ladder that does not reduce its scalar mod r.  The two must agree before any device output is compared.

tests/test_emulated_point_validity.py runs the same bodies on the emulated library.
"""
import ctypes as C
import functools
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import generator as GEN
from bellman_b200 import params_io as PIO
from bellman_b200 import r1cs as RC
from bellman_b200 import verifier as V
from oracle import o1
from oracle.oracle0 import bellman as B
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

import test_gpu_params_read as GP
import test_gpu_proof_read as GR
import test_gpu_verify as GV
from test_gpu_parity import _AssemblyAdapter

pytestmark = pytest.mark.gpu

P, R, X = F.FP_MODULUS, F.FR_MODULUS, F.BLS_X
F2 = F.Fp2Ops
OK, FLAGS, NONCANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, IDENTITY = range(6)

# #E(Fp) = h1 r and #E'(Fp2) = h2 r
H1 = (X - 1) ** 2 // 3
H2 = (X ** 8 - 4 * X ** 7 + 5 * X ** 6 - 4 * X ** 4 + 6 * X ** 3 - 4 * X ** 2 - 4 * X + 13) // 9
Q1 = (11, 10177, 859267, 52437899)                               # h1 = 3 * q^2 over these
Q2 = (13, 23, 2713, 11953, 262069)                               # h2 = 13^2 23^2 2713 11953 262069 q135
Q2_BIG = H2 // (13 ** 2 * 23 ** 2 * 2713 * 11953 * 262069)
T_FROB = X + 1                                                   # trace of Frobenius of E / Fp


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# exact arithmetic: no reduction of scalars mod r
# --------------------------------------------------------------------------------------------
def mul(G, pt, k):
    """[k] pt for an integer k >= 0, by double-and-add over the integer itself"""
    acc, add = None, pt
    while k:
        if k & 1:
            acc = G.add(acc, add)
        add = G.add(add, add)
        k >>= 1
    return acc


def has_order(G, pt, n, primes):
    """pt has order exactly n, the primes being those of n"""
    return pt is not None and mul(G, pt, n) is None and all(mul(G, pt, n // q) is not None for q in primes)


def _fp2_pow(a, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = F2.mul(r, a)
        a = F2.mul(a, a)
        e >>= 1
    return r


def _beta():
    """the cube root of unity of the G1 check: [x^2] P = (beta x, -y) on G1"""
    g = F.G1_GEN
    want = F.G1.mul(g, X * X)
    for b in (pow(2, (P - 1) // 3, P), pow(pow(2, (P - 1) // 3, P), 2, P)):
        if b != 1 and want == (b * g[0] % P, (P - g[1]) % P):
            return b
    raise AssertionError("no cube root of unity gives [x^2] G = -phi(G)")


BETA = _beta()
PSI_X = F2.inv(_fp2_pow((1, 1), (P - 1) // 3))
PSI_Y = F2.inv(_fp2_pow((1, 1), (P - 1) // 2))


def phi(pt):
    return None if pt is None else (BETA * pt[0] % P, pt[1])


def psi(pt):
    """untwist-Frobenius-twist: psi(P) = [x] P on G2"""
    if pt is None:
        return None
    conj = lambda a: (a[0], (P - a[1]) % P)
    return F2.mul(conj(pt[0]), PSI_X), F2.mul(conj(pt[1]), PSI_Y)


assert psi(F.G2_GEN) == F.G2.mul(F.G2_GEN, X % R)


def random_curve_point(group, rng):
    """a uniform point of E(Fp) or E'(Fp2), cofactor part included"""
    while True:
        if group == 1:
            x = rng.randrange(P)
            y = PR._fp_sqrt((x * x * x + 4) % P)
            if y is not None:
                return x, y if rng.random() < 0.5 else (P - y) % P
        else:
            x = (rng.randrange(P), rng.randrange(P))
            y = PR._fp2_sqrt(F2.add(F2.mul(F2.mul(x, x), x), F.G2_B))
            if y is not None:
                return x, y if rng.random() < 0.5 else F2.neg(y)


def cube_root_of_unity_mod(q):
    """a root of t^2 + t + 1 mod q (q = 1 mod 3)"""
    for g in range(2, q):
        w = pow(g, (q - 1) // 3, q)
        if w != 1:
            assert (w * w + w + 1) % q == 0
            return w


def quadratic_roots_mod(a1, a0, q):
    """the roots of t^2 + a1 t + a0 mod a small prime q"""
    return [t for t in range(q) if (t * t + a1 * t + a0) % q == 0]


def point_of_order(G, q, cofactor, rng):
    """a point of order q (q a prime with q^k | cofactor): [r cofactor / q^k] of a random point, then [q] until its
    order is q"""
    k = 0
    while cofactor % q ** (k + 1) == 0:
        k += 1
    group = 1 if G is F.G1 else 2
    while True:
        t = mul(G, random_curve_point(group, rng), R * cofactor // q ** k)
        while t is not None and mul(G, t, q) is not None:
            t = mul(G, t, q)
        if t is not None:
            assert has_order(G, t, q, (q,))
            return t


# --------------------------------------------------------------------------------------------
# the families: (name, point, order); order None = on the curve but of order divisible by r and a cofactor prime
# --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def g1_family():
    rng = random.Random(901)
    G = F.G1
    assert H1 == 3 * (11 * 10177 * 859267 * 52437899) ** 2 and abs(X - 1) == 3 * 11 * 10177 * 859267 * 52437899
    out = [("T3", (0, 2), 3), ("-T3", (0, P - 2), 3)]            # the only points of order 3: x = 0
    for pt in (out[0][1], out[1][1]):
        assert G.is_on_curve(pt) and has_order(G, pt, 3, (3,)) and phi(pt) == pt
    for q in Q1:
        t = point_of_order(G, q, H1, rng)
        # phi^2 + phi + 1 = 0 on E: confirmed on t, so an eigenvalue of phi mod q is a root of t^2 + t + 1
        assert G.add(G.add(phi(phi(t)), phi(t)), t) is None
        if q % 3 == 1:
            lam = cube_root_of_unity_mod(q)
            lam2 = (-1 - lam) % q
            assert phi(t) not in (mul(G, t, lam), mul(G, t, lam2))     # t is no eigenvector: t, phi(t) independent
            for a, b in ((lam, lam2), (lam2, lam)):
                e = G.add(phi(t), G.neg(mul(G, t, b)))                 # (phi - b) t is in the kernel of phi - a
                assert has_order(G, e, q, (q,)) and phi(e) == mul(G, e, a)
                out.append((f"T{q}_eigen{a}", e, q))
        # else: t^2 + t + 1 has no root mod q, so phi(t) is not in <t>
        # two independent points of order q and q^2 exactly dividing h1: the q-part of E(Fp) is Z/q x Z/q
        assert H1 % q ** 2 == 0 and H1 % q ** 3 != 0
        out += [(f"T{q}", t, q), (f"phi(T{q})", phi(t), q)]
    primes = (3,) + Q1
    while True:                                                  # the largest order the cofactor part holds: |x - 1|
        t = mul(G, random_curve_point(1, rng), R)
        if has_order(G, t, abs(X - 1), primes):
            out.append(("T_max", t, abs(X - 1)))
            break
    return tuple(out)


@functools.lru_cache(maxsize=None)
def g2_family():
    rng = random.Random(902)
    G = F.G2
    assert H2 == 13 ** 2 * 23 ** 2 * 2713 * 11953 * 262069 * Q2_BIG and len(str(Q2_BIG)) == 135
    assert pow(3, Q2_BIG - 1, Q2_BIG) == 1
    # psi^2 - t psi + p = 0 on E'(Fp2), t = x + 1: confirmed on points with their cofactor part
    for _ in range(2):
        pt = random_curve_point(2, rng)
        assert G.add(G.add(psi(psi(pt)), mul(G, psi(pt), -T_FROB)), mul(G, pt, P)) is None
    out = []
    for q in Q2 + (Q2_BIG,):
        t = point_of_order(G, q, H2, rng)
        out.append((f"T{q if q < 10 ** 9 else 'q135'}", t, q))
        if q > 10 ** 9:
            continue
        roots = quadratic_roots_mod(-T_FROB % q, P % q, q)
        if H2 % q ** 2 == 0 and len(roots) == 2 and psi(t) not in [mul(G, t, m) for m in roots]:
            for a, b in (roots, roots[::-1]):
                e = G.add(psi(t), G.neg(mul(G, t, b)))
                assert has_order(G, e, q, (q,)) and psi(e) == mul(G, e, a)
                out.append((f"T{q}_eigen{a}", e, q))
        elif H2 % q ** 2 != 0:                                   # a cyclic q-part: t is an eigenvector
            assert psi(t) in [mul(G, t, m) for m in roots]
    # square-root branches and zero coordinates (not of small order; each outside G2)
    for k in range(2):                                           # y purely imaginary: alpha = -1 in the Fp2 square root
        while True:
            y1 = rng.randrange(1, P)
            x = GR._fp2_cbrt(((-y1 * y1 - 4) % P, P - 4))
            if x is not None:
                pt = (x, (0, y1))
                assert G.is_on_curve(pt)
                out += [(f"y_imaginary{k}", pt, None), (f"-y_imaginary{k}", G.neg(pt), None)]
                break
    for k, pt in enumerate(GR.g2_points_with_real_y(rng, 1)):
        out += [(f"y_real{k}", pt, None), (f"-y_real{k}", G.neg(pt), None)]
    for name, mk in (("x.c1=0", lambda v: (v, 0)), ("x.c0=0", lambda v: (0, v))):
        while True:
            x = mk(rng.randrange(1, P))
            y = PR._fp2_sqrt(F2.add(F2.mul(F2.mul(x, x), x), F.G2_B))
            if y is not None:
                out.append((name, (x, y), None))
                break
    return tuple(out)


@functools.lru_cache(maxsize=None)
def family(group):
    """the torsion / special points, and each torsion point T also as P + T (P random in the subgroup) and G + T"""
    G = F.G1 if group == 1 else F.G2
    base = g1_family() if group == 1 else g2_family()
    rng = random.Random(903 + group)
    out = list(base)
    for name, t, order in base:
        if order is not None:
            p = G.mul(G.gen, rng.randrange(1, R))
            out += [(f"P+{name}", G.add(p, t), None), (f"G+{name}", G.add(G.gen, t), None)]
    for name, pt, order in out:
        assert G.is_on_curve(pt)
        assert mul(G, pt, R) is not None, name                   # outside the subgroup, by the exact order
        assert G.mul(pt, R - 1) != G.neg(pt), name               # and by the oracle's test
    return tuple(out)


def abi(group, pts):
    return (o1.g1_from_affine_ints if group == 1 else o1.g2_from_affine_ints)(list(pts))


def compress(group, pt):
    return F.g1_compress(pt) if group == 1 else F.g2_compress(pt)


def uncompressed(group, pt):
    return F.g1_uncompressed(pt) if group == 1 else F.g2_uncompressed(pt)


def decompress_unchecked(group, b):
    """from_compressed_unchecked over Python integers: (why, point)"""
    why, pt = GR.classify_point(group, b)
    if why != NOT_IN_SUBGROUP:
        return why, pt
    x = int.from_bytes(bytes([b[0] & 0x1F]) + b[1:48], "big")
    if group == 1:
        y = PR._fp_sqrt((x * x * x + 4) % P)
        if (y > (P - 1) // 2) != bool(b[0] & 0x20):
            y = P - y
        return OK, (x, y)
    x = (int.from_bytes(b[48:], "big"), x)
    y = PR._fp2_sqrt(F2.add(F2.mul(F2.mul(x, x), x), F.G2_B))
    if F._fp2_lexi_larger(y) != bool(b[0] & 0x20):
        y = F2.neg(y)
    return OK, (x, y)


def near_p():
    """p + 2^(32k) - 1 and p + 2^(32k) (not canonical) and p - 2^(32k) (canonical), k = 1..11"""
    return [(P + (1 << 32 * k) - 1, False) for k in range(1, 12)] + [(P + (1 << 32 * k), False) for k in range(1, 12)] + \
           [(P - (1 << 32 * k), True) for k in range(1, 12)]


def compressed_edges(group):
    """compressed encodings at the decoder's edges: the all-zero x under each flag combination, and each coordinate of a
    torsion point's x next to p"""
    size = 48 if group == 1 else 96
    out = [(f"zero x, flags {f:#04x}", bytes([f]) + bytes(size - 1)) for f in range(0, 256, 32)]
    ref = compress(group, family(group)[2][1])
    for v, _ in near_p():
        for j in range(size // 48):                              # G2: x.c1, then x.c0
            b = bytearray(ref)
            b[48 * j:48 * (j + 1)] = v.to_bytes(48, "big")
            if j == 0:
                b[0] |= ref[0] & 0xE0
            out.append((f"coordinate {j} = {v - P:+#x} + p", bytes(b)))
    return out


# --------------------------------------------------------------------------------------------
# 1 and 4: bb_diag_points_decompress, bb_points_validate
# --------------------------------------------------------------------------------------------
def validate(worker, group, pts, check_subgroup):
    first_bad, why = C.c_size_t(), C.c_int()
    arr = np.ascontiguousarray(pts, np.uint64)
    assert bb.load_library().bb_points_validate(worker._h, C.c_int(group), arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.shape[0]),
                                                C.c_int(check_subgroup), C.byref(first_bad), C.byref(why)) == 0
    return first_bad.value, why.value


@pytest.mark.parametrize("group", [1, 2])
def test_decompress_and_validate(worker, group):
    """every family point, and its negation (the other sort bit): rejected by the checked decoder, decoded exactly by the
    unchecked one, and rejected by [r]P; at each subgroup point beside them all three accept"""
    G = F.G1 if group == 1 else F.G2
    pts = [pt for _, pt, _ in family(group)]
    pts += [G.neg(pt) for pt in pts]
    good = [G.gen, G.mul(G.gen, 12345)]
    encs = [compress(group, pt) for pt in pts + good]
    assert {e[0] & 0x20 for e in encs} == {0, 0x20}
    want = [NOT_IN_SUBGROUP] * len(pts) + [OK] * len(good)
    assert [GR.classify_point(group, e)[0] for e in encs] == want
    data = b"".join(encs)
    out, why = V.points_decompress(worker, group, data)
    assert list(why) == want
    assert not out[:len(pts)].any() and np.array_equal(out[len(pts):], abi(group, good))
    out_u, why_u = V.points_decompress(worker, group, data, check_subgroup=False)
    assert not why_u.any() and np.array_equal(out_u, abi(group, pts + good))
    for i in range(len(encs)):                                   # path 4 agrees point by point with path 1
        assert validate(worker, group, out_u[i:i + 1], 1)[1] == (2 if why[i] == NOT_IN_SUBGROUP else 0), i
        assert validate(worker, group, out_u[i:i + 1], 0)[1] == 0, i
    first, w = validate(worker, group, out_u[len(pts) - 1:], 1)
    assert (first, w) == (0, 2)
    first, w = validate(worker, group, np.concatenate([out_u[len(pts):], out_u[:3]]), 1)
    assert (first, w) == (len(good), 2)


@pytest.mark.parametrize("group", [1, 2])
def test_decompress_edges(worker, group):
    """the all-zero x under every flag byte and coordinates next to p, with and without the subgroup check; G1's x = 0
    decodes to (0, +-2), G2's to nothing (4(u + 1) is not a square)"""
    edges = compressed_edges(group)
    encs = [e for _, e in edges]
    data = b"".join(encs)
    for check in (True, False):
        want = [(GR.classify_point(group, e) if check else decompress_unchecked(group, e)) for e in encs]
        out, why = V.points_decompress(worker, group, data, check_subgroup=check)
        assert list(why) == [w for w, _ in want], [(n, int(g), w) for (n, _), g, (w, _) in zip(edges, why, want) if g != w]
        for i, (w, pt) in enumerate(want):
            assert np.array_equal(out[i], abi(group, [pt])[0] if w == OK else np.zeros(out.shape[1], np.uint64)), edges[i][0]
    zero = {f: GR.classify_point(group, bytes([f]) + bytes(47 if group == 1 else 95))[0] for f in range(0, 256, 32)}
    if group == 1:
        assert zero == {0x00: FLAGS, 0x20: FLAGS, 0x40: FLAGS, 0x60: FLAGS, 0x80: NOT_IN_SUBGROUP, 0xa0: NOT_IN_SUBGROUP,
                        0xc0: IDENTITY, 0xe0: FLAGS}
        assert decompress_unchecked(1, bytes([0x80]) + bytes(47)) == (OK, (0, 2))
        assert decompress_unchecked(1, bytes([0xa0]) + bytes(47)) == (OK, (0, P - 2))
    else:
        assert PR._fp2_sqrt(F.G2_B) is None
        assert zero[0x80] == zero[0xa0] == NOT_ON_CURVE and zero[0xc0] == IDENTITY
    whys = [GR.classify_point(group, e)[0] for _, e in edges[8:]]
    canonical = [c for v, c in near_p() for _ in range(1 if group == 1 else 2)]
    assert [w == NONCANONICAL for w in whys] == [not c for c in canonical]


# --------------------------------------------------------------------------------------------
# 2: Proof::read and the batch verifier's queue
# --------------------------------------------------------------------------------------------
def test_proofs_read(worker, seed=904):
    """each family point and edge encoding as A, as B and as C of a proof whose other points are valid; valid proofs
    between them decode exactly"""
    rng = random.Random(seed)
    a, b, c = GR.random_g1(rng), GR.random_g2(rng), GR.random_g1(rng)
    ga, gb, gc = F.g1_compress(a), F.g2_compress(b), F.g1_compress(c)
    bad1 = [compress(1, pt) for _, pt, _ in family(1)] + [e for _, e in compressed_edges(1)]
    bad2 = [compress(2, pt) for _, pt, _ in family(2)] + [e for _, e in compressed_edges(2)]
    proofs = [ga + gb + gc]
    for e in bad1:
        proofs += [e + gb + gc, ga + gb + e]
    for e in bad2:
        proofs += [ga + e + gc]
    proofs.append(ga + gb + gc)
    want = [GR.classify(p) for p in proofs]
    assert want[0] == want[-1] == 0 and all(want[1:-1])
    da, db, dc, status = V.read_proofs(worker, b"".join(proofs))
    assert list(status) == want
    for i in (0, len(proofs) - 1):
        assert np.array_equal(da[i], abi(1, [a])[0]) and np.array_equal(db[i], abi(2, [b])[0]) and np.array_equal(dc[i], abi(1, [c])[0])
    assert not da[1:-1].any() and not db[1:-1].any() and not dc[1:-1].any()


def test_queue_bytes_reports_the_index(worker, seed=21):
    """a torsion point as A, B or C of the k-th queued proof: InvalidProofEncoding with index k, before any pairing"""
    vk, vk_int, items = GV.mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    encoded = [(GR.proof_bytes(*proof), x) for proof, x in items]
    t1 = dict((n, pt) for n, pt, _ in family(1))
    t2 = dict((n, pt) for n, pt, _ in family(2))
    cases = [(0, 0, compress(1, t1["T3"]), 0x14), (2, 48, compress(2, t2["y_imaginary0"]), 0x24),
             (len(encoded) - 1, 144, compress(1, t1["P+T11"]), 0x34), (1, 48, compress(2, t2["T13"]), 0x24)]
    for k, off, enc, st in cases:
        bv = bb.BatchVerifier()
        for i, (pb, x) in enumerate(encoded):
            bv.queue_bytes(pb[:off] + enc + pb[off + len(enc):] if i == k else pb, x)
        launches = worker.kernel_launches
        with pytest.raises(bb.InvalidProofEncoding) as ei:
            bv.verify(random.Random(k), pvk)
        assert ei.value.index == k and ei.value.status == st
        assert worker.kernel_launches - launches == 3            # the decoding kernels only
    pvk.free()


# --------------------------------------------------------------------------------------------
# 3 and 7: Parameters::read / VerifyingKey::read, the host reader, write-back
# --------------------------------------------------------------------------------------------
G1_SECTIONS = [s for s, n in enumerate(PIO.SECTIONS) if n not in GP.G2_SECTIONS]
G2_SECTIONS = [s for s, n in enumerate(PIO.SECTIONS) if n in GP.G2_SECTIONS]


def host_accepts(data, checked, worker):
    try:
        PIO.read_parameters(data, checked=checked, worker=worker)
        return True
    except PIO.InvalidData:
        return False


def uncompressed_edges(group, ref):
    """uncompressed encodings at the reader's edges: zero coordinates under each flag byte, (0, +-2), and each coordinate
    of a valid point next to p"""
    size = 96 if group == 1 else 192
    out = [(f"zeros, flags {f:#04x}", bytes([f]) + bytes(size - 1)) for f in range(0, 256, 32)]
    if group == 1:
        out += [("(0, 2)", F.g1_uncompressed((0, 2))), ("(0, -2)", F.g1_uncompressed((0, P - 2)))]
    for v, _ in near_p():
        for j in range(size // 48):
            b = bytearray(ref)
            b[48 * j:48 * (j + 1)] = v.to_bytes(48, "big")
            out.append((f"coordinate {j} = {v - P:+#x} + p", bytes(b)))
    return out


def check_key_file(worker, bad, name, section, index, back=None):
    """the device reader against restate, both modes, host and device bytes; bb_vk_read on the verifying key; the host
    reader accepts the same files; a file read unchecked writes back byte for byte (as `back` where it differs)"""
    for checked in (True, False):
        want = GP.restate(bad, checked)
        for on_device in (False, True):
            got, _ = GP.raw_read(worker, bad, checked, on_device=on_device)
            assert got == want, (name, checked, on_device, got, want)
        if want[0] == "invalid":
            assert want[1:3] == (section, index) or (not checked and section > 6), (name, want)
        assert host_accepts(bad, checked, worker) == (want[0] == "ok"), (name, checked)
        if want[0] == "ok" and not checked:
            params, pvk = PIO.read_parameters_device(worker, bad, checked=False, verifying_key=True)
            assert PIO.write_parameters_device(params, pvk) == (bad if back is None else back), name
            params.free()
            pvk.free()
    if section <= 6:
        got, _ = GP.raw_read(worker, bad, vk_only=True)
        assert got == GP.restate(bad, True, sections=7), name


def test_params_read_families(worker):
    """each family point (uncompressed) in a section of its group, every section of both groups visited, both modes"""
    data = PIO.write_parameters(GP.small_key((2, 3, 2, 3, 2, 2), seed=905))
    pts, _ = GP.offsets(data)
    for group, sections in ((1, G1_SECTIONS), (2, G2_SECTIONS)):
        size = 96 if group == 1 else 192
        for i, (name, pt, _) in enumerate(family(group)):
            s = sections[i % len(sections)]
            idx = 1 if s >= 6 else 0
            o = pts[(s, idx)]
            bad = data[:o] + uncompressed(group, pt) + data[o + size:]
            assert GP.restate(bad, True) == ("invalid", s, idx, NOT_IN_SUBGROUP)
            assert GP.restate(bad, False) == (("invalid", s, idx, NOT_IN_SUBGROUP) if s <= 6 else ("ok", len(data)))
            check_key_file(worker, bad, name, s, idx)


def test_params_read_edges(worker):
    """zero coordinates under each flag byte, (0, +-2) and coordinates next to p, in every section"""
    data = PIO.write_parameters(GP.small_key((2, 3, 2, 3, 2, 2), seed=906))
    pts, _ = GP.offsets(data)
    for group, sections in ((1, G1_SECTIONS), (2, G2_SECTIONS)):
        size = 96 if group == 1 else 192
        for s in sections:
            idx = 1 if s >= 6 else 0
            o = pts[(s, idx)]
            edges = uncompressed_edges(group, data[o:o + size])
            for k, (name, enc) in enumerate(edges):
                if k >= 10 and k % len(sections) != sections.index(s) % len(sections):
                    continue                                     # the near-p cases rotate over the sections
                back = None
                if enc == bytes(size):                           # (0, 0) is held as the identity: pinned below
                    back = data[:o] + bytes([0x40]) + bytes(size - 1) + data[o + size:]
                check_key_file(worker, data[:o] + enc + data[o + size:], f"{PIO.SECTIONS[s]}: {name}", s, idx, back)


def test_params_read_zero_point_without_flag(worker):
    """pinned: uncompressed zeros without the infinity flag.  from_uncompressed_unchecked gives (0, 0) with infinity =
    false, which the reference holds as a point off the curve; the device reads it as its all-zero identity, and a
    key read unchecked writes it back as the identity encoding 0x40 || 0.  Checked, and in the verifying key, it is
    not on the curve, as in the reference."""
    data = PIO.write_parameters(GP.small_key((2, 3, 2, 3, 2, 2), seed=907))
    pts, _ = GP.offsets(data)
    o = pts[(7, 1)]                                              # h[1]
    bad = data[:o] + bytes(96) + data[o + 96:]
    assert GP.restate(bad, False) == ("ok", len(data)) and GP.raw_read(worker, bad, False)[0] == ("ok", len(data))
    assert GP.restate(bad, True) == GP.raw_read(worker, bad, True)[0] == ("invalid", 7, 1, NOT_ON_CURVE)
    params, pvk = PIO.read_parameters_device(worker, bad, checked=False, verifying_key=True)
    assert not PIO.download_parameters(params)["h"][1].any()
    back = PIO.write_parameters_device(params, pvk)
    assert back == data[:o] + bytes([0x40]) + bytes(95) + data[o + 96:]
    params.free()
    pvk.free()
    assert not PIO.read_parameters(bad, checked=False, worker=worker)["h"][1].any()
    with pytest.raises(PIO.InvalidData, match="not on the curve"):
        PIO.read_parameters(bad, checked=True, worker=worker)
    for s in (0, 2, 6):                                          # alpha_g1, beta_g2, ic[1]
        size = 192 if s == 2 else 96
        o = pts[(s, 1 if s == 6 else 0)]
        bad = data[:o] + bytes(size) + data[o + size:]
        assert GP.raw_read(worker, bad, False)[0] == GP.restate(bad, False) == ("invalid", s, 1 if s == 6 else 0, NOT_ON_CURVE)
        with pytest.raises(PIO.InvalidData, match="not on the curve"):
            PIO.read_parameters(bad, checked=False, worker=worker)


@pytest.mark.parametrize("first", [0, 63, 64, 65, 199])
def test_params_read_first_failure(worker, first):
    """200 points in h (DECODE_THREADS = 64 per block) with a bad point at `first` and a second one after it: the earlier
    ordinal wins, whichever block or section holds the later one"""
    data = PIO.write_parameters(GP.small_key((2, 200, 3, 2, 1, 1), seed=908))
    pts, _ = GP.offsets(data)
    t11 = uncompressed(1, dict((n, pt) for n, pt, _ in family(1))["T11"])
    second = (7, first + 1) if first + 1 < 200 else (8, 0)
    for enc1, enc2 in ((t11, None), (None, t11)):
        bad = bytearray(data)
        o1_, o2_ = pts[(7, first)], pts[second]
        bad[o1_:o1_ + 96] = enc1 if enc1 else bytes([bad[o1_] | 0x80]) + bad[o1_ + 1:o1_ + 96]
        bad[o2_:o2_ + 96] = enc2 if enc2 else bytes([bad[o2_] | 0x80]) + bad[o2_ + 1:o2_ + 96]
        bad = bytes(bad)
        for checked in (True, False):
            want = GP.restate(bad, checked)
            if checked or enc1 is None:
                assert want == ("invalid", 7, first, FLAGS if enc1 is None else NOT_IN_SUBGROUP)
            else:
                assert want == ("invalid", second[0], second[1], FLAGS)
            for on_device in (False, True):
                assert GP.raw_read(worker, bad, checked, on_device=on_device)[0] == want, (checked, on_device)


# --------------------------------------------------------------------------------------------
# 5: a caller's generator
# --------------------------------------------------------------------------------------------
def test_generate_rejects_torsion_generators(worker, seed=909):
    rng = random.Random(seed)
    asm = GEN.KeypairAssembly()
    asm.alloc_input()
    B.xor_demo(1, 0)(_AssemblyAdapter(asm))
    r1cs = RC.R1CS.from_assembly(worker, asm)
    tox = [rng.randrange(1, R) for _ in range(5)]
    launches = worker.kernel_launches
    for group in (1, 2):
        for name, pt, _ in family(group):
            g = abi(group, [pt])[0]
            with pytest.raises(bb.BackendError, match="not in the prime-order subgroup"):
                GEN.generate_parameters_device(worker, r1cs, *tox, **{"g1" if group == 1 else "g2": g})
    assert worker.kernel_launches == launches
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 6: host helpers
# --------------------------------------------------------------------------------------------
def point_mul(group, pt_abi, k):
    w = 12 if group == 1 else 24
    a = np.ascontiguousarray(pt_abi, np.uint64).reshape(1, w)
    s = np.array([(k >> (64 * j)) & (2 ** 64 - 1) for j in range(4)], np.uint64)
    out = np.zeros((1, w), np.uint64)
    assert bb.load_library().bb_point_mul(C.c_int(group), a.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), C.c_int(0),
                                          out.ctypes.data_as(C.c_void_p)) == 0
    return out[0]


@pytest.mark.parametrize("group", [1, 2])
def test_host_helpers(group):
    """sums with doublings and cancellations, multiples at and around the order, compression, all on torsion points"""
    G = F.G1 if group == 1 else F.G2
    fam = family(group)
    tors = [(n, pt, q) for n, pt, q in fam if q is not None]
    zero = np.zeros(12 if group == 1 else 24, np.uint64)
    enc = lambda pt: zero if pt is None else abi(group, [pt])[0]
    rng = random.Random(910 + group)
    for name, t, q in tors:
        others = [t, G.neg(t), mul(G, t, 2), G.gen, None] + [rng.choice(fam)[1]]
        for u in others:
            got = bb.point_add(group, enc(t), enc(u))[0]
            assert np.array_equal(got, enc(G.add(t, u))), name
            got = bb.point_add(group, enc(u), enc(t))[0]
            assert np.array_equal(got, enc(G.add(u, t))), name
        ks = [1, 2, q - 1, q, q + 1, 2 * q + 1, R - 1, rng.randrange(R)] if q < R else [1, 2, R - 1, rng.randrange(R)]
        for k in ks:
            if k < 2 ** 255:
                assert np.array_equal(point_mul(group, enc(t), k), enc(mul(G, t, k))), (name, k)
        assert bb.point_compress(group, enc(t)) == compress(group, t)
        assert bb.point_compress(group, enc(G.neg(t))) == compress(group, G.neg(t))
    for name, pt, _ in fam:
        assert bb.point_compress(group, enc(pt)) == compress(group, pt), name


# --------------------------------------------------------------------------------------------
# 7: proofs write-back
# --------------------------------------------------------------------------------------------
def test_proofs_write_back(worker):
    """points decoded unchecked come back byte for byte through bb_proofs_write, as A, B and C"""
    e1 = [compress(1, pt) for _, pt, _ in family(1)] + [bytes([0x80]) + bytes(47), bytes([0xa0]) + bytes(47)]
    e2 = [compress(2, pt) for _, pt, _ in family(2)]
    n = max(len(e1), len(e2))
    e1, e2 = (e1 * 2)[:n], (e2 * 3)[:n]
    p1, w1 = V.points_decompress(worker, 1, b"".join(e1), check_subgroup=False)
    p2, w2 = V.points_decompress(worker, 2, b"".join(e2), check_subgroup=False)
    assert not w1.any() and not w2.any()
    got = V.write_proofs(worker, p1, p2, p1[::-1].copy())
    assert got == b"".join(a + b + c for a, b, c in zip(e1, e2, e1[::-1]))
