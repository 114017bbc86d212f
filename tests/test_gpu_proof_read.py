"""Proof::read / Proof::write over a batch on the device (bb_proofs_read, bb_proofs_write, csrc/decode.cu) against the
oracle's restatement of Proof::read (oracle/oracle0/pairing.py: g1_decompress, g2_decompress, proof_read).

Every expected status comes from `classify`, which maps the oracle's decoders onto the (which, why) codes of
include/bellman_b200.h.  tests/test_emulated_proof_read.py runs the same bodies on the emulated device (tests/native/);
this file adds the sizes only a device reaches.
"""
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import verifier as V
from oracle import o1
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

import test_gpu_verify as GV

pytestmark = pytest.mark.gpu

P, R = F.FP_MODULUS, F.FR_MODULUS
OK, FLAGS, NONCANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, IDENTITY = range(6)


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# the oracle's view: Proof::read as (which, why) codes
# --------------------------------------------------------------------------------------------
_ORACLE_WHY = {"not compressed": FLAGS, "invalid infinity encoding": FLAGS, "x not canonical": NONCANONICAL,
               "not on curve": NOT_ON_CURVE, "not in the prime-order subgroup": NOT_IN_SUBGROUP}


def classify_point(group, b):
    """why code of one encoding by the oracle's from_compressed (5 = a valid identity encoding), and the point"""
    try:
        pt = (PR.g1_decompress if group == 1 else PR.g2_decompress)(bytes(b))
    except ValueError as e:
        return _ORACLE_WHY[str(e)], None
    return (IDENTITY, None) if pt is None else (OK, pt)


def classify(b192):
    """the status byte Proof::read implies: A, then B, then C; the first failing element decides"""
    for which, group, lo, hi in ((1, 1, 0, 48), (2, 2, 48, 144), (3, 1, 144, 192)):
        why, _ = classify_point(group, b192[lo:hi])
        if why:
            return (which << 4) | why
    return 0


def g1_abi(pts):
    return o1.g1_from_affine_ints(list(pts))


def g2_abi(pts):
    return o1.g2_from_affine_ints(list(pts))


def random_g1(rng):
    return F.G1.mul(F.G1_GEN, rng.randrange(1, R))


def random_g2(rng):
    return F.G2.mul(F.G2_GEN, rng.randrange(1, R))


def off_subgroup_g1(rng):
    """a point of y^2 = x^3 + 4 with random x and no cofactor cleared, confirmed outside G1 by the oracle"""
    while True:
        x = rng.randrange(P)
        y = PR._fp_sqrt((x * x * x + 4) % P)
        if y is not None:
            pt = (x, y if rng.random() < 0.5 else (P - y) % P)
            assert F.G1.mul(pt, R - 1) != F.G1.neg(pt)
            return pt


def off_subgroup_g2(rng):
    while True:
        x = (rng.randrange(P), rng.randrange(P))
        y = PR._fp2_sqrt(F.Fp2Ops.add(F.Fp2Ops.mul(F.Fp2Ops.mul(x, x), x), F.G2_B))
        if y is not None:
            pt = (x, y if rng.random() < 0.5 else F.Fp2Ops.neg(y))
            assert F.G2.mul(pt, R - 1) != F.G2.neg(pt)
            return pt


def no_root_x(group, rng):
    """an x (canonical) whose x^3 + b has no square root"""
    while True:
        if group == 1:
            x = rng.randrange(P)
            if PR._fp_sqrt((x * x * x + 4) % P) is None:
                return x
        else:
            x = (rng.randrange(P), rng.randrange(P))
            if PR._fp2_sqrt(F.Fp2Ops.add(F.Fp2Ops.mul(F.Fp2Ops.mul(x, x), x), F.G2_B)) is None:
                return x


def _fp2_cbrt(c):
    """a cube root in Fp2 (None if there is none): p^2 - 1 = 9 t with 3 not dividing t, so c^(3^-1 mod t) is a root up to a
    factor in the 9-element 3-Sylow subgroup, found by trying all of them"""
    q = P * P
    t = (q - 1) // 9
    assert t % 3 != 0
    pw = _fp2_pow
    if pw(c, (q - 1) // 3) != (1, 0):
        return None
    r = pw(c, pow(3, -1, t))
    z = next(pw((k, 1), t) for k in range(2, 50) if pw((k, 1), (q - 1) // 3) != (1, 0))      # generator of the 3-Sylow
    g = (1, 0)
    for _ in range(9):
        cand = F.Fp2Ops.mul(r, g)
        if F.Fp2Ops.mul(F.Fp2Ops.mul(cand, cand), cand) == c:
            return cand
        g = F.Fp2Ops.mul(g, z)
    return None


def _fp2_pow(a, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = F.Fp2Ops.mul(r, a)
        a = F.Fp2Ops.mul(a, a)
        e >>= 1
    return r


def g2_points_with_real_y(rng, count):
    """points of E' with y.c1 = 0 (so y.c0 decides the sort bit): y = (y0, 0), x a cube root of y0^2 - 4(u + 1)"""
    out = []
    while len(out) < count:
        y0 = rng.randrange(1, P)
        x = _fp2_cbrt(((y0 * y0 - 4) % P, P - 4))
        if x is not None:
            pt = (x, (y0, 0))
            assert F.G2.is_on_curve(pt)
            out.append(pt)
    return out


def compress(group, pt):
    return F.g1_compress(pt) if group == 1 else F.g2_compress(pt)


def proof_bytes(a, b, c):
    return F.g1_compress(a) + F.g2_compress(b) + F.g1_compress(c)


# --------------------------------------------------------------------------------------------
# bodies shared with the emulated file
# --------------------------------------------------------------------------------------------
def test_round_trip(worker, n_random=3, seed=11):
    """the generators and random subgroup points: oracle compression -> device decode; device encode
    (bb_proofs_write) == bb_point_compress == oracle compression, byte for byte"""
    rng = random.Random(seed)
    g1 = [F.G1_GEN] + [random_g1(rng) for _ in range(2 * n_random)]
    g2 = [F.G2_GEN] + [random_g2(rng) for _ in range(n_random)]
    for group, pts, abi in ((1, g1, g1_abi), (2, g2, g2_abi)):
        out, why = V.points_decompress(worker, group, b"".join(compress(group, p) for p in pts))
        assert list(why) == [OK] * len(pts)
        assert np.array_equal(out, abi(pts))
    n = n_random + 1
    a, b, c = g1[:n], g2, g1[n:] + [F.G1_GEN]
    want = b"".join(proof_bytes(*t) for t in zip(a, b, c))
    got = V.write_proofs(worker, g1_abi(a), g2_abi(b), g1_abi(c))
    assert got == want
    for i in range(n):
        assert got[192 * i:192 * i + 48] == bb.point_compress(bb.G1, g1_abi([a[i]]))
        assert got[192 * i + 48:192 * i + 144] == bb.point_compress(bb.G2, g2_abi([b[i]]))
    da, db, dc, status = V.read_proofs(worker, got)
    assert list(status) == [0] * n
    assert np.array_equal(da, g1_abi(a)) and np.array_equal(db, g2_abi(b)) and np.array_equal(dc, g1_abi(c))
    for i in range(n):                                           # the oracle's Proof::read agrees
        assert PR.proof_read(got[192 * i:192 * (i + 1)]) == (a[i], b[i], c[i])


def test_sign_choice(worker, seed=12):
    """both sort-bit values in both groups; G2 points whose y.c1 = 0, where y.c0 decides (decoded without the subgroup
    check, since such points are not in G2)"""
    rng = random.Random(seed)
    for group, pts in ((1, [random_g1(rng), F.G1_GEN]), (2, [random_g2(rng), F.G2_GEN])):
        G = F.G1 if group == 1 else F.G2
        both = pts + [G.neg(p) for p in pts]
        encs = [compress(group, p) for p in both]
        assert {e[0] & 0x20 for e in encs} == {0, 0x20}
        out, why = V.points_decompress(worker, group, b"".join(encs))
        assert list(why) == [OK] * len(both)
        assert np.array_equal(out, (g1_abi if group == 1 else g2_abi)(both))
    real = g2_points_with_real_y(rng, 2)
    real += [F.G2.neg(p) for p in real]
    encs = [F.g2_compress(p) for p in real]
    assert {e[0] & 0x20 for e in encs} == {0, 0x20}
    out, why = V.points_decompress(worker, 2, b"".join(encs), check_subgroup=False)
    assert list(why) == [OK] * len(real)
    assert np.array_equal(out, g2_abi(real))
    for e in encs:                                               # and with the check: outside the subgroup
        assert classify_point(2, e)[0] == NOT_IN_SUBGROUP
    _, why = V.points_decompress(worker, 2, b"".join(encs))
    assert list(why) == [NOT_IN_SUBGROUP] * len(real)


def bad_encodings(group, rng):
    """one encoding per rejection class (and the identity), as (name, bytes, why)"""
    size = 48 if group == 1 else 96
    good = compress(group, random_g1(rng) if group == 1 else random_g2(rng))
    out = []
    out.append(("compression bit clear", bytes([good[0] & 0x7f]) + good[1:], FLAGS))
    out.append(("infinity with the sort bit", bytes([0xe0]) + bytes(size - 1), FLAGS))
    out.append(("infinity with a non-zero x", bytes([0xc0]) + bytes(size - 2) + b"\x01", FLAGS))
    out.append(("infinity, compression bit clear", bytes([0x40]) + bytes(size - 1), FLAGS))
    for k in (0, 1):                                             # x = p, x = p + 1 (G2: in x.c1)
        xb = bytearray((P + k).to_bytes(48, "big"))
        xb[0] |= 0x80
        out.append((f"x = p + {k}", bytes(xb) + good[48:], NONCANONICAL))
    if group == 2:
        out.append(("x.c0 = p", good[:48] + P.to_bytes(48, "big"), NONCANONICAL))
        out.append(("x.c0 = 2^384 - 1", good[:48] + b"\xff" * 48, NONCANONICAL))
    x = no_root_x(group, rng)
    nr = bytearray(x.to_bytes(48, "big") if group == 1 else x[1].to_bytes(48, "big") + x[0].to_bytes(48, "big"))
    nr[0] |= 0x80
    out.append(("x^3 + b is not a square", bytes(nr), NOT_ON_CURVE))
    off = off_subgroup_g1(rng) if group == 1 else off_subgroup_g2(rng)
    out.append(("on the curve, outside the subgroup", compress(group, off), NOT_IN_SUBGROUP))
    out.append(("the identity", bytes([0xc0]) + bytes(size - 1), IDENTITY))
    return out


def test_every_rejection_class(worker, seed=13):
    """each class of the table for A, B and C: the status byte, the classifier, the zeroed points and read_proof's message"""
    rng = random.Random(seed)
    a, b, c = random_g1(rng), random_g2(rng), random_g1(rng)
    ga, gb, gc = F.g1_compress(a), F.g2_compress(b), F.g1_compress(c)
    proofs, want = [proof_bytes(a, b, c)], [0]
    for which in (1, 2, 3):
        for name, enc, why in bad_encodings(2 if which == 2 else 1, rng):
            assert classify_point(2 if which == 2 else 1, enc)[0] == why, name
            pb = {1: enc + gb + gc, 2: ga + enc + gc, 3: ga + gb + enc}[which]
            proofs.append(pb)
            want.append((which << 4) | why)
    data = b"".join(proofs)
    assert [classify(p) for p in proofs] == want
    da, db, dc, status = V.read_proofs(worker, data)
    assert list(status) == want
    assert np.array_equal(da[0], g1_abi([a])[0]) and np.array_equal(db[0], g2_abi([b])[0])
    assert not da[1:].any() and not db[1:].any() and not dc[1:].any()     # nothing of an invalid proof leaks out
    for pb, st in zip(proofs[1:], want[1:]):
        with pytest.raises(bb.InvalidProofEncoding) as ei:
            V.read_proof(worker, pb)
        msg = "point at infinity" if st & 15 == IDENTITY else ("invalid G2" if st >> 4 == 2 else "invalid G1")
        assert str(ei.value) == msg and isinstance(ei.value, ValueError) and ei.value.status == st
    got = V.read_proof(worker, proofs[0])
    assert np.array_equal(got[2], g1_abi([c])[0])


def test_priority(worker, seed=14):
    """A and C bad: A is reported; B bad and C the identity: B is reported"""
    rng = random.Random(seed)
    a, b, c = random_g1(rng), random_g2(rng), random_g1(rng)
    ga, gb, gc = F.g1_compress(a), F.g2_compress(b), F.g1_compress(c)
    ident1, bad1 = bytes([0xc0]) + bytes(47), bytes([ga[0] & 0x7f]) + ga[1:]
    off2 = F.g2_compress(off_subgroup_g2(rng))
    cases = [(bad1 + gb + ident1, 0x11), (bad1 + gb + bad1, 0x11), (ident1 + gb + bad1, 0x15), (ga + off2 + ident1, 0x24), (ga + gb + ident1, 0x35)]
    _, _, _, status = V.read_proofs(worker, b"".join(p for p, _ in cases))
    assert list(status) == [s for _, s in cases] == [classify(p) for p, _ in cases]


def test_fast_subgroup_check_matches_rP(worker, count=64, seed=15):
    """on points of the curve outside the subgroup, and on subgroup points, the fast checks (phi / psi) agree with
    bb_points_validate's [r]P"""
    rng = random.Random(seed)
    for group, off, good in ((1, off_subgroup_g1, random_g1), (2, off_subgroup_g2, random_g2)):
        pts = [off(rng) for _ in range(count)] + [good(rng) for _ in range(2)]
        encs = b"".join(compress(group, p) for p in pts)
        _, why = V.points_decompress(worker, group, encs)
        assert list(why) == [NOT_IN_SUBGROUP] * count + [OK] * 2
        abi = (g1_abi if group == 1 else g2_abi)(pts)
        unchecked, why_u = V.points_decompress(worker, group, encs, check_subgroup=False)
        assert list(why_u) == [OK] * len(pts) and np.array_equal(unchecked, abi)
        for i in range(len(pts)):
            first_bad, why_v = _validate(worker, group, abi[i:i + 1])
            assert (why_v == 2) == (i < count), i


def _validate(worker, group, pts):
    import ctypes as C
    first_bad, why = C.c_size_t(), C.c_int()
    arr = np.ascontiguousarray(pts, np.uint64)
    assert bb.load_library().bb_points_validate(worker._h, C.c_int(group), arr.ctypes.data_as(C.c_void_p), C.c_size_t(arr.shape[0]),
                                                C.c_int(1), C.byref(first_bad), C.byref(why)) == 0
    return first_bad.value, why.value


def test_mixed_batch(worker, seed=16):
    """valid and invalid proofs interleaved, read at stride 192 and at stride 384 with the proof at offset 128 among
    random padding; argument errors; n = 0"""
    rng = random.Random(seed)
    proofs = []
    for k in range(8):
        a, b, c = random_g1(rng), random_g2(rng), random_g1(rng)
        pb = bytearray(proof_bytes(a, b, c))
        if k % 3 == 1:
            pb[48 + 95] ^= 1                                     # a flipped x byte of B
        elif k % 3 == 2:
            pb[144] &= 0x7f                                      # C without the compression bit
        proofs.append(bytes(pb))
    want = [classify(p) for p in proofs]
    assert sum(1 for s in want if s) >= 4
    a192, b192, c192, st192 = V.read_proofs(worker, b"".join(proofs))
    assert list(st192) == want
    for i, s in enumerate(want):
        if s:
            assert not a192[i].any() and not b192[i].any() and not c192[i].any()
        else:
            pa, pbb, pc = PR.proof_read(proofs[i])
            assert np.array_equal(a192[i], g1_abi([pa])[0]) and np.array_equal(b192[i], g2_abi([pbb])[0])
            assert np.array_equal(c192[i], g1_abi([pc])[0])
    recs = b"".join(bytes(rng.randrange(256) for _ in range(128)) + p + bytes(rng.randrange(256) for _ in range(64)) for p in proofs)
    a384, b384, c384, st384 = V.read_proofs(worker, memoryview(recs)[128:], stride=384)
    assert list(st384) == want
    assert np.array_equal(a384, a192) and np.array_equal(b384, b192) and np.array_equal(c384, c192)
    _check_n_invalid(worker, b"".join(proofs), len(proofs), sum(1 for s in want if s))
    _check_arg_errors(worker, b"".join(proofs))
    a0, b0, c0, s0 = V.read_proofs(worker, b"", n=0)
    assert a0.shape == (0, 12) and b0.shape == (0, 24) and s0.shape == (0,)
    assert V.write_proofs(worker, a0, b0, c0) == b""


def _raw_read(worker, data, n, stride, nulls=()):
    import ctypes as C
    buf = np.frombuffer(data, np.uint8) if data else None
    pb = V._ProofBytes()
    pb.bytes = None if "bytes" in nulls or buf is None else buf.ctypes.data
    pb.n, pb.stride, pb.on_device = n, stride, 0
    a, b, c = np.zeros((max(n, 1), 12), np.uint64), np.zeros((max(n, 1), 24), np.uint64), np.zeros((max(n, 1), 12), np.uint64)
    status = np.zeros(max(n, 1), np.uint8)
    n_invalid = C.c_size_t(12345)
    ptr = lambda arr, name: None if name in nulls else arr.ctypes.data_as(C.c_void_p)
    rc = bb.load_library().bb_proofs_read(worker._h, C.byref(pb), ptr(a, "a"), ptr(b, "b"), ptr(c, "c"), C.c_int(0), ptr(status, "status"),
                                          C.byref(n_invalid))
    return rc, n_invalid.value


def _check_n_invalid(worker, data, n, bad):
    rc, n_invalid = _raw_read(worker, data, n, 0)
    assert rc == 0 and n_invalid == bad


def _check_arg_errors(worker, data):
    for stride in (1, 191):
        assert _raw_read(worker, data, 1, stride)[0] == 16
    for name in ("bytes", "a", "b", "c", "status"):
        assert _raw_read(worker, data, 1, 192, nulls=(name,))[0] == 16, name
    rc, n_invalid = _raw_read(worker, b"", 0, 0, nulls=("bytes", "a", "b", "c", "status"))
    assert rc == 0 and n_invalid == 0


def test_verifier_from_bytes(worker, seed=21):
    """MiMC-322 proofs queued as bytes are accepted; a tampered but well-encoded proof is rejected with InvalidProof; a
    badly encoded one raises InvalidProofEncoding with bellman's message and its queue index, before any pairing work"""
    vk, vk_int, items = GV.mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    encoded = [(proof_bytes(*proof), x) for proof, x in items]
    for (b192, _), (proof, _) in zip(encoded, items):
        a, b, c = V.read_proof(worker, b192)
        want = GV.abi_proof(proof)
        assert np.array_equal(a, want[0]) and np.array_equal(b, want[1]) and np.array_equal(c, want[2])

    def verdict(queue_items, rng):
        bv = bb.BatchVerifier()
        for kind, item in queue_items:
            if kind == "bytes":
                bv.queue_bytes(*item)
            else:
                bv.queue(item)
        try:
            bv.verify(rng, pvk)
            return True
        except bb.InvalidProof:
            return False

    assert verdict([("bytes", e) for e in encoded], random.Random(1))
    assert verdict([("bytes", e) for e in encoded], None)
    mixed = [("bytes", encoded[0]), ("arrays", (GV.abi_proof(items[1][0]), items[1][1]))] + [("bytes", e) for e in encoded[2:]]
    assert verdict(mixed, random.Random(2))
    bad_proof, bad_x = GV.tampered(*items[2], "c")
    tampered = [("bytes", e) for e in encoded[:2]] + [("bytes", (proof_bytes(*bad_proof), bad_x))] + [("bytes", e) for e in encoded[3:]]
    assert not verdict(tampered, random.Random(3))
    broken = bytearray(encoded[3][0])
    broken[48] &= 0x7f                                           # B without its compression bit
    bv = bb.BatchVerifier()
    for k, (b192, x) in enumerate(encoded):
        bv.queue_bytes(bytes(broken) if k == 3 else b192, x)
    launches = worker.kernel_launches
    with pytest.raises(bb.InvalidProofEncoding) as ei:
        bv.verify(random.Random(4), pvk)
    assert str(ei.value).startswith("invalid G2") and ei.value.index == 3 and "3" in str(ei.value)
    assert worker.kernel_launches - launches == 3                # the decoding kernels only: no pairing work
    pvk.free()


# --------------------------------------------------------------------------------------------
# GPU only: sizes the emulation cannot reach
# --------------------------------------------------------------------------------------------
def test_gpu_prover_proofs_read_and_verify(worker):
    """bytes from bb_groth16_prove decode to the oracle's points and verify from their bytes"""
    rng = random.Random(81)
    mc = o1.Mimc(322, seed=4)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    p = mc.export_params()
    params = bb.Parameters(worker, p)
    wit = mc.witness()
    asg = bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"], wit["a_aux_density"],
                               wit["b_input_density"], wit["b_aux_density"])
    vk = {"alpha_g1": p["vk_g1"][0], "beta_g2": p["vk_g2"][0], "gamma_g2": p["vk_g2"][1], "delta_g2": p["vk_g2"][2], "ic": p["ic"]}
    pvk = bb.prepare_verifying_key(worker, vk)
    x = o1.fr_to_ints(wit["inputs"][1:])
    proofs = [bb.create_proof(asg, params, rng.randrange(R), rng.randrange(R)) for _ in range(4)]
    a, b, c, status = V.read_proofs(worker, b"".join(proofs))
    assert not status.any()
    for i, pb in enumerate(proofs):
        want = GV.abi_proof(PR.proof_read(pb))
        assert np.array_equal(a[i], want[0]) and np.array_equal(b[i], want[1]) and np.array_equal(c[i], want[2])
    bv = bb.BatchVerifier()
    for pb in proofs:
        bv.queue_bytes(pb, x)
    bv.verify(random.Random(5), pvk)
    pvk.free()
    params.free()


def _flip(data, idx, offset):
    out = bytearray(data)
    out[192 * idx + offset] ^= 1
    return bytes(out)


def test_gpu_large_batch(worker, log_n=16, n_inputs=2):
    """a 2^16-proof synthetic batch written with bb_proofs_write decodes back to the identical points, from HBM and from
    host memory; with a corrupted proof at the first, middle and last index exactly those statuses are set"""
    n = 1 << log_n
    vk, pvk, d, host = GV.synth_batch(worker, 41, n, n_inputs)
    a, b, c, _ = host
    d_bytes = worker.device_alloc(n * 192)
    import ctypes as C
    assert bb.load_library().bb_proofs_write(worker._h, d["a"], d["b"], d["c"], C.c_size_t(n), C.c_int(1), d_bytes) == 0
    data = np.zeros(n * 192, np.uint8)
    worker.download(d_bytes, data)
    data = data.tobytes()
    assert data == V.write_proofs(worker, a, b, c)
    ha, hb, hc, hs = V.read_proofs(worker, data)
    assert not hs.any() and np.array_equal(ha, a) and np.array_equal(hb, b) and np.array_equal(hc, c)
    outs = {k: worker.device_alloc(n * w * 8) for k, w in (("a", 12), ("b", 24), ("c", 12))}
    _, _, _, ds = V.read_proofs(worker, d_bytes, n=n, on_device=True, out_device=(outs["a"], outs["b"], outs["c"]))
    assert not ds.any()
    for key, ref in (("a", a), ("b", b), ("c", c)):
        got = np.zeros_like(ref)
        worker.download(outs[key], got)
        assert np.array_equal(got, ref), key
    bad = data
    for pos, off in ((0, 5), (n // 2, 48 + 95), (n - 1, 144 + 47)):
        bad = _flip(bad, pos, off)
    want = {i: classify(bad[192 * i:192 * (i + 1)]) for i in (0, n // 2, n - 1)}
    assert all(want.values()) and want[n // 2] >> 4 == 2
    _, _, _, st = V.read_proofs(worker, bad)
    assert set(np.flatnonzero(st)) == set(want) and all(st[i] == s for i, s in want.items())
    worker.upload(d_bytes, np.frombuffer(bad, np.uint8))
    _, _, _, st_d = V.read_proofs(worker, d_bytes, n=n, on_device=True, out_device=(outs["a"], outs["b"], outs["c"]))
    assert np.array_equal(st_d, st)
    for p in list(outs.values()) + [d_bytes]:
        worker.device_free(p)
    GV.free_batch(worker, pvk, d)


def test_gpu_fast_subgroup_check_many(worker, count=1 << 12, seed=17):
    """2^12 points per group outside the subgroup: the fast checks and [r]P (bb_points_validate) reject every one"""
    rng = random.Random(seed)
    for group in (1, 2):
        pts = _cheap_off_subgroup(group, rng, count)
        encs = b"".join(compress(group, p) for p in pts)
        out, why = V.points_decompress(worker, group, encs, check_subgroup=False)
        assert not why.any()
        _, why_fast = V.points_decompress(worker, group, encs)
        assert (why_fast == NOT_IN_SUBGROUP).all()
        flags = [_validate(worker, group, out[i:i + 1])[1] for i in range(count)]
        assert all(f == 2 for f in flags)


def _cheap_off_subgroup(group, rng, count):
    """points on the curve without the oracle's (slow) order check: a random point lies in the subgroup with
    probability 1 / cofactor (below 2^-126), and [r]P on the device confirms each one above"""
    out = []
    while len(out) < count:
        if group == 1:
            x = rng.randrange(P)
            y = PR._fp_sqrt((x * x * x + 4) % P)
        else:
            x = (rng.randrange(P), rng.randrange(P))
            y = PR._fp2_sqrt(F.Fp2Ops.add(F.Fp2Ops.mul(F.Fp2Ops.mul(x, x), x), F.G2_B))
        if y is not None:
            out.append((x, y))
    return out
