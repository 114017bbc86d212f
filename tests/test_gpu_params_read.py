"""Parameters::read / VerifyingKey::read on the device (bb_params_read, bb_vk_read, csrc/decode.cu;
params_io.read_parameters_device / read_verifying_key_device) against params_io.read_parameters + Parameters(...) and
against `restate`, a small pure-Python restatement of the reference's reader (groth16/src/lib.rs:158-218, 289-398) over
the oracle's curve arithmetic.  tests/test_emulated_params_read.py runs the same bodies on the emulated device
(tests/native/) at small sizes.
"""
import ctypes as C
import random
import struct

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import generator as GEN
from bellman_b200 import params_io as PIO
from oracle import o1
from oracle.oracle0 import bellman as B
from oracle.oracle0 import fields as F

from test_gpu_parity import _AssemblyAdapter
from test_gpu_proof_read import off_subgroup_g1, off_subgroup_g2
from test_gpu_verify import abi_proof

pytestmark = pytest.mark.gpu

P, R = F.FP_MODULUS, F.FR_MODULUS
OK, FLAGS, NONCANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, IDENTITY = range(6)
SECTIONS = PIO.SECTIONS
G2_SECTIONS = {"beta_g2", "gamma_g2", "delta_g2", "b_g2"}
ARG, INVALID, EOF = 16, 8, 3


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# the reference's reader, restated
# --------------------------------------------------------------------------------------------
_CLASSIFIED = {}


def classify(g2, b, checked, allow_identity):
    """why code of one uncompressed point: from_uncompressed (checked) / from_uncompressed_unchecked, then bellman's
    identity rule"""
    key = (g2, bytes(b), checked, allow_identity)
    if key in _CLASSIFIED:
        return _CLASSIFIED[key]
    flags = b[0]
    coords = [int.from_bytes(bytes([b[0] & 0x1F]) + bytes(b[1:48]), "big")] + [int.from_bytes(b[j:j + 48], "big") for j in range(48, len(b), 48)]
    if flags & 0xA0:
        why = FLAGS
    elif flags & 0x40:
        why = FLAGS if any(coords) else (OK if allow_identity else IDENTITY)
    elif any(v >= P for v in coords):
        why = NONCANONICAL
    elif checked:
        curve = F.G2 if g2 else F.G1
        pt = ((coords[1], coords[0]), (coords[3], coords[2])) if g2 else (coords[0], coords[1])
        why = NOT_ON_CURVE if not curve.is_on_curve(pt) else NOT_IN_SUBGROUP if curve.mul(pt, R - 1) != curve.neg(pt) else OK
    else:
        why = OK
    _CLASSIFIED[key] = why
    return why


def restate(data, checked, sections=12):
    """Parameters::read (sections=12) / VerifyingKey::read (7), point by point: ("ok", consumed),
    ("invalid", section, index, why) of the first failing point, or ("eof", section, index, offset)"""
    off = 0
    for s in range(sections):
        size = 192 if SECTIONS[s] in G2_SECTIONS else 96
        n = 1
        if s >= 6:
            if len(data) - off < 4:
                return ("eof", s, 0, off)
            n = struct.unpack_from(">I", data, off)[0]
            off += 4
        for i in range(n):
            if len(data) - off < size:
                return ("eof", s, i, off)
            why = classify(size == 192, data[off:off + size], checked or s <= 6, s <= 5)
            if why:
                return ("invalid", s, i, why)
            off += size
    return ("ok", off)


# --------------------------------------------------------------------------------------------
# the library's view
# --------------------------------------------------------------------------------------------
def live_bytes(worker):
    lib = bb.load_library()
    lib.bb_diag_ctx_live_bytes.restype = C.c_uint64
    return int(lib.bb_diag_ctx_live_bytes(worker._h))


def device_copy(worker, data):
    p = worker.device_alloc(max(len(data), 16))
    if len(data):
        worker.upload(p, np.frombuffer(bytes(data), np.uint8))
    return p


def raw_read(worker, data, checked=True, on_device=False, vk_only=False):
    """bb_params_read (or bb_vk_read) with both out pointers: the outcome in restate's form.  A failure must leave both
    out pointers NULL and the context's live bytes where they were."""
    lib = bb.load_library()
    d = device_copy(worker, data) if on_device else None
    buf = np.frombuffer(bytes(data), np.uint8)
    ptr = C.c_void_p(bb._addr(d)) if on_device else C.c_void_p(buf.ctypes.data if buf.size else None)
    crs, vk = C.c_void_p(0x1000), C.c_void_p(0x2000)
    rep = PIO.ParamsReport()
    before = live_bytes(worker)
    if vk_only:
        rc = lib.bb_vk_read(worker._h, ptr, C.c_size_t(len(data)), C.c_int(1 if on_device else 0), C.byref(vk), C.byref(rep))
        crs = C.c_void_p(None)
    else:
        rc = lib.bb_params_read(worker._h, ptr, C.c_size_t(len(data)), C.c_int(1 if on_device else 0), C.c_int(1 if checked else 0),
                                C.byref(crs), C.byref(vk), C.byref(rep))
    if rc == 0:
        lib.bb_crs_destroy(crs)
        lib.bb_vk_destroy(vk)
        out = ("ok", int(rep.consumed))
    else:
        assert crs.value is None and vk.value is None, (rc, crs.value, vk.value)
        assert live_bytes(worker) == before, lib.bb_last_error()
        if rc == INVALID:
            out = ("invalid", rep.section, int(rep.index), rep.why)
        elif rc == EOF:
            assert rep.why == 0
            out = ("eof", rep.section, int(rep.index), int(rep.consumed))
        else:
            raise AssertionError(f"status {rc}: {lib.bb_last_error()}")
    if d is not None:
        worker.device_free(d)
    return out, rep


# --------------------------------------------------------------------------------------------
# keys
# --------------------------------------------------------------------------------------------
def small_key(sizes=(2, 3, 2, 3, 1, 1), seed=1):
    """random points in the shape of the reference's one-constraint key (ic 2, h 3, l 2, a 3, b_g1 1, b_g2 1: 2136 bytes)"""
    rng = random.Random(seed)
    mk1 = lambda n: o1.g1_fixed_mul(o1.fr_from_ints([rng.randrange(1, R) for _ in range(n)])) if n else np.zeros((0, 12), np.uint64)
    mk2 = lambda n: o1.g2_fixed_mul(o1.fr_from_ints([rng.randrange(1, R) for _ in range(n)])) if n else np.zeros((0, 24), np.uint64)
    return dict(vk_g1=mk1(3), vk_g2=mk2(3), ic=mk1(sizes[0]), h=mk1(sizes[1]), l=mk1(sizes[2]), a=mk1(sizes[3]),
                b_g1=mk1(sizes[4]), b_g2=mk2(sizes[5]))


def mimc_key(rounds, seed=5, rng_seed=4):
    rng = random.Random(rng_seed)
    mc = o1.Mimc(rounds, seed=seed)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    return mc


def generated_key(worker, seed=41):
    rng = random.Random(seed)
    asm = GEN.KeypairAssembly()
    asm.alloc_input()
    B.xor_demo(0, 1)(_AssemblyAdapter(asm))
    return GEN.generate_parameters(worker, asm, *[rng.randrange(1, R) for _ in range(5)])


def offsets(data):
    """byte offset of every point and prefix: {(section, index): offset}, {section: prefix offset}"""
    pts, pre, off = {}, {}, 0
    for s, name in enumerate(SECTIONS):
        size = 192 if name in G2_SECTIONS else 96
        n = 1
        if s >= 6:
            pre[s] = off
            n = struct.unpack_from(">I", data, off)[0]
            off += 4
        for i in range(n):
            pts[(s, i)] = off
            off += size
    return pts, pre


def pinned(data):
    """a page-locked copy of data where a CUDA device is present (a plain copy otherwise)"""
    import torch
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8)
    if torch.cuda.is_available():
        t = t.pin_memory()
    return t, t.numpy()


def assert_same_key(worker, got, want_dict):
    """a resident Parameters holds exactly the points of read_parameters' dict, and those of Parameters(dict)"""
    old = bb.Parameters(worker, want_dict)
    for held in (PIO.download_parameters(got), PIO.download_parameters(old)):
        for name in ("h", "l", "a", "b_g1", "b_g2"):
            assert np.array_equal(held[name], np.asarray(want_dict[name], np.uint64).reshape(held[name].shape)), name
        vk1 = np.asarray(want_dict["vk_g1"], np.uint64).reshape(3, 12)
        vk2 = np.asarray(want_dict["vk_g2"], np.uint64).reshape(3, 24)
        assert np.array_equal(held["vk_g1"], vk1)
        assert np.array_equal(held["vk_g2"], vk2[[0, 2]])
    assert got.lens == old.lens
    old.free()


# --------------------------------------------------------------------------------------------
# 1. round trip
# --------------------------------------------------------------------------------------------
def round_trip(worker, data, chunks=(0, 97, 1000, 579)):
    """every input form, both modes, several staging chunk sizes (0 = the default): the resident key equals the host
    reader's, and bb_vk_read / the returned PreparedVerifyingKey hold |ic| points"""
    for checked in (True, False):
        want = PIO.read_parameters(data, checked=checked, worker=worker)
        keep, pin = pinned(data)
        d = device_copy(worker, data)
        try:
            inputs = [("bytes", bytes(data)), ("bytearray", bytearray(data)), ("memoryview", memoryview(bytes(data))), ("pinned", pin),
                      ("device", (d, len(data)))]
            for chunk in chunks:
                worker.set_option("params_read_chunk", chunk or (64 << 20))
                for name, src in inputs:
                    if chunk and name in ("bytearray", "memoryview", "device"):
                        continue
                    params, pvk = PIO.read_parameters_device(worker, src, checked=checked, verifying_key=True)
                    assert pvk.ic_len == want["ic"].shape[0], name
                    assert_same_key(worker, params, want)
                    params.free()
                    pvk.free()
        finally:
            worker.set_option("params_read_chunk", 64 << 20)
            worker.device_free(d)
    pvk, consumed = PIO.read_verifying_key_device(worker, data)
    assert consumed == 868 + 96 * want["ic"].shape[0] and pvk.ic_len == want["ic"].shape[0]
    pvk.free()


def test_round_trip_small_keys(worker):
    data = PIO.write_parameters(small_key())
    assert len(data) == 2136
    round_trip(worker, data)
    round_trip(worker, PIO.write_parameters(small_key((1, 0, 0, 0, 0, 0), seed=2)), chunks=(0, 97))
    round_trip(worker, PIO.write_parameters(small_key((0, 0, 0, 0, 0, 0), seed=3)), chunks=(0,))


def test_round_trip_mimc_and_generated(worker, rounds=322):
    round_trip(worker, PIO.write_parameters(mimc_key(rounds).export_params()), chunks=(0, 4099))
    round_trip(worker, PIO.write_parameters(generated_key(worker)), chunks=(0, 97))


# --------------------------------------------------------------------------------------------
# 2. proofs from the read key, verified under the read verifying key
# --------------------------------------------------------------------------------------------
def test_proofs(worker, rounds=322):
    from bellman_b200.r1cs import R1CS
    mc = mimc_key(rounds)
    data = PIO.write_parameters(mc.export_params())
    host = bb.Parameters(worker, PIO.read_parameters(data, worker=worker))
    dev, pvk = PIO.read_parameters_device(worker, data, checked=True, verifying_key=True)
    wit = mc.witness()
    asg = bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"], wit["a_aux_density"],
                               wit["b_input_density"], wit["b_aux_density"])
    rng = random.Random(7)
    r, s = rng.randrange(R), rng.randrange(R)
    proof = bb.create_proof(asg, dev, r, s)
    assert proof == bb.create_proof(asg, host, r, s) == mc.expected_proof(r, s)
    r1cs = R1CS.synth_mimc(worker, rounds, 5)
    assert bb.create_proof_r1cs(r1cs, dev, wit["inputs"], wit["aux"], r, s) == proof
    r1cs.free()
    rs, ss = [r, rng.randrange(R), rng.randrange(R)], [s, rng.randrange(R), rng.randrange(R)]
    batch = bb.create_proof_batch([asg] * 3, dev, rs, ss)
    assert batch == bb.create_proof_batch([asg] * 3, host, rs, ss) and batch[0] == proof
    from oracle.oracle0 import pairing as PR
    x = o1.fr_to_ints(wit["inputs"][1:])
    bv = bb.BatchVerifier()
    for p in batch:
        bb.verify_proof(pvk, abi_proof(PR.proof_read(p)), x)
        bv.queue((abi_proof(PR.proof_read(p)), x))
    bv.queue_bytes(batch[1], x)
    bv.verify(rng, pvk)
    assert bv.verify_each(pvk) == [None] * 4
    bad = abi_proof(PR.proof_read(batch[2]))
    with pytest.raises(bb.InvalidProof):
        bb.verify_proof(pvk, (bad[0], bad[1], abi_proof(PR.proof_read(batch[1]))[2]), x)
    pvk2, _ = PIO.read_verifying_key_device(worker, data)
    bb.verify_proof(pvk2, abi_proof(PR.proof_read(proof)), x)
    for obj in (pvk, pvk2, dev, host):
        obj.free()


# --------------------------------------------------------------------------------------------
# 3. every rejection class in every section
# --------------------------------------------------------------------------------------------
def corruptions(g2, rng):
    """name -> function(point bytes) -> corrupted bytes"""
    n = 4 if g2 else 2
    enc = (lambda p: F.g2_uncompressed(p)) if g2 else (lambda p: F.g1_uncompressed(p))
    off = off_subgroup_g2(rng) if g2 else off_subgroup_g1(rng)
    out = {"compressed": lambda b: bytes([b[0] | 0x80]) + b[1:], "sort": lambda b: bytes([b[0] | 0x20]) + b[1:],
           "infinity_with_coordinates": lambda b: bytes([b[0] | 0x40]) + b[1:],
           "identity": lambda b: bytes([0x40]) + bytes(len(b) - 1),
           "off_curve": lambda b: b[:-48] + ((int.from_bytes(b[-48:], "big") + 1) % P).to_bytes(48, "big"),
           "off_subgroup": lambda b, e=enc(off): e}
    for j in range(n):
        out[f"non_canonical_{j}"] = lambda b, j=j: b[:48 * j] + P.to_bytes(48, "big") + b[48 * (j + 1):]
    return out


def test_every_rejection_class(worker):
    rng = random.Random(11)
    p = small_key()
    data = PIO.write_parameters(p)
    pts, _ = offsets(data)
    cor = {False: corruptions(False, rng), True: corruptions(True, rng)}
    seen = set()
    for s, name in enumerate(SECTIONS):
        g2 = name in G2_SECTIONS
        size = 192 if g2 else 96
        idx = {6: 1, 7: 1, 9: 2}.get(s, 0)                   # a point inside the vector where there is one
        o = pts[(s, idx)]
        for kind, fn in cor[g2].items():
            bad = data[:o] + fn(data[o:o + size]) + data[o + size:]
            assert len(bad) == len(data)
            for checked in (True, False):
                want = restate(bad, checked)
                got, _ = raw_read(worker, bad, checked)
                assert got == want, (name, kind, checked, got, want)
                seen.add((want[0], want[3] if want[0] == "invalid" else None))
                strict = s <= 6 or checked
                if kind == "identity":
                    assert want == (("ok", len(data)) if s <= 5 else ("invalid", s, idx, IDENTITY))
                elif kind in ("off_curve", "off_subgroup") and not strict:
                    assert want == ("ok", len(data))                  # loaded as-is, as read_parameters(checked=False) does
                    params = PIO.read_parameters_device(worker, bad, checked=False)
                    host = PIO.read_parameters(bad, checked=False, worker=worker)
                    assert np.array_equal(PIO.download_parameters(params)[name], host[name])
                    params.free()
                else:
                    assert want[0] == "invalid" and want[1:3] == (s, idx), (name, kind, checked, want)
                # single faults: the host reader accepts and rejects the same files
                try:
                    PIO.read_parameters(bad, checked=checked, worker=worker)
                    host_ok = True
                except PIO.InvalidData:
                    host_ok = False
                assert host_ok == (want[0] == "ok"), (name, kind, checked)
    assert {w for k, w in seen if k == "invalid"} == {FLAGS, NONCANONICAL, NOT_ON_CURVE, NOT_IN_SUBGROUP, IDENTITY}
    # the exception of the Python reader carries the section, index, code and the reference's text
    o = pts[(7, 1)]
    bad = data[:o] + bytes([0x40]) + bytes(95) + data[o + 96:]
    with pytest.raises(PIO.InvalidData, match=r"^h\[1\]: point at infinity$") as ei:
        PIO.read_parameters_device(worker, bad)
    assert (ei.value.section, ei.value.index, ei.value.why) == ("h", 1, IDENTITY)
    o = pts[(11, 0)]
    bad = data[:o] + corruptions(True, rng)["off_subgroup"](data[o:o + 192]) + data[o + 192:]
    with pytest.raises(PIO.InvalidData, match=r"^b_g2\[0\]: invalid G2 \(not in the prime-order subgroup\)$"):
        PIO.read_parameters_device(worker, bad)
    o = pts[(0, 0)]
    bad = data[:o] + bytes([data[o] | 0x80]) + data[o + 1:]
    with pytest.raises(PIO.InvalidData, match=r"^alpha_g1: invalid G1"):
        PIO.read_verifying_key_device(worker, bad)


# --------------------------------------------------------------------------------------------
# 4. precedence, truncation, prefixes
# --------------------------------------------------------------------------------------------
def put(data, o, b):
    return data[:o] + b + data[o + len(b):]


def test_precedence(worker):
    rng = random.Random(12)
    data = PIO.write_parameters(small_key(seed=4))
    pts, pre = offsets(data)
    c1, c2 = corruptions(False, rng), corruptions(True, rng)
    seg = lambda s, i: data[pts[(s, i)]:pts[(s, i)] + (192 if SECTIONS[s] in G2_SECTIONS else 96)]
    cases = []
    # two faults in one vector: the earlier index wins whatever its class
    bad = put(put(data, pts[(7, 1)], c1["identity"](seg(7, 1))), pts[(7, 2)], c1["compressed"](seg(7, 2)))
    cases.append((bad, True, ("invalid", 7, 1, IDENTITY)))
    bad = put(put(data, pts[(9, 0)], c1["off_curve"](seg(9, 0))), pts[(9, 2)], c1["sort"](seg(9, 2)))
    cases += [(bad, True, ("invalid", 9, 0, NOT_ON_CURVE)), (bad, False, ("invalid", 9, 2, FLAGS))]
    # faults in two sections: the earlier section wins
    bad = put(put(data, pts[(11, 0)], c2["compressed"](seg(11, 0))), pts[(9, 1)], c1["off_subgroup"](seg(9, 1)))
    cases += [(bad, True, ("invalid", 9, 1, NOT_IN_SUBGROUP)), (bad, False, ("invalid", 11, 0, FLAGS))]
    bad = put(put(data, pts[(6, 1)], c1["identity"](seg(6, 1))), pts[(3, 0)], c2["off_curve"](seg(3, 0)))
    cases.append((bad, False, ("invalid", 3, 0, NOT_ON_CURVE)))
    # an invalid point before a truncation in the same vector is InvalidData, not EOF (read_parameters reports EOF here)
    bad = put(data, pts[(7, 1)], c1["non_canonical_1"](seg(7, 1)))[:pts[(7, 2)] + 10]
    cases.append((bad, True, ("invalid", 7, 1, NONCANONICAL)))
    with pytest.raises(EOFError):
        PIO.read_parameters(bad, worker=worker)
    # truncations: inside the key head, inside a point, inside a prefix, right after a prefix, at the end
    cases += [(data[:500], True, ("eof", 3, 0, 384)), (data[:pts[(9, 1)] + 50], True, ("eof", 9, 1, pts[(9, 1)])),
              (data[:pre[8] + 2], True, ("eof", 8, 0, pre[8])), (data[:pre[10] + 4], True, ("eof", 10, 0, pre[10] + 4)),
              (data[:-1], False, ("eof", 11, 0, pts[(11, 0)])), (data[:0], True, ("eof", 0, 0, 0))]
    # trailing bytes are not read
    cases.append((data + b"\xff" * 100, True, ("ok", len(data))))
    for bad, checked, want in cases:
        assert restate(bad, checked) == want
        for on_device in (False, True):
            got, _ = raw_read(worker, bad, checked, on_device=on_device)
            assert got == want, (checked, on_device, got, want)
    with pytest.raises(EOFError, match=r"^l: unexpected end of file in the length prefix"):
        PIO.read_parameters_device(worker, data[:pre[8] + 2])
    # a forged prefix: EOF after the points the buffer holds, no OOM and nothing allocated beyond the buffer
    for forged, k, want in ((put(data, pre[11], struct.pack(">I", 0xFFFFFFFF)), 5, ("eof", 11, 1, pts[(11, 0)] + 192)),
                            (put(data, pre[7], struct.pack(">I", 0xFFFFFFFF))[:pre[7] + 4], 1, ("eof", 7, 0, pre[7] + 4))):
        assert restate(forged, True) == want
        for on_device in (False, True):
            got, rep = raw_read(worker, forged, on_device=on_device)
            assert got == want and rep.len[k] == 0xFFFFFFFF and rep.len[0] == 2
    # bb_vk_read on a Parameters file reads its VerifyingKey and stops there
    got, rep = raw_read(worker, data, vk_only=True)
    assert got == ("ok", 868 + 96 * 2) and list(rep.len) == [2, 0, 0, 0, 0, 0]
    assert raw_read(worker, data[:868 + 96 + 10], vk_only=True)[0] == ("eof", 6, 1, 868 + 96)


# --------------------------------------------------------------------------------------------
# 5. argument errors, before any device work
# --------------------------------------------------------------------------------------------
def test_argument_errors(worker):
    lib = bb.load_library()
    data = np.frombuffer(PIO.write_parameters(small_key(seed=5)), np.uint8)
    crs, vk = C.c_void_p(0x1000), C.c_void_p(0x2000)
    rep = PIO.ParamsReport()
    launches, copied, live = worker.kernel_launches, worker.bytes_copied(), live_bytes(worker)
    assert lib.bb_params_read(worker._h, None, C.c_size_t(10), 0, 1, C.byref(crs), C.byref(vk), C.byref(rep)) == ARG
    assert crs.value is None and vk.value is None and rep.section == -1
    assert b"null" in lib.bb_last_error()
    assert lib.bb_params_read(worker._h, data.ctypes.data_as(C.c_void_p), C.c_size_t(data.size), 0, 1, None, None, None) == ARG
    assert lib.bb_vk_read(worker._h, data.ctypes.data_as(C.c_void_p), C.c_size_t(data.size), 0, None, None) == ARG
    assert lib.bb_params_read(None, data.ctypes.data_as(C.c_void_p), C.c_size_t(data.size), 0, 1, C.byref(crs), None, None) == ARG
    assert (worker.kernel_launches, worker.bytes_copied(), live_bytes(worker)) == (launches, copied, live)
    with pytest.raises(bb.BackendError):
        worker.set_option("params_read_chunk", 0)


# --------------------------------------------------------------------------------------------
# 6. profile stages and bytes copied
# --------------------------------------------------------------------------------------------
def test_profile_and_bytes(worker):
    data = PIO.write_parameters(small_key(seed=6))
    worker.set_option("profile", 1)
    worker.profile_reset()
    h2d0, _ = worker.bytes_copied()
    PIO.read_parameters_device(worker, data).free()
    h2d1, _ = worker.bytes_copied()
    assert h2d1 - h2d0 == len(data) - 6 * 4                   # every point, none of the prefixes
    for stage in ("params.upload", "params.g1", "params.g2"):
        assert worker.profile_read(stage)[1] > 0, stage
    worker.set_option("profile", 0)


# --------------------------------------------------------------------------------------------
# GPU sizes
# --------------------------------------------------------------------------------------------
def test_large_synthetic_key(worker, log_size=17):
    """a bench-shaped key at 2^17 constraints: round trip against the host reader from pinned memory and HBM"""
    import bench_params_read as BP
    data = BP.make_key_file(worker, log_size)
    want = PIO.read_parameters(data, checked=False, worker=worker)
    keep, pin = pinned(data)
    d = device_copy(worker, data)
    for src in (pin, (d, len(data))):
        params = PIO.read_parameters_device(worker, src, checked=True)
        assert_same_key(worker, params, want)
        params.free()
    worker.device_free(d)
