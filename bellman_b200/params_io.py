"""groth16::Parameters / VerifyingKey files (groth16/src/lib.rs:143-219, 258-398).

Format (all integers big-endian): VerifyingKey = alpha_g1, beta_g1 (96 B), beta_g2, gamma_g2 (192 B),
delta_g1 (96 B), delta_g2 (192 B), u32 |ic|, ic points (96 B each); Parameters = VerifyingKey, then
u32-length-prefixed h, l, a, b_g1 (G1) and b_g2 (G2).  Points use the uncompressed ZCash encoding
(`UncompressedEncoding::to_uncompressed`): x | y big-endian canonical coordinates, G2 as
x.c1 | x.c0 | y.c1 | y.c0; byte 0 carries the flags (bit 7 compressed = 0, bit 6 infinity).

`read_parameters` returns the arrays `bellman_b200.Parameters` uploads (Montgomery little-endian
limbs, identity = all-zero) and applies the reference's acceptance rules:

* encoding (both modes; what `from_uncompressed_unchecked` of the bls12_381 crate rejects): the
  compression and sort flags must be clear, coordinates must be canonical (< p), and an infinity
  flag requires every other bit of the encoding to be zero;
* the point at infinity is rejected in h, l, a, b_g1, b_g2 and ic in BOTH modes (lib.rs:199-207,
  303-315,337-345) and accepted for alpha, beta, gamma, delta (so that the prover can report the
  subversion CRS itself, prover.rs:320-324);
* curve equation and subgroup membership (`from_uncompressed`): always for the VerifyingKey
  (lib.rs:158-183 has no unchecked mode), for the five vectors when `checked=True`
  (lib.rs:294-298,328-332).  This is curve arithmetic, so it runs on the device
  (`bb_points_validate`): pass the `Worker` to use, or one is created on device 0 -- without a CUDA
  device the call fails, there is no CPU fallback.  Zero coordinates without the infinity flag are
  the point (0, 0), off the curve, and fail this check; unchecked, they load as the all-zero
  identity (DESIGN.md section 7).

`read_parameters_device` / `read_verifying_key_device` read the same files on the device
(`bb_params_read` / `bb_vk_read`): the bytes are decoded and checked there, straight into a
resident `Parameters` (and `PreparedVerifyingKey`), with no host arrays.  They follow
Parameters::read / VerifyingKey::read exactly, point by point: the first failing point in file
order decides, and a short file is EOF only when every complete point before its end is valid.
"""
import ctypes as C
import struct

import numpy as np

from . import _addr, _check, _ERRORS, load_library


def _coords_to_abi(raw, ncoord, g2):
    """raw: (n, ncoord*48) uint8 big-endian canonical coordinates -> (n, ncoord*6) uint64 Montgomery"""
    n = raw.shape[0]
    be = raw.reshape(n, ncoord, 48).copy()
    be[:, 0, 0] &= 0x1F                                   # strip the flag bits of byte 0
    le = np.ascontiguousarray(be[:, :, ::-1])             # little-endian bytes per coordinate
    if g2:                                                # file: x.c1 x.c0 y.c1 y.c0 -> ABI: x.c0 x.c1 y.c0 y.c1
        le = np.ascontiguousarray(le[:, [1, 0, 3, 2], :])
    limbs = le.reshape(n, ncoord * 48).view(np.uint64).reshape(n, ncoord * 6).copy()
    _check(load_library().bb_fp_convert(limbs.ctypes.data_as(C.c_void_p), C.c_size_t(n * ncoord), C.c_int(1)))
    return limbs


def _abi_to_coords(limbs, ncoord, g2):
    arr = np.ascontiguousarray(limbs, dtype=np.uint64).reshape(-1, ncoord * 6).copy()
    n = arr.shape[0]
    ident = ~arr.any(axis=1)
    _check(load_library().bb_fp_convert(arr.ctypes.data_as(C.c_void_p), C.c_size_t(n * ncoord), C.c_int(0)))
    le = arr.view(np.uint8).reshape(n, ncoord, 48)
    if g2:
        le = le[:, [1, 0, 3, 2], :]
    be = np.ascontiguousarray(le[:, :, ::-1]).reshape(n, ncoord * 48).copy()
    be[ident] = 0
    be[ident, 0] = 0x40
    return be


class InvalidData(ValueError):
    """io::ErrorKind::InvalidData of Parameters::read / VerifyingKey::read.  From the device reader: `section` (its name,
    e.g. "h"), `index` within it and `why` (BB_READ_* code: 1 flags, 2 coordinate >= p, 3 off the curve, 4 outside the
    subgroup, 5 identity)."""

    def __init__(self, message, section=None, index=None, why=None):
        super().__init__(message)
        self.section, self.index, self.why = section, index, why


BB_ERR_IO_INVALID_DATA = 8
_ERRORS[BB_ERR_IO_INVALID_DATA] = InvalidData


def _read_points(buf, off, count, g2, what, allow_infinity, validate):
    """validate: None, or a callable (group_is_g2, points, what) applying the curve checks"""
    size = 192 if g2 else 96
    name = "G2" if g2 else "G1"
    end = off + count * size
    if end > len(buf):
        raise EOFError(f"{what}: file ends inside the vector")
    raw = np.frombuffer(buf, dtype=np.uint8, count=count * size, offset=off).reshape(count, size)
    inf = np.zeros(count, bool)
    if count:
        flags = raw[:, 0]
        if (flags & 0x80).any():
            raise InvalidData(f"invalid {name}: {what} holds a compressed encoding")
        if (flags & 0x20).any():
            raise InvalidData(f"invalid {name}: {what} has the sort flag set on an uncompressed point")
        inf = (flags & 0x40) != 0
        if inf.any():
            rest = raw[inf].copy()
            rest[:, 0] &= 0x3F & ~0x40
            if rest.any():
                raise InvalidData(f"invalid {name}: {what} has an infinity flag with non-zero coordinates")
            if not allow_infinity:
                raise InvalidData(f"point at infinity in {what}")                 # lib.rs:199-207,303-315
    try:
        out = _coords_to_abi(raw, 4 if g2 else 2, g2)                              # rejects coordinates >= p
    except Exception as e:
        raise InvalidData(f"invalid {name}: {what}: {e}") from None
    if count:
        out[inf] = 0
    if validate is not None and count:
        # zeros without the infinity flag are the point (0, 0), which is not on the curve; the ABI's all-zero identity
        # cannot stand for it, so it is rejected here, after the points before it are checked
        zero = np.flatnonzero(~out.any(axis=1) & ~inf)
        if zero.size:
            validate(g2, out[:zero[0]], what)
            raise InvalidData(f"invalid {name}: {what}[{int(zero[0])}] is not on the curve")
        validate(g2, out, what)
    return out, end


def _read_u32(buf, off):
    if off + 4 > len(buf):
        raise EOFError("file ends inside a length prefix")
    return struct.unpack_from(">I", buf, off)[0], off + 4


class _Validator:
    """curve + subgroup checks on the device, with a Worker made on demand"""

    def __init__(self, worker):
        self.worker, self.own = worker, None

    def __call__(self, g2, points, what):
        if self.worker is None:
            from . import Worker
            self.own = self.worker = Worker(0)
        first, why = C.c_size_t(), C.c_int()
        pts = np.ascontiguousarray(points, dtype=np.uint64)
        _check(load_library().bb_points_validate(self.worker._h, C.c_int(2 if g2 else 1), pts.ctypes.data_as(C.c_void_p),
                                                 C.c_size_t(pts.shape[0]), C.c_int(1), C.byref(first), C.byref(why)))
        if why.value:
            reason = "not on the curve" if why.value == 1 else "not in the prime-order subgroup"
            raise InvalidData(f"invalid {'G2' if g2 else 'G1'}: {what}[{first.value}] is {reason}")

    def close(self):
        if self.own is not None:
            self.own.close()


def read_verifying_key(buf, off=0, worker=None, _validator=None):
    """VerifyingKey::read (lib.rs:158-218): always curve- and subgroup-checked."""
    val = _validator or _Validator(worker)
    try:
        vk = {}
        g1 = lambda o, w: _read_points(buf, o, 1, False, w, True, val)
        g2 = lambda o, w: _read_points(buf, o, 1, True, w, True, val)
        vk["alpha_g1"], off = g1(off, "alpha_g1")
        vk["beta_g1"], off = g1(off, "beta_g1")
        vk["beta_g2"], off = g2(off, "beta_g2")
        vk["gamma_g2"], off = g2(off, "gamma_g2")
        vk["delta_g1"], off = g1(off, "delta_g1")
        vk["delta_g2"], off = g2(off, "delta_g2")
        n, off = _read_u32(buf, off)
        vk["ic"], off = _read_points(buf, off, n, False, "ic", False, val)
    finally:
        if _validator is None:
            val.close()
    return vk, off


def read_parameters(data, checked=True, worker=None):
    """bytes of Parameters::write -> dict for bellman_b200.Parameters (+ 'gamma_g2', 'ic');
    Parameters::read(reader, checked), lib.rs:289-398."""
    buf = memoryview(data)
    val = _Validator(worker)
    try:
        vk, off = read_verifying_key(buf, 0, _validator=val)
        p = dict(vk_g1=np.concatenate([vk["alpha_g1"], vk["beta_g1"], vk["delta_g1"]]),
                 vk_g2=np.concatenate([vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"]]), ic=vk["ic"])
        for name, is_g2 in (("h", False), ("l", False), ("a", False), ("b_g1", False), ("b_g2", True)):
            n, off = _read_u32(buf, off)
            p[name], off = _read_points(buf, off, n, is_g2, name, False, val if checked else None)
    finally:
        val.close()
    return p


SECTIONS = ("alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "delta_g1", "delta_g2", "ic", "h", "l", "a", "b_g1", "b_g2")


class ParamsReport(C.Structure):
    """bb_params_report"""
    _fields_ = [("len", C.c_size_t * 6), ("consumed", C.c_size_t), ("section", C.c_int), ("index", C.c_size_t), ("why", C.c_int)]


def _device_read(worker, data, checked, want_crs, want_vk):
    """bb_params_read (want_crs) or bb_vk_read of `data` -> (crs handle, vk handle, report); raises InvalidData / EOFError"""
    lib = load_library()
    keep = None
    if isinstance(data, tuple):                                   # (device pointer, length): bytes in HBM
        ptr, n, on_device = _addr(data[0]), int(data[1]), 1
    else:
        keep = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8).reshape(-1)
        ptr, n, on_device = (keep.ctypes.data if keep.size else None), keep.size, 0
    rep = ParamsReport()
    crs, vk = C.c_void_p(), C.c_void_p()
    if want_crs:
        rc = lib.bb_params_read(worker._h, C.c_void_p(ptr), C.c_size_t(n), C.c_int(on_device), C.c_int(1 if checked else 0), C.byref(crs),
                                C.byref(vk) if want_vk else None, C.byref(rep))
    else:
        rc = lib.bb_vk_read(worker._h, C.c_void_p(ptr), C.c_size_t(n), C.c_int(on_device), C.byref(vk), C.byref(rep))
    if rc == BB_ERR_IO_INVALID_DATA:
        raise InvalidData(lib.bb_last_error().decode(errors="replace"), section=SECTIONS[rep.section], index=int(rep.index), why=int(rep.why))
    if rc == 3:                                                   # BB_ERR_IO_UNEXPECTED_EOF
        raise EOFError(lib.bb_last_error().decode(errors="replace"))
    _check(rc)
    return crs, vk, rep


def read_parameters_device(worker, data, checked=True, verifying_key=False):
    """Parameters::read(reader, checked) on the device (bb_params_read) -> a resident Parameters, or with
    verifying_key=True (Parameters, PreparedVerifyingKey).  data: bytes, bytearray, memoryview or a uint8 array (host,
    pageable or pinned), or (device_ptr, length) for bytes in HBM.  Bytes after the key are not read.  Raises InvalidData
    (with .section, .index, .why) or EOFError as read_parameters does, in the reference's precedence."""
    from . import Parameters
    from .verifier import PreparedVerifyingKey
    crs, vk, rep = _device_read(worker, data, checked, True, verifying_key)
    lens = dict(zip(("ic", "h", "l", "a", "b_g1", "b_g2"), (int(v) for v in rep.len)))
    params = Parameters._from_handle(worker, crs, lens)
    if not verifying_key:
        return params
    return params, PreparedVerifyingKey._from_handle(worker, vk, lens["ic"])


def read_verifying_key_device(worker, data):
    """VerifyingKey::read + prepare_verifying_key on the device (bb_vk_read) -> (PreparedVerifyingKey, bytes consumed).
    data as for read_parameters_device; a Parameters file starts with its VerifyingKey."""
    from .verifier import PreparedVerifyingKey
    _, vk, rep = _device_read(worker, data, True, False, True)
    return PreparedVerifyingKey._from_handle(worker, vk, int(rep.len[0])), int(rep.consumed)


def download_parameters(params):
    """diagnostic (bb_diag_crs_download): the points a resident Parameters holds, as the dict read_parameters returns
    (without gamma_g2 and ic, which bb_crs does not keep): vk_g1 (alpha, beta, delta), vk_g2 (beta, delta), h, l, a,
    b_g1, b_g2"""
    lib = load_library()
    out = {}
    for which, (name, width) in enumerate((("h", 12), ("l", 12), ("a", 12), ("b_g1", 12), ("b_g2", 24))):
        arr = np.zeros((max(params.lens[name], 1), width), np.uint64)
        _check(lib.bb_diag_crs_download(params._h, C.c_int(which), arr.ctypes.data_as(C.c_void_p)))
        out[name] = arr[:params.lens[name]]
    vk = np.zeros(3 * 12 + 2 * 24, np.uint64)
    _check(lib.bb_diag_crs_download(params._h, C.c_int(5), vk.ctypes.data_as(C.c_void_p)))
    out["vk_g1"], out["vk_g2"] = vk[:36].reshape(3, 12), vk[36:].reshape(2, 24)
    return out


def write_parameters(p):
    """inverse of read_parameters (Parameters::write, lib.rs:258-287)"""
    vk1 = np.asarray(p["vk_g1"], dtype=np.uint64).reshape(3, 12)
    vk2 = np.asarray(p["vk_g2"], dtype=np.uint64).reshape(3, 24)
    out = bytearray()
    out += _abi_to_coords(vk1[0:1], 2, False).tobytes()       # alpha_g1
    out += _abi_to_coords(vk1[1:2], 2, False).tobytes()       # beta_g1
    out += _abi_to_coords(vk2[0:1], 4, True).tobytes()        # beta_g2
    out += _abi_to_coords(vk2[1:2], 4, True).tobytes()        # gamma_g2
    out += _abi_to_coords(vk1[2:3], 2, False).tobytes()       # delta_g1
    out += _abi_to_coords(vk2[2:3], 4, True).tobytes()        # delta_g2
    for name, g2 in (("ic", False), ("h", False), ("l", False), ("a", False), ("b_g1", False), ("b_g2", True)):
        arr = np.asarray(p[name], dtype=np.uint64).reshape(-1, 24 if g2 else 12)
        out += struct.pack(">I", arr.shape[0])
        out += _abi_to_coords(arr, 4 if g2 else 2, g2).tobytes()
    return bytes(out)


def write_parameters_device(params, pvk, verifying_key_only=False, out=None):
    """Parameters::write (or with verifying_key_only=True VerifyingKey::write) of a resident key, encoded on the device
    (bb_params_write): byte for byte write_parameters of the same points.  params: a single-GPU Parameters; pvk: its
    PreparedVerifyingKey (it holds gamma_g2 and ic).  Returns the bytes; or with out = (device_ptr, capacity) writes them
    there and returns their length.  A sharded key, a verifying key of another key or too small a buffer raise
    BackendError."""
    lib = load_library()
    n = C.c_size_t()
    _check(lib.bb_params_write(params.worker._h, params._h, pvk._h, C.c_int(1 if verifying_key_only else 0), None, C.c_size_t(0),
                               C.c_int(0), C.byref(n)))
    if out is not None:
        _check(lib.bb_params_write(params.worker._h, params._h, pvk._h, C.c_int(1 if verifying_key_only else 0), C.c_void_p(_addr(out[0])),
                                   C.c_size_t(int(out[1])), C.c_int(1), C.byref(n)))
        return int(n.value)
    buf = np.empty(n.value, np.uint8)
    _check(lib.bb_params_write(params.worker._h, params._h, pvk._h, C.c_int(1 if verifying_key_only else 0), buf.ctypes.data_as(C.c_void_p),
                               C.c_size_t(buf.size), C.c_int(0), C.byref(n)))
    return buf.tobytes()
