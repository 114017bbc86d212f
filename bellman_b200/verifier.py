"""Groth16 verification on the device: the host-side mirror of bellman's groth16 verifier
(groth16/src/verifier.rs, groth16/src/verifier/batch.rs) over bb_vk_prepare / bb_groth16_verify /
bb_groth16_verify_batch.

    pvk = prepare_verifying_key(worker, vk)            # vk: the dict params_io.read_verifying_key returns
    verify_proof(pvk, (a, b, c), inputs)               # raises InvalidProof / InvalidVerifyingKey
    bv = BatchVerifier(); bv.queue(((a, b, c), inputs)); bv.verify(rng, pvk)
    bv.verify_each(pvk)                                # verify_single per item, one device call: [None | exception, ...]

Proofs are ABI-format affine point arrays (A, C: 12 u64, B: 24 u64); public inputs are Fr, either
Python integers or an (L, 4) uint64 array in Montgomery form.

Proofs as bytes (Proof::read / Proof::write, groth16/src/lib.rs:39-99, over bb_proofs_read / bb_proofs_write):

    a, b, c, status = read_proofs(worker, data, stride=384)     # status: one byte per proof, 0 = valid
    proof = read_proof(worker, b192)                           # raises InvalidProofEncoding like Proof::read
    bv.queue_bytes((b192, inputs)); bv.verify(rng, pvk)        # decoded on the device at verify() time
"""
import contextlib
import ctypes as C

import numpy as np

from . import BackendError, EvaluationDomain, _addr, _c64, _check, _DeviceObject, _ERRORS, _ptr, load_library


class VerificationError(Exception):
    """groth16::VerificationError (src/lib.rs:353-358)"""


class InvalidVerifyingKey(VerificationError):
    """inputs.len() + 1 != ic.len() (verifier.rs:28-30, batch.rs:105-111)"""


class InvalidProof(VerificationError):
    """the pairing equation does not hold"""


_ERRORS.update({6: InvalidVerifyingKey, 7: InvalidProof})

R_MODULUS = EvaluationDomain.FR_MODULUS
GT_WORDS = 72                                   # 12 Fp coordinates of 6 u64


class _VkDesc(C.Structure):
    _fields_ = [("alpha_g1", C.c_void_p), ("beta_g2", C.c_void_p), ("gamma_g2", C.c_void_p), ("delta_g2", C.c_void_p),
                ("ic", C.c_void_p), ("ic_len", C.c_size_t)]


class _ProofBatch(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("c", C.c_void_p), ("n", C.c_size_t),
                ("inputs", C.c_void_p), ("n_inputs", C.c_size_t), ("on_device", C.c_int)]


class PreparedVerifyingKey(_DeviceObject):
    """groth16::PreparedVerifyingKey (groth16/src/lib.rs:400-409): the key resident on the device."""

    _destroy = "bb_vk_destroy"

    def __init__(self, worker, vk):
        self.worker = worker
        g1 = lambda v: _c64(v, 12)
        g2 = lambda v: _c64(v, 24)
        keep = [g1(vk["alpha_g1"]), g2(vk["beta_g2"]), g2(vk["gamma_g2"]), g2(vk["delta_g2"]), g1(vk["ic"])]
        d = _VkDesc()
        d.alpha_g1, d.beta_g2, d.gamma_g2, d.delta_g2, d.ic = (a.ctypes.data for a in keep)
        d.ic_len = keep[4].shape[0]
        self.ic_len = int(d.ic_len)
        h = C.c_void_p()
        _check(load_library().bb_vk_prepare(worker._h, C.byref(d), C.byref(h)))
        self._own(worker, h)


    @classmethod
    def _from_handle(cls, worker, h, ic_len):
        """a bb_vk built by the library itself (params_io.read_parameters_device / read_verifying_key_device)"""
        self = cls.__new__(cls)
        self.worker, self.ic_len = worker, int(ic_len)
        self._own(worker, h)
        return self


def prepare_verifying_key(worker, vk):
    """verifier.rs:11-21"""
    return PreparedVerifyingKey(worker, vk)


def fr_inputs(inputs):
    """public inputs -> (L, 4) uint64 Montgomery array (Python integers are reduced mod r)"""
    if isinstance(inputs, np.ndarray):
        return _c64(inputs, 4)
    vals = list(inputs)
    if not vals:
        return np.zeros((0, 4), np.uint64)
    return np.stack([EvaluationDomain._to_mont(int(v)) for v in vals])


def _z_bytes(z):
    """list of Python integers -> n x 32 canonical little-endian bytes"""
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in z), np.uint8).copy() if len(z) else np.zeros(32, np.uint8)


def verify_proof(pvk, proof, inputs):
    """verifier.rs:23-58.  Returns None; raises InvalidProof or InvalidVerifyingKey."""
    a, b, c = (_c64(proof[0], 12), _c64(proof[1], 24), _c64(proof[2], 12))
    x = fr_inputs(inputs)
    _check(load_library().bb_groth16_verify(pvk.worker._h, pvk._h, _ptr(a), _ptr(b), _ptr(c), _ptr(x), C.c_size_t(x.shape[0])))


def verify_batch_arrays(pvk, a, b, c, inputs, z=None, on_device=False, n=None, n_inputs=None, gt=False):
    """bb_groth16_verify_batch over whole arrays: a (n,12), b (n,24), c (n,12), inputs (n, L, 4) or (n*L, 4) Montgomery; or,
    with on_device=True, device addresses and explicit n / n_inputs.  z: None (OS randomness) or n Python integers.
    gt=True also returns the G_T value the verdict was taken from ((72,) uint64: 12 canonical Fp, tower order);
    then the verdict is returned as a bool instead of raising InvalidProof."""
    lib = load_library()
    keep = []
    bt, n = _proof_batch(a, b, c, inputs, on_device, n, n_inputs, keep)
    zb = None
    if z is not None:
        assert len(z) == n
        zb = _z_bytes(z)
    if not gt:
        _check(lib.bb_groth16_verify_batch(pvk.worker._h, pvk._h, C.byref(bt), _ptr(zb)))
        return None
    out = np.zeros(GT_WORDS, np.uint64)
    rc = lib.bb_diag_verify_batch_gt(pvk.worker._h, pvk._h, C.byref(bt), _ptr(zb), _ptr(out))
    if rc == 7:
        return False, out
    _check(rc)
    return True, out


def _proof_batch(a, b, c, inputs, on_device, n, n_inputs, keep):
    """the bb_proof_batch of verify_batch_arrays' arguments, and n; host arrays are appended to keep"""
    bt = _ProofBatch()
    if on_device:
        bt.a, bt.b, bt.c, bt.inputs = (_addr(p) for p in (a, b, c, inputs))
        bt.n, bt.n_inputs, bt.on_device = n, n_inputs, 1
        return bt, n
    a, b, c = _c64(a, 12), _c64(b, 24), _c64(c, 12)
    n = a.shape[0]
    x = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(n, -1, 4) if n else np.zeros((0, 0, 4), np.uint64)
    L = x.shape[1] if n_inputs is None else n_inputs
    keep += [a, b, c, x]
    bt.a, bt.b, bt.c, bt.inputs = (arr.ctypes.data for arr in (a, b, c, x))
    bt.n, bt.n_inputs, bt.on_device = n, L, 0
    return bt, n


def verify_each_arrays(pvk, a, b, c, inputs, on_device=False, n=None, n_inputs=None, gt=False):
    """bb_groth16_verify_each: verify_proof for every proof of the arrays (arguments as for verify_batch_arrays, without z).
    Returns the (n,) uint8 verdicts, 0 = valid, 1 = the equation fails; raises InvalidVerifyingKey for a wrong input count.
    gt=True also returns the n + 1 G_T values ((n + 1, 72) uint64: every proof's final-exponentiated three-pair product,
    then the key's e(alpha, beta)^k, k = gt_exponent())."""
    lib = load_library()
    keep = []
    bt, n = _proof_batch(a, b, c, inputs, on_device, n, n_inputs, keep)
    verdicts = np.zeros(max(n, 1), np.uint8)
    n_invalid = C.c_size_t()
    _check(lib.bb_groth16_verify_each(pvk.worker._h, pvk._h, C.byref(bt), _ptr(verdicts), C.byref(n_invalid)))
    if n_invalid.value != int(np.count_nonzero(verdicts[:n])):
        raise BackendError(f"bb_groth16_verify_each: n_invalid = {n_invalid.value} for {int(np.count_nonzero(verdicts[:n]))} invalid verdicts")
    if not gt:
        return verdicts[:n]
    out = np.zeros((n + 1, GT_WORDS), np.uint64)
    _check(lib.bb_diag_verify_each_gt(pvk.worker._h, pvk._h, C.byref(bt), _ptr(out)))
    return verdicts[:n], out


class InvalidProofEncoding(ValueError):
    """Proof::read failed (groth16/src/lib.rs:47-99): bellman's io::Error of kind InvalidData.  The message starts with
    bellman's text ("invalid G1", "invalid G2" or "point at infinity"); `status` is the byte of bb_proofs_read and
    `index` the proof's position (in the queue, for BatchVerifier.queue_bytes)."""

    def __init__(self, message, status=None, index=None):
        super().__init__(message)
        self.status, self.index = status, index


# the status byte of bb_proofs_read: (which << 4) | why
READ_OK, READ_BAD_FLAGS, READ_NON_CANONICAL, READ_NOT_ON_CURVE, READ_NOT_IN_SUBGROUP, READ_IDENTITY = range(6)
PROOF_BYTES = 192


def read_error_message(status):
    """bellman's io::Error text for a non-zero status byte"""
    if status & 15 == READ_IDENTITY:
        return "point at infinity"
    return "invalid G2" if status >> 4 == 2 else "invalid G1"


class _ProofBytes(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("n", C.c_size_t), ("stride", C.c_size_t), ("on_device", C.c_int)]


def read_proofs(worker, data, n=None, stride=PROOF_BYTES, on_device=False, out_device=None):
    """Proof::read over a batch on the device (bb_proofs_read).  Proof i is the 192 bytes at data[i * stride:].
    data: bytes-like or a uint8 array (host), or with on_device=True a device address (then n is required).
    n: number of proofs (default: every whole record of data).  out_device: None, or three device addresses (n x 96 B,
    n x 192 B, n x 96 B) that receive A, B, C.  Returns (a, b, c, status): the points as (n, 12) / (n, 24) / (n, 12)
    uint64 arrays (ABI format) or the three device addresses, and the (n,) uint8 status bytes."""
    lib = load_library()
    pb = _ProofBytes()
    keep = None
    if on_device:
        if n is None:
            raise ValueError("read_proofs: n is required for bytes in device memory")
        pb.bytes = _addr(data)
    else:
        keep = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, np.uint8).reshape(-1)
        whole = 0 if keep.size < PROOF_BYTES or stride < PROOF_BYTES else 1 + (keep.size - PROOF_BYTES) // stride
        n = whole if n is None else n
        if n > whole:
            raise ValueError(f"read_proofs: {keep.size} bytes hold {whole} proofs at stride {stride}, not {n}")
        pb.bytes = keep.ctypes.data if keep.size else None
    pb.n, pb.stride, pb.on_device = n, stride, 1 if on_device else 0
    status = np.zeros(max(n, 1), np.uint8)
    n_invalid = C.c_size_t()
    if out_device is not None:
        da, db, dc = (C.c_void_p(_addr(p)) for p in out_device)
        _check(lib.bb_proofs_read(worker._h, C.byref(pb), da, db, dc, C.c_int(1), _ptr(status), C.byref(n_invalid)))
        return out_device[0], out_device[1], out_device[2], status[:n]
    a, b, c = np.zeros((n, 12), np.uint64), np.zeros((n, 24), np.uint64), np.zeros((n, 12), np.uint64)
    _check(lib.bb_proofs_read(worker._h, C.byref(pb), _ptr(a), _ptr(b), _ptr(c), C.c_int(0), _ptr(status), C.byref(n_invalid)))
    return a, b, c, status[:n]


def read_proof(worker, b192):
    """Proof::read of one proof: the ABI triple (a, b, c), or InvalidProofEncoding with bellman's message"""
    if len(b192) != PROOF_BYTES:
        raise ValueError("a proof is 192 bytes")
    a, b, c, status = read_proofs(worker, bytes(b192), n=1)
    if status[0]:
        raise InvalidProofEncoding(read_error_message(int(status[0])), status=int(status[0]), index=0)
    return a[0], b[0], c[0]


def write_proofs(worker, a, b, c):
    """Proof::write over a batch on the device (bb_proofs_write): ABI point arrays -> n x 192 bytes"""
    a, b, c = _c64(a, 12), _c64(b, 24), _c64(c, 12)
    n = a.shape[0]
    assert b.shape[0] == n and c.shape[0] == n
    out = np.zeros(max(n, 1) * PROOF_BYTES, np.uint8)
    _check(load_library().bb_proofs_write(worker._h, _ptr(a), _ptr(b), _ptr(c), C.c_size_t(n), C.c_int(0), _ptr(out)))
    return bytes(out[:n * PROOF_BYTES])


def write_proofs_device(worker, d_a, d_b, d_c, n, d_out):
    """bb_proofs_write with everything in HBM: n proofs of the device arrays d_a, d_b, d_c -> d_out (n x 192 B)"""
    ptrs = (C.c_void_p(_addr(p)) for p in (d_a, d_b, d_c))
    _check(load_library().bb_proofs_write(worker._h, *ptrs, C.c_size_t(n), C.c_int(1), C.c_void_p(_addr(d_out))))


def points_decompress(worker, group, data, check_subgroup=True):
    """diagnostic (bb_diag_points_decompress): from_compressed, or from_compressed_unchecked with check_subgroup=False,
    of packed 48-byte (G1) or 96-byte (G2) encodings -> ((n, 12 | 24) uint64 points, (n,) uint8 codes)"""
    enc, width = (48, 12) if group == 1 else (96, 24)
    buf = np.frombuffer(bytes(data), np.uint8)
    n = buf.size // enc
    out = np.zeros((n, width), np.uint64)
    why = np.zeros(max(n, 1), np.uint8)
    _check(load_library().bb_diag_points_decompress(worker._h, C.c_int(group), _ptr(buf) if n else None, C.c_size_t(n),
                                                    C.c_int(1 if check_subgroup else 0), _ptr(out), _ptr(why)))
    return out, why[:n]


class BatchVerifier:
    """groth16::batch::Verifier (batch.rs:72-173)."""

    def __init__(self):
        self.items = []

    def queue(self, item):
        """batch.rs:89-98: item = (proof, inputs), proof = (a, b, c)"""
        proof, inputs = item
        self.items.append(((_c64(proof[0], 12), _c64(proof[1], 24), _c64(proof[2], 12)), fr_inputs(inputs)))

    def queue_bytes(self, proof_bytes, inputs):
        """queue a proof in its 192-byte Proof::write encoding.  It is read on the device at verify() time, together with
        every other proof queued this way (one bb_proofs_read), and its points stay there for the verification."""
        if len(proof_bytes) != PROOF_BYTES:
            raise ValueError("a proof is 192 bytes")
        self.items.append((bytes(proof_bytes), fr_inputs(inputs)))

    def verify(self, rng, pvk):
        """batch.rs:100-173 against a PreparedVerifyingKey.  rng: None = z from the operating system (getrandom); any
        object with randrange gives reproducible z.  Returns None; raises InvalidProof or InvalidVerifyingKey, and
        InvalidProofEncoding (naming the queue index) for a proof of queue_bytes that does not read -- before any pairing
        work, as bellman's Proof::read fails before its proof could be queued."""
        n = len(self.items)
        if any(isinstance(p, bytes) for p, _ in self.items):
            return self._verify_from_bytes(rng, pvk)
        if n and any(x.shape[0] + 1 != pvk.ic_len for _, x in self.items):
            raise InvalidVerifyingKey(f"[bb_status 6] InvalidVerifyingKey: a key with {pvk.ic_len} ic entries")
        L = pvk.ic_len - 1
        z = None if rng is None else [rng.randrange(1, R_MODULUS) for _ in range(n)]
        verify_batch_arrays(pvk, *self._points(range(n)), self._inputs(range(n), L), z, n_inputs=max(L, 0))

    def _verify_from_bytes(self, rng, pvk):
        """the batch in device buffers (see _staged); the verdict of a batch does not depend on the order of its items"""
        n, L = len(self.items), pvk.ic_len - 1
        enc, dec = self._split()
        with self._staged(pvk.worker, enc, dec, self._inputs(enc + dec, L)) as (d, status):
            bad = np.flatnonzero(status)
            if bad.size:
                k = int(bad[0])
                raise InvalidProofEncoding(f"{read_error_message(int(status[k]))} (queued proof {enc[k]})", status=int(status[k]), index=enc[k])
            if any(x.shape[0] + 1 != pvk.ic_len for _, x in self.items):
                raise InvalidVerifyingKey(f"[bb_status 6] InvalidVerifyingKey: a key with {pvk.ic_len} ic entries")
            z = None if rng is None else [rng.randrange(1, R_MODULUS) for _ in range(n)]
            verify_batch_arrays(pvk, *d, z, on_device=True, n=n, n_inputs=L)

    def _split(self):
        """the queue indices of the queue_bytes items and of the queue() items"""
        enc = [i for i, (p, _) in enumerate(self.items) if isinstance(p, bytes)]
        return enc, [i for i, (p, _) in enumerate(self.items) if not isinstance(p, bytes)]

    def _points(self, order):
        """the a (k, 12), b (k, 24), c (k, 12) arrays of the queue() items at the queue indices `order`"""
        return [np.stack([self.items[i][0][k].reshape(w) for i in order]) if len(order) else np.zeros((0, w), np.uint64)
                for k, w in ((0, 12), (1, 24), (2, 12))]

    def _inputs(self, order, L):
        """the (k, L, 4) public inputs of the items at the queue indices `order`; zero rows for items of another length"""
        x = np.zeros((len(order), max(L, 0), 4), np.uint64)
        for k, i in enumerate(order):
            if self.items[i][1].shape[0] == L:
                x[k] = self.items[i][1].reshape(L, 4)
        return x

    @contextlib.contextmanager
    def _staged(self, worker, enc, dec, x):
        """the queue in device buffers a, b, c, x, freed on exit: the queue_bytes items `enc` decoded in place by one
        read_proofs, the queue() items `dec` uploaded behind them, and the inputs x (rows in the order enc + dec).
        Yields the four buffers and the status bytes of the enc items."""
        n, nb = len(enc) + len(dec), len(enc)
        d = [worker.device_alloc(n * 96), worker.device_alloc(n * 192), worker.device_alloc(n * 96), worker.device_alloc(max(1, x.size // 4) * 32)]
        try:
            _, _, _, status = read_proofs(worker, b"".join(self.items[i][0] for i in enc), n=nb, out_device=d[:3])
            if dec:
                for buf, rows in zip(d, self._points(dec)):
                    worker.upload(C.c_void_p(_addr(buf) + nb * rows.shape[1] * 8), rows)
            if x.size:
                worker.upload(d[3], x)
            yield d, status
        finally:
            for p in d:
                worker.device_free(p)

    def verify_each(self, pvk):
        """Item::verify_single (batch.rs:57-65) for every queued item, in one device call (bb_groth16_verify_each): the
        fallback that finds the bad proofs of a rejected batch.  Returns one entry per item, in queue order: None, or the
        exception verify_single would raise for it -- InvalidProof; InvalidVerifyingKey for an item with the wrong number
        of inputs (the other items are still verified); InvalidProofEncoding (with its queue index) for a queue_bytes item
        that does not read.  The queue_bytes items are decoded in one bb_proofs_read into device buffers and verified
        there.  Only back-end failures raise."""
        n, L = len(self.items), pvk.ic_len - 1
        out = [None] * n
        for i, (_, x) in enumerate(self.items):
            if x.shape[0] != L:
                out[i] = InvalidVerifyingKey(f"[bb_status 6] InvalidVerifyingKey: {x.shape[0]} public inputs for a key with "
                                             f"{pvk.ic_len} ic entries (queued item {i})")
        if n == 0 or L < 0:
            return out
        enc, dec = self._split()
        order = enc + dec                                       # device row k holds queue item order[k]
        x = self._inputs(order, L)                              # zero rows for the items of a wrong input count
        if not enc:
            verdicts = verify_each_arrays(pvk, *self._points(order), x, n_inputs=L)
        else:
            with self._staged(pvk.worker, enc, dec, x) as (d, status):
                for k, i in enumerate(enc):                     # Proof::read fails before the item could be queued
                    if status[k]:
                        out[i] = InvalidProofEncoding(f"{read_error_message(int(status[k]))} (queued proof {i})", status=int(status[k]), index=i)
                verdicts = verify_each_arrays(pvk, *d, on_device=True, n=n, n_inputs=L)
        for k, i in enumerate(order):
            if out[i] is None and verdicts[k]:
                out[i] = InvalidProof(f"[bb_status 7] InvalidProof: queued item {i} does not verify")
        return out


def multi_pairing(worker, g1, g2):
    """diagnostic: prod e(P_i, Q_i)^k after the final exponentiation (k = gt_exponent()); (72,) uint64 of 12 canonical Fp"""
    p, q = _c64(g1, 12), _c64(g2, 24)
    out = np.zeros(GT_WORDS, np.uint64)
    _check(load_library().bb_diag_multi_pairing(worker._h, C.c_size_t(p.shape[0]), _ptr(p), _ptr(q), _ptr(out)))
    return out


def gt_exponent():
    return int(load_library().bb_diag_gt_exponent())


def synth_proof_batch(worker, seed, n, n_inputs, d_a, d_b, d_c, d_inputs):
    """bench / test generator: a synthetic verifying key (returned as a read_verifying_key-style dict) and n valid proofs
    written to the device buffers d_a (n*96 B), d_b (n*192 B), d_c (n*96 B), d_inputs (n*n_inputs*32 B, Montgomery)."""
    vk = {"alpha_g1": np.zeros(12, np.uint64), "beta_g2": np.zeros(24, np.uint64), "gamma_g2": np.zeros(24, np.uint64),
          "delta_g2": np.zeros(24, np.uint64), "ic": np.zeros((n_inputs + 1, 12), np.uint64)}
    _check(load_library().bb_synth_proof_batch(worker._h, C.c_uint64(seed), C.c_size_t(n), C.c_size_t(n_inputs),
                                               _ptr(vk["alpha_g1"]), _ptr(vk["beta_g2"]), _ptr(vk["gamma_g2"]), _ptr(vk["delta_g2"]),
                                               _ptr(vk["ic"]), d_a, d_b, d_c, d_inputs))
    return vk
