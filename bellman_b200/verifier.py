"""Groth16 verification on the device: the host-side mirror of bellman's groth16 verifier
(groth16/src/verifier.rs, groth16/src/verifier/batch.rs) over bb_vk_prepare / bb_groth16_verify /
bb_groth16_verify_batch.

    pvk = prepare_verifying_key(worker, vk)            # vk: the dict params_io.read_verifying_key returns
    verify_proof(pvk, (a, b, c), inputs)               # raises InvalidProof / InvalidVerifyingKey
    bv = BatchVerifier(); bv.queue(((a, b, c), inputs)); bv.verify(rng, pvk)

Proofs are ABI-format affine point arrays (A, C: 12 u64, B: 24 u64); public inputs are Fr, either
Python integers or an (L, 4) uint64 array in Montgomery form.
"""
import ctypes as C

import numpy as np

from . import EvaluationDomain, _c64, _check, _ERRORS, _ptr, load_library


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


class PreparedVerifyingKey:
    """groth16::PreparedVerifyingKey (groth16/src/lib.rs:400-409): the key resident on the device."""

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
        self._h = h
        worker._children.add(self)

    def free(self):
        if getattr(self, "_h", None):
            if getattr(self.worker, "_h", None):
                load_library().bb_vk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


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
    bt = _ProofBatch()
    keep = []
    if on_device:
        bt.a, bt.b, bt.c, bt.inputs = (p.value if isinstance(p, C.c_void_p) else p for p in (a, b, c, inputs))
        bt.n, bt.n_inputs, bt.on_device = n, n_inputs, 1
    else:
        a, b, c = _c64(a, 12), _c64(b, 24), _c64(c, 12)
        n = a.shape[0]
        x = np.ascontiguousarray(inputs, dtype=np.uint64).reshape(n, -1, 4) if n else np.zeros((0, 0, 4), np.uint64)
        L = x.shape[1] if n_inputs is None else n_inputs
        keep += [a, b, c, x]
        bt.a, bt.b, bt.c, bt.inputs = (arr.ctypes.data for arr in (a, b, c, x))
        bt.n, bt.n_inputs, bt.on_device = n, L, 0
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


class BatchVerifier:
    """groth16::batch::Verifier (batch.rs:72-173)."""

    def __init__(self):
        self.items = []

    def queue(self, item):
        """batch.rs:89-98: item = (proof, inputs), proof = (a, b, c)"""
        proof, inputs = item
        self.items.append(((_c64(proof[0], 12), _c64(proof[1], 24), _c64(proof[2], 12)), fr_inputs(inputs)))

    def verify(self, rng, pvk):
        """batch.rs:100-173 against a PreparedVerifyingKey.  rng: None = z from the operating system (getrandom); any
        object with randrange gives reproducible z.  Returns None; raises InvalidProof or InvalidVerifyingKey."""
        n = len(self.items)
        if n and any(x.shape[0] + 1 != pvk.ic_len for _, x in self.items):
            raise InvalidVerifyingKey(f"[bb_status 6] InvalidVerifyingKey: a key with {pvk.ic_len} ic entries")
        L = pvk.ic_len - 1
        a = np.stack([p[0].reshape(12) for p, _ in self.items]) if n else np.zeros((0, 12), np.uint64)
        b = np.stack([p[1].reshape(24) for p, _ in self.items]) if n else np.zeros((0, 24), np.uint64)
        c = np.stack([p[2].reshape(12) for p, _ in self.items]) if n else np.zeros((0, 12), np.uint64)
        x = np.stack([xi.reshape(L, 4) for _, xi in self.items]) if n and L else np.zeros((n, max(L, 0), 4), np.uint64)
        z = None if rng is None else [rng.randrange(1, R_MODULUS) for _ in range(n)]
        verify_batch_arrays(pvk, a, b, c, x, z, n_inputs=max(L, 0))


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
