"""bellman_b200 -- host-side mirror of bellman's hot-path interface over the CUDA back-end.

The names follow the reference (bellman/src/multiexp.rs, src/domain.rs,
src/multicore.rs, groth16/src/prover.rs) so that tests read like the reference's own:

    worker = Worker()                                    # multicore::Worker::new()
    fast = multiexp(worker, (bases, 0), FullDensity, exponents).wait()
    dom = EvaluationDomain.from_coeffs(worker, coeffs); dom.ifft(); dom.coset_fft()
    proof = create_proof(assignment, params, r, s)       # prover.rs:182 after synthesis

Everything here is plumbing over the C ABI in include/bellman_b200.h (ctypes).  There is no
CPU implementation behind it: importing works without a GPU (so the ABI can be inspected),
but creating a Worker without the built library or without a CUDA device raises.
"""
import ctypes as C
import os
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbellman_b200.so")

BB_OK = 0
FORM_CANONICAL, FORM_MONTGOMERY = 0, 1
NTT_FFT, NTT_IFFT, NTT_COSET_FFT, NTT_ICOSET_FFT = 0, 1, 2, 3
G1, G2 = 1, 2
PARTIALS_BYTES = 960


class SynthesisError(Exception):
    """bellman::SynthesisError (src/lib.rs:304-319)"""


class PolynomialDegreeTooLarge(SynthesisError):
    pass


class UnexpectedIdentity(SynthesisError):
    pass


class IoError(SynthesisError):
    """SynthesisError::IoError(UnexpectedEof) -- 'expected more bases from source'"""


class DensityMismatch(AssertionError):
    """the assert! at src/multiexp.rs:324-329 (a panic upstream)"""


class BackendError(RuntimeError):
    pass


_ERRORS = {1: PolynomialDegreeTooLarge, 2: UnexpectedIdentity, 3: IoError, 5: DensityMismatch}

_lib = None


def load_library():
    """Load libbellman_b200.so; fail loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BackendError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(bellman_b200 has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.bb_last_error.restype = C.c_char_p
    lib.bb_ctx_kernel_launches.restype = C.c_uint64
    lib.bb_ctx_kernel_launches.argtypes = [C.c_void_p]
    _lib = lib
    return lib


def _check(rc):
    if rc == BB_OK:
        return
    msg = load_library().bb_last_error().decode(errors="replace")
    raise _ERRORS.get(rc, BackendError)(f"[bb_status {rc}] {msg}")


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _addr(p):
    """device address as an int (None for a null one), from an int or a ctypes void pointer (Worker.device_alloc returns
    the latter)"""
    return p.value if isinstance(p, C.c_void_p) else None if p is None else int(p)


def _c64(a, width):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a.reshape(-1, width)


def pack_density(bools):
    """list/array of bools -> (uint64 words LSB-first, length): DensityTracker's BitVec storage"""
    b = np.ascontiguousarray(bools, dtype=np.uint8)
    n = b.shape[0]
    packed = np.packbits(b, bitorder="little")
    pad = (-packed.shape[0]) % 8
    if pad or packed.shape[0] == 0:
        packed = np.concatenate([packed, np.zeros(pad if packed.shape[0] else 8, np.uint8)])
    return packed.view(np.uint64).copy(), n


class Worker:
    """multicore::Worker (src/multicore.rs:21-92): here, one CUDA device."""

    def __init__(self, device=0):
        lib = load_library()
        h = C.c_void_p()
        _check(lib.bb_ctx_create(C.c_int(device), C.byref(h)))
        self._h = h
        self.device = device
        self._children = weakref.WeakSet()      # the _DeviceObjects living on this context

    def close(self):
        if getattr(self, "_h", None):
            for child in list(self._children):  # device objects must go before their context
                child.free()
            load_library().bb_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key, value):
        _check(load_library().bb_ctx_set_option(self._h, key.encode(), C.c_long(value)))

    def synchronize(self):
        _check(load_library().bb_ctx_synchronize(self._h))

    @property
    def kernel_launches(self):
        return int(load_library().bb_ctx_kernel_launches(self._h))

    def profile_read(self, what):
        ms, launches, units = C.c_double(), C.c_uint64(), C.c_uint64()
        _check(load_library().bb_profile_read(self._h, what.encode(), C.byref(ms), C.byref(launches), C.byref(units)))
        return ms.value, launches.value, units.value

    def profile_reset(self):
        _check(load_library().bb_profile_reset(self._h))

    def bytes_copied(self):
        h2d, d2h = C.c_uint64(), C.c_uint64()
        _check(load_library().bb_ctx_bytes_copied(self._h, C.byref(h2d), C.byref(d2h)))
        return h2d.value, d2h.value

    # raw device buffers (bench: inputs resident in HBM before the timed region)
    def device_alloc(self, nbytes):
        p = C.c_void_p()
        _check(load_library().bb_device_alloc(self._h, C.c_size_t(nbytes), C.byref(p)))
        return p

    def device_free(self, p):
        _check(load_library().bb_device_free(self._h, p))

    def upload(self, d_ptr, host_array):
        a = np.ascontiguousarray(host_array)
        _check(load_library().bb_device_upload(self._h, d_ptr, _ptr(a), C.c_size_t(a.nbytes)))

    def download(self, d_ptr, host_array):
        _check(load_library().bb_device_download(self._h, _ptr(host_array), d_ptr, C.c_size_t(host_array.nbytes)))


class _DeviceObject:
    """An object living on a Worker's context: freed by free(), when collected, or with the Worker (close() frees its
    children before the context).  A subclass names its destroy call in _destroy and calls _own once it holds a handle."""

    _destroy = None

    def _own(self, worker, h):
        self.worker, self._h = worker, h
        worker._children.add(self)

    def free(self):
        if getattr(self, "_h", None):
            if getattr(self.worker, "_h", None):     # a context that is already gone took the device memory with it
                getattr(load_library(), self._destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Bases(_DeviceObject):
    """Arc<Vec<G::Affine>> resident in HBM (a SourceBuilder's backing store, multiexp.rs:45-51)."""

    _destroy = "bb_bases_free"

    def __init__(self, worker, group, points, global_offset=0, global_len=None):
        width = 12 if group == G1 else 24
        pts = _c64(points, width)
        self.worker, self.group, self.n = worker, group, pts.shape[0]
        if global_len is None:
            global_len = pts.shape[0]
        h = C.c_void_p()
        _check(load_library().bb_bases_upload(worker._h, C.c_int(group), _ptr(pts), C.c_size_t(pts.shape[0]),
                                              C.c_size_t(global_offset), C.c_size_t(global_len), C.byref(h)))
        self._own(worker, h)

    @classmethod
    def synthetic(cls, worker, group, seed, n, global_offset=0, global_len=None):
        """bench-only: [k_i]G with counter-based pseudorandom k_i, generated in HBM (no host copy)."""
        self = cls.__new__(cls)
        self.worker, self.group, self.n = worker, group, n
        h = C.c_void_p()
        _check(load_library().bb_synth_bases(worker._h, C.c_int(group), C.c_uint64(seed), C.c_size_t(n), C.c_size_t(global_offset),
                                             C.c_size_t(n if global_len is None else global_len), C.byref(h)))
        self._own(worker, h)
        return self

    def precompute(self):
        """resident window multiples 2^(c w) P_i: one bucket set for all windows (bb_bases_precompute)"""
        _check(load_library().bb_bases_precompute(self.worker._h, self._h))
        return self

    def drop_table(self):
        """bb_bases_drop_table: frees the window multiples again (no MSM over these bases may be in flight)"""
        _check(load_library().bb_bases_drop_table(self._h))
        return self


class _FullDensity:
    """multiexp::FullDensity (src/multiexp.rs:97-116)"""

    def __repr__(self):
        return "FullDensity"


FullDensity = _FullDensity()


class DensityTracker:
    """multiexp::DensityTracker (src/multiexp.rs:118-157)"""

    def __init__(self, bits=()):
        self.bv = [bool(b) for b in bits]

    def add_element(self):
        self.bv.append(False)

    def inc(self, idx):
        self.bv[idx] = True

    def get_total_density(self):
        return sum(self.bv)


class Waiter:
    """multicore::Waiter (src/multicore.rs:94-118)"""

    def __init__(self, job, group, keepalive):
        self._job, self._group, self._keep = job, group, keepalive

    def wait(self):
        if self._job is None:
            raise RuntimeError("wait() called twice")
        out = np.zeros((1, 12 if self._group == G1 else 24), dtype=np.uint64)
        job, self._job = self._job, None
        rc = load_library().bb_msm_wait(job, _ptr(out))
        self._keep = None
        _check(rc)
        return out


def multiexp(pool, bases, density_map, exponents, form=FORM_MONTGOMERY):
    """bellman::multiexp::multiexp (src/multiexp.rs:305-332).

    bases: (Bases, offset) -- the (Arc<Vec<G>>, usize) SourceBuilder.
    density_map: FullDensity or a DensityTracker.
    exponents: (n,4) uint64 Fr array; Montgomery (Scalar's memory form) or canonical
               (Exponent::Bits) according to `form`.
    """
    b, offset = bases
    ex = _c64(exponents, 4)
    n = ex.shape[0]
    dens_words, dens_len = None, 0
    if density_map is not FullDensity:
        bits = density_map.bv if isinstance(density_map, DensityTracker) else density_map
        dens_words, dens_len = pack_density(bits)
    job = C.c_void_p()
    _check(load_library().bb_msm_async(pool._h, b._h, C.c_size_t(offset), _ptr(dens_words), C.c_size_t(dens_len),
                                       _ptr(ex), C.c_size_t(n), C.c_int(form), C.byref(job)))
    return Waiter(job, b.group, (b, ex, dens_words))


def multiexp_device(pool, bases, d_scalars, n, form=FORM_MONTGOMERY):
    """multiexp over scalars already resident in HBM (FullDensity)."""
    b, offset = bases
    job = C.c_void_p()
    _check(load_library().bb_msm_async_device(pool._h, b._h, C.c_size_t(offset), None, C.c_size_t(0),
                                              d_scalars, C.c_size_t(n), C.c_int(form), C.byref(job)))
    return Waiter(job, b.group, (b,))


class EvaluationDomain:
    """bellman::domain::EvaluationDomain<Fr, Scalar<Fr>> (src/domain.rs:21-190); coefficients
    live on the host as an (m,4) uint64 Montgomery array, every method runs on the device."""

    def __init__(self, worker, coeffs, exp):
        self.worker, self.coeffs, self.exp = worker, coeffs, exp

    @classmethod
    def from_coeffs(cls, worker, coeffs):                  # domain.rs:47-79
        c = _c64(coeffs, 4)
        m, exp = 1, 0
        while m < c.shape[0]:
            m *= 2
            exp += 1
            if exp >= 32:
                raise PolynomialDegreeTooLarge()
        padded = np.zeros((m, 4), dtype=np.uint64)
        padded[: c.shape[0]] = c
        return cls(worker, padded, exp)

    def into_coeffs(self):
        return self.coeffs

    def _run(self, mode):
        _check(load_library().bb_ntt(self.worker._h, _ptr(self.coeffs), C.c_uint32(self.exp), C.c_int(mode),
                                     C.c_int(FORM_MONTGOMERY)))

    # Fr as Python integers <-> the Montgomery limbs of the buffers (host helpers of the mirror)
    FR_MODULUS = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
    MULTIPLICATIVE_GENERATOR = 7

    @classmethod
    def _to_mont(cls, v):
        m = (v % cls.FR_MODULUS) * (1 << 256) % cls.FR_MODULUS
        return np.array([(m >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)

    def _pointwise(self, op, other=None, k=None):
        b = None if other is None else _c64(other, 4)
        if b is not None:
            assert b.shape == self.coeffs.shape                # assert_eq!(self.coeffs.len(), other.coeffs.len())
        kk = None if k is None else self._to_mont(k)
        _check(load_library().bb_domain_pointwise(self.worker._h, C.c_int(op), _ptr(self.coeffs), _ptr(b),
                                                  C.c_size_t(self.coeffs.shape[0]), _ptr(kk)))

    def mul_assign(self, other):                           # domain.rs:154-170
        self._pointwise(0, other.coeffs if isinstance(other, EvaluationDomain) else other)

    def sub_assign(self, other):                           # :173-189
        self._pointwise(1, other.coeffs if isinstance(other, EvaluationDomain) else other)

    def distribute_powers(self, g):                        # :101-113 (g: Python integer)
        self._pointwise(3, k=g)

    def z(self, tau):                                      # :129-134, tau^m - 1 as a Python integer
        return (pow(tau, self.coeffs.shape[0], self.FR_MODULUS) - 1) % self.FR_MODULUS

    def divide_by_z_on_coset(self):                        # :139-151
        self._pointwise(2, k=pow(self.z(self.MULTIPLICATIVE_GENERATOR), -1, self.FR_MODULUS))

    def fft(self): self._run(NTT_FFT)                      # domain.rs:81-83
    def ifft(self): self._run(NTT_IFFT)                    # :85-99
    def coset_fft(self): self._run(NTT_COSET_FFT)          # :115-118
    def icoset_fft(self): self._run(NTT_ICOSET_FFT)        # :120-125


def ntt_device(worker, d_ptr, log_n, mode):
    _check(load_library().bb_ntt_device(worker._h, d_ptr, C.c_uint32(log_n), C.c_int(mode)))


def h_poly(worker, a, b, c):
    """The H block of create_proof (groth16/src/prover.rs:221-240): returns the m-1 quotient
    coefficients as canonical integers (Exponent::Bits form), shape (m-1, 4)."""
    a, b, c = _c64(a, 4), _c64(b, 4), _c64(c, 4)
    n = a.shape[0]
    m = 1
    while m < n:
        m *= 2
    out = np.zeros((max(m - 1, 1), 4), dtype=np.uint64)
    m_out = C.c_size_t()
    _check(load_library().bb_h_poly(worker._h, _ptr(a), _ptr(b), _ptr(c), C.c_size_t(n), _ptr(out), C.byref(m_out)))
    return out[: m_out.value - 1]


def fixed_base_mul(worker, group, scalars, form=FORM_MONTGOMERY):
    k = _c64(scalars, 4)
    out = np.zeros((k.shape[0], 12 if group == G1 else 24), dtype=np.uint64)
    _check(load_library().bb_fixed_base_mul(worker._h, C.c_int(group), _ptr(k), C.c_size_t(k.shape[0]), C.c_int(form), _ptr(out)))
    return out


def point_add(group, a, b):
    w = 12 if group == G1 else 24
    a, b = _c64(a, w), _c64(b, w)
    out = np.zeros((1, w), dtype=np.uint64)
    _check(load_library().bb_point_add(C.c_int(group), _ptr(a), _ptr(b), _ptr(out)))
    return out


def point_compress(group, a):
    w = 12 if group == G1 else 24
    a = _c64(a, w)
    out = np.zeros(48 if group == G1 else 96, dtype=np.uint8)
    _check(load_library().bb_point_compress(C.c_int(group), _ptr(a), _ptr(out)))
    return bytes(out)


class _CrsDesc(C.Structure):
    _fields_ = [("alpha_g1", C.c_void_p), ("beta_g1", C.c_void_p), ("delta_g1", C.c_void_p),
                ("beta_g2", C.c_void_p), ("delta_g2", C.c_void_p),
                ("h", C.c_void_p), ("h_len", C.c_size_t), ("l", C.c_void_p), ("l_len", C.c_size_t),
                ("a", C.c_void_p), ("a_len", C.c_size_t), ("b_g1", C.c_void_p), ("b_g1_len", C.c_size_t),
                ("b_g2", C.c_void_p), ("b_g2_len", C.c_size_t),
                ("shard_index", C.c_uint32), ("shard_count", C.c_uint32)]


class _Witness(C.Structure):
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("c", C.c_void_p), ("n_constraints", C.c_size_t),
                ("input_assignment", C.c_void_p), ("n_inputs", C.c_size_t),
                ("aux_assignment", C.c_void_p), ("n_aux", C.c_size_t),
                ("a_aux_density", C.c_void_p), ("b_input_density", C.c_void_p), ("b_aux_density", C.c_void_p),
                ("on_device", C.c_int)]


class Parameters(_DeviceObject):
    """groth16::Parameters made device-resident (groth16/src/lib.rs:222-244).  `p` maps
    vk_g1 (alpha,beta,delta), vk_g2 (beta,gamma,delta), h, l, a, b_g1, b_g2 to uint64 arrays."""

    _destroy = "bb_crs_destroy"

    def __init__(self, worker, p, shard_index=0, shard_count=1):
        self.worker = worker
        self._keep = {k: np.ascontiguousarray(v, dtype=np.uint64) for k, v in p.items()}
        k = self._keep
        vk1, vk2 = k["vk_g1"].reshape(3, 12), k["vk_g2"].reshape(3, 24)
        self._vk = [np.ascontiguousarray(vk1[0]), np.ascontiguousarray(vk1[1]), np.ascontiguousarray(vk1[2]),
                    np.ascontiguousarray(vk2[0]), np.ascontiguousarray(vk2[2])]
        d = _CrsDesc()
        d.alpha_g1, d.beta_g1, d.delta_g1 = (self._vk[i].ctypes.data for i in range(3))
        d.beta_g2, d.delta_g2 = self._vk[3].ctypes.data, self._vk[4].ctypes.data
        self.lens = {"ic": int(np.asarray(p["ic"]).reshape(-1, 12).shape[0])} if "ic" in p else {}
        for name, width in (("h", 12), ("l", 12), ("a", 12), ("b_g1", 12), ("b_g2", 24)):
            arr = k[name].reshape(-1, width)
            setattr(d, name, arr.ctypes.data)
            setattr(d, name + "_len", arr.shape[0])
            self.lens[name] = int(arr.shape[0])
        d.shard_index, d.shard_count = shard_index, shard_count
        h = C.c_void_p()
        _check(load_library().bb_crs_create(worker._h, C.byref(d), C.byref(h)))
        self._own(worker, h)
        self._keep = None                    # the vectors are resident in HBM now

    @classmethod
    def _from_handle(cls, worker, h, lens):
        """a bb_crs built by the library itself (params_io.read_parameters_device); lens: the vector lengths"""
        self = cls.__new__(cls)
        self.worker, self._keep, self.lens = worker, None, dict(lens)
        self._own(worker, h)
        return self

    @classmethod
    def synthetic(cls, worker, seed, shape, shard_index=0, shard_count=1):
        """bench-only: Parameters-shaped vectors [k_i]G generated on the device for this rank's
        base-range shard (lengths as generate_parameters would produce for `shape`)."""
        self = cls.__new__(cls)
        self.worker, self._keep = worker, None
        h = C.c_void_p()
        _check(load_library().bb_synth_crs(worker._h, C.c_uint64(seed), C.c_size_t(shape["m"] - 1), C.c_size_t(shape["num_aux"]),
                                           C.c_size_t(shape["num_inputs"] + shape["a_aux_total"]),
                                           C.c_size_t(shape["b_in_total"] + shape["b_aux_total"]),
                                           C.c_uint32(shard_index), C.c_uint32(shard_count), C.byref(h)))
        self._own(worker, h)
        return self

    def precompute(self):
        """bb_crs_precompute: window multiples of all five vectors resident (msm_precompute forms)"""
        _check(load_library().bb_crs_precompute(self.worker._h, self._h))
        return self

    def drop_tables(self):
        _check(load_library().bb_crs_drop_tables(self._h))
        return self

    def apply_tuning(self, index):
        """bb_crs_apply_tuning: select MSM form `index` (see tuning_names()) for this key and its worker"""
        _check(load_library().bb_crs_apply_tuning(self.worker._h, self._h, C.c_int(index)))

    def autotune(self, assignment, reps=3, device_ptrs=None):
        """bb_groth16_autotune: prove `assignment` with every MSM form, keep the fastest whose partial sums equal the
        default form's.  Returns {"chosen": index, "name": ..., "ms": [per form; negative = not eligible]}.
        A sharded key (shard_count > 1) is only measured and stays on the default form: all shards must run the same
        form (see distributed.autotune_sharded)."""
        lib = load_library()
        n = lib.bb_tuning_count()
        ms = (C.c_double * n)()
        chosen = C.c_int(0)
        w = assignment._struct(device_ptrs)
        _check(lib.bb_groth16_autotune(self.worker._h, self._h, C.byref(w), C.c_int(reps), C.byref(chosen), ms))
        return {"chosen": chosen.value, "name": tuning_names()[chosen.value], "ms": [round(float(x), 3) for x in ms]}


def tuning_names():
    """the MSM forms bb_groth16_autotune chooses from (index 0 = default)"""
    lib = load_library()
    lib.bb_tuning_name.restype = C.c_char_p
    return [lib.bb_tuning_name(C.c_int(i)).decode() for i in range(lib.bb_tuning_count())]


class ProvingAssignment:
    """What groth16's ProvingAssignment holds once synthesis is done (prover.rs:57-71,
    193-215): a, b, c evaluations (incl. the input constraints), assignments, densities."""

    def __init__(self, a, b, c, input_assignment, aux_assignment, a_aux_density, b_input_density, b_aux_density):
        self.a, self.b, self.c = _c64(a, 4), _c64(b, 4), _c64(c, 4)
        self.input_assignment, self.aux_assignment = _c64(input_assignment, 4), _c64(aux_assignment, 4)
        self.a_aux_density, _ = pack_density(a_aux_density)
        self.b_input_density, _ = pack_density(b_input_density)
        self.b_aux_density, _ = pack_density(b_aux_density)

    def _struct(self, device_ptrs=None):
        """device_ptrs: optional dict a,b,c,inputs,aux -> device addresses (inputs resident in HBM)"""
        p = device_ptrs if device_ptrs is not None else {
            "a": self.a.ctypes.data, "b": self.b.ctypes.data, "c": self.c.ctypes.data,
            "inputs": self.input_assignment.ctypes.data, "aux": self.aux_assignment.ctypes.data}
        w = _Witness()
        w.a, w.b, w.c = p["a"], p["b"], p["c"]
        w.n_constraints = self.a.shape[0]
        w.input_assignment, w.n_inputs = p["inputs"], self.input_assignment.shape[0]
        w.aux_assignment, w.n_aux = p["aux"], self.aux_assignment.shape[0]
        w.a_aux_density = self.a_aux_density.ctypes.data
        w.b_input_density = self.b_input_density.ctypes.data
        w.b_aux_density = self.b_aux_density.ctypes.data
        w.on_device = 0 if device_ptrs is None else 1
        return w


def _scalar_bytes(v):
    return (C.c_uint8 * 32).from_buffer_copy(int(v).to_bytes(32, "little"))


def prove_partials(assignment, params, device_ptrs=None):
    """NTT pipeline + the eight MSMs over this process's CRS shard -> 960 bytes of partial sums."""
    out = (C.c_uint8 * PARTIALS_BYTES)()
    w = assignment._struct(device_ptrs)
    _check(load_library().bb_groth16_prove_partials(params.worker._h, params._h, C.byref(w), out))
    return bytes(out)


def prove_begin(assignment, params, device_ptrs=None):
    """bb_groth16_prove_begin: uploads the assignments and queues the seven witness MSMs; returns the state
    (keep `assignment` alive until prove_end)."""
    w = assignment._struct(device_ptrs)
    h = C.c_void_p()
    _check(load_library().bb_groth16_prove_begin(params.worker._h, params._h, C.byref(w), C.byref(h)))
    return h


def prove_end(state, evals=None):
    """bb_groth16_prove_end: `evals` = device addresses of the coset evaluations of a, b, c (bb_h_coset_evals on
    whichever rank computed them), or None to run the whole H pipeline here -> 960 bytes of partial sums."""
    out = (C.c_uint8 * PARTIALS_BYTES)()
    ea, eb, ec = (C.c_void_p(_addr(p)) for p in evals) if evals is not None else (None, None, None)
    _check(load_library().bb_groth16_prove_end(state, ea, eb, ec, out))
    return bytes(out)


def h_coset_evals_async(worker, poly, n_constraints, d_out, on_device=False):
    """bb_h_coset_evals_async: queue the upload and the two transforms of one polynomial, return at once; the
    caller keeps `poly` and the output buffer alive until h_coset_evals_wait(worker)."""
    src = C.c_void_p(_addr(poly)) if on_device else _ptr(poly)
    _check(load_library().bb_h_coset_evals_async(worker._h, src, C.c_size_t(n_constraints), C.c_int(1 if on_device else 0), C.c_void_p(_addr(d_out))))


def h_coset_evals_wait(worker):
    _check(load_library().bb_h_coset_evals_wait(worker._h))


def h_coset_evals(worker, poly, n_constraints, d_out, on_device=False):
    """coset_fft(ifft(from_coeffs(poly))) of ONE of a, b, c (prover.rs:225-230) into the device buffer d_out
    (m Fr).  `poly`: numpy array (host) or a device address with on_device=True."""
    src = C.c_void_p(_addr(poly)) if on_device else _ptr(poly)
    _check(load_library().bb_h_coset_evals(worker._h, src, C.c_size_t(n_constraints), C.c_int(1 if on_device else 0), C.c_void_p(_addr(d_out))))


PROOF_STATIC_BYTES = 768


def finalize_static(params, r, s):
    """the terms of A, B, C that need no MSM result (prover.rs:326-337); host only, callable from a
    thread while the devices work (ctypes releases the GIL)"""
    out = (C.c_uint8 * PROOF_STATIC_BYTES)()
    _check(load_library().bb_groth16_finalize_static(params._h, _scalar_bytes(r), _scalar_bytes(s), out))
    return bytes(out)


def finalize(params, partial_sets, r, s, static=None):
    """prover.rs:320-360 + Proof::write; partial_sets: list of 960-byte blobs (one per shard);
    `static`: the result of finalize_static(params, r, s) if it was computed ahead."""
    blob = b"".join(partial_sets)
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
    proof = (C.c_uint8 * 192)()
    if static is None:
        _check(load_library().bb_groth16_finalize(params._h, buf, C.c_size_t(len(partial_sets)), _scalar_bytes(r), _scalar_bytes(s), proof))
    else:
        assert len(static) == PROOF_STATIC_BYTES
        st = (C.c_uint8 * PROOF_STATIC_BYTES).from_buffer_copy(static)
        _check(load_library().bb_groth16_finalize_with(params._h, buf, C.c_size_t(len(partial_sets)), _scalar_bytes(r), _scalar_bytes(s),
                                                        st, proof))
    return bytes(proof)


def create_proof(assignment, params, r, s, device_ptrs=None):
    """groth16::create_proof after synthesis (prover.rs:217-360) + Proof::write: 192 bytes.
    r, s are Python integers in [0, r)."""
    proof = (C.c_uint8 * 192)()
    w = assignment._struct(device_ptrs)
    _check(load_library().bb_groth16_prove(params.worker._h, params._h, C.byref(w), _scalar_bytes(r), _scalar_bytes(s), proof))
    return bytes(proof)


def create_random_proof(assignment, params, rng=None, device_ptrs=None):
    """groth16::create_random_proof (prover.rs:164-179): r, s <- Fr::random, then create_proof.
    `rng`: anything with randrange (default: the operating system's CSPRNG)."""
    import secrets
    draw = rng.randrange if rng is not None else secrets.randbelow
    q = EvaluationDomain.FR_MODULUS
    return create_proof(assignment, params, draw(q), draw(q), device_ptrs)


def _batch_result(params, rc, proofs, status):
    """one entry per item: its 192 proof bytes, or the exception create_proof raises for it alone"""
    _check(rc)
    raw = bytes(proofs)
    out = []
    for i, st in enumerate(status):
        if st == BB_OK:
            out.append(raw[192 * i:192 * (i + 1)])
        else:
            out.append(_ERRORS.get(st, BackendError)(f"[bb_status {st}] {_status_message(params, st)}"))
    return out


def _status_message(params, st):
    """the message bb_groth16_prove reports with status `st` for this key (bb_groth16_prove_message); a back-end failure
    of a sub-batch keeps the call's bb_last_error"""
    lib = load_library()
    lib.bb_groth16_prove_message.restype = C.c_char_p
    msg = lib.bb_groth16_prove_message(params._h, C.c_int(st))
    return (msg if msg is not None else lib.bb_last_error()).decode(errors="replace")


def _scalars_bytes(vals):
    return (C.c_uint8 * (32 * len(vals))).from_buffer_copy(b"".join(int(v).to_bytes(32, "little") for v in vals))


def create_proof_batch(assignments, params, rs, ss, device_ptrs=None):
    """bb_groth16_prove_batch: create_proof for every assignment of one circuit against `params`, in one call.
    `device_ptrs`: None, or one dict per item as create_proof takes it.  Returns one entry per item: the 192 bytes
    create_proof returns for it alone, or the exception it would raise (an instance, not raised)."""
    n = len(assignments)
    if not (len(rs) == len(ss) == n) or (device_ptrs is not None and len(device_ptrs) != n):
        raise ValueError("create_proof_batch: one r, one s (and one device_ptrs entry) per assignment")
    ws = (_Witness * max(n, 1))()
    for i, asg in enumerate(assignments):
        ws[i] = asg._struct(None if device_ptrs is None else device_ptrs[i])
    proofs = (C.c_uint8 * (192 * max(n, 1)))()
    status = (C.c_int * max(n, 1))()
    rc = load_library().bb_groth16_prove_batch(params.worker._h, params._h, ws, C.c_size_t(n), _scalars_bytes(rs), _scalars_bytes(ss),
                                               proofs, status)
    return _batch_result(params, rc, proofs, list(status)[:n])


def create_random_proof_batch(assignments, params, rng=None, device_ptrs=None):
    """create_random_proof for every assignment: fresh (r, s) per item, then create_proof_batch"""
    import secrets
    draw = rng.randrange if rng is not None else secrets.randbelow
    q = EvaluationDomain.FR_MODULUS
    rs, ss = [], []
    for _ in assignments:
        rs.append(draw(q))
        ss.append(draw(q))
    return create_proof_batch(assignments, params, rs, ss, device_ptrs)


def synth_mimc(rounds, seed, pinned=False):
    """bench-only: the MiMC-chain witness of `rounds` rounds as a ProvingAssignment (product-side
    generator, bellman_b200/csrc/synth.cu).  pinned=True places the arrays in page-locked host
    memory (torch) so that cudaMemcpyAsync runs at full PCIe speed."""
    lib = load_library()
    shape = np.zeros(7, np.uint64)
    _check(lib.bb_synth_mimc_shape(C.c_size_t(rounds), _ptr(shape)))
    ni, na, n = int(shape[0]), int(shape[1]), int(shape[2])

    def buf(rows):
        if pinned:
            import torch
            t = torch.zeros((rows, 4), dtype=torch.int64).pin_memory()
            return t, t.numpy().view(np.uint64)
        return None, np.zeros((rows, 4), np.uint64)

    keep, arrs = [], []
    for rows in (n, n, n, ni, na):
        t, a = buf(rows)
        keep.append(t)
        arrs.append(a)
    a, b, c, inputs, aux = arrs
    words = (na + 63) // 64
    ad, bd, bi = np.zeros(words, np.uint64), np.zeros(words, np.uint64), np.zeros(1, np.uint64)
    _check(lib.bb_synth_mimc_witness(C.c_size_t(rounds), C.c_uint64(seed), _ptr(a), _ptr(b), _ptr(c), _ptr(inputs), _ptr(aux),
                                     _ptr(ad), _ptr(bi), _ptr(bd)))
    asg = ProvingAssignment.__new__(ProvingAssignment)
    asg.a, asg.b, asg.c, asg.input_assignment, asg.aux_assignment = a, b, c, inputs, aux
    asg.a_aux_density, asg.b_input_density, asg.b_aux_density = ad, bi, bd
    asg._keep = keep
    return asg, dict(num_inputs=ni, num_aux=na, num_constraints=n, m=int(shape[3]), a_aux_total=int(shape[4]),
                     b_in_total=int(shape[5]), b_aux_total=int(shape[6]))


def synth_scalars_device(worker, seed, n, d_ptr):
    """bench-only: fill a device buffer with n pseudorandom canonical scalars (< 2^254)."""
    _check(load_library().bb_synth_scalars_device(worker._h, C.c_uint64(seed), C.c_size_t(n), d_ptr))


def fr_dot_device(worker, d_a, d_b, n):
    """diagnostic: sum a_i b_i mod r of two device arrays of canonical Fr -> (4,) uint64 canonical"""
    out = np.zeros(4, np.uint64)
    _check(load_library().bb_diag_fr_dot(worker._h, d_a, d_b, C.c_size_t(n), _ptr(out)))
    return out


# groth16 verification (groth16/src/verifier.rs, verifier/batch.rs)
from .verifier import (BatchVerifier, InvalidProof, InvalidVerifyingKey, PreparedVerifyingKey,  # noqa: E402
                       VerificationError, prepare_verifying_key, verify_proof)
# Proof::read / Proof::write over a batch (groth16/src/lib.rs:39-99)
from .verifier import InvalidProofEncoding, read_proof, read_proofs, write_proofs  # noqa: E402
# the constraint system on the device: prove from the witness alone (groth16/src/prover.rs:19-55,105-145)
from .r1cs import (R1CS, check_r1cs_batch, create_proof_r1cs, create_proof_r1cs_batch, create_random_proof_r1cs,  # noqa: E402
                   create_random_proof_r1cs_batch)
# Parameters::read / VerifyingKey::read on the device (groth16/src/lib.rs:158-218, 289-398)
from .params_io import InvalidData, read_parameters_device, read_verifying_key_device  # noqa: E402
