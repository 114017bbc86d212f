"""The constraint system resident on the device (bb_r1cs_*, csrc/r1cs.cu): prove from the witness alone.

ProvingAssignment::enforce (groth16/src/prover.rs:19-55,105-145) evaluates every linear combination of every
constraint during synthesis.  With the A, B, C matrices in HBM beside the key -- the ones KeypairAssembly records for
generate_parameters -- a proof needs only input_assignment and aux_assignment; a, b, c and the densities come from the
device:

    r1cs = R1CS.from_assembly(worker, asm)          # the KeypairAssembly synthesis left, as for generate_parameters
    proof = create_proof_r1cs(r1cs, params, input_assignment, aux_assignment, r, s)

Matrices are CSR by constraint: (row_offsets uint64 (n+1,), vars uint32 (nnz,), coeffs (nnz, 4) uint64 Montgomery Fr),
variables numbered inputs first (ONE = 0), then aux.  The input rows of prover.rs:208-215 are appended by the library.
"""
import ctypes as C

import numpy as np

from . import EvaluationDomain, _addr, _c64, _check, _DeviceObject, _ptr, _scalar_bytes, load_library

FR_MODULUS = EvaluationDomain.FR_MODULUS
SHAPE_WORDS = 9
_MASK64 = (1 << 64) - 1


class _Matrix(C.Structure):
    _fields_ = [("row_offsets", C.c_void_p), ("vars", C.c_void_p), ("coeffs", C.c_void_p)]


class _Desc(C.Structure):
    _fields_ = [("a", _Matrix), ("b", _Matrix), ("c", _Matrix),
                ("n_constraints", C.c_size_t), ("n_inputs", C.c_size_t), ("n_aux", C.c_size_t)]


def _unpack(words, n):
    return np.unpackbits(np.ascontiguousarray(words, np.uint64).view(np.uint8), bitorder="little")[:n].astype(bool)


def _mont_limbs(ints):
    """Python integers mod r -> (n, 4) uint64 Montgomery limbs"""
    out = np.zeros((len(ints), 4), np.uint64)
    for i, v in enumerate(ints):
        out[i] = EvaluationDomain._to_mont(v)
    return out


class R1CS(_DeviceObject):
    """bb_r1cs: the A, B, C matrices of one circuit in HBM.  a, b, c: (row_offsets, vars, coeffs) per matrix."""

    _destroy = "bb_r1cs_destroy"

    def __init__(self, worker, n_inputs, n_aux, a, b, c):
        mats = []
        for off, var, cf in (a, b, c):
            off = np.ascontiguousarray(off, np.uint64)
            var = np.ascontiguousarray(var, np.uint32)
            cf = _c64(cf, 4) if len(cf) else np.zeros((0, 4), np.uint64)
            mats.append((off, var, cf))
        n = mats[0][0].shape[0] - 1
        if n < 0 or any(m[0].shape[0] != n + 1 for m in mats):
            raise ValueError("the three matrices need the same number of rows")
        d = _Desc()
        for name, (off, var, cf) in zip("abc", mats):
            setattr(d, name, _Matrix(off.ctypes.data, var.ctypes.data if var.size else None, cf.ctypes.data if cf.size else None))
        d.n_constraints, d.n_inputs, d.n_aux = n, n_inputs, n_aux
        h = C.c_void_p()
        _check(load_library().bb_r1cs_create(worker._h, C.byref(d), C.byref(h)))
        self._own(worker, h)
        shape = np.zeros(SHAPE_WORDS, np.uint64)
        _check(load_library().bb_r1cs_info(h, _ptr(shape), None, None, None))
        self.n_constraints, self.n_inputs, self.n_aux = (int(x) for x in shape[:3])
        self.nnz = tuple(int(x) for x in shape[3:6])              # terms the evaluation reads, per matrix
        self.unit = tuple(int(x) for x in shape[6:9])             # of those, coefficient one

    @classmethod
    def from_assembly(cls, worker, asm):
        """generator.KeypairAssembly as synthesis leaves it (ONE allocated as input 0, no input rows): its per-variable
        (coefficient, constraint) lists transposed into rows.  Duplicate and zero-coefficient terms are kept as
        recorded, so the densities are bellman's."""
        ni, n = asm.num_inputs, asm.num_constraints
        mats = []
        for inputs, aux in ((asm.at_inputs, asm.at_aux), (asm.bt_inputs, asm.bt_aux), (asm.ct_inputs, asm.ct_aux)):
            rows, vars_, coeffs = [], [], []
            for base, per_var in ((0, inputs), (ni, aux)):
                for j, terms in enumerate(per_var):
                    for coeff, row in terms:
                        rows.append(row)
                        vars_.append(base + j)
                        coeffs.append(coeff)
            order = np.argsort(np.array(rows, np.int64), kind="stable")
            off = np.zeros(n + 1, np.uint64)
            off[1:] = np.cumsum(np.bincount(np.array(rows, np.int64), minlength=n)[:n])
            cf = _mont_limbs(coeffs)[order] if coeffs else np.zeros((0, 4), np.uint64)
            mats.append((off, np.array(vars_, np.uint32)[order], cf))
        return cls(worker, ni, asm.num_aux, *mats)

    @classmethod
    def synth_mimc(cls, worker, rounds, seed):
        """bench-only: the MiMC circuit of bb_synth_mimc_witness(rounds, seed) (same constants), from bb_synth_mimc_r1cs"""
        return cls(worker, 2, 2 * rounds + 1, *synth_mimc_matrices(rounds, seed))

    def density_words(self):
        """(a_aux_density, b_input_density, b_aux_density) as bb_witness's LSB-first uint64 words"""
        aw, iw = max(1, (self.n_aux + 63) // 64), max(1, (self.n_inputs + 63) // 64)
        a, bi, b = np.zeros(aw, np.uint64), np.zeros(iw, np.uint64), np.zeros(aw, np.uint64)
        _check(load_library().bb_r1cs_info(self._h, _ptr(np.zeros(SHAPE_WORDS, np.uint64)), _ptr(a), _ptr(bi), _ptr(b)))
        return a, bi, b

    def densities(self):
        """(a_aux_density, b_input_density, b_aux_density) as bool arrays of n_aux, n_inputs, n_aux entries"""
        a, bi, b = self.density_words()
        return _unpack(a, self.n_aux), _unpack(bi, self.n_inputs), _unpack(b, self.n_aux)

    def eval(self, input_assignment, aux_assignment, on_device=False, out=None):
        """a, b, c for the witness (bb_r1cs_eval).  Host arrays of Montgomery Fr, or with on_device=True device addresses
        (lengths taken from the constraint system).  out: None -> three (n, 4) host arrays returned; or a dict a, b, c
        of device addresses written in place."""
        src, keep = self._witness_args(input_assignment, aux_assignment, on_device)
        if out is None:
            res = [np.zeros((self.n_constraints, 4), np.uint64) for _ in range(3)]
            dst = [_ptr(x) for x in res]
        else:
            res = None
            dst = [C.c_void_p(_addr(out[k])) for k in "abc"]
        _check(load_library().bb_r1cs_eval(self.worker._h, self._h, *src, *dst, C.c_int(0 if out is None else 1)))
        del keep
        return None if res is None else tuple(res)

    def unsatisfied(self, input_assignment, aux_assignment, on_device=False, bits=False):
        """bb_r1cs_check: (first, count) -- the lowest row k with <A_k,z> <B_k,z> != <C_k,z> (None if every row holds) and
        how many rows fail; with bits=True also a bool array of n_constraints marking them.  Rows are numbered as eval's
        outputs (the appended input rows never fail).  Witness arguments as eval's."""
        src, keep = self._witness_args(input_assignment, aux_assignment, on_device)
        first, count = C.c_size_t(), C.c_size_t()
        words = np.zeros((self.n_constraints + 63) // 64, np.uint64) if bits else None
        _check(load_library().bb_r1cs_check(self.worker._h, self._h, *src, C.byref(first), C.byref(count), _ptr(words)))
        del keep
        res = (_first_or_none(first.value), count.value)
        return res + (_unpack(words, self.n_constraints),) if bits else res

    def which_is_unsatisfied(self, input_assignment, aux_assignment, on_device=False):
        """TestConstraintSystem::which_is_unsatisfied (src/gadgets/test/mod.rs:254-267) on the device: the index of the
        first failing constraint, or None (constraints have no names here)"""
        return self.unsatisfied(input_assignment, aux_assignment, on_device)[0]

    def is_satisfied(self, input_assignment, aux_assignment, on_device=False):
        """TestConstraintSystem::is_satisfied (src/gadgets/test/mod.rs:269-272) on the device"""
        return self.which_is_unsatisfied(input_assignment, aux_assignment, on_device) is None

    def _witness_args(self, input_assignment, aux_assignment, on_device):
        """the (input, n_inputs, aux, n_aux, on_device) arguments of bb_r1cs_eval and bb_groth16_prove_r1cs, and the host
        arrays they point into: device addresses (lengths taken from the constraint system), or host arrays"""
        if on_device:
            return (C.c_void_p(_addr(input_assignment)), C.c_size_t(self.n_inputs), C.c_void_p(_addr(aux_assignment)),
                    C.c_size_t(self.n_aux), C.c_int(1)), ()
        inp, aux = _c64(input_assignment, 4), _c64(aux_assignment, 4)
        return (_ptr(inp), C.c_size_t(inp.shape[0]), _ptr(aux), C.c_size_t(aux.shape[0]), C.c_int(0)), (inp, aux)

    def assignment(self, input_assignment, aux_assignment):
        """the ProvingAssignment bellman's synthesis would have built, evaluated on the device"""
        from . import ProvingAssignment
        a, b, c = self.eval(input_assignment, aux_assignment)
        asg = ProvingAssignment.__new__(ProvingAssignment)
        asg.a, asg.b, asg.c = a, b, c
        asg.input_assignment, asg.aux_assignment = _c64(input_assignment, 4), _c64(aux_assignment, 4)
        asg.a_aux_density, asg.b_input_density, asg.b_aux_density = self.density_words()
        return asg


def synth_mimc_matrices(rounds, seed):
    """bench-only: the A, B, C matrices of bb_synth_mimc_r1cs(rounds, seed), (row_offsets, vars, coeffs) each, as
    R1CS.synth_mimc uploads them (2 inputs, 2 rounds + 1 aux, 2 rounds constraints before the input rows)"""
    mats = []
    for terms in (3 * rounds, 4 * rounds, 3 * rounds):
        mats.append((np.zeros(2 * rounds + 1, np.uint64), np.zeros(terms, np.uint32), np.zeros((terms, 4), np.uint64)))
    args = [_ptr(x) for m in mats for x in m]
    _check(load_library().bb_synth_mimc_r1cs(C.c_size_t(rounds), C.c_uint64(seed), *args))
    return mats


def _first_or_none(v):
    return None if v == C.c_size_t(-1).value else int(v)


def _batch_witness_args(r1cs, inputs, aux, count, device_ptrs):
    """the (inputs, n_inputs, aux, n_aux, count, on_device) arguments of bb_r1cs_check_batch, and the host arrays they point
    into (count = 0: null pointers, nothing to read)"""
    if device_ptrs is not None or not count:
        d = device_ptrs or {"inputs": None, "aux": None}
        return (C.c_void_p(_addr(d["inputs"])), C.c_size_t(r1cs.n_inputs), C.c_void_p(_addr(d["aux"])),
                C.c_size_t(r1cs.n_aux), C.c_size_t(count), C.c_int(device_ptrs is not None)), ()
    inp = np.ascontiguousarray(np.asarray(inputs, dtype=np.uint64).reshape(count, -1, 4))
    ax = np.ascontiguousarray(np.asarray(aux, dtype=np.uint64).reshape(count, -1, 4))
    return (_ptr(inp), C.c_size_t(inp.shape[1]), _ptr(ax), C.c_size_t(ax.shape[1]), C.c_size_t(count), C.c_int(0)), (inp, ax)


def check_r1cs_batch(r1cs, inputs, aux, count=None, device_ptrs=None):
    """bb_r1cs_check_batch: R1CS.unsatisfied for `count` witnesses in one call (count defaults to len(inputs); with
    device_ptrs it must be given).  inputs / aux / device_ptrs as create_proof_r1cs_batch takes them.  Returns one
    (first or None, count) per item."""
    if count is None:
        if device_ptrs is not None:
            raise ValueError("check_r1cs_batch: count is required with device_ptrs")
        count = len(inputs)
    src, keep = _batch_witness_args(r1cs, inputs, aux, count, device_ptrs)
    first = np.zeros(max(count, 1), np.uint64)
    n_unsat = np.zeros(max(count, 1), np.uint64)
    _check(load_library().bb_r1cs_check_batch(r1cs.worker._h, r1cs._h, *src, _ptr(first), _ptr(n_unsat)))
    del keep
    return [(_first_or_none(int(f)), int(k)) for f, k in zip(first[:count], n_unsat[:count])]


def create_proof_r1cs(r1cs, params, input_assignment, aux_assignment, r, s, device_ptrs=None):
    """create_proof from the witness alone (bb_groth16_prove_r1cs): the bytes create_proof gives for the
    ProvingAssignment synthesis would have built.  device_ptrs: optional dict inputs, aux -> device addresses (the
    witness resident in HBM; input_assignment / aux_assignment are then ignored)."""
    if device_ptrs is not None:
        input_assignment, aux_assignment = device_ptrs["inputs"], device_ptrs["aux"]
    src, keep = r1cs._witness_args(input_assignment, aux_assignment, device_ptrs is not None)
    proof = (C.c_uint8 * 192)()
    _check(load_library().bb_groth16_prove_r1cs(params.worker._h, params._h, r1cs._h, *src, _scalar_bytes(r), _scalar_bytes(s), proof))
    del keep
    return bytes(proof)


class _ProveState(C.c_void_p):
    """a bb_prove handle that keeps the host witness it was begun from alive until prove_end"""


def prove_r1cs_begin(r1cs, params, input_assignment, aux_assignment, own=0, evals=None, device_ptrs=None):
    """bb_groth16_prove_r1cs_begin on any key, sharded or not -> the state bellman_b200.prove_end(state, evals) ends.
    evals = three device addresses (m Fr each; split mode): the polynomials whose bit is set in `own` (1 = a, 2 = b, 4 = c)
    are evaluated from the witness straight into theirs and taken through ifft + coset_fft, ahead of the witness MSMs;
    h_coset_evals_wait(worker) waits for them, and prove_end takes the three vectors once every rank's are there.
    evals = None (replicated mode, own = 0): the whole H pipeline runs here and prove_end takes no vectors.  Witness
    arguments as create_proof_r1cs's."""
    if device_ptrs is not None:
        input_assignment, aux_assignment = device_ptrs["inputs"], device_ptrs["aux"]
    src, keep = r1cs._witness_args(input_assignment, aux_assignment, device_ptrs is not None)
    d_evals = None if evals is None else (C.c_void_p * 3)(*(_addr(p) for p in evals))
    state = _ProveState()
    _check(load_library().bb_groth16_prove_r1cs_begin(params.worker._h, params._h, r1cs._h, *src, C.c_uint(own), d_evals, C.byref(state)))
    state.keep = keep
    return state


def create_random_proof_r1cs(r1cs, params, input_assignment, aux_assignment, rng=None, device_ptrs=None):
    """create_random_proof (prover.rs:164-179) from the witness alone: r, s <- Fr::random, then create_proof_r1cs"""
    import secrets
    draw = rng.randrange if rng is not None else secrets.randbelow
    return create_proof_r1cs(r1cs, params, input_assignment, aux_assignment, draw(FR_MODULUS), draw(FR_MODULUS), device_ptrs)



def create_proof_r1cs_batch(r1cs, params, inputs, aux, rs, ss, device_ptrs=None):
    """bb_groth16_prove_r1cs_batch: create_proof_r1cs for len(rs) witnesses of this constraint system in one call.
    inputs / aux: one witness per item (count x n_inputs and count x n_aux Fr), or device_ptrs = dict inputs, aux -> device
    addresses of those two row-major arrays.  Returns one entry per item: its 192 bytes, or the exception
    create_proof_r1cs would raise for it alone (an instance, not raised)."""
    from . import _batch_result, _scalars_bytes
    count = len(rs)
    if len(ss) != count:
        raise ValueError("create_proof_r1cs_batch: one r and one s per item")
    if device_ptrs is not None:
        src = (C.c_void_p(_addr(device_ptrs["inputs"])), C.c_size_t(r1cs.n_inputs), C.c_void_p(_addr(device_ptrs["aux"])),
               C.c_size_t(r1cs.n_aux), C.c_size_t(count), C.c_int(1))
        keep = ()
    else:
        inp = np.ascontiguousarray(np.asarray(inputs, dtype=np.uint64).reshape(count, -1, 4))
        ax = np.ascontiguousarray(np.asarray(aux, dtype=np.uint64).reshape(count, -1, 4))
        src = (_ptr(inp), C.c_size_t(inp.shape[1]), _ptr(ax), C.c_size_t(ax.shape[1]), C.c_size_t(count), C.c_int(0))
        keep = (inp, ax)
    proofs = (C.c_uint8 * (192 * max(count, 1)))()
    status = (C.c_int * max(count, 1))()
    rc = load_library().bb_groth16_prove_r1cs_batch(params.worker._h, params._h, r1cs._h, *src, _scalars_bytes(rs), _scalars_bytes(ss),
                                                    proofs, status)
    del keep
    return _batch_result(params, rc, proofs, list(status)[:count])


def create_random_proof_r1cs_batch(r1cs, params, inputs, aux, count=None, rng=None, device_ptrs=None):
    """create_random_proof_r1cs for each witness: fresh (r, s) per item, then create_proof_r1cs_batch"""
    import secrets
    draw = rng.randrange if rng is not None else secrets.randbelow
    count = len(inputs) if count is None else count
    rs, ss = [], []
    for _ in range(count):
        rs.append(draw(FR_MODULUS))
        ss.append(draw(FR_MODULUS))
    return create_proof_r1cs_batch(r1cs, params, inputs, aux, rs, ss, device_ptrs)
