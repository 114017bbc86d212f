"""groth16::generate_parameters on the device (SURVEY.md section 8f, rank 3).

Mirrors bellman/groth16/src/generator.rs:159-507 from the point where the circuit has
been synthesised into a KeypairAssembly (:43-155, :188-191):

  * the powers of tau (:249-264) and the H-query scalars tau^i t(tau)/delta (:267-296) are
    produced by the domain kernels (`distribute_powers`, scale);
  * the Lagrange coefficients L_j(tau) come from one inverse NTT (:300);
  * every group element -- h, a, b_g1, b_g2, ic/l and the verifying key -- is a fixed-base
    multiplication on the device (`bb_fixed_base_mul`; the reference uses a wNAF table per thread
    and batch normalisation, :209-226,271-296,310-415);
  * the per-variable QAP evaluations (:376-415) are sparse dot products with L_j(tau); they are
    O(non-zeros) field operations and stay on the host, as integers.

g1 and g2 are the standard generators scaled by `g1_scalar` / `g2_scalar` (generate_random_parameters
draws random generators, :21-40; a random multiple of a fixed generator is the same distribution).
The result maps the names of groth16::Parameters (vk_g1 = alpha, beta, delta; vk_g2 = beta, gamma,
delta; ic, h, l, a, b_g1, b_g2) to Montgomery-limb arrays, the layout `Parameters(worker, p)` and
`params_io.write_parameters` take.
"""
import ctypes as C

import numpy as np

from . import (EvaluationDomain, G1, G2, FORM_CANONICAL, SynthesisError, UnexpectedIdentity, _c64, _check, _ERRORS, fixed_base_mul,
               load_library)

FR_MODULUS = EvaluationDomain.FR_MODULUS
_R = 1 << 256
_R_INV = pow(_R, -1, FR_MODULUS)


class UnconstrainedVariable(SynthesisError):
    """SynthesisError::UnconstrainedVariable (generator.rs:466-470).  From the device generator: `index`, the first aux
    variable whose l element is the identity."""

    def __init__(self, message, index=None):
        super().__init__(message)
        self.index = index


BB_ERR_UNCONSTRAINED_VARIABLE = 4
_ERRORS[BB_ERR_UNCONSTRAINED_VARIABLE] = UnconstrainedVariable


class KeypairAssembly:
    """generator.rs:43-155: per variable, the (coefficient, constraint index) pairs of the A, B and
    C matrices.  Variables are ("input", i) or ("aux", i); linear combinations are lists of
    (variable, coefficient)."""

    def __init__(self):
        self.num_inputs = self.num_aux = self.num_constraints = 0
        self.at_inputs, self.bt_inputs, self.ct_inputs = [], [], []
        self.at_aux, self.bt_aux, self.ct_aux = [], [], []

    def alloc(self):                                          # :58-75
        self.num_aux += 1
        for m in (self.at_aux, self.bt_aux, self.ct_aux):
            m.append([])
        return ("aux", self.num_aux - 1)

    def alloc_input(self):                                    # :77-94
        self.num_inputs += 1
        for m in (self.at_inputs, self.bt_inputs, self.ct_inputs):
            m.append([])
        return ("input", self.num_inputs - 1)

    def enforce(self, a, b, c):                               # :96-138
        for lc, inputs, aux in ((a, self.at_inputs, self.at_aux), (b, self.bt_inputs, self.bt_aux), (c, self.ct_inputs, self.ct_aux)):
            for (kind, idx), coeff in lc:
                (inputs if kind == "input" else aux)[idx].append((coeff % FR_MODULUS, self.num_constraints))
        self.num_constraints += 1


def _to_limbs(values):
    out = np.zeros((len(values), 4), dtype=np.uint64)
    for i, v in enumerate(values):
        for j in range(4):
            out[i, j] = (v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    return out


def _mont_to_ints(arr):
    a = np.ascontiguousarray(arr, dtype=np.uint64).reshape(-1, 4)
    return [(int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192) * _R_INV % FR_MODULUS for r in a]


def generate_parameters(worker, assembly, alpha, beta, gamma, delta, tau, g1_scalar=1, g2_scalar=1):
    """`assembly`: the KeypairAssembly as `circuit.synthesize` leaves it (ONE already allocated as
    input 0, generator.rs:188-191).  alpha..tau: integers mod r."""
    q = FR_MODULUS
    import copy
    asm = copy.deepcopy(assembly)                             # the caller's assembly is left as synthesis made it
    for i in range(asm.num_inputs):                           # x_i * 0 = 0, :195-202
        asm.enforce([(("input", i), 1)], [], [])
    dom = EvaluationDomain.from_coeffs(worker, np.zeros((asm.num_constraints, 4), dtype=np.uint64))   # :205-206
    m = dom.coeffs.shape[0]
    if gamma % q == 0 or delta % q == 0:                      # :228-243
        raise UnexpectedIdentity("gamma or delta is not invertible")
    gamma_inverse, delta_inverse = pow(gamma, -1, q), pow(delta, -1, q)
    g1s, g2s = g1_scalar % q, g2_scalar % q

    def g1_mul(ints):
        return fixed_base_mul(worker, G1, _to_limbs([v * g1s % q for v in ints]), FORM_CANONICAL)

    def g2_mul(ints):
        return fixed_base_mul(worker, G2, _to_limbs([v * g2s % q for v in ints]), FORM_CANONICAL)

    # powers of tau (:249-264), then the H query g1^(tau^i t(tau)/delta) for i < m-1 (:267-296)
    dom.coeffs[:] = EvaluationDomain._to_mont(1)
    dom.distribute_powers(tau)
    hq = EvaluationDomain(worker, dom.coeffs.copy(), dom.exp)
    hq._pointwise(2, k=dom.z(tau) * delta_inverse * g1s % q)
    h = fixed_base_mul(worker, G1, hq.coeffs[: m - 1])        # Montgomery scalars straight from the kernel
    dom.ifft()                                                # Lagrange coefficients at tau, :300
    lag = _mont_to_ints(dom.coeffs)

    def eval_at_tau(terms):                                   # :376-389
        acc = 0
        for coeff, index in terms:
            acc += lag[index] * coeff
        return acc % q

    def evaluate(at, bt, ct, inv):                            # :310-415
        a_t = [eval_at_tau(t) for t in at]
        b_t = [eval_at_tau(t) for t in bt]
        c_t = [eval_at_tau(t) for t in ct]
        ext = [(a * beta + b * alpha + c) % q * inv % q for a, b, c in zip(a_t, b_t, c_t)]
        return a_t, b_t, ext

    a_in, b_in, ic_k = evaluate(asm.at_inputs, asm.bt_inputs, asm.ct_inputs, gamma_inverse)
    a_aux, b_aux, l_k = evaluate(asm.at_aux, asm.bt_aux, asm.ct_aux, delta_inverse)
    if any(v == 0 for v in l_k):                              # an identity in L, :466-470
        raise UnconstrainedVariable("auxiliary variable %d is unconstrained" % l_k.index(0))
    a_k = [v for v in a_in + a_aux if v]                      # identities are filtered out, :491-505
    b_k = [v for v in b_in + b_aux if v]
    return dict(
        vk_g1=g1_mul([alpha, beta, delta]), vk_g2=g2_mul([beta, gamma, delta]),
        ic=g1_mul(ic_k), h=h, l=g1_mul(l_k), a=g1_mul(a_k), b_g1=g1_mul(b_k), b_g2=g2_mul(b_k),
        num_inputs=asm.num_inputs, num_aux=asm.num_aux, m=m)


# --------------------------------------------------------------------------------------------
# the whole generator on the device (bb_groth16_generate, csrc/generate.cu)
# --------------------------------------------------------------------------------------------
class _Toxic(C.Structure):
    """bb_toxic"""
    _fields_ = [("g1", C.c_void_p), ("g2", C.c_void_p), ("alpha", C.c_uint8 * 32), ("beta", C.c_uint8 * 32), ("gamma", C.c_uint8 * 32),
                ("delta", C.c_uint8 * 32), ("tau", C.c_uint8 * 32)]


class GenerateReport(C.Structure):
    """bb_generate_report"""
    _fields_ = [("len", C.c_size_t * 6), ("m", C.c_size_t), ("unconstrained", C.c_size_t)]


def _device_generate(worker, r1cs, toxic):
    from . import Parameters
    from .verifier import PreparedVerifyingKey
    crs, vk, rep = C.c_void_p(), C.c_void_p(), GenerateReport()
    rc = load_library().bb_groth16_generate(worker._h, r1cs._h, C.byref(toxic) if toxic is not None else None, C.byref(crs), C.byref(vk),
                                            C.byref(rep))
    if rc == BB_ERR_UNCONSTRAINED_VARIABLE:
        raise UnconstrainedVariable(load_library().bb_last_error().decode(errors="replace"), index=int(rep.unconstrained))
    _check(rc)
    lens = dict(zip(("ic", "h", "l", "a", "b_g1", "b_g2"), (int(v) for v in rep.len)))
    return Parameters._from_handle(worker, crs, lens), PreparedVerifyingKey._from_handle(worker, vk, lens["ic"])


def generate_parameters_device(worker, r1cs, alpha, beta, gamma, delta, tau, g1=None, g2=None):
    """generate_parameters (generator.rs:159-507) for the constraint system resident in `r1cs` (an R1CS of this worker),
    computed on the device -> (Parameters, PreparedVerifyingKey).  alpha..tau: integers in [0, r).  g1, g2: the generators
    as affine points in the library's format ((12,) / (24,) uint64 Montgomery), None = the standard ones.  The same points
    generate_parameters gives for the KeypairAssembly the constraint system was built from (with g1_scalar, g2_scalar:
    g1 = [g1_scalar] G1).  Raises UnexpectedIdentity (gamma or delta zero), UnconstrainedVariable (with .index) or
    BackendError for bad arguments."""
    t = _Toxic()
    keep = []
    for name, g, width in (("g1", g1, 12), ("g2", g2, 24)):
        if g is not None:
            arr = _c64(g, width).copy()
            keep.append(arr)
            setattr(t, name, arr.ctypes.data)
    for name, v in (("alpha", alpha), ("beta", beta), ("gamma", gamma), ("delta", delta), ("tau", tau)):
        v = int(v)
        if not 0 <= v < 1 << 256:
            raise ValueError(f"{name} is not a 256-bit integer")
        getattr(t, name)[:] = v.to_bytes(32, "little")
    try:
        return _device_generate(worker, r1cs, t)
    finally:
        C.memset(C.addressof(t), 0, C.sizeof(t))
        del keep


def generate_random_parameters_device(worker, r1cs):
    """generate_random_parameters (generator.rs:21-40) on the device: the toxic waste and the generators are drawn by the
    library from the operating system and never leave it -> (Parameters, PreparedVerifyingKey)"""
    return _device_generate(worker, r1cs, None)
