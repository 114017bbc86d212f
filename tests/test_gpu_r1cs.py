"""The constraint system on the device (bb_r1cs_*, bb_groth16_prove_r1cs, csrc/r1cs.cu; bellman_b200.r1cs) against
oracle-0's ProvingAssignment (oracle/oracle0/bellman.py: synthesize_witness): a, b, c element for element, the three
densities bit for bit, and proofs byte for byte against create_proof on the host-evaluated assignment and the oracle's
prover.  tests/test_emulated_r1cs.py runs the same bodies on the emulated device (tests/native/) at the sizes a host
reaches; this file adds the sizes only a device reaches (a row of 2^16 terms, the 2^20 MiMC workload).
"""
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import generator as GEN
from bellman_b200 import r1cs as RC
from oracle import o1
from oracle.oracle0 import bellman as B
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

from test_gpu_parity import _AssemblyAdapter
from test_gpu_verify import abi_proof

pytestmark = pytest.mark.gpu

R = F.FR_MODULUS
ARG = "[bb_status 16]"


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def fr(ints):
    return o1.fr_from_ints([int(v) % R for v in ints]) if len(ints) else np.zeros((0, 4), np.uint64)


def synthesize(circuit):
    """one circuit through both recorders: oracle-0's ProvingAssignment (the witness) and the product's KeypairAssembly"""
    pa = B.synthesize_witness(B.Bls12, circuit)
    asm = GEN.KeypairAssembly()
    asm.alloc_input()                                          # ONE, generator.rs:188
    circuit(_AssemblyAdapter(asm))
    return pa, asm


def device_copy(worker, arr):
    p = worker.device_alloc(max(arr.nbytes, 32))
    if arr.nbytes:
        worker.upload(p, arr)
    return p


def check_eval(worker, r1cs, inputs, aux, want_abc, want_dens):
    """a, b, c from host and from device witness memory, into host and into device memory, and the densities"""
    inp, ax = fr(inputs), fr(aux)
    want = [fr(v) for v in want_abc]
    n = r1cs.n_constraints
    assert n == len(want_abc[0])
    results = [r1cs.eval(inp, ax)]
    d_in, d_aux = device_copy(worker, inp), device_copy(worker, ax)
    results.append(r1cs.eval(d_in, d_aux, on_device=True))
    outs = {k: worker.device_alloc(n * 32) for k in "abc"}
    r1cs.eval(d_in, d_aux, on_device=True, out=outs)
    got = []
    for k in "abc":
        h = np.zeros((n, 4), np.uint64)
        worker.download(outs[k], h)
        got.append(h)
    results.append(tuple(got))
    for p in (d_in, d_aux, *outs.values()):
        worker.device_free(p)
    for res in results:
        for name, g, w in zip("abc", res, want):
            assert np.array_equal(g, w), name
    for name, g, w in zip(("a_aux", "b_input", "b_aux"), r1cs.densities(), want_dens):
        assert g.tolist() == [bool(x) for x in w], name


def check_circuit(worker, circuit):
    pa, asm = synthesize(circuit)
    r1cs = RC.R1CS.from_assembly(worker, asm)
    assert (r1cs.n_inputs, r1cs.n_aux) == (len(pa.input_assignment), len(pa.aux_assignment))
    check_eval(worker, r1cs, pa.input_assignment, pa.aux_assignment, (pa.a, pa.b, pa.c),
               (pa.a_aux_density, pa.b_input_density, pa.b_aux_density))
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 1. bb_r1cs_eval against ProvingAssignment
# --------------------------------------------------------------------------------------------
def test_eval_xor_demo(worker):
    for a, b in ((0, 0), (1, 0), (1, 1)):
        check_circuit(worker, B.xor_demo(a, b))


def test_eval_zero_coeffs(worker):
    """groth16/src/tests/mod.rs:375-440: a zero coefficient marks no density, whether on ONE or on an aux variable"""
    for one_var in (True, False):
        check_circuit(worker, B.mult_with_zero_coeffs(5, 6, 30, one_var))


def test_eval_mimc322(worker):
    rng = random.Random(30)
    constants = [rng.randrange(R) for _ in range(322)]
    check_circuit(worker, B.mimc_circuit(B.Bls12.fr, rng.randrange(R), rng.randrange(R), constants))


def random_system(rng, n_rows, n_inputs, n_aux, lengths):
    """rows of (var, coeff) per matrix: `lengths` planted in each matrix, plus empty rows, all-zero-coefficient rows and
    cancelling duplicate terms; coefficients 0, 1, r - 1 and random values"""
    nv = n_inputs + n_aux

    def coeff():
        return rng.choice((0, 1, 1, R - 1, rng.randrange(R), rng.randrange(R)))

    mats = []
    for _ in range(3):
        rows = [[(rng.randrange(nv), coeff()) for _ in range(rng.randrange(4))] for _ in range(n_rows)]
        slots = rng.sample(range(n_rows), len(lengths) + 3)
        for slot, ln in zip(slots, lengths):
            rows[slot] = [(rng.randrange(nv), coeff()) for _ in range(ln)]
        rows[slots[-3]] = []                                                   # empty
        rows[slots[-2]] = [(rng.randrange(nv), 0) for _ in range(3)]           # all coefficients zero
        v, k = rng.randrange(nv), rng.randrange(1, R)
        rows[slots[-1]] = [(v, k), (rng.randrange(nv), 0), (v, R - k)]         # cancels: value 0, density set
        mats.append(rows)
    return mats


def reference(mats, z, n_inputs, n_aux):
    """ProvingAssignment::enforce (prover.rs:19-55,105-145) over the rows, then the input rows of :208-215"""
    vals = [[sum(c * z[v] for v, c in row) % R for row in rows] + ([z[i] for i in range(n_inputs)] if m == 0 else [0] * n_inputs)
            for m, rows in enumerate(mats)]
    a_aux, b_in, b_aux = [False] * n_aux, [False] * n_inputs, [False] * n_aux
    for m, rows in enumerate(mats):
        for row in rows:
            for v, c in row:
                if c % R == 0:
                    continue
                if v >= n_inputs and m == 0:
                    a_aux[v - n_inputs] = True
                if m == 1:
                    if v < n_inputs:
                        b_in[v] = True
                    else:
                        b_aux[v - n_inputs] = True
    return vals, (a_aux, b_in, b_aux)


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    terms = [t for r in rows for t in r]
    return off, np.array([v for v, _ in terms], np.uint32), RC._mont_limbs([c for _, c in terms])


def check_random(worker, seed, total_rows, lengths, n_inputs=3, n_aux=50):
    rng = random.Random(seed)
    n_rows = total_rows - n_inputs
    mats = random_system(rng, n_rows, n_inputs, n_aux, lengths)
    z = [1] + [rng.randrange(R) for _ in range(n_inputs + n_aux - 1)]
    vals, dens = reference(mats, z, n_inputs, n_aux)
    r1cs = RC.R1CS(worker, n_inputs, n_aux, *(csr(rows) for rows in mats))
    assert r1cs.n_constraints == total_rows
    check_eval(worker, r1cs, z[:n_inputs], z[n_inputs:], vals, dens)
    r1cs.free()


EMU_LENGTHS = (1, 31, 32, 33, 1000, 4096)


def test_eval_random(worker, big=True):
    """row lengths across the three kernels (one thread, one warp, one CTA per row); 2^k and 2^k + 1 constraints"""
    lengths = EMU_LENGTHS + ((1 << 16),) if big else EMU_LENGTHS
    for seed, total in ((1, 1 << 9), (2, (1 << 9) + 1)):
        check_random(worker, seed, total, lengths)


# --------------------------------------------------------------------------------------------
# 2. proof bytes
# --------------------------------------------------------------------------------------------
def assignment(wit):
    return bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"], wit["a_aux_density"],
                                wit["b_input_density"], wit["b_aux_density"])


def test_prove_mimc322(worker):
    """bb_synth_mimc_r1cs is the circuit of the oracle's MiMC case of the same seed: create_proof_r1cs from the witness
    equals create_proof on the host-evaluated assignment and the oracle's prover, from host and from device memory"""
    rng = random.Random(31)
    mc = o1.Mimc(322, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    wit = mc.witness()
    r1cs = RC.R1CS.synth_mimc(worker, 322, 5)
    got = r1cs.eval(wit["inputs"], wit["aux"])
    for k, g in zip("abc", got):
        assert np.array_equal(g, wit[k]), k
    for g, k in zip(r1cs.densities(), ("a_aux_density", "b_input_density", "b_aux_density")):
        assert g.tolist() == [bool(x) for x in wit[k]], k
    r, s = rng.randrange(R), rng.randrange(R)
    want = mc.prove(r, s)
    assert bb.create_proof(assignment(wit), params, r, s) == want
    assert RC.create_proof_r1cs(r1cs, params, wit["inputs"], wit["aux"], r, s) == want
    d = {"inputs": device_copy(worker, wit["inputs"]), "aux": device_copy(worker, wit["aux"])}
    assert RC.create_proof_r1cs(r1cs, params, None, None, r, s, device_ptrs=d) == want
    for p in d.values():
        worker.device_free(p)


def test_prove_generated_key_verifies(worker, rounds=40):
    """one synthesis gives the key (generate_parameters) and the device R1CS (from_assembly); the proof from the witness
    equals create_proof on the oracle's assignment and verifies with the device verify_proof"""
    from bellman_b200 import params_io
    rng = random.Random(32)
    constants = [rng.randrange(R) for _ in range(rounds)]
    circuit = B.mimc_circuit(B.Bls12.fr, rng.randrange(R), rng.randrange(R), constants)
    pa, asm = synthesize(circuit)
    toxic = [rng.randrange(1, R) for _ in range(5)]
    key = GEN.generate_parameters(worker, asm, *toxic)
    params = bb.Parameters(worker, params_io.read_parameters(params_io.write_parameters(key), worker=worker))
    r1cs = RC.R1CS.from_assembly(worker, asm)
    inp, aux = fr(pa.input_assignment), fr(pa.aux_assignment)
    asg = bb.ProvingAssignment(fr(pa.a), fr(pa.b), fr(pa.c), inp, aux, pa.a_aux_density, pa.b_input_density, pa.b_aux_density)
    r, s = rng.randrange(R), rng.randrange(R)
    proof = RC.create_proof_r1cs(r1cs, params, inp, aux, r, s)
    assert proof == bb.create_proof(asg, params, r, s)
    pvk = bb.prepare_verifying_key(worker, {"alpha_g1": key["vk_g1"][0], "beta_g2": key["vk_g2"][0], "gamma_g2": key["vk_g2"][1],
                                            "delta_g2": key["vk_g2"][2], "ic": key["ic"]})
    x = pa.input_assignment[1:]
    bb.verify_proof(pvk, abi_proof(PR.proof_read(proof)), x)
    other = RC.create_random_proof_r1cs(r1cs, params, inp, aux, rng=rng)       # fresh (r, s): a different, valid proof
    assert other != proof
    bb.verify_proof(pvk, abi_proof(PR.proof_read(other)), x)
    with pytest.raises(bb.InvalidProof):
        bb.verify_proof(pvk, abi_proof(PR.proof_read(proof)), [(x[0] + 1) % R])
    pvk.free()


# --------------------------------------------------------------------------------------------
# 3. errors
# --------------------------------------------------------------------------------------------
def test_errors(worker):
    rng = random.Random(33)
    good = [[[(0, 1), (4, 5)], [(3, R - 1)]], [[(1, 7)], []], [[], [(4, 1)]]]     # 2 rows; 2 inputs, 3 aux

    def make(mats, n_inputs=2, n_aux=3, edit=None):
        parts = [list(csr(rows)) for rows in mats]
        if edit:
            edit(parts)
        return RC.R1CS(worker, n_inputs, n_aux, *parts)

    def no_device_work(fn, match):
        l0, b0 = worker.kernel_launches, worker.bytes_copied()
        with pytest.raises(bb.BackendError, match=match) as e:
            fn()
        assert ARG in str(e.value)
        assert (worker.kernel_launches, worker.bytes_copied()) == (l0, b0)

    def set_off(m, k, v):
        def f(parts):
            parts[m][0][k] = v
        return f

    def big_coeff(parts):
        parts[0][2][1] = np.array([(R >> (64 * j)) & RC._MASK64 for j in range(4)], np.uint64)   # the integer r itself

    no_device_work(lambda: make(good, n_inputs=0, n_aux=5), "no inputs")
    no_device_work(lambda: make([[[(5, 1)], []], good[1], good[2]]), "variable 5 of 5")
    no_device_work(lambda: make(good, edit=set_off(1, 0, 1)), "row_offsets")
    no_device_work(lambda: make(good, edit=set_off(0, 2, 1)), "decrease")
    no_device_work(lambda: make(good, edit=big_coeff), "coefficient not below r")
    r1cs = make(good)
    z = fr([1] + [rng.randrange(R) for _ in range(4)])
    r1cs.eval(z[:2], z[2:])
    no_device_work(lambda: r1cs.eval(z[:2], z[2:4]), "witness has 2 inputs and 2 aux")
    no_device_work(lambda: r1cs.eval(z[:1], z[1:]), "witness has 1 inputs and 4 aux")

    # key errors: exactly bb_groth16_prove's, in its precedence
    mc = o1.Mimc(20, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    wit = mc.witness()
    asg = assignment(wit)
    mimc = RC.R1CS.synth_mimc(worker, 20, 5)
    base = mc.export_params()
    r, s = rng.randrange(R), rng.randrange(R)
    params = bb.Parameters(worker, base)
    no_device_work(lambda: RC.create_proof_r1cs(mimc, params, wit["inputs"], wit["aux"][:-1], r, s), "witness has")

    def variant(**changes):
        p = {k: np.array(v, copy=True) for k, v in base.items()}
        for k, f in changes.items():
            p[k] = f(p[k])
        return bb.Parameters(worker, p)

    def short(v):                       # the B query no longer matches the densities: the MSM runs out of bases
        return v.reshape(-1, v.shape[-1])[:-1]

    def zero_delta(v):
        v = v.reshape(3, -1).copy()
        v[2] = 0
        return v

    for key, exc in ((variant(b_g1=short), bb.IoError), (variant(a=short), bb.IoError),
                     (variant(vk_g1=zero_delta), bb.UnexpectedIdentity),
                     (variant(vk_g1=zero_delta, b_g1=short), bb.UnexpectedIdentity)):
        with pytest.raises(exc) as want:
            bb.create_proof(asg, key, r, s)
        with pytest.raises(exc) as got:
            RC.create_proof_r1cs(mimc, key, wit["inputs"], wit["aux"], r, s)
        assert str(got.value) == str(want.value)


# --------------------------------------------------------------------------------------------
# 4. the bench workload: bb_synth_mimc_r1cs against bb_synth_mimc_witness
# --------------------------------------------------------------------------------------------
def check_synth(worker, log_n):
    rounds = (1 << (log_n - 1)) - 1
    asg, shape = bb.synth_mimc(rounds, seed=20)
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    assert r1cs.n_constraints == shape["num_constraints"] == 1 << log_n
    assert r1cs.nnz == (3 * rounds + 2, 4 * rounds, 3 * rounds) and r1cs.unit[0] == 2 * rounds + 2
    for k, g in zip("abc", r1cs.eval(asg.input_assignment, asg.aux_assignment)):
        assert np.array_equal(g, getattr(asg, k)), k
    for g, k in zip(r1cs.density_words(), ("a_aux_density", "b_input_density", "b_aux_density")):
        assert np.array_equal(g, getattr(asg, k)), k
    params = bb.Parameters.synthetic(worker, 21, shape)
    r, s = 0x1234567, 0x7654321
    assert RC.create_proof_r1cs(r1cs, params, asg.input_assignment, asg.aux_assignment, r, s) == bb.create_proof(asg, params, r, s)
    params.free()
    r1cs.free()


def test_synth_mimc_2_20(worker):
    check_synth(worker, 20)
