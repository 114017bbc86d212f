"""Checking witnesses against the constraint system on the device (bb_r1cs_check, bb_r1cs_check_batch, csrc/r1cs.cu;
R1CS.unsatisfied / which_is_unsatisfied / is_satisfied and check_r1cs_batch in bellman_b200.r1cs) against a Python-integer
evaluation of every row (test_gpu_r1cs.reference): the first failing row, the count and the bitmap, from host and from
device witnesses.  tests/test_emulated_r1cs_check.py runs the same bodies on the emulated device at the sizes a host
reaches; this file adds rows of more than 2048 terms and the 2^20 MiMC workload.
"""
import ctypes as C
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import r1cs as RC
from oracle import o1
from oracle.oracle0 import bellman as B

from test_gpu_r1cs import ARG, csr, device_copy, fr, random_system, reference, synthesize

pytestmark = pytest.mark.gpu

R = o1.FR_MODULUS


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def failing_rows(mats, z, n_inputs, n_aux):
    """which_is_unsatisfied over every row in Python integers: the rows k with a_k b_k != c_k, input rows included"""
    vals, _ = reference(mats, z, n_inputs, n_aux)
    return [k for k, (a, b, c) in enumerate(zip(*vals)) if a * b % R != c]


def check_unsat(worker, r1cs, z, rows):
    """bb_r1cs_check from host and from device witnesses against the failing `rows`: first, count and bitmap, the
    bellman-named forms, and a one-item batch of each kind"""
    ni, n = r1cs.n_inputs, r1cs.n_constraints
    inp, ax = fr(z[:ni]), fr(z[ni:])
    want = (rows[0] if rows else None, len(rows))
    want_bits = np.zeros(n, bool)
    want_bits[rows] = True
    d = {"inputs": device_copy(worker, inp), "aux": device_copy(worker, ax)}
    for args in ((inp, ax, False), (d["inputs"], d["aux"], True)):
        first, count, bits = r1cs.unsatisfied(*args, bits=True)
        assert (first, count) == want
        assert np.array_equal(bits, want_bits)
        assert r1cs.unsatisfied(*args) == want
        assert r1cs.which_is_unsatisfied(*args) == want[0]
        assert r1cs.is_satisfied(*args) == (not rows)
    assert RC.check_r1cs_batch(r1cs, inp[None], ax[None]) == [want]
    assert RC.check_r1cs_batch(r1cs, None, None, count=1, device_ptrs=d) == [want]
    for p in d.values():
        worker.device_free(p)


def changed(rng, v):
    return (v + rng.randrange(1, R)) % R


def corruptions(rng, z, n_inputs, n_aux):
    """the witness as given, one aux value changed, three aux values changed, input 0 = 2"""
    one = list(z)
    j = n_inputs + rng.randrange(n_aux)
    one[j] = changed(rng, one[j])
    several = list(z)
    for j in rng.sample(range(n_inputs, n_inputs + n_aux), min(3, n_aux)):
        several[j] = changed(rng, several[j])
    bad_one = list(z)
    bad_one[0] = 2
    return [list(z), one, several, bad_one]


def check_cases(worker, r1cs, mats, cases, n_inputs, n_aux):
    """check_unsat for each witness against the Python evaluation; the first holds, and some later one does not"""
    fails = [failing_rows(mats, zz, n_inputs, n_aux) for zz in cases]
    assert not fails[0] and any(fails[1:])
    for zz, rows in zip(cases, fails):
        check_unsat(worker, r1cs, zz, rows)
    return fails


def assembly_rows(asm):
    """KeypairAssembly's per-variable (coefficient, row) lists as rows of (variable, coefficient) per matrix"""
    mats = []
    for inputs, aux in ((asm.at_inputs, asm.at_aux), (asm.bt_inputs, asm.bt_aux), (asm.ct_inputs, asm.ct_aux)):
        rows = [[] for _ in range(asm.num_constraints)]
        for base, per_var in ((0, inputs), (asm.num_inputs, aux)):
            for j, terms in enumerate(per_var):
                for coeff, row in terms:
                    rows[row].append((base + j, coeff))
        mats.append(rows)
    return mats


def check_circuit(worker, circuit, seed):
    rng = random.Random(seed)
    pa, asm = synthesize(circuit)
    r1cs = RC.R1CS.from_assembly(worker, asm)
    mats, ni, na = assembly_rows(asm), asm.num_inputs, asm.num_aux
    z = [int(v) % R for v in list(pa.input_assignment) + list(pa.aux_assignment)]
    check_cases(worker, r1cs, mats, corruptions(rng, z, ni, na), ni, na)
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 1. circuits: satisfied and corrupted witnesses
# --------------------------------------------------------------------------------------------
def test_check_xor_demo(worker):
    for a, b in ((0, 0), (1, 0), (1, 1)):
        check_circuit(worker, B.xor_demo(a, b), 40 + 2 * a + b)


def test_check_zero_coeffs(worker):
    for one_var in (True, False):
        check_circuit(worker, B.mult_with_zero_coeffs(5, 6, 30, one_var), 44 + one_var)


def test_check_mimc322_circuit(worker):
    rng = random.Random(30)
    constants = [rng.randrange(R) for _ in range(322)]
    check_circuit(worker, B.mimc_circuit(B.Bls12.fr, rng.randrange(R), rng.randrange(R), constants), 46)


def test_check_mimc322_oracle(worker):
    """oracle-1's MiMC-322 witness against bb_synth_mimc_r1cs of the same seed: satisfied, then corrupted (rows from
    the matrices in Python integers)"""
    rng = random.Random(47)
    wit = o1.Mimc(322, seed=5).witness()
    r1cs = RC.R1CS.synth_mimc(worker, 322, 5)
    mats = []
    for off, var, cf in RC.synth_mimc_matrices(322, 5):
        terms = list(zip(var.tolist(), o1.fr_to_ints(cf)))
        mats.append([terms[int(off[k]):int(off[k + 1])] for k in range(len(off) - 1)])
    z = o1.fr_to_ints(wit["inputs"]) + o1.fr_to_ints(wit["aux"])
    ni, na = r1cs.n_inputs, r1cs.n_aux
    check_cases(worker, r1cs, mats, corruptions(rng, z, ni, na), ni, na)
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 2. random systems over the three row kernels
# --------------------------------------------------------------------------------------------
def satisfiable_system(rng, total_rows, n_inputs, n_free, lengths):
    """random_system's rows over n_inputs + n_free variables, plus one aux variable per row that C_k holds with coefficient
    one and no other row reads: set to a_k b_k - (the rest of C_k) it satisfies row k, changed it fails row k alone.
    Returns the rows, a satisfying z and n_aux."""
    n_rows = total_rows - n_inputs
    mats = random_system(rng, n_rows, n_inputs, n_free, lengths)
    nv = n_inputs + n_free
    for k, row in enumerate(mats[2]):
        row.append((nv + k, 1))
    z = [1] + [rng.randrange(R) for _ in range(nv - 1)] + [0] * n_rows
    vals, _ = reference(mats, z, n_inputs, n_free + n_rows)
    for k in range(n_rows):
        z[nv + k] = (vals[0][k] * vals[1][k] - vals[2][k]) % R
    return mats, z, n_free + n_rows


def check_random(worker, seed, total_rows, lengths, n_inputs=3, n_free=50):
    rng = random.Random(seed)
    mats, z, na = satisfiable_system(rng, total_rows, n_inputs, n_free, lengths)
    r1cs = RC.R1CS(worker, n_inputs, na, *(csr(rows) for rows in mats))
    assert r1cs.n_constraints == total_rows
    n_rows, own = total_rows - n_inputs, n_inputs + n_free
    first, last = list(z), list(z)
    first[own] = changed(rng, z[own])                             # row 0 alone
    last[own + n_rows - 1] = changed(rng, z[own + n_rows - 1])    # the last constraint row alone
    fails = check_cases(worker, r1cs, mats, corruptions(rng, z, n_inputs, na) + [first, last], n_inputs, na)
    assert fails[-2:] == [[0], [n_rows - 1]]
    r1cs.free()


EMU_LENGTHS = (1, 31, 32, 33, 1000, 2048)


def test_check_random(worker, big=True):
    """rows of <= 32, 33..2048 and (GPU only) more than 2048 terms; 2^k and 2^k + 1 constraints"""
    lengths = EMU_LENGTHS + (2049, 4096, 1 << 16) if big else EMU_LENGTHS
    for seed, total in ((51, 1 << 9), (52, (1 << 9) + 1)):
        check_random(worker, seed, total, lengths)


# --------------------------------------------------------------------------------------------
# 3. batches
# --------------------------------------------------------------------------------------------
def test_check_batch(worker, lengths=(1, 40, 3000)):
    """satisfied and corrupted items mixed, from host and from device memory: item i's (first, count) is its single
    call's and the Python evaluation's; count = 0 is BB_OK and touches nothing"""
    rng = random.Random(53)
    ni = 2
    mats, z, na = satisfiable_system(rng, 200, ni, 20, lengths)
    r1cs = RC.R1CS(worker, ni, na, *(csr(rows) for rows in mats))
    own = ni + 20
    items = corruptions(rng, z, ni, na)
    for k in (0, 5, 197):
        zz = list(z)
        zz[own + k] = changed(rng, zz[own + k])
        items.append(zz)
    items.insert(3, list(z))
    want = []
    for zz in items:
        rows = failing_rows(mats, zz, ni, na)
        want.append((rows[0] if rows else None, len(rows)))
    assert want[0] == want[3] == (None, 0) and want[-3:] == [(0, 1), (5, 1), (197, 1)]
    inputs = np.stack([fr(zz[:ni]) for zz in items])
    aux = np.stack([fr(zz[ni:]) for zz in items])
    assert [r1cs.unsatisfied(i, a) for i, a in zip(inputs, aux)] == want
    assert RC.check_r1cs_batch(r1cs, inputs, aux) == want
    d = {"inputs": device_copy(worker, inputs), "aux": device_copy(worker, aux)}
    assert RC.check_r1cs_batch(r1cs, None, None, count=len(items), device_ptrs=d) == want
    assert RC.check_r1cs_batch(r1cs, None, None, count=3, device_ptrs=d) == want[:3]
    l0, b0 = worker.kernel_launches, worker.bytes_copied()
    assert RC.check_r1cs_batch(r1cs, [], [], count=0) == []
    assert RC.check_r1cs_batch(r1cs, None, None, count=0, device_ptrs=d) == []
    assert (worker.kernel_launches, worker.bytes_copied()) == (l0, b0)
    for p in d.values():
        worker.device_free(p)
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 4. argument errors: before any device work
# --------------------------------------------------------------------------------------------
def test_check_errors(worker):
    rng = random.Random(54)
    ni = 3
    mats, z, na = satisfiable_system(rng, 64, ni, 10, (1, 40))
    r1cs = RC.R1CS(worker, ni, na, *(csr(rows) for rows in mats))
    inp, ax = fr(z[:ni]), fr(z[ni:])
    lib = bb.load_library()
    first, count = C.c_size_t(), C.c_size_t()
    firsts = np.zeros(2, np.uint64)

    def no_device_work(fn, match, workers=(worker,)):
        before = [(w.kernel_launches, w.bytes_copied()) for w in workers]
        with pytest.raises(bb.BackendError, match=match) as e:
            fn()
        assert ARG in str(e.value)
        assert [(w.kernel_launches, w.bytes_copied()) for w in workers] == before

    def check(ctx, r, i, n_i, a, n_a, on_device, f, c, bits=None):
        bb._check(lib.bb_r1cs_check(ctx, r, i, C.c_size_t(n_i), a, C.c_size_t(n_a), C.c_int(on_device), f, c, bits))

    def check_batch(ctx, r, i, n_i, a, n_a, cnt, on_device, f, c=None):
        bb._check(lib.bb_r1cs_check_batch(ctx, r, i, C.c_size_t(n_i), a, C.c_size_t(n_a), C.c_size_t(cnt), C.c_int(on_device), f, c))

    assert r1cs.unsatisfied(inp, ax) == (None, 0)
    # the witness's shape
    no_device_work(lambda: r1cs.unsatisfied(inp, ax[:-1]), f"witness has 3 inputs and {na - 1} aux")
    no_device_work(lambda: r1cs.unsatisfied(inp[:2], ax), f"witness has 2 inputs and {na} aux")
    no_device_work(lambda: RC.check_r1cs_batch(r1cs, inp[None], ax[None, 1:]), "bb_r1cs_check_batch: witness has")
    # a constraint system of another context
    other = bb.Worker(0)
    no_device_work(lambda: check(other._h, r1cs._h, bb._ptr(inp), ni, bb._ptr(ax), na, 0, C.byref(first), C.byref(count)),
                   "another context", (worker, other))
    no_device_work(lambda: check_batch(other._h, r1cs._h, bb._ptr(inp), ni, bb._ptr(ax), na, 1, 0, bb._ptr(firsts)),
                   "another context", (worker, other))
    other.close()
    # NULL pointers
    args = (bb._ptr(inp), ni, bb._ptr(ax), na, 0)
    no_device_work(lambda: check(worker._h, None, *args, C.byref(first), C.byref(count)), "bb_r1cs_check: null argument")
    no_device_work(lambda: check(worker._h, r1cs._h, *args, None, C.byref(count)), "bb_r1cs_check: null argument")
    no_device_work(lambda: check(worker._h, r1cs._h, *args, C.byref(first), None), "bb_r1cs_check: null argument")
    no_device_work(lambda: check(worker._h, r1cs._h, None, ni, bb._ptr(ax), na, 0, C.byref(first), C.byref(count)), "null witness pointer")
    no_device_work(lambda: check(worker._h, r1cs._h, bb._ptr(inp), ni, None, na, 0, C.byref(first), C.byref(count)), "null witness pointer")
    no_device_work(lambda: check_batch(worker._h, r1cs._h, *args[:4], 2, 0, None), "bb_r1cs_check_batch: null argument")
    no_device_work(lambda: check_batch(worker._h, r1cs._h, None, ni, bb._ptr(ax), na, 2, 0, bb._ptr(firsts)), "null witness pointer")
    # misaligned device witnesses
    d_in, d_aux = device_copy(worker, np.concatenate([inp, inp])), device_copy(worker, np.concatenate([ax, ax]))
    assert r1cs.unsatisfied(d_in, d_aux, on_device=True) == (None, 0)
    no_device_work(lambda: r1cs.unsatisfied(d_in.value + 8, d_aux, on_device=True), "16-byte aligned")
    no_device_work(lambda: r1cs.unsatisfied(d_in, d_aux.value + 8, on_device=True), "16-byte aligned")
    no_device_work(lambda: RC.check_r1cs_batch(r1cs, None, None, count=2, device_ptrs={"inputs": d_in.value + 4, "aux": d_aux}),
                   "16-byte aligned")
    assert RC.check_r1cs_batch(r1cs, None, None, count=2, device_ptrs={"inputs": d_in, "aux": d_aux}) == [(None, 0)] * 2
    for p in (d_in, d_aux):
        worker.device_free(p)
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 5. the bench workload: 2^20 MiMC constraints
# --------------------------------------------------------------------------------------------
def mimc_rows_of(mats, var):
    """the rows of the bb_synth_mimc_r1cs matrices whose terms read variable `var`"""
    rows = set()
    for off, v, _ in mats:
        rows.update((np.searchsorted(off, np.nonzero(v == var)[0], side="right") - 1).tolist())
    return sorted(rows)


def mimc_row_holds(mats, k, z_of):
    vals = []
    for off, var, cf in mats:
        lo, hi = int(off[k]), int(off[k + 1])
        coeffs = o1.fr_to_ints(cf[lo:hi]) if hi > lo else []
        vals.append(sum(x * z_of(v) for v, x in zip(var[lo:hi].tolist(), coeffs)) % R)
    return vals[0] * vals[1] % R == vals[2]


def check_mimc(worker, log_n):
    """the synthetic MiMC witness holds; then single corruptions at the first, middle and last aux index fail exactly the
    rows of that variable's CSR columns that no longer hold (those rows evaluated in Python integers)"""
    rng = random.Random(55)
    rounds = (1 << (log_n - 1)) - 1
    asg, _ = bb.synth_mimc(rounds, seed=20)
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    mats = RC.synth_mimc_matrices(rounds, 20)
    n, ni, na = r1cs.n_constraints, r1cs.n_inputs, r1cs.n_aux
    inp, aux0 = np.ascontiguousarray(asg.input_assignment), np.ascontiguousarray(asg.aux_assignment)
    d_in, d_aux = device_copy(worker, inp), device_copy(worker, aux0)
    first, count, bits = r1cs.unsatisfied(d_in, d_aux, on_device=True, bits=True)
    assert (first, count, bits.any()) == (None, 0, False)
    assert r1cs.unsatisfied(inp, aux0) == (None, 0)
    for j in (0, na // 2, na - 1):
        aux = aux0.copy()
        old = o1.fr_to_ints(aux0[j:j + 1])[0]
        aux[j] = fr([changed(rng, old)])[0]
        new = o1.fr_to_ints(aux[j:j + 1])[0]

        def z_of(v):
            if v == ni + j:
                return new
            return o1.fr_to_ints(inp[v:v + 1] if v < ni else aux0[v - ni:v - ni + 1])[0]

        rows = [k for k in mimc_rows_of(mats, ni + j) if not mimc_row_holds(mats, k, z_of)]
        assert rows
        worker.upload(d_aux, aux)
        want_bits = np.zeros(n, bool)
        want_bits[rows] = True
        first, count, bits = r1cs.unsatisfied(d_in, d_aux, on_device=True, bits=True)
        assert (first, count) == (rows[0], len(rows)) and np.array_equal(bits, want_bits)
        assert r1cs.unsatisfied(inp, aux) == (rows[0], len(rows))
    for p in (d_in, d_aux):
        worker.device_free(p)
    r1cs.free()


def test_check_mimc_2_20(worker):
    check_mimc(worker, 20)
