"""Many witnesses of one circuit against one key in one call (bb_groth16_prove_batch, bb_groth16_prove_r1cs_batch;
bellman_b200.create_proof_batch, r1cs.create_proof_r1cs_batch): every item's bytes and status against create_proof of that
item alone.  tests/test_emulated_prove_batch.py runs the same bodies on the emulated device (tests/native/) at the sizes a
host reaches; this file adds the sizes only a device reaches (2^17 and 2^20 constraints).
"""
import ctypes as C
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


def assignment(wit, aux=None):
    return bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"] if aux is None else aux, wit["a_aux_density"],
                                wit["b_input_density"], wit["b_aux_density"])


def single(asg, params, r, s, device_ptrs=None):
    """create_proof of one item: its bytes, or the exception it raises"""
    try:
        return bb.create_proof(asg, params, r, s, device_ptrs)
    except (bb.SynthesisError, bb.DensityMismatch, bb.BackendError) as e:
        return e


def same(got, want):
    if isinstance(want, bytes):
        return got == want
    return type(got) is type(want) and str(got) == str(want)


def check_batch(params, asgs, rng, device=None, worker=None):
    """create_proof_batch against create_proof per item, from host or (device=worker) HBM; returns the batch"""
    rs = [rng.randrange(R) for _ in asgs]
    ss = [rng.randrange(R) for _ in asgs]
    ptrs, held = None, []
    if device is not None:
        ptrs = []
        for asg in asgs:
            d = {k: device_copy(device, v) for k, v in (("a", asg.a), ("b", asg.b), ("c", asg.c), ("inputs", asg.input_assignment),
                                                        ("aux", asg.aux_assignment))}
            ptrs.append(d)
            held += list(d.values())
    got = bb.create_proof_batch(asgs, params, rs, ss, ptrs)
    assert len(got) == len(asgs)
    for i, asg in enumerate(asgs):
        want = single(asg, params, rs[i], ss[i], None if ptrs is None else ptrs[i])
        assert same(got[i], want), (i, got[i], want)
    for p in held:
        device.device_free(p)
    return got


def device_copy(worker, arr):
    p = worker.device_alloc(max(arr.nbytes, 32))
    if arr.nbytes:
        worker.upload(p, arr)
    return p


def mimc_key(worker, rounds=322, seed=5, rng=None):
    mc = o1.Mimc(rounds, seed=seed)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    return mc


def mimc_items(rounds, count, mont_one):
    """`count` witnesses of the MiMC shape: distinct seeds, then an all-zero aux, an all-one aux and one with every other aux
    value zeroed -- items that differ in their Exponent::Zero / Exponent::One patterns"""
    wits = [o1.Mimc(rounds, seed=10 + k).witness() for k in range(max(count - 3, 1))]
    base = wits[0]
    asgs = [assignment(w) for w in wits]
    na = base["aux"].shape[0]
    zeros = np.zeros_like(base["aux"])
    ones = np.tile(mont_one, (na, 1))
    every_other = base["aux"].copy()
    every_other[::2] = 0
    asgs += [assignment(base, zeros), assignment(base, ones), assignment(base, every_other)]
    return asgs[:count]


# --------------------------------------------------------------------------------------------
# 1. bytes
# --------------------------------------------------------------------------------------------
def test_bytes_mimc322(worker, rounds=322, sizes=(1, 2, 5, 33)):
    """B in {1, 2, 5, 33}, prove_batch_max = 2 (uneven sub-batches), the three MSM forms, host and device witnesses"""
    rng = random.Random(40)
    mc = mimc_key(worker, rounds, 5, rng)
    params = bb.Parameters(worker, mc.export_params())
    one = fr([1])[0]
    items = mimc_items(rounds, max(sizes), one)
    forms = {"default": lambda: params.apply_tuning(0),
             "precompute 1": lambda: (params.apply_tuning(0), params.precompute(), worker.set_option("msm_precompute", 1)),
             "precompute 2": lambda: params.apply_tuning(1)}
    try:
        for name, form in forms.items():
            form()
            for b in sizes:
                check_batch(params, items[:b], rng)
            worker.set_option("prove_batch_max", 2)
            check_batch(params, items[:5], rng)
            check_batch(params, items[:5], rng, device=worker)
            worker.set_option("prove_batch_max", 0)
    finally:
        worker.set_option("prove_batch_max", 0)
        params.apply_tuning(0)
    params.free()


def test_bytes_xor_demo(worker):
    """the xor circuit (groth16/src/tests/mod.rs:13-89) for all four inputs, against a generated key"""
    from bellman_b200 import params_io
    rng = random.Random(41)
    asm = GEN.KeypairAssembly()
    asm.alloc_input()
    B.xor_demo(0, 0)(_AssemblyAdapter(asm))
    key = GEN.generate_parameters(worker, asm, *[rng.randrange(1, R) for _ in range(5)])
    params = bb.Parameters(worker, params_io.read_parameters(params_io.write_parameters(key), worker=worker))
    asgs = []
    for a, b in ((0, 0), (0, 1), (1, 0), (1, 1)):
        pa = B.synthesize_witness(B.Bls12, B.xor_demo(a, b))
        asgs.append(bb.ProvingAssignment(fr(pa.a), fr(pa.b), fr(pa.c), fr(pa.input_assignment), fr(pa.aux_assignment),
                                         pa.a_aux_density, pa.b_input_density, pa.b_aux_density))
    check_batch(params, asgs, rng)
    params.free()


def test_generated_key_verifies(worker, rounds=40, count=4):
    """distinct witnesses of one MiMC circuit against generate_parameters' key: bytes as create_proof, and each verifies"""
    from bellman_b200 import params_io
    rng = random.Random(42)
    constants = [rng.randrange(R) for _ in range(rounds)]
    circuits = [B.mimc_circuit(B.Bls12.fr, rng.randrange(R), rng.randrange(R), constants) for _ in range(count)]
    asm = GEN.KeypairAssembly()
    asm.alloc_input()
    circuits[0](_AssemblyAdapter(asm))
    key = GEN.generate_parameters(worker, asm, *[rng.randrange(1, R) for _ in range(5)])
    params = bb.Parameters(worker, params_io.read_parameters(params_io.write_parameters(key), worker=worker))
    pas = [B.synthesize_witness(B.Bls12, c) for c in circuits]
    asgs = [bb.ProvingAssignment(fr(pa.a), fr(pa.b), fr(pa.c), fr(pa.input_assignment), fr(pa.aux_assignment), pa.a_aux_density,
                                 pa.b_input_density, pa.b_aux_density) for pa in pas]
    proofs = check_batch(params, asgs, rng)
    pvk = bb.prepare_verifying_key(worker, {"alpha_g1": key["vk_g1"][0], "beta_g2": key["vk_g2"][0], "gamma_g2": key["vk_g2"][1],
                                            "delta_g2": key["vk_g2"][2], "ic": key["ic"]})
    for pa, proof in zip(pas, proofs):
        bb.verify_proof(pvk, abi_proof(PR.proof_read(proof)), pa.input_assignment[1:])
    with pytest.raises(bb.InvalidProof):                    # proof 0 does not hold for proof 1's statement
        bb.verify_proof(pvk, abi_proof(PR.proof_read(proofs[0])), pas[1].input_assignment[1:])
    pvk.free()
    params.free()


# --------------------------------------------------------------------------------------------
# 2. status per item
# --------------------------------------------------------------------------------------------
def test_status_per_item(worker, rounds=20):
    rng = random.Random(43)
    mc = mimc_key(worker, rounds, 5, rng)
    base = mc.export_params()
    items = mimc_items(rounds, 5, fr([1])[0])            # 2 distinct witnesses, all-zero aux, all-one aux, every other aux zero
    na = items[0].aux_assignment.shape[0]
    j = next(k for k in range(0, na, 2) if items[0].aux_assignment[k].any())   # aux[j] = 0 only in the zeroed items
    b_in = int(np.unpackbits(items[0].b_input_density.view(np.uint8), bitorder="little")[:items[0].input_assignment.shape[0]].sum())
    b_aux_bits = np.unpackbits(items[0].b_aux_density.view(np.uint8), bitorder="little")[:na]
    first_b_aux = 0                                          # the base of the first b-aux variable is row b_in of b_g1
    jb = int(np.flatnonzero(b_aux_bits)[0])
    hole = items[0].aux_assignment.copy()
    hole[jb] = 0                                             # this item never reads that base
    items.append(bb.ProvingAssignment.__new__(bb.ProvingAssignment))
    items[-1].__dict__.update(items[0].__dict__)
    items[-1].aux_assignment = hole

    def variant(**changes):
        p = {k: np.array(v, copy=True) for k, v in base.items()}
        for k, f in changes.items():
            p[k] = f(p[k])
        return bb.Parameters(worker, p)

    def zero_row(idx):
        def f(v):
            v = v.reshape(-1, v.shape[-1] if v.ndim > 1 else 12).copy()
            v[idx] = 0
            return v
        return f

    def short(v):
        return v.reshape(-1, v.shape[-1])[:-1]

    def zero_delta(v):
        v = v.reshape(3, -1).copy()
        v[2] = 0
        return v

    cases = {
        "identity in l": (variant(l=zero_row(j)), {bytes: {2, 4}, bb.UnexpectedIdentity: {0, 1, 3}}),
        "identity in b_g2 under ones": (variant(b_g2=zero_row(-1)), None),
        "short key": (variant(b_g1=short), None),
        "delta identity": (variant(vk_g1=zero_delta), None),
        "delta identity and short": (variant(vk_g1=zero_delta, b_g1=short), None),
        "short and identity in l": (variant(a=short, l=zero_row(j)), None),
        # both faults in ONE job: b_g1 runs out of bases and holds an identity at the first b-aux variable's base; items
        # differ in whether that variable's scalar is zero, so each is classified over its own scalars
        "short and identity in b_g1": (variant(b_g1=lambda v: short(zero_row(b_in + first_b_aux)(v))), None),
    }
    for name, (params, expect) in cases.items():
        got = check_batch(params, items, rng)
        if expect:
            for kind, idx in expect.items():
                for i in idx:
                    assert isinstance(got[i], kind), (name, i, got[i])
        if name == "identity in b_g2 under ones":
            assert isinstance(got[3], bb.UnexpectedIdentity) and isinstance(got[2], bytes), name
        if name == "short key":
            assert all(isinstance(g, bb.IoError) for g in got), name
        if name.startswith("delta"):
            assert all(isinstance(g, bb.UnexpectedIdentity) and "delta" in str(g) for g in got), name
        params.free()


def test_argument_errors(worker):
    """argument errors come before any device work: no launch, no copy"""
    rng = random.Random(44)
    mc = mimc_key(worker, 20, 5, rng)
    p = mc.export_params()
    params = bb.Parameters(worker, p)
    items = mimc_items(20, 2, fr([1])[0])
    lib = bb.load_library()

    def no_device_work(fn, match):
        l0, b0 = worker.kernel_launches, worker.bytes_copied()
        with pytest.raises(bb.BackendError, match=match) as e:
            fn()
        assert ARG in str(e.value)
        assert (worker.kernel_launches, worker.bytes_copied()) == (l0, b0)

    wit = mc.witness()
    other = bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"][:-1], wit["a_aux_density"][:-1],
                                 wit["b_input_density"], wit["b_aux_density"][:-1])
    no_device_work(lambda: bb.create_proof_batch([items[0], items[1], other], params, [1, 2, 3], [4, 5, 6]), "item 2 differs")
    sharded = bb.Parameters(worker, p, shard_index=0, shard_count=2)
    no_device_work(lambda: bb.create_proof_batch(items, sharded, [1, 2], [3, 4]), "unsharded")
    ws = (bb._Witness * 2)(items[0]._struct(), items[1]._struct())
    sc = bb._scalars_bytes([1, 2])
    no_device_work(lambda: bb._check(lib.bb_groth16_prove_batch(worker._h, params._h, ws, C.c_size_t(2), sc, sc, None, None)), "null")
    no_device_work(lambda: bb._check(lib.bb_groth16_prove_batch(worker._h, params._h, None, C.c_size_t(2), sc, sc,
                                                                 (C.c_uint8 * 384)(), (C.c_int * 2)())), "null")
    l0 = worker.kernel_launches
    assert bb.create_proof_batch([], params, [], []) == []
    assert worker.kernel_launches == l0
    mimc = RC.R1CS.synth_mimc(worker, 20, 5)
    inp = np.stack([wit["inputs"]] * 2)
    no_device_work(lambda: RC.create_proof_r1cs_batch(mimc, params, inp, np.stack([wit["aux"][:-1]] * 2), [1, 2], [3, 4]), "witness has")
    no_device_work(lambda: RC.create_proof_r1cs_batch(mimc, sharded, inp, np.stack([wit["aux"]] * 2), [1, 2], [3, 4]), "unsharded")
    mimc.free()
    sharded.free()
    params.free()


def test_launches_shared(worker):
    """one launch sequence for the sub-batch: 16 proofs in one sub-batch launch at most 1.25 x what one proof launches"""
    rng = random.Random(45)
    mc = mimc_key(worker, 322, 5, rng)
    params = bb.Parameters(worker, mc.export_params())
    items = mimc_items(322, 16, fr([1])[0])
    counts = {}
    bb.create_proof_batch(items[:1], params, [1], [2])     # the NTT tables of the domain are built once, not counted
    for b in (1, 16):
        l0 = worker.kernel_launches
        assert all(isinstance(p, bytes) for p in bb.create_proof_batch(items[:b], params, [1] * b, [2] * b))
        counts[b] = worker.kernel_launches - l0
    assert counts[16] <= 1.25 * counts[1], counts
    params.free()


# --------------------------------------------------------------------------------------------
# 3. R1CS form
# --------------------------------------------------------------------------------------------
def test_r1cs_batch(worker, rounds=322, count=5):
    rng = random.Random(46)
    mc = mimc_key(worker, rounds, 5, rng)
    params = bb.Parameters(worker, mc.export_params())
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    wits = [o1.Mimc(rounds, seed=20 + k).witness() for k in range(count)]
    inp = np.stack([w["inputs"] for w in wits])
    aux = np.stack([w["aux"] for w in wits])
    aux[-1] = 0
    rs = [rng.randrange(R) for _ in wits]
    ss = [rng.randrange(R) for _ in wits]
    want = [RC.create_proof_r1cs(r1cs, params, inp[i], aux[i], rs[i], ss[i]) for i in range(count)]
    assert RC.create_proof_r1cs_batch(r1cs, params, inp, aux, rs, ss) == want
    d = {"inputs": device_copy(worker, inp), "aux": device_copy(worker, aux)}
    worker.set_option("prove_batch_max", 2)
    try:
        assert RC.create_proof_r1cs_batch(r1cs, params, None, None, rs, ss, device_ptrs=d) == want
    finally:
        worker.set_option("prove_batch_max", 0)
    for p in d.values():
        worker.device_free(p)
    r1cs.free()
    params.free()


# --------------------------------------------------------------------------------------------
# 4. the sizes only a device reaches
# --------------------------------------------------------------------------------------------
def check_large(worker, log_n, count):
    rounds = (1 << (log_n - 1)) - 1
    asgs = [bb.synth_mimc(rounds, seed=30 + k)[0] for k in range(count)]
    shape = bb.synth_mimc(rounds, seed=30)[1]
    params = bb.Parameters.synthetic(worker, 31, shape)
    rs = [0x1234567 + k for k in range(count)]
    ss = [0x7654321 + k for k in range(count)]
    got = bb.create_proof_batch(asgs, params, rs, ss)
    for asg, r, s, g in zip(asgs, rs, ss, got):
        assert g == bb.create_proof(asg, params, r, s)
    params.free()


def test_large_2_17(worker):
    check_large(worker, 17, 16)


def test_large_2_20(worker):
    check_large(worker, 20, 3)
