"""Groth16 verification on the device (bellman_b200/verifier.py, csrc/verify.cu, csrc/tower.cuh) against the
Python-integer pairing and verifier of the oracle (oracle/oracle0/pairing.py).

The pairing is checked value for value: G_T from bb_diag_multi_pairing must equal the oracle's pairing raised to
k = bb_diag_gt_exponent().  The verifiers are checked verdict for verdict against oracle0.pairing.verify_proof on
MiMC-322 proofs of the CPU oracle (groth16/tests/mimc.rs), on proofs of the GPU prover and on synthetic batches.
tests/test_emulated_verify.py runs the same bodies on the emulated device (tests/native/).
"""
import functools
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import verifier as V
from oracle import o1
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

pytestmark = pytest.mark.gpu

R = F.FR_MODULUS


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


# --------------------------------------------------------------------------------------------
# G_T values
# --------------------------------------------------------------------------------------------
def gt_to_oracle(out):
    """12 canonical Fp in tower order -> the oracle's Fp12 (w^12 = 2 w^6 - 2, u = w^6 - 1): the Fp2 coefficient
    c0 + c1 u of v^i w^j is c0 - c1 at w^(2i+j) plus c1 at w^(2i+j+6)"""
    ints = o1.limbs_to_ints(np.asarray(out, dtype=np.uint64).reshape(12, 6))
    c = [0] * 12
    for t, val in enumerate(ints):
        j, i, part = t // 6, (t % 6) // 2, t % 2
        k = 2 * i + j
        if part == 0:
            c[k] += val
        else:
            c[k] -= val
            c[k + 6] += val
    return PR.Fp12(c)


def _device_pairing(worker, pairs):
    g1 = o1.g1_from_affine_ints([p for p, _ in pairs])
    g2 = o1.g2_from_affine_ints([q for _, q in pairs])
    return gt_to_oracle(V.multi_pairing(worker, g1, g2))


def _fp12_to_mont(f):
    """oracle Fp12 -> 12 Montgomery Fp in tower order (inverse of gt_to_oracle's map)"""
    c = [x % F.FP_MODULUS for x in f.c]
    tower = [0] * 12
    for j in range(2):
        for i in range(3):
            k = 2 * i + j
            c1 = c[k + 6]
            tower[6 * j + 2 * i + 1] = c1
            tower[6 * j + 2 * i] = (c[k] + c1) % F.FP_MODULUS
    return o1.fp_from_ints(tower).reshape(72)


def _fp12_from_mont(words):
    return gt_to_oracle(o1.ints_to_limbs(o1.fp_to_ints(np.asarray(words, dtype=np.uint64).reshape(12, 6)), 6))


def _device_fp12(worker, op, a, b):
    import ctypes as C
    x, y = _fp12_to_mont(a), _fp12_to_mont(b)
    out = np.zeros(72, np.uint64)
    assert bb.load_library().bb_diag_fp12(worker._h, C.c_int(op), x.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p),
                                          out.ctypes.data_as(C.c_void_p), C.c_size_t(1)) == 0
    return _fp12_from_mont(out)


def test_tower_operations(worker, seed=3):
    """the Fp12 operations of tower.cuh one by one against the oracle's Fp12"""
    rng = random.Random(seed)
    P = F.FP_MODULUS
    a = PR.Fp12([rng.randrange(P) for _ in range(12)])
    b = PR.Fp12([rng.randrange(P) for _ in range(12)])
    assert _device_fp12(worker, 0, a, b) == a * b
    assert _device_fp12(worker, 1, a, b) == a * a
    assert _device_fp12(worker, 2, a, b) * a == PR.Fp12.one()
    assert _device_fp12(worker, 4, a, b) == a.pow(P)
    assert _device_fp12(worker, 5, a, b) == a.pow(P * P)
    t = a.pow((P ** 6 - 1) * (P ** 2 + 1))                        # in the cyclotomic subgroup
    assert _device_fp12(worker, 3, t, b) == t * t
    bw = _fp12_to_mont(b).reshape(12, 6).copy()                 # the sparse line made of b's c0.c0, c0.c1, c1.c1
    bw[[4, 5, 6, 7, 10, 11]] = 0
    line = _fp12_from_mont(bw.reshape(72))
    assert _device_fp12(worker, 7, a, b) == a * line
    assert _device_fp12(worker, 6, a, b) == a.pow(3 * PR.FINAL_EXP)


def test_gt_convention(worker):
    k = V.gt_exponent()
    assert k in (1, -1, 3, -3)
    want = PR.pairing(F.G1_GEN, F.G2_GEN)
    assert _device_pairing(worker, [(F.G1_GEN, F.G2_GEN)]) == want.pow(k % R)


def test_gt_matches_oracle(worker, n_random=2, seed=5):
    rng = random.Random(seed)
    k = V.gt_exponent() % R
    for _ in range(n_random):                                    # random multiples on both sides
        p = F.G1.mul(F.G1_GEN, rng.randrange(1, R))
        q = F.G2.mul(F.G2_GEN, rng.randrange(1, R))
        assert _device_pairing(worker, [(p, q)]) == PR.pairing(p, q).pow(k)
    a, b = rng.randrange(1, R), rng.randrange(1, R)              # e(aP, Q) e(bP, Q) e(-(a+b)P, Q) = 1
    pairs = [(F.G1.mul(F.G1_GEN, a), F.G2_GEN), (F.G1.mul(F.G1_GEN, b), F.G2_GEN), (F.G1.mul(F.G1_GEN, (-(a + b)) % R), F.G2_GEN)]
    assert _device_pairing(worker, pairs) == PR.Fp12.one()
    one = PR.Fp12.one()                                          # an identity on either side contributes one
    assert _device_pairing(worker, [(None, F.G2_GEN)]) == one and _device_pairing(worker, [(F.G1_GEN, None)]) == one
    p = F.G1.mul(F.G1_GEN, 77)
    assert _device_pairing(worker, [(None, F.G2_GEN), (p, F.G2_GEN), (F.G1_GEN, None)]) == PR.pairing(p, F.G2_GEN).pow(k)
    assert _device_pairing(worker, []) == one


# --------------------------------------------------------------------------------------------
# MiMC-322 proofs of the CPU oracle
# --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def mimc_case(seed=21, n_proofs=5):
    """a MiMC-322 key (toxic waste and witness from `seed`) and n proofs made with different (r, s): ABI arrays plus the
    oracle's view"""
    rng = random.Random(seed)
    mc = o1.Mimc(322, seed=seed)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    p = mc.export_params()
    vk = {"alpha_g1": p["vk_g1"][0], "beta_g2": p["vk_g2"][0], "gamma_g2": p["vk_g2"][1], "delta_g2": p["vk_g2"][2], "ic": p["ic"]}
    g1, g2 = o1.g1_to_affine_ints(p["vk_g1"]), o1.g2_to_affine_ints(p["vk_g2"])
    vk_int = dict(alpha_g1=g1[0], beta_g2=g2[0], gamma_g2=g2[1], delta_g2=g2[2], ic=o1.g1_to_affine_ints(p["ic"]))
    x = o1.fr_to_ints(mc.witness()["inputs"][1:])               # public inputs without the leading one
    items = [(PR.proof_read(mc.prove(rng.randrange(R), rng.randrange(R))), x) for _ in range(n_proofs)]
    return vk, vk_int, items


def abi_proof(proof):
    a, b, c = proof
    return o1.g1_from_affine_ints([a])[0], o1.g2_from_affine_ints([b])[0], o1.g1_from_affine_ints([c])[0]


def batch_verdict(pvk, items, rng=None):
    bv = bb.BatchVerifier()
    for proof, x in items:
        bv.queue((abi_proof(proof), x))
    try:
        bv.verify(rng, pvk)
        return True
    except bb.InvalidProof:
        return False


def tampered(proof, x, what):
    a, b, c = proof
    if what == "a":
        return (F.G1.add(a, F.G1_GEN), b, c), x
    if what == "b":
        return (a, F.G2.add(b, F.G2_GEN), c), x
    if what == "c":
        return (a, b, F.G1.add(c, F.G1_GEN)), x
    return proof, [(x[0] + 1) % R] + list(x[1:])


def test_batch_verifies_mimc_proofs(worker, seed=21):
    vk, vk_int, items = mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    rng = random.Random(1)
    assert all(PR.verify_proof(vk_int, proof, x) for proof, x in items[:2])
    _, _, other = mimc_case(seed + 1, 1)                         # another key's witness and toxic waste
    assert not batch_verdict(pvk, items[:2] + other, rng)
    assert batch_verdict(pvk, items, rng)
    assert batch_verdict(pvk, items, None)                       # z from the operating system
    for what in ("a", "b", "c", "input"):                        # one bad item in turn, at position 2 of 5
        bad = tampered(*items[2], what)
        assert not PR.verify_proof(vk_int, *bad), what
        batch = items[:2] + [bad] + items[3:]
        for zseed in (2, 3):                                     # the verdict does not depend on z
            assert not batch_verdict(pvk, batch, random.Random(zseed)), what
    assert batch_verdict(pvk, [], rng)                           # empty batch
    for proof, x in items[:2]:                                   # verify_proof == the batch of one
        bb.verify_proof(pvk, abi_proof(proof), x)
        assert batch_verdict(pvk, [(proof, x)], rng)
    with pytest.raises(bb.InvalidProof):
        bb.verify_proof(pvk, abi_proof(items[0][0]), [(items[0][1][0] + 1) % R])
    pvk.free()


def test_batch_edge_cases(worker, seed=21):
    vk, vk_int, items = mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    (a, b, c), x = items[0]
    ident = ((None, b, c), x)                                    # identity A: whatever the oracle says
    want = PR.verify_proof(vk_int, *ident)
    assert batch_verdict(pvk, [ident], random.Random(4)) == want
    assert batch_verdict(pvk, items[1:3] + [ident], random.Random(4)) == want
    with pytest.raises(bb.InvalidVerifyingKey):                  # wrong input count, checked before any device work
        bb.verify_proof(pvk, abi_proof(items[0][0]), [])
    with pytest.raises(bb.InvalidVerifyingKey):
        batch_verdict(pvk, items[:2] + [(items[2][0], list(items[2][1]) + [5])], random.Random(4))
    pa, pb, pc = abi_proof(items[0][0])
    xs = V.fr_inputs(items[0][1])
    for z in ([0], [R], [R + 1]):                                # z must lie in [1, r)
        with pytest.raises(bb.BackendError) as ei:
            V.verify_batch_arrays(pvk, pa[None], pb[None], pc[None], xs[None], z=z)
        assert "[bb_status 16]" in str(ei.value)
    V.verify_batch_arrays(pvk, pa[None], pb[None], pc[None], xs[None], z=[R - 1])
    pvk.free()


def test_synthetic_batch_generator(worker, n=3, n_inputs=2, seed=9):
    """bb_synth_proof_batch: its proofs pass the oracle's verify_proof, so the generator is checked independently of
    the device verifier; then the device verifier accepts them and rejects one bad C"""
    vk, pvk, d, host = synth_batch(worker, seed, n, n_inputs)
    vk_int = dict(alpha_g1=o1.g1_to_affine_ints(vk["alpha_g1"])[0], beta_g2=o1.g2_to_affine_ints(vk["beta_g2"])[0],
                  gamma_g2=o1.g2_to_affine_ints(vk["gamma_g2"])[0], delta_g2=o1.g2_to_affine_ints(vk["delta_g2"])[0],
                  ic=o1.g1_to_affine_ints(vk["ic"]))
    a, b, c, x = host
    for i in range(min(n, 2)):
        proof = (o1.g1_to_affine_ints(a[i])[0], o1.g2_to_affine_ints(b[i])[0], o1.g1_to_affine_ints(c[i])[0])
        assert PR.verify_proof(vk_int, proof, o1.fr_to_ints(x[i]))
    z = [random.Random(3).randrange(1, R) for _ in range(n)]
    assert V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=z, on_device=True, n=n, n_inputs=n_inputs) is None
    V.verify_batch_arrays(pvk, a, b, c, x, z=z)
    c2 = c.copy()
    c2[n - 1] = c[0]
    with pytest.raises(bb.InvalidProof):
        V.verify_batch_arrays(pvk, a, b, c2, x, z=z)
    free_batch(worker, pvk, d)


def synth_batch(worker, seed, n, n_inputs):
    """bb_synth_proof_batch into fresh device buffers; also returns host copies (a, b, c, x)"""
    d = {"a": worker.device_alloc(n * 96), "b": worker.device_alloc(n * 192), "c": worker.device_alloc(n * 96),
         "x": worker.device_alloc(max(1, n * n_inputs) * 32)}
    vk = V.synth_proof_batch(worker, seed, n, n_inputs, d["a"], d["b"], d["c"], d["x"])
    pvk = bb.prepare_verifying_key(worker, vk)
    host = (np.zeros((n, 12), np.uint64), np.zeros((n, 24), np.uint64), np.zeros((n, 12), np.uint64), np.zeros((n, n_inputs, 4), np.uint64))
    for arr, key in zip(host, ("a", "b", "c", "x")):
        if arr.size:
            worker.download(d[key], arr)
    return vk, pvk, d, host


def free_batch(worker, pvk, d):
    pvk.free()
    for p in d.values():
        worker.device_free(p)


# --------------------------------------------------------------------------------------------
# GPU only: sizes the emulation cannot reach
# --------------------------------------------------------------------------------------------
def test_gpu_gt_random_pairs(worker):
    test_gt_matches_oracle(worker, n_random=6, seed=77)


def test_gpu_prover_proofs_verify(worker):
    """proofs made by bb.create_proof on MiMC-322 are accepted; tampered ones are rejected"""
    rng = random.Random(71)
    mc = o1.Mimc(322, seed=3)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    p = mc.export_params()
    params = bb.Parameters(worker, p)
    wit = mc.witness()
    asg = bb.ProvingAssignment(wit["a"], wit["b"], wit["c"], wit["inputs"], wit["aux"], wit["a_aux_density"],
                               wit["b_input_density"], wit["b_aux_density"])
    vk = {"alpha_g1": p["vk_g1"][0], "beta_g2": p["vk_g2"][0], "gamma_g2": p["vk_g2"][1], "delta_g2": p["vk_g2"][2], "ic": p["ic"]}
    pvk = bb.prepare_verifying_key(worker, vk)
    x = o1.fr_to_ints(wit["inputs"][1:])
    items = [(PR.proof_read(bb.create_proof(asg, params, rng.randrange(R), rng.randrange(R))), x) for _ in range(4)]
    assert batch_verdict(pvk, items, random.Random(5))
    bb.verify_proof(pvk, abi_proof(items[0][0]), x)
    for what in ("a", "b", "c", "input"):
        assert not batch_verdict(pvk, items[:1] + [tampered(*items[1], what)] + items[2:], random.Random(5)), what
    pvk.free()
    params.free()


def test_gpu_large_synthetic_batch(worker, log_n=16, n_inputs=2):
    """a 2^16-proof batch is accepted; one bad C at the first, the middle and the last position is rejected; the batch
    resident in HBM and the same batch from host buffers give the same verdicts"""
    n = 1 << log_n
    vk, pvk, d, host = synth_batch(worker, 31, n, n_inputs)
    a, b, c, x = host
    z = [random.Random(8).randrange(1, R) for _ in range(n)]
    V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=z, on_device=True, n=n, n_inputs=n_inputs)
    V.verify_batch_arrays(pvk, a, b, c, x, z=z)
    V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=None, on_device=True, n=n, n_inputs=n_inputs)
    for pos in (0, n // 2, n - 1):
        c2 = c.copy()
        c2[pos] = c[(pos + 1) % n]
        worker.upload(d["c"], c2)
        with pytest.raises(bb.InvalidProof):
            V.verify_batch_arrays(pvk, d["a"], d["b"], d["c"], d["x"], z=z, on_device=True, n=n, n_inputs=n_inputs)
        with pytest.raises(bb.InvalidProof):
            V.verify_batch_arrays(pvk, a, b, c2, x, z=z)
    worker.upload(d["c"], c)
    free_batch(worker, pvk, d)
