"""verify_proof for every proof of a batch on the device (bb_groth16_verify_each, BatchVerifier.verify_each,
csrc/verify.cu: k_each_psi, k_each_miller, k_each_final_exp) against the oracle's Python pairing and verifier
(oracle/oracle0/pairing.py) and against the batch-of-one path (bb_groth16_verify), proof by proof.

The G_T values are pinned: bb_diag_verify_each_gt's value i must equal the oracle's
multi_pairing([(A, B), (Psi, -gamma), (C, -delta)]) raised to k = gt_exponent(), and the last value e(alpha, beta)^k.
tests/test_emulated_verify_each.py runs the same bodies on the emulated device (tests/native/).
"""
import ctypes as C
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import verifier as V
from oracle import o1
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

from test_gpu_proof_read import proof_bytes
from test_gpu_verify import abi_proof, batch_verdict, gt_to_oracle, mimc_case, synth_batch, tampered

pytestmark = pytest.mark.gpu

R = F.FR_MODULUS


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def oracle_psi(vk_int, x):
    acc = vk_int["ic"][0]
    for xj, icj in zip(x, vk_int["ic"][1:]):
        acc = F.G1.add(acc, F.G1.mul(icj, xj))
    return acc


def oracle_gt(vk_int, proof, x, k):
    """FE(ML(A, B) ML(Psi, -gamma) ML(C, -delta))^k in the oracle"""
    a, b, c = proof
    pairs = [(a, b), (oracle_psi(vk_int, x), F.G2.neg(vk_int["gamma_g2"])), (c, F.G2.neg(vk_int["delta_g2"]))]
    return PR.multi_pairing(pairs).pow(k)


def arrays(items):
    """(proof, inputs) items of the oracle's view -> the ABI arrays of verify_each_arrays"""
    pts = [abi_proof(p) for p, _ in items]
    a, b, c = (np.stack([t[k] for t in pts]) for k in range(3))
    x = np.stack([V.fr_inputs(xi) for _, xi in items])
    return a, b, c, x


def raw_batch(a, b, c, x):
    """the bb_proof_batch of host arrays, for calls of the C entry point; keep the second value alive"""
    keep = []
    bt, _ = V._proof_batch(a, b, c, x, False, None, None, keep)
    return bt, keep


def each(pvk, items, gt=False):
    return V.verify_each_arrays(pvk, *arrays(items), gt=gt)


def one_by_one(pvk, items):
    """the batch-of-one path, an independent implementation: 0 = valid, 1 = InvalidProof"""
    out = []
    for proof, x in items:
        try:
            bb.verify_proof(pvk, abi_proof(proof), x)
            out.append(0)
        except bb.InvalidProof:
            out.append(1)
    return out


def check_gt(pvk, vk_int, items):
    """verdicts and G_T values of one call against the oracle; returns the verdicts"""
    k = V.gt_exponent() % R
    verdicts, gt = each(pvk, items, gt=True)
    assert gt.shape == (len(items) + 1, 72)
    target = PR.pairing(vk_int["alpha_g1"], vk_int["beta_g2"])
    assert gt_to_oracle(gt[-1]) == target.pow(k)
    for i, (proof, x) in enumerate(items):
        got = gt_to_oracle(gt[i])
        assert got == oracle_gt(vk_int, proof, x, k), i
        assert verdicts[i] == (0 if PR.verify_proof(vk_int, proof, x) else 1), i
    return verdicts


# --------------------------------------------------------------------------------------------
# a key from trapdoor scalars: valid proofs with identities, and a Psi that is the identity
# --------------------------------------------------------------------------------------------
def trapdoor_key(rng, t):
    """alpha, beta, gamma, delta random; ic[j] = [t_j] G1 (t_j = 0: the identity).  Returns (scalars, vk, vk_int)."""
    s = {k: rng.randrange(1, R) for k in ("alpha", "beta", "gamma", "delta")}
    vk_int = {"alpha_g1": F.G1.mul(F.G1_GEN, s["alpha"]), "beta_g2": F.G2.mul(F.G2_GEN, s["beta"]),
              "gamma_g2": F.G2.mul(F.G2_GEN, s["gamma"]), "delta_g2": F.G2.mul(F.G2_GEN, s["delta"]),
              "ic": [F.G1.mul(F.G1_GEN, tj) if tj % R else None for tj in t]}
    vk = {"alpha_g1": o1.g1_from_affine_ints([vk_int["alpha_g1"]])[0], "beta_g2": o1.g2_from_affine_ints([vk_int["beta_g2"]])[0],
          "gamma_g2": o1.g2_from_affine_ints([vk_int["gamma_g2"]])[0], "delta_g2": o1.g2_from_affine_ints([vk_int["delta_g2"]])[0],
          "ic": o1.g1_from_affine_ints(vk_int["ic"])}
    s["t"] = list(t)
    return s, vk, vk_int


def trapdoor_proof(s, x, a=None, b=None):
    """a valid proof for inputs x: a b = alpha beta + gamma psi + delta c, psi = t_0 + sum x_j t_j.  a = 0 or b = 0 gives
    an identity A or B; c comes out as zero (an identity C) when a b = alpha beta + gamma psi."""
    psi = (s["t"][0] + sum(xj * tj for xj, tj in zip(x, s["t"][1:]))) % R
    rest = (s["alpha"] * s["beta"] + s["gamma"] * psi) % R
    if a is None and b is None:                                  # make c = 0
        a = 7
        b = rest * pow(a, -1, R) % R
    c = ((a * b - rest) * pow(s["delta"], -1, R)) % R
    g1 = lambda k: F.G1.mul(F.G1_GEN, k) if k else None
    g2 = lambda k: F.G2.mul(F.G2_GEN, k) if k else None
    return (g1(a), g2(b), g1(c)), list(x)


# --------------------------------------------------------------------------------------------
# bodies shared with the emulated file
# --------------------------------------------------------------------------------------------
def test_each_gt_matches_oracle(worker, seed=21, n_proofs=3):
    """value i of bb_diag_verify_each_gt is the oracle's three-pair product, the last one e(alpha, beta)^k, for valid
    and for tampered proofs"""
    vk, vk_int, items = mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    batch = items[:n_proofs - 1] + [tampered(*items[n_proofs - 1], "c")]
    verdicts = check_gt(pvk, vk_int, batch)
    assert verdicts.tolist() == [0] * (n_proofs - 1) + [1]
    pvk.free()


def test_each_verdicts_mimc(worker, seed=21):
    """items tampered in A, B, C or an input at the first, middle and last position: every verdict is the oracle's and
    the batch of one's; n_invalid counts them; all zero exactly when the batch verifier accepts"""
    vk, vk_int, items = mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    n = len(items)
    assert each(pvk, items).tolist() == [0] * n
    assert batch_verdict(pvk, items, random.Random(1))
    for what in ("a", "b", "c", "input"):
        bad = {0, n // 2, n - 1}
        batch = [tampered(*it, what) if i in bad else it for i, it in enumerate(items)]
        want = [0 if PR.verify_proof(vk_int, p, x) else 1 for p, x in batch]
        assert want == [1 if i in bad else 0 for i in range(n)], what
        got = each(pvk, batch)
        assert got.tolist() == want, what
        assert one_by_one(pvk, batch) == want, what
        assert not batch_verdict(pvk, batch, random.Random(2)), what
        bt, keep = raw_batch(*arrays(batch))
        verdicts, n_invalid = np.full(n, 9, np.uint8), C.c_size_t(99)
        assert bb.load_library().bb_groth16_verify_each(worker._h, pvk._h, C.byref(bt), V._ptr(verdicts), C.byref(n_invalid)) == 0
        assert n_invalid.value == 3 and verdicts.tolist() == want
    bv = bb.BatchVerifier()
    for it in items:
        bv.queue((abi_proof(it[0]), it[1]))
    assert bv.verify_each(pvk) == [None] * n
    pvk.free()


def test_each_identities(worker, seed=13):
    """identity A, B or C, an identity ic[j], and a Psi that is the identity: verdicts and values are the oracle's
    (valid proofs among them, so a pair that should contribute one cannot hide behind a wrong zero)"""
    rng = random.Random(seed)
    t0 = rng.randrange(1, R)
    # ic[2] is the identity; inputs x = (1, *) give Psi = ic[0] + ic[1] = the identity
    s, vk, vk_int = trapdoor_key(rng, [t0, R - t0, 0])
    pvk = bb.prepare_verifying_key(worker, vk)
    x = [rng.randrange(R), rng.randrange(R)]
    items = [
        trapdoor_proof(s, x, a=rng.randrange(1, R), b=rng.randrange(1, R)),       # a valid proof, no identity
        trapdoor_proof(s, x, a=0, b=rng.randrange(1, R)),                         # identity A, valid
        trapdoor_proof(s, x, a=rng.randrange(1, R), b=0),                         # identity B, valid
        trapdoor_proof(s, x),                                                     # identity C, valid
        trapdoor_proof(s, [1, x[1]], a=rng.randrange(1, R), b=rng.randrange(1, R)),  # Psi = the identity, valid
        trapdoor_proof(s, [1, x[1]]),                                             # Psi and C the identity, valid
    ]
    assert items[1][0][0] is None and items[2][0][1] is None and items[3][0][2] is None and items[5][0][2] is None
    assert oracle_psi(vk_int, items[4][1]) is None
    bad_a = ((None, items[0][0][1], items[0][0][2]), x)                           # identity A where it does not belong
    bad_c = ((items[0][0][0], items[0][0][1], None), x)
    batch = items + [bad_a, bad_c]
    verdicts = check_gt(pvk, vk_int, batch)
    assert verdicts.tolist() == [0] * len(items) + [1, 1]
    assert one_by_one(pvk, batch) == verdicts.tolist()
    pvk.free()


def test_each_errors(worker, seed=21):
    """a wrong input count (before device work), NULL arrays, n = 0; BatchVerifier.verify_each with a wrong input count
    and an undecodable queue_bytes item among valid ones"""
    vk, vk_int, items = mimc_case(seed)
    pvk = bb.prepare_verifying_key(worker, vk)
    lib = bb.load_library()
    a, b, c, x = arrays(items[:2])
    launches = worker.kernel_launches
    with pytest.raises(bb.InvalidVerifyingKey):
        V.verify_each_arrays(pvk, a, b, c, x, n_inputs=0)
    with pytest.raises(bb.InvalidVerifyingKey):
        V.verify_each_arrays(pvk, a, b, c, np.zeros((2, 2, 4), np.uint64), n_inputs=2)
    assert worker.kernel_launches == launches
    verdicts, n_invalid = np.zeros(2, np.uint8), C.c_size_t()
    for nulls in ("a", "b", "c", "inputs", "verdicts", "n_invalid"):
        bt, keep = raw_batch(a, b, c, x)
        if nulls in ("a", "b", "c", "inputs"):
            setattr(bt, nulls, None)
        rc = lib.bb_groth16_verify_each(worker._h, pvk._h, C.byref(bt), None if nulls == "verdicts" else V._ptr(verdicts),
                                        None if nulls == "n_invalid" else C.byref(n_invalid))
        assert rc == 16, nulls                                  # BB_ERR_ARG
    empty = V.verify_each_arrays(pvk, a[:0], b[:0], c[:0], x[:0])
    assert empty.shape == (0,)
    bt, keep = raw_batch(a[:0], b[:0], c[:0], x[:0])
    n_invalid.value = 5
    assert lib.bb_groth16_verify_each(worker._h, pvk._h, C.byref(bt), None, C.byref(n_invalid)) == 0 and n_invalid.value == 0
    assert bb.BatchVerifier().verify_each(pvk) == []
    # the queue: valid bytes, a wrong input count, valid arrays, an undecodable proof, a tampered proof, valid bytes
    enc = [(proof_bytes(*p), xi) for p, xi in items]
    broken = bytearray(enc[3][0])
    broken[0] &= 0x7f                                            # A without its compression bit
    bad_proof, bad_x = tampered(*items[4], "b")
    bv = bb.BatchVerifier()
    bv.queue_bytes(*enc[0])
    bv.queue((abi_proof(items[1][0]), list(items[1][1]) + [5]))
    bv.queue((abi_proof(items[2][0]), items[2][1]))
    bv.queue_bytes(bytes(broken), items[3][1])
    bv.queue_bytes(proof_bytes(*bad_proof), bad_x)
    bv.queue_bytes(*enc[4])
    got = bv.verify_each(pvk)
    assert [type(e) for e in got] == [type(None), bb.InvalidVerifyingKey, type(None), bb.InvalidProofEncoding, bb.InvalidProof,
                                      type(None)]
    assert got[3].index == 3 and str(got[3]).startswith("invalid G1")
    plain = bb.BatchVerifier()                                   # the same without bytes: the host-array path
    plain.queue((abi_proof(items[0][0]), items[0][1]))
    plain.queue((abi_proof(items[1][0]), []))
    plain.queue((abi_proof(bad_proof), bad_x))
    assert [type(e) for e in plain.verify_each(pvk)] == [type(None), bb.InvalidVerifyingKey, bb.InvalidProof]
    pvk.free()


# --------------------------------------------------------------------------------------------
# GPU only: sizes the emulation cannot reach
# --------------------------------------------------------------------------------------------
def test_gpu_each_prover_proofs(worker):
    """proofs made by bb.create_proof on MiMC-322: valid ones pass, each tampered one is flagged alone"""
    rng = random.Random(72)
    mc = o1.Mimc(322, seed=6)
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
    assert each(pvk, items).tolist() == [0] * 4
    for k, what in enumerate(("a", "b", "c", "input")):
        batch = [tampered(*it, what) if i == k else it for i, it in enumerate(items)]
        want = [1 if i == k else 0 for i in range(4)]
        assert each(pvk, batch).tolist() == want, what
        assert one_by_one(pvk, batch) == want, what
    pvk.free()
    params.free()


def test_gpu_each_large_synthetic_batch(worker, log_n=16, n_inputs=2):
    """2^16 proofs with bad C at the first, middle and last index: exactly those are flagged, from HBM, from host buffers
    and through the bytes path (bb_proofs_write, then BatchVerifier.queue_bytes)"""
    n = 1 << log_n
    vk, pvk, d, host = synth_batch(worker, 33, n, n_inputs)
    a, b, c, x = host
    assert not V.verify_each_arrays(pvk, d["a"], d["b"], d["c"], d["x"], on_device=True, n=n, n_inputs=n_inputs).any()
    bad = [0, n // 2, n - 1]
    c2 = c.copy()
    for pos in bad:
        c2[pos] = c[(pos + 1) % n]
    worker.upload(d["c"], c2)
    got = V.verify_each_arrays(pvk, d["a"], d["b"], d["c"], d["x"], on_device=True, n=n, n_inputs=n_inputs)
    assert np.flatnonzero(got).tolist() == bad
    got = V.verify_each_arrays(pvk, a, b, c2, x)
    assert np.flatnonzero(got).tolist() == bad
    data = V.write_proofs(worker, a, b, c2)
    bv = bb.BatchVerifier()
    for i in range(n):
        bv.queue_bytes(data[192 * i:192 * (i + 1)], x[i])
    res = bv.verify_each(pvk)
    assert [i for i, e in enumerate(res) if e is not None] == bad
    assert all(isinstance(res[i], bb.InvalidProof) for i in bad)
    worker.upload(d["c"], c)
    pvk.free()
    for p in d.values():
        worker.device_free(p)
