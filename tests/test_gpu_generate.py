"""Groth16 parameters generated on the device (bb_groth16_generate, csrc/generate.cu; generator.generate_parameters_device /
generate_random_parameters_device) against the host generator (generator.generate_parameters, the reference's algorithm
over Python integers) and the oracle's MiMC key, and resident keys written as parameter files (bb_params_write, decode.cu;
params_io.write_parameters_device) against params_io.write_parameters.  tests/test_emulated_generate.py runs the same bodies
on the emulated device (tests/native/) at small sizes; this file adds the sizes only a device reaches.
"""
import ctypes as C
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import generator as GEN
from bellman_b200 import params_io as PIO
from bellman_b200 import r1cs as RC
from oracle import o1
from oracle.oracle0 import bellman as B
from oracle.oracle0 import fields as F
from oracle.oracle0 import pairing as PR

from test_gpu_parity import _AssemblyAdapter
from test_gpu_r1cs import csr, random_system
from test_gpu_verify import abi_proof

pytestmark = pytest.mark.gpu

R = F.FR_MODULUS
ARG = "[bb_status 16]"


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def live_bytes(worker):
    lib = bb.load_library()
    lib.bb_diag_ctx_live_bytes.restype = C.c_uint64
    return int(lib.bb_diag_ctx_live_bytes(worker._h))


def assembly(circuit):
    asm = GEN.KeypairAssembly()
    asm.alloc_input()                                          # ONE, generator.rs:188
    circuit(_AssemblyAdapter(asm))
    return asm


def assembly_from_rows(mats, n_inputs, n_aux):
    """the KeypairAssembly of rows of (variable, coefficient) per matrix (inputs first, then aux)"""
    asm = GEN.KeypairAssembly()
    for _ in range(n_inputs):
        asm.alloc_input()
    for _ in range(n_aux):
        asm.alloc()
    for k in range(len(mats[0])):
        lcs = [[(("input", v) if v < n_inputs else ("aux", v - n_inputs), c) for v, c in rows[k]] for rows in mats]
        asm.enforce(*lcs)
    return asm


def g_points(g1s, g2s):
    """[g1s] G1 and [g2s] G2 in the library's format, or None for the standard generator"""
    g1 = None if g1s == 1 else o1.g1_fixed_mul(o1.fr_from_ints([g1s]))[0]
    g2 = None if g2s == 1 else o1.g2_fixed_mul(o1.fr_from_ints([g2s]))[0]
    return g1, g2


def assert_same_key(params, pvk, want):
    """the resident key holds the host dict's points, all twelve sections: the vectors and the crs's verifying-key points
    element for element, ic and gamma_g2 through the written file"""
    got = PIO.download_parameters(params)
    for name in ("h", "l", "a", "b_g1", "b_g2"):
        w = np.asarray(want[name], np.uint64).reshape(got[name].shape)
        assert np.array_equal(got[name], w), name
    vk1, vk2 = np.asarray(want["vk_g1"]).reshape(3, 12), np.asarray(want["vk_g2"]).reshape(3, 24)
    assert np.array_equal(got["vk_g1"], vk1), "vk_g1"
    assert np.array_equal(got["vk_g2"], vk2[[0, 2]]), "vk_g2"
    assert PIO.write_parameters_device(params, pvk) == PIO.write_parameters(want)


def check_parity(worker, asm, toxic, g1s=1, g2s=1, r1cs=None):
    """device key == host key for one assembly (or a constraint system built otherwise from the same rows)"""
    want = GEN.generate_parameters(worker, asm, *toxic, g1_scalar=g1s, g2_scalar=g2s)
    own = r1cs is None
    r1cs = RC.R1CS.from_assembly(worker, asm) if own else r1cs
    params, pvk = GEN.generate_parameters_device(worker, r1cs, *toxic, *g_points(g1s, g2s))
    assert params.lens == {"ic": want["ic"].shape[0], "h": want["h"].shape[0], "l": want["l"].shape[0], "a": want["a"].shape[0],
                           "b_g1": want["b_g1"].shape[0], "b_g2": want["b_g2"].shape[0]}
    assert_same_key(params, pvk, want)
    params.free()
    pvk.free()
    if own:
        r1cs.free()
    return want


def toxic_of(rng):
    return [rng.randrange(1, R) for _ in range(5)]


# --------------------------------------------------------------------------------------------
# 1. parity with the host generator
# --------------------------------------------------------------------------------------------
def test_parity_small_circuits(worker):
    rng = random.Random(50)
    check_parity(worker, assembly(B.xor_demo(0, 1)), toxic_of(rng))
    for one_var in (True, False):                              # a zero coefficient on ONE or on an aux variable
        check_parity(worker, assembly(B.mult_with_zero_coeffs(5, 6, 30, one_var)), toxic_of(rng))
    want = check_parity(worker, assembly(lambda cs: None), toxic_of(rng))     # no aux, no constraints: m = 1
    assert want["m"] == 1 and want["h"].shape[0] == 0 and want["l"].shape[0] == 0
    # non-standard generators: [g1s] G1, [g2s] G2
    check_parity(worker, assembly(B.xor_demo(1, 1)), toxic_of(rng), g1s=rng.randrange(2, R), g2s=rng.randrange(2, R))


def test_parity_xor_demo_oracle0(worker):
    """xor_demo with non-standard generators against oracle-0's restatement of generate_parameters"""
    rng = random.Random(51)
    tox = toxic_of(rng)
    g1s, g2s = rng.randrange(2, R), rng.randrange(2, R)
    E = B.Bls12
    g1, g2 = E.g1.mul(F.G1_GEN, g1s), E.g2.mul(F.G2_GEN, g2s)
    prm = B.generate_parameters(E, B.xor_demo(1, 0), g1, g2, *tox)
    params, pvk = GEN.generate_parameters_device(worker, RC.R1CS.from_assembly(worker, assembly(B.xor_demo(1, 0))), *tox, *g_points(g1s, g2s))
    got = PIO.download_parameters(params)
    conv1 = lambda pts: o1.g1_from_affine_ints([None if E.g1.is_identity(p) else p for p in pts]) if pts else np.zeros((0, 12), np.uint64)
    conv2 = lambda pts: o1.g2_from_affine_ints([None if E.g2.is_identity(p) else p for p in pts]) if pts else np.zeros((0, 24), np.uint64)
    for name, conv in (("h", conv1), ("l", conv1), ("a", conv1), ("b_g1", conv1), ("b_g2", conv2)):
        assert np.array_equal(got[name], conv(getattr(prm, name))), name
    assert np.array_equal(got["vk_g1"], conv1([prm.alpha_g1, prm.beta_g1, prm.delta_g1]))
    assert np.array_equal(got["vk_g2"], conv2([prm.beta_g2, prm.delta_g2]))
    params.free()
    pvk.free()


def test_parity_mimc(worker, rounds=322):
    """MiMC: the key equals the host generator's and the oracle's export; a proof from it equals the trapdoor-expected bytes
    and verifies under the generated verifying key"""
    rng = random.Random(52)
    tox = toxic_of(rng)
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic(tox)
    mc.generate()
    want = mc.export_params()
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    params, pvk = GEN.generate_parameters_device(worker, r1cs, *tox)
    assert_same_key(params, pvk, want)
    wit = mc.witness()
    r, s = rng.randrange(R), rng.randrange(R)
    proof = RC.create_proof_r1cs(r1cs, params, wit["inputs"], wit["aux"], r, s)
    assert proof == mc.expected_proof(r, s)
    x = o1.fr_to_ints(wit["inputs"][1:])
    bb.verify_proof(pvk, abi_proof(PR.proof_read(proof)), x)
    bv = bb.BatchVerifier()
    bv.queue((abi_proof(PR.proof_read(proof)), x))
    bv.verify(rng, pvk)
    params.free()
    pvk.free()
    r1cs.free()


def check_random(worker, seed, total_rows, lengths, n_inputs=3, n_aux=50):
    """a random system: empty rows, zero coefficients, cancelling duplicates, 0 / 1 / r - 1, long rows; one C row per aux
    variable keeps l free of identities"""
    rng = random.Random(seed)
    n_rows = total_rows - n_inputs - n_aux
    mats = random_system(rng, n_rows, n_inputs, n_aux, lengths)
    for j in range(n_aux):
        mats[0].append([])
        mats[1].append([])
        mats[2].append([(n_inputs + j, 1)])
    v, k = n_inputs + rng.randrange(n_aux), rng.randrange(1, R)
    for rows in mats:                                          # variable v: the A terms cancel in every row it has
        rows[:] = [[t for t in row if t[0] != v or rows is not mats[0]] for row in rows]
    mats[0][0] = mats[0][0] + [(v, k), (v, R - k)]
    asm = assembly_from_rows(mats, n_inputs, n_aux)
    r1cs = RC.R1CS(worker, n_inputs, n_aux, *(csr(rows) for rows in mats))
    assert r1cs.n_constraints == total_rows
    assert r1cs.densities()[0][v - n_inputs]                   # density bit set, a element filtered
    want = check_parity(worker, asm, toxic_of(rng), r1cs=r1cs)
    assert want["a"].shape[0] < n_inputs + n_aux
    r1cs.free()


EMU_LENGTHS = (1, 31, 32, 33, 1000, 4096)


def test_parity_random(worker, big=True):
    """column lengths across the three evaluation kernels; 2^9 and 2^9 + 1 constraints; on the device a variable in 2^16
    rows"""
    for seed, total in ((1, 1 << 9), (2, (1 << 9) + 1)):
        check_random(worker, seed, total, EMU_LENGTHS)
    if big:
        rng = random.Random(3)
        n_rows = 1 << 16
        a = [[(1, rng.randrange(1, R))] for _ in range(n_rows)]        # variable 1 (an input) in every A row
        b = [[(2 + (k % 7), 1)] for k in range(n_rows)]
        c = [[(2 + (k % 7), rng.randrange(R))] for k in range(n_rows)]
        mats = [a, b, c]
        r1cs = RC.R1CS(worker, 2, 7, *(csr(rows) for rows in mats))
        check_parity(worker, assembly_from_rows(mats, 2, 7), toxic_of(rng), r1cs=r1cs)
        r1cs.free()


# --------------------------------------------------------------------------------------------
# 2. edge toxic waste and errors
# --------------------------------------------------------------------------------------------
def root_of_unity(m):
    w = pow(7, (R - 1) // m, R)                                # 7 generates Fr^*: w has order m
    assert pow(w, m, R) == 1
    return w


def test_edge_toxic(worker):
    rng = random.Random(53)
    asm = assembly(B.mimc_circuit(B.Bls12.fr, 3, 4, [rng.randrange(R) for _ in range(5)]))     # every aux is some C's output
    base = toxic_of(rng)
    m = GEN.generate_parameters(worker, asm, *base)["m"]
    for k, v in ((4, 0), (4, root_of_unity(m)), (0, 0), (1, 0)):        # tau = 0, tau^m = 1, alpha = 0, beta = 0
        tox = list(base)
        tox[k] = v
        try:
            want = check_parity(worker, asm, tox)
        except GEN.UnconstrainedVariable as e:                 # such toxic waste can leave an l scalar zero: the same error
            r1cs = RC.R1CS.from_assembly(worker, asm)
            with pytest.raises(GEN.UnconstrainedVariable) as dev:
                GEN.generate_parameters_device(worker, r1cs, *tox)
            r1cs.free()
            assert str(e).split()[2] == str(dev.value.index)
            continue
        if k == 4 and v:
            assert not np.asarray(want["h"]).any()                   # every h element the identity


def test_errors(worker):
    rng = random.Random(54)
    asm = assembly(B.xor_demo(1, 0))
    r1cs = RC.R1CS.from_assembly(worker, asm)
    tox = toxic_of(rng)
    before = live_bytes(worker)
    launches = worker.kernel_launches
    for k in (2, 3):                                           # gamma = 0, then delta = 0: before any device work
        bad = list(tox)
        bad[k] = 0
        with pytest.raises(bb.UnexpectedIdentity):
            GEN.generate_parameters_device(worker, r1cs, *bad)
    for k in range(5):                                         # a scalar >= r
        bad = list(tox)
        bad[k] = R + (k == 0)
        with pytest.raises(bb.BackendError, match="not below r"):
            GEN.generate_parameters_device(worker, r1cs, *bad)
    g1 = o1.g1_fixed_mul(o1.fr_from_ints([3]))[0]
    off_curve = g1.copy()
    off_curve[0] ^= 1
    for bad_g1, why in ((np.zeros(12, np.uint64), "identity"), (off_curve, "curve")):
        with pytest.raises(bb.BackendError, match=why):
            GEN.generate_parameters_device(worker, r1cs, *tox, g1=bad_g1)
    with pytest.raises(bb.BackendError, match="identity"):
        GEN.generate_parameters_device(worker, r1cs, *tox, g2=np.zeros(24, np.uint64))
    p_limbs = np.array([(F.FP_MODULUS >> (64 * k)) % (1 << 64) for k in range(6)], np.uint64)
    x_is_p = g1.copy()
    x_is_p[:6] = p_limbs
    with pytest.raises(bb.BackendError, match="not below p"):
        GEN.generate_parameters_device(worker, r1cs, *tox, g1=x_is_p)
    y1_is_p = o1.g2_fixed_mul(o1.fr_from_ints([3]))[0].copy()
    y1_is_p[18:] = p_limbs                                     # y.c1, the last of x.c0 | x.c1 | y.c0 | y.c1
    with pytest.raises(bb.BackendError, match="not below p"):
        GEN.generate_parameters_device(worker, r1cs, *tox, g2=y1_is_p)
    from test_gpu_proof_read import off_subgroup_g1, off_subgroup_g2
    with pytest.raises(bb.BackendError, match="subgroup"):
        GEN.generate_parameters_device(worker, r1cs, *tox, g1=o1.g1_from_affine_ints([off_subgroup_g1(rng)])[0])
    with pytest.raises(bb.BackendError, match="subgroup"):
        GEN.generate_parameters_device(worker, r1cs, *tox, g2=o1.g2_from_affine_ints([off_subgroup_g2(rng)])[0])
    assert worker.kernel_launches == launches and live_bytes(worker) == before
    lib = bb.load_library()
    crs = C.c_void_p(0x1000)
    assert lib.bb_groth16_generate(None, r1cs._h, None, C.byref(crs), None, None) == 16
    assert lib.bb_groth16_generate(worker._h, None, None, C.byref(crs), None, None) == 16 and crs.value is None
    assert lib.bb_groth16_generate(worker._h, r1cs._h, None, None, None, None) == 16
    other = bb.Worker(0)
    with pytest.raises(bb.BackendError, match="another context"):
        GEN.generate_parameters_device(other, r1cs, *tox)
    other.close()
    # an unconstrained aux variable: reported with its index after the evaluation, nothing left allocated
    asm2 = GEN.KeypairAssembly()
    one = asm2.alloc_input()
    x, y, z = asm2.alloc(), asm2.alloc(), asm2.alloc()
    asm2.enforce([(x, 1)], [(one, 1)], [(x, 1)])
    asm2.enforce([(z, 2)], [(one, 1)], [(z, 2)])
    with pytest.raises(GEN.UnconstrainedVariable):
        GEN.generate_parameters(worker, asm2, *tox)
    r2 = RC.R1CS.from_assembly(worker, asm2)
    before = live_bytes(worker)
    with pytest.raises(GEN.UnconstrainedVariable) as ei:
        GEN.generate_parameters_device(worker, r2, *tox)
    assert ei.value.index == 1 and "auxiliary variable 1" in str(ei.value)    # y appears in no constraint
    assert live_bytes(worker) == before
    r2.free()
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 3. random keys
# --------------------------------------------------------------------------------------------
def test_random_keys(worker, rounds=30):
    rng = random.Random(55)
    mc = o1.Mimc(rounds, seed=5)
    wit = mc.witness()
    x = o1.fr_to_ints(wit["inputs"][1:])
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    keys = [GEN.generate_random_parameters_device(worker, r1cs) for _ in range(2)]
    files = [PIO.write_parameters_device(p, v) for p, v in keys]
    assert files[0] != files[1]
    proofs = [abi_proof(PR.proof_read(RC.create_random_proof_r1cs(r1cs, p, wit["inputs"], wit["aux"], rng=rng))) for p, _ in keys]
    for i, (_, pvk) in enumerate(keys):
        bb.verify_proof(pvk, proofs[i], x)
        with pytest.raises(bb.InvalidProof):
            bb.verify_proof(pvk, proofs[1 - i], x)
    for p, v in keys:
        p.free()
        v.free()
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 4. writing resident keys
# --------------------------------------------------------------------------------------------
def raw_write(worker, params, pvk, vk_only=0, out=None, cap=0):
    n = C.c_size_t(0)
    rc = bb.load_library().bb_params_write(worker._h, params._h, pvk._h, C.c_int(vk_only), out, C.c_size_t(cap), C.c_int(0), C.byref(n))
    return rc, n.value


def test_write(worker, rounds=30):
    rng = random.Random(56)
    tox = toxic_of(rng)
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic(tox)
    mc.generate()
    p = mc.export_params()
    data = PIO.write_parameters(p)
    vk_len = 868 + 96 * p["ic"].shape[0]
    # a key from bb_crs_create + bb_vk_prepare
    made = bb.Parameters(worker, p)
    made_vk = bb.prepare_verifying_key(worker, {"alpha_g1": p["vk_g1"][0], "beta_g2": p["vk_g2"][0], "gamma_g2": p["vk_g2"][1],
                                                "delta_g2": p["vk_g2"][2], "ic": p["ic"]})
    assert PIO.write_parameters_device(made, made_vk) == data
    assert PIO.write_parameters_device(made, made_vk, verifying_key_only=True) == data[:vk_len]
    # a key read by bb_params_read, and a generated one
    read, read_vk = PIO.read_parameters_device(worker, data, verifying_key=True)
    assert PIO.write_parameters_device(read, read_vk) == data
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    gen, gen_vk = GEN.generate_parameters_device(worker, r1cs, *tox)
    assert PIO.write_parameters_device(gen, gen_vk) == data
    # device output
    d = worker.device_alloc(len(data) + 64)
    assert PIO.write_parameters_device(gen, gen_vk, out=(d, len(data))) == len(data)
    host = np.zeros(len(data), np.uint8)
    worker.download(d, host)
    assert host.tobytes() == data
    worker.device_free(d)
    # NULL, short capacity, foreign verifying key
    assert raw_write(worker, gen, gen_vk) == (0, len(data))
    assert raw_write(worker, gen, gen_vk, vk_only=1) == (0, vk_len)
    buf = np.zeros(len(data), np.uint8)
    assert raw_write(worker, gen, gen_vk, out=buf.ctypes.data_as(C.c_void_p), cap=len(data) - 1) == (16, len(data))
    other, other_vk = GEN.generate_parameters_device(worker, r1cs, *toxic_of(rng))
    assert raw_write(worker, gen, other_vk)[0] == 16
    assert "not this key's verifying key" in bb.load_library().bb_last_error().decode()
    # a sharded key
    sharded = bb.Parameters(worker, p, shard_index=0, shard_count=2)
    assert raw_write(worker, sharded, made_vk)[0] == 16
    for obj in (made, made_vk, read, read_vk, gen, gen_vk, other, other_vk, sharded, r1cs):
        obj.free()


def test_write_identity_h(worker):
    """tau a root of unity (here 1): every h element the identity, and the key matches the host generator's; written and
    read back, bb_params_read reports h[0] as the point at infinity, as Parameters::read does"""
    rng = random.Random(57)
    asm = GEN.KeypairAssembly()
    one = asm.alloc_input()
    x = asm.alloc()
    asm.enforce([(x, 1)], [(one, 1)], [(x, 1)])                # x * 1 = x: x is in row 0, where L(1) is one
    tox = toxic_of(rng)
    tox[4] = 1
    want = check_parity(worker, asm, tox)
    assert want["h"].shape[0] == 1 and not np.asarray(want["h"]).any()
    r1cs = RC.R1CS.from_assembly(worker, asm)
    params, pvk = GEN.generate_parameters_device(worker, r1cs, *tox)
    data = PIO.write_parameters_device(params, pvk)
    with pytest.raises(PIO.InvalidData, match=r"h\[0\]: point at infinity"):
        PIO.read_parameters_device(worker, data)
    params.free()
    pvk.free()
    r1cs.free()


def test_profile_stages(worker):
    r1cs = RC.R1CS.synth_mimc(worker, 30, 5)
    worker.set_option("profile", 1)
    worker.profile_reset()
    try:
        params, pvk = GEN.generate_random_parameters_device(worker, r1cs)
        for stage in ("generate.transpose", "generate.lagrange", "generate.qap", "generate.g1", "generate.g2"):
            assert worker.profile_read(stage)[1] == 1, stage
    finally:
        worker.set_option("profile", 0)
    params.free()
    pvk.free()
    r1cs.free()


# --------------------------------------------------------------------------------------------
# 5. sizes only a device reaches
# --------------------------------------------------------------------------------------------
def test_mimc_2_20(worker):
    """the 2^20 MiMC constraint system of bb_synth_mimc_r1cs: the generated key proves the trapdoor-expected bytes"""
    rounds = (1 << 19) - 1
    rng = random.Random(58)
    tox = toxic_of(rng)
    mc = o1.Mimc(rounds, seed=20)
    mc.set_toxic(tox)
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    params, pvk = GEN.generate_parameters_device(worker, r1cs, *tox)
    assert params.lens["h"] == (1 << 20) - 1
    wit = mc.witness()
    r, s = rng.randrange(R), rng.randrange(R)
    proof = RC.create_proof_r1cs(r1cs, params, wit["inputs"], wit["aux"], r, s)
    assert proof == mc.expected_proof(r, s)
    bb.verify_proof(pvk, abi_proof(PR.proof_read(proof)), o1.fr_to_ints(wit["inputs"][1:]))
    params.free()
    pvk.free()
    r1cs.free()
