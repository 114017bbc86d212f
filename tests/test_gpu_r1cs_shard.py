"""Proving from the witness on a sharded key (bb_groth16_prove_r1cs_begin, csrc/r1cs.cu; r1cs.prove_r1cs_begin): the
owner of polynomial i evaluates matrix i alone straight into its transform buffer, and the partial sums of all shards give
bb_groth16_prove_r1cs's bytes on the unsharded key.  Ranks are simulated in one process on one device: every rank gets its
own device copy of each broadcast vector (prove_end clobbers evals_a).  tests/test_emulated_r1cs_shard.py runs the same
bodies on the emulated device at the sizes a host reaches.
"""
import ctypes as C
import random

import numpy as np
import pytest

import bellman_b200 as bb
from bellman_b200 import r1cs as RC
from bellman_b200.distributed import h_owner
from oracle import o1

import test_gpu_r1cs as G

pytestmark = pytest.mark.gpu

R = o1.FR_MODULUS
ARG = "[bb_status 16]"


@pytest.fixture(scope="module")
def worker():
    w = bb.Worker(0)
    yield w
    w.close()


def domain(n):
    m = 1
    while m < n:
        m *= 2
    return m


def popcount(words):
    return int(sum(bin(int(x)).count("1") for x in words))


def synthetic_key(worker, r1cs, seed, shard=(0, 1)):
    """a key of the constraint system's shape (synthetic vectors), shard `shard` of it"""
    a, bi, b = r1cs.density_words()
    shape = {"m": domain(r1cs.n_constraints), "num_inputs": r1cs.n_inputs, "num_aux": r1cs.n_aux, "a_aux_total": popcount(a),
             "b_in_total": popcount(bi), "b_aux_total": popcount(b)}
    return bb.Parameters.synthetic(worker, seed, shape, *shard)


class Vectors:
    """three device buffers of m Fr: one rank's copies of the coset evaluations of a, b, c"""

    def __init__(self, worker, m, fill=None):
        self.worker, self.m = worker, m
        self.ptrs = [worker.device_alloc(m * 32) for _ in range(3)]
        for i, v in enumerate(fill or ()):
            if v is not None:
                worker.upload(self.ptrs[i], v)

    def get(self, i):
        h = np.zeros((self.m, 4), np.uint64)
        self.worker.download(self.ptrs[i], h)
        return h

    def free(self):
        for p in self.ptrs:
            self.worker.device_free(p)


class Witness:
    """a witness as host arrays and as a device copy"""

    def __init__(self, worker, inputs, aux):
        self.worker = worker
        self.inp, self.aux = (x if isinstance(x, np.ndarray) else G.fr(x) for x in (inputs, aux))
        self.dev = {"inputs": G.device_copy(worker, self.inp), "aux": G.device_copy(worker, self.aux)}

    def args(self, device):
        return (None, None, self.dev) if device else (self.inp, self.aux, None)

    def free(self):
        for p in self.dev.values():
            self.worker.device_free(p)


def begin(r1cs, params, wit, device, own=0, vecs=None):
    inp, aux, d = wit.args(device)
    return RC.prove_r1cs_begin(r1cs, params, inp, aux, own, None if vecs is None else vecs.ptrs, device_ptrs=d)


def want_vectors(worker, r1cs, wit):
    """what an owner does without this call: bb_r1cs_eval, then bb_h_coset_evals of each polynomial from HBM"""
    m = domain(r1cs.n_constraints)
    out = Vectors(worker, m)
    for i, p in enumerate(r1cs.eval(wit.inp, wit.aux)):
        bb.h_coset_evals(worker, p, r1cs.n_constraints, out.ptrs[i])
    res = [out.get(i) for i in range(3)]
    out.free()
    return res


def counted(worker, fn):
    l0, (h0, _) = worker.kernel_launches, worker.bytes_copied()
    res = fn()
    worker.synchronize()
    return res, worker.kernel_launches - l0, worker.bytes_copied()[0] - h0


# --------------------------------------------------------------------------------------------
# 1. the owner's vectors: bb_h_coset_evals of bb_r1cs_eval's polynomial, byte for byte
# --------------------------------------------------------------------------------------------
def check_owner(worker, r1cs, inputs, aux, params=None):
    own_params = params is None
    params = params or synthetic_key(worker, r1cs, 3)
    wit = Witness(worker, inputs, aux)
    want = want_vectors(worker, r1cs, wit)
    m = domain(r1cs.n_constraints)
    for device in (False, True):
        for own in (1, 2, 4, 7):
            vecs = Vectors(worker, m)
            state = begin(r1cs, params, wit, device, own, vecs)
            bb.h_coset_evals_wait(worker)
            for i in range(3):
                if own >> i & 1:
                    assert np.array_equal(vecs.get(i), want[i]), (device, own, "abc"[i])
            bb.prove_end(state, vecs.ptrs)                          # (the unowned vectors are whatever the buffers held)
            vecs.free()
    wit.free()
    if own_params:
        params.free()


def test_owner_mimc322(worker, rounds=322):
    """the MiMC system of test_gpu_r1cs.py (646 rows: N < m) with its own key"""
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic([random.Random(40).randrange(1, R) for _ in range(5)])
    mc.generate()
    params = bb.Parameters(worker, mc.export_params())
    wit = mc.witness()
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    check_owner(worker, r1cs, wit["inputs"], wit["aux"], params)
    r1cs.free()
    params.free()


def test_owner_from_assembly(worker, rounds=40):
    rng = random.Random(41)
    constants = [rng.randrange(R) for _ in range(rounds)]
    pa, asm = G.synthesize(G.B.mimc_circuit(G.B.Bls12.fr, rng.randrange(R), rng.randrange(R), constants))
    r1cs = RC.R1CS.from_assembly(worker, asm)
    check_owner(worker, r1cs, pa.input_assignment, pa.aux_assignment)
    r1cs.free()


def random_r1cs(worker, seed, total_rows, lengths, cta_only_in=None, empty=None, n_inputs=3, n_aux=50):
    """test_gpu_r1cs.random_system's rows; cta_only_in: one matrix gets the one row above R1CS_WARP_MAX terms; empty: a
    matrix with no terms"""
    rng = random.Random(seed)
    mats = G.random_system(rng, total_rows - n_inputs, n_inputs, n_aux, lengths)
    nv = n_inputs + n_aux
    if cta_only_in is not None:
        mats[cta_only_in][rng.randrange(total_rows - n_inputs)] = [(rng.randrange(nv), rng.randrange(1, R)) for _ in range(4096)]
    if empty is not None:
        mats[empty] = [[] for _ in mats[empty]]
    z = [1] + [rng.randrange(R) for _ in range(nv - 1)]
    return RC.R1CS(worker, n_inputs, n_aux, *(G.csr(rows) for rows in mats)), z[:n_inputs], z[n_inputs:]


def test_owner_random(worker, lengths=G.EMU_LENGTHS, log_rows=9):
    """rows in all three bins in every matrix, N = m and N < m; CTA rows in one matrix only; a matrix with no terms"""
    for seed, total, kw in ((1, 1 << log_rows, {}), (2, (1 << log_rows) - 5, {}),
                            (3, 1 << log_rows, {"cta_only_in": 1}), (4, (1 << log_rows) + 1, {"cta_only_in": 2, "empty": 0}),
                            (5, 1 << log_rows, {"empty": 2})):
        ls = tuple(x for x in lengths if x <= 2048) if "cta_only_in" in kw else lengths
        r1cs, inp, aux = random_r1cs(worker, seed, total, ls, **kw)
        if "empty" in kw:
            assert r1cs.nnz[kw["empty"]] == (r1cs.n_inputs if kw["empty"] == 0 else 0)
        check_owner(worker, r1cs, inp, aux)
        r1cs.free()


# --------------------------------------------------------------------------------------------
# 2. sharded proofs on one device
# --------------------------------------------------------------------------------------------
def owned(rank, count):
    return sum(1 << i for i in range(3) if h_owner(i, count) == rank)


def prove_shards(worker, r1cs, keys, wit, device, r, s):
    """every shard through begin (split, own = its h_owner polynomials) / wait / end, the broadcast as uploads of the
    owners' vectors into each rank's own buffers, then finalize over all partial sums"""
    count, m = len(keys), domain(r1cs.n_constraints)
    bcast = [None] * 3
    for k in range(count):                              # the owners' vectors, as each owner rank computes them
        if owned(k, count):
            vecs = Vectors(worker, m)
            state = begin(r1cs, keys[k], wit, device, owned(k, count), vecs)
            bb.h_coset_evals_wait(worker)
            for i in range(3):
                if owned(k, count) >> i & 1:
                    bcast[i] = vecs.get(i)
            bb.prove_end(state, vecs.ptrs)
            vecs.free()
    partials = []
    for k in range(count):
        own = owned(k, count)
        vecs = Vectors(worker, m)
        state = begin(r1cs, keys[k], wit, device, own, vecs)
        bb.h_coset_evals_wait(worker)
        for i in range(3):
            if own >> i & 1:
                assert np.array_equal(vecs.get(i), bcast[i])
            else:
                worker.upload(vecs.ptrs[i], bcast[i])
        partials.append(bb.prove_end(state, vecs.ptrs))
        vecs.free()
    return bb.finalize(keys[0], partials, r, s)


def prove_replicated(r1cs, keys, wit, device, r, s):
    return bb.finalize(keys[0], [bb.prove_end(begin(r1cs, key, wit, device)) for key in keys], r, s)


def test_sharded_mimc(worker, rounds=322, counts=(1, 2, 3, 5, 8)):
    rng = random.Random(42)
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    p = mc.export_params()
    w = mc.witness()
    wit = Witness(worker, w["inputs"], w["aux"])
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    r, s = rng.randrange(R), rng.randrange(R)
    whole = bb.Parameters(worker, p)
    want = RC.create_proof_r1cs(r1cs, whole, wit.inp, wit.aux, r, s)
    assert want == mc.expected_proof(r, s)
    for windows, cnts in ((4, counts), (1, counts[-2:])):
        worker.set_option("shard_windows", windows)
        try:
            for count in cnts:
                keys = [bb.Parameters(worker, p, shard_index=k, shard_count=count) for k in range(count)]
                for device in (False, True):
                    assert prove_shards(worker, r1cs, keys, wit, device, r, s) == want, (windows, count, device)
                    assert prove_replicated(r1cs, keys, wit, device, r, s) == want, (windows, count, device)
                for key in keys:
                    key.free()
        finally:
            worker.set_option("shard_windows", 4)
    whole.free()
    r1cs.free()
    wit.free()


def check_synth_sharded(worker, log_n, count):
    """the bench workload's key (bb_synth_crs) in `count` shards, its witness from HBM"""
    rounds = (1 << (log_n - 1)) - 1
    asg, shape = bb.synth_mimc(rounds, seed=20)
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 20)
    wit = Witness(worker, asg.input_assignment, asg.aux_assignment)
    r, s = 0x1234567, 0x7654321
    whole = bb.Parameters.synthetic(worker, 21, shape)
    want = RC.create_proof_r1cs(r1cs, whole, None, None, r, s, device_ptrs=wit.dev)
    assert want == bb.create_proof(asg, whole, r, s)
    whole.free()
    keys = [bb.Parameters.synthetic(worker, 21, shape, k, count) for k in range(count)]
    assert prove_shards(worker, r1cs, keys, wit, True, r, s) == want
    assert prove_replicated(r1cs, keys, wit, True, r, s) == want
    for key in keys:
        key.free()
    r1cs.free()
    wit.free()


def test_sharded_synth_2_16(worker):
    check_synth_sharded(worker, 16, 3)


# --------------------------------------------------------------------------------------------
# 3. counters and profile stages
# --------------------------------------------------------------------------------------------
def test_counters(worker, rounds=322):
    rng = random.Random(43)
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    p = mc.export_params()
    w = mc.witness()
    wit = Witness(worker, w["inputs"], w["aux"])
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    asg = r1cs.assignment(wit.inp, wit.aux)
    n, m = r1cs.n_constraints, domain(r1cs.n_constraints)
    want = want_vectors(worker, r1cs, wit)
    _, l_eval, _ = counted(worker, lambda: r1cs.eval(wit.inp, wit.aux))
    scratch = Vectors(worker, m)
    _, l_coset, _ = counted(worker, lambda: bb.h_coset_evals(worker, asg.a, n, scratch.ptrs[0]))
    scratch.free()
    for count in (1, 3):
        keys = [bb.Parameters(worker, p, shard_index=k, shard_count=count) for k in range(count)]
        for device in (False, True):
            for k in range(count):
                def old():                                   # bb_groth16_prove_begin + prove_end of this shard, same vectors
                    vecs = Vectors(worker, m, want)
                    d = None if not device else {"a": 0, "b": 0, "c": 0, **wit.dev}
                    res = bb.prove_end(bb.prove_begin(asg, keys[k], d), vecs.ptrs)
                    vecs.free()
                    return res

                def new(own):
                    vecs = Vectors(worker, m, [None if own >> i & 1 else want[i] for i in range(3)])
                    state = begin(r1cs, keys[k], wit, device, own, vecs)
                    bb.h_coset_evals_wait(worker)
                    res = bb.prove_end(state, vecs.ptrs)
                    vecs.free()
                    return res

                old()                                        # (a key's first proof builds what it keeps for the next)
                base, l_old, h_old = counted(worker, old)
                got, l_none, h_none = counted(worker, lambda: new(0))
                assert got == base and l_none == l_old and h_none == h_old, (count, k, device)
                for i in range(3):
                    got, l_own, h_own = counted(worker, lambda: new(1 << i))
                    assert got == base and h_own == h_old, (count, k, device, i)
                    assert 0 < l_own - l_old <= l_eval + l_coset, (l_own - l_old, l_eval, l_coset)
        for key in keys:
            key.free()
    # profile mode: the owner stage's stages
    key = bb.Parameters(worker, p)
    worker.set_option("profile", 1)
    worker.profile_reset()
    try:
        vecs = Vectors(worker, m)
        state = begin(r1cs, key, wit, False, 7, vecs)
        bb.h_coset_evals_wait(worker)
        bb.prove_end(state, vecs.ptrs)
        vecs.free()
        assert worker.profile_read("r1cs_owner.upload")[1:] == (1, 0)
        assert worker.profile_read("r1cs_owner.eval")[1:] == (3, sum(r1cs.nnz))            # each matrix's own terms
        assert worker.profile_read("r1cs_owner.transforms")[1:] == (3, 3 * m)
        worker.profile_reset()                                  # bb_groth16_prove_r1cs: its r1cs.* stages
        RC.create_proof_r1cs(r1cs, key, wit.inp, wit.aux, 1, 2)
        for stage in ("r1cs.upload", "r1cs.eval"):
            assert worker.profile_read(stage)[1:] == (1, sum(r1cs.nnz)), stage
    finally:
        worker.set_option("profile", 0)
        worker.profile_reset()
    key.free()
    r1cs.free()
    wit.free()


# --------------------------------------------------------------------------------------------
# 4. errors
# --------------------------------------------------------------------------------------------
def test_errors(worker, rounds=20):
    rng = random.Random(44)
    mc = o1.Mimc(rounds, seed=5)
    mc.set_toxic([rng.randrange(1, R) for _ in range(5)])
    mc.generate()
    base = mc.export_params()
    w = mc.witness()
    wit = Witness(worker, w["inputs"], w["aux"])
    r1cs = RC.R1CS.synth_mimc(worker, rounds, 5)
    params = bb.Parameters(worker, base)
    m = domain(r1cs.n_constraints)
    vecs = Vectors(worker, m)
    lib = bb.load_library()
    r, s = rng.randrange(R), rng.randrange(R)

    def no_device_work(fn, match):
        l0, b0 = worker.kernel_launches, worker.bytes_copied()
        with pytest.raises(bb.BackendError, match=match) as e:
            fn()
        assert ARG in str(e.value)
        assert (worker.kernel_launches, worker.bytes_copied()) == (l0, b0)

    def raw(ctx=worker._h, crs=params._h, rc=r1cs._h, inp=None, n_in=None, aux=None, n_aux=None, on_device=0, own=0, evals=None, out=True):
        h = C.c_void_p()
        inp = wit.inp.ctypes.data if inp is None else inp
        aux = wit.aux.ctypes.data if aux is None else aux
        n_in = r1cs.n_inputs if n_in is None else n_in
        n_aux = r1cs.n_aux if n_aux is None else n_aux
        d = None if evals is None else (C.c_void_p * 3)(*evals)
        bb._check(lib.bb_groth16_prove_r1cs_begin(ctx, crs, rc, C.c_void_p(inp), C.c_size_t(n_in), C.c_void_p(aux), C.c_size_t(n_aux),
                                                  C.c_int(on_device), C.c_uint(own), d, C.byref(h) if out else None))
        assert h.value is not None
        bb.prove_end(h, None if evals is None else vecs.ptrs)

    raw()                                                                      # the helper itself is sound
    no_device_work(lambda: raw(ctx=None), "null argument")
    no_device_work(lambda: raw(crs=None), "null argument")
    no_device_work(lambda: raw(rc=None), "null argument")
    no_device_work(lambda: raw(out=False), "null argument")
    other = bb.Worker(0)
    foreign_key = bb.Parameters(other, base)
    foreign_r1cs = RC.R1CS.synth_mimc(other, rounds, 5)
    no_device_work(lambda: raw(crs=foreign_key._h), "another context")
    no_device_work(lambda: raw(rc=foreign_r1cs._h), "another context")
    no_device_work(lambda: raw(n_aux=r1cs.n_aux - 1), "witness has")
    no_device_work(lambda: raw(n_in=r1cs.n_inputs + 1), "witness has")
    no_device_work(lambda: raw(inp=0), "null witness pointer")
    no_device_work(lambda: raw(aux=0), "null witness pointer")
    d_in, d_aux = bb._addr(wit.dev["inputs"]), bb._addr(wit.dev["aux"])
    raw(inp=d_in, aux=d_aux, on_device=1)
    no_device_work(lambda: raw(inp=d_in + 8, aux=d_aux, on_device=1), "aligned")
    no_device_work(lambda: raw(inp=d_in, aux=d_aux + 8, on_device=1), "aligned")
    ev = [bb._addr(p) for p in vecs.ptrs]
    raw(own=7, evals=ev)
    no_device_work(lambda: raw(own=8, evals=ev), "own = 8")
    no_device_work(lambda: raw(own=1), "without evaluation vectors")
    no_device_work(lambda: raw(own=2, evals=[ev[0], None, ev[2]]), "vector b is null")
    no_device_work(lambda: raw(own=4, evals=[ev[0], ev[1], ev[2] + 8]), "vector c is not 16-byte aligned")
    raw(own=3, evals=[ev[0], ev[1], ev[2] + 8])                              # an unowned vector is not checked (ended with vecs)
    foreign_r1cs.free()
    foreign_key.free()
    other.close()
    # ending a state the wrong way: BB_ERR_ARG, the state freed
    with pytest.raises(bb.BackendError, match="three evaluation vectors are needed"):
        bb.prove_end(begin(r1cs, params, wit, False, 1, vecs), None)
    with pytest.raises(bb.BackendError, match="no evaluation vectors"):
        bb.prove_end(begin(r1cs, params, wit, False), vecs.ptrs)

    # MSM errors: a shard with an identity base in l; delta = identity first
    def variant(**changes):
        q = {k: np.array(v, copy=True) for k, v in base.items()}
        for k, f in changes.items():
            q[k] = f(q[k])
        return q

    def identity_l(v):
        v = v.reshape(-1, 12).copy()
        v[-1] = 0
        return v

    def zero_delta(v):
        v = v.reshape(3, -1).copy()
        v[2] = 0
        return v

    def short(v):
        return v.reshape(-1, v.shape[-1])[:-1]

    good, bad = bb.Parameters(worker, base, 0, 2), bb.Parameters(worker, variant(l=identity_l), 1, 2)
    assert len(bb.prove_end(begin(r1cs, good, wit, False, 5, vecs), vecs.ptrs)) == bb.PARTIALS_BYTES
    with pytest.raises(bb.UnexpectedIdentity):
        bb.prove_end(begin(r1cs, bad, wit, False, 2, vecs), vecs.ptrs)
    good.free()
    bad.free()
    for q in (variant(vk_g1=zero_delta), variant(vk_g1=zero_delta, b_g1=short)):
        key = bb.Parameters(worker, q)
        with pytest.raises(bb.UnexpectedIdentity) as want:
            RC.create_proof_r1cs(r1cs, key, wit.inp, wit.aux, r, s)
        for split in (True, False):
            with pytest.raises(bb.UnexpectedIdentity) as got:
                bb.prove_end(begin(r1cs, key, wit, False, 7 if split else 0, vecs if split else None), vecs.ptrs if split else None)
            assert str(got.value) == str(want.value)
        key.free()
    # an unsatisfied witness proves, as in the reference
    aux = wit.aux.copy()
    aux[3] = G.fr([rng.randrange(R)])[0]
    assert r1cs.which_is_unsatisfied(wit.inp, aux) is not None
    broken = Witness(worker, wit.inp, aux)
    want = RC.create_proof_r1cs(r1cs, params, broken.inp, broken.aux, r, s)
    for count in (1, 2):
        keys = [bb.Parameters(worker, base, k, count) for k in range(count)]
        assert prove_shards(worker, r1cs, keys, broken, False, r, s) == want
        assert prove_replicated(r1cs, keys, broken, True, r, s) == want
        for key in keys:
            key.free()
    broken.free()
    vecs.free()
    params.free()
    r1cs.free()
    wit.free()
