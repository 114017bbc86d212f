"""Multi-GPU plumbing for the base-range sharded MSM (SURVEY.md 8e): one process per GPU,
torch.distributed for the single exchange step.  The data path has exactly one collective per
proof: an all-gather of the per-shard partial sums (960 bytes per rank)."""
import numpy as np

from . import PARTIALS_BYTES

MSG_BYTES = 159          # error text a failing rank shares with the others (960 + 1 + 159 = 1120 bytes per rank)


def shard_range(length, index, count):
    """Contiguous range `index` of `count` over `length` items:
    [length*index/count, length*(index+1)/count) -- the split bb_crs_create applies to the base
    vectors (after it has set aside up to 4 window groups, see prover.cu: shard_policy)."""
    return length * index // count, length * (index + 1) // count


def all_gather_partials(partials, group=None):
    """All-gather one 960-byte partial-sum blob per rank; returns the list ordered by rank.
    Works on NCCL (blob staged through a CUDA tensor) and on gloo (CPU tensor)."""
    import torch
    import torch.distributed as dist

    assert len(partials) == PARTIALS_BYTES
    world = dist.get_world_size(group)
    backend = dist.get_backend(group)
    device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    mine = torch.frombuffer(bytearray(partials), dtype=torch.uint8).to(device)
    out = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(out, mine, group=group)
    return [bytes(t.cpu().numpy()) for t in out]


def max_over_ranks(seconds, group=None):
    import torch
    import torch.distributed as dist

    backend = dist.get_backend(group)
    device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    t = torch.tensor([seconds], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


def _all_reduce(value, op, group=None):
    import torch
    import torch.distributed as dist

    backend = dist.get_backend(group)
    device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=getattr(dist.ReduceOp, op), group=group)
    return float(t.item())


def autotune_sharded(assignment, params, r, s, device_ptrs=None, reps=3, group=None, split_h=True):
    """bb_groth16_autotune for a sharded key: every MSM form (bellman_b200.tuning_names()) proves `assignment` through
    create_proof_sharded on all ranks; a form is eligible only if every rank could set it up and rank 0's proof bytes
    equal the default form's; the time of a form is the fastest of `reps` proofs, each the MAX over ranks between two
    barriers; all ranks end up configured for the same, fastest form.  Collective: call it on every rank.
    Returns {"chosen", "name", "ms"} (ms < 0: -1 not available on some rank, -2 failed, -3 different proof)."""
    import time

    import torch.distributed as dist

    from . import BackendError, SynthesisError, tuning_names

    names = tuning_names()
    rank = dist.get_rank(group)
    ms, ref = [], None
    for index in range(len(names)):
        ok = 1.0
        try:
            params.apply_tuning(index)
        except BackendError:
            if index == 0:
                raise
            ok = 0.0
        if _all_reduce(ok, "MIN", group) < 1.0:
            ms.append(-1.0)
            continue
        def prove():
            """one sharded proof; every rank learns whether ANY rank failed (rank 0 alone can fail in finalize), so that
            all ranks leave this form together and the collectives below stay matched"""
            proof, err = None, None
            try:
                proof = create_proof_sharded(assignment, params, params, r, s, device_ptrs, group, split_h)
                params.worker.synchronize()
            except (BackendError, SynthesisError, AssertionError) as e:
                err = e
            done = time.perf_counter()                   # the status exchange below is not part of the proof
            if _all_reduce(1.0 if err else 0.0, "MAX", group) > 0.0:
                raise err if err is not None else BackendError("the sharded proof failed on another rank")
            return proof, done

        try:
            proof, _ = prove()
            same = 1.0
            if rank == 0:
                if index == 0:
                    ref = proof
                same = 1.0 if proof == ref else 0.0
            if _all_reduce(same, "MIN", group) < 1.0:
                ms.append(-3.0)
                continue
            best = None
            for _ in range(reps):
                params.worker.synchronize()
                dist.barrier(group)
                t0 = time.perf_counter()
                _, t1 = prove()
                dt = _all_reduce(t1 - t0, "MAX", group)
                best = dt if best is None or dt < best else best
            ms.append(round(1e3 * best, 3))
        except (BackendError, SynthesisError, AssertionError):
            if index == 0:
                raise
            ms.append(-2.0)
    chosen = min((i for i in range(len(names)) if ms[i] > 0), key=lambda i: ms[i])
    ok = 1.0
    try:
        params.apply_tuning(chosen)
    except BackendError:
        ok = 0.0
    if _all_reduce(ok, "MIN", group) < 1.0:              # (a table that no longer fits on one rank:) everybody back to the default
        ms[chosen] = -1.0
        chosen = 0
        params.apply_tuning(0)
    HOST_MS.clear()
    return {"chosen": chosen, "name": names[chosen], "ms": ms}


_EVAL_BUFFERS = {}       # (device, m) -> three tensors of m Fr: the coset evaluations of a, b, c on this rank
HOST_MS = {}             # accumulated host milliseconds of create_proof_sharded's phases on this rank (bench.py reads and resets it)


def _mark(name, t0):
    import time
    now = time.perf_counter()
    HOST_MS[name] = HOST_MS.get(name, 0.0) + 1e3 * (now - t0)
    return now


def h_owner(poly_index, world):
    """Which rank takes polynomial 0 = a, 1 = b, 2 = c through ifft + coset_fft: one each from three ranks on;
    with two ranks the first takes a and c."""
    return poly_index % world if world < 3 else poly_index


def create_proof_sharded(assignment, params, full_vk_params, r, s, device_ptrs=None, group=None, split_h=True):
    """One proof over all ranks of `group` (create_proof, groth16/src/prover.rs:217-360, with the MSMs
    sharded): every rank runs its shard of the eight MSMs, the 960-byte partial sums AND each rank's status and
    error text are all-gathered in one collective, and rank 0 finalises.  A SynthesisError on any rank is
    re-raised on every rank (nobody is left waiting in a collective).  Returns the 192 proof bytes on rank
    0, None elsewhere.  `full_vk_params` is any Parameters object of this rank (only its verifying-key elements
    are read by finalize).

    split_h: the H pipeline is divided by polynomial instead of being replicated.  Each NTT stays on one GPU:
    rank h_owner(i) takes polynomial i of (a, b, c) through ifft + coset_fft (two transforms) and broadcasts
    the m evaluations; every rank then runs the last transform (a b - c, / Z, icoset_fft) itself.  The longest
    chain drops from seven transforms to three, and a rank uploads only the polynomials it owns.  The seven
    witness MSMs are queued first and run underneath."""
    import bellman_b200 as bb

    def start(bufs, own, lap):
        n = assignment.a.shape[0]
        for i, name in enumerate(("a", "b", "c")):
            if own >> i & 1:
                if device_ptrs is not None:
                    bb.h_coset_evals_async(params.worker, device_ptrs[name], n, bufs[i].data_ptr(), on_device=True)
                else:
                    bb.h_coset_evals_async(params.worker, getattr(assignment, name), n, bufs[i].data_ptr())
        lap("h_stage1_launch")
        state = bb.prove_begin(assignment, params, device_ptrs)
        lap("queue_witness_msms")
        return state

    return _prove_collective(lambda: assignment.a.shape[0], start, lambda: bb.prove_partials(assignment, params, device_ptrs),
                             params, full_vk_params, r, s, group, split_h)


def create_proof_r1cs_sharded(r1cs, params, full_vk_params, input_assignment, aux_assignment, r, s, device_ptrs=None, group=None,
                              split_h=True):
    """create_proof_sharded from the witness alone (bb_groth16_prove_r1cs_begin on every rank's key shard): the same
    collective -- the h_owner split, every rank in every broadcast, one all-gather of partial sums, status and error text,
    finalize on rank 0 -- but no rank evaluates a, b, c on the host or uploads them.  With split_h, rank h_owner(i)
    evaluates matrix i alone straight into the buffer it broadcasts and transforms it there, launched before its witness
    MSMs are queued; otherwise (or with one rank) every rank runs the whole H pipeline from its own copy of the witness.
    Witness arguments as r1cs.create_proof_r1cs's.  Returns the 192 proof bytes on rank 0, None elsewhere."""
    import bellman_b200 as bb
    from . import r1cs as RC

    def begin(own=0, evals=None):
        return RC.prove_r1cs_begin(r1cs, params, input_assignment, aux_assignment, own, evals, device_ptrs)

    def start(bufs, own, lap):
        state = begin(own, [b.data_ptr() for b in bufs])      # the owner stage launched, then the witness MSMs queued
        lap("r1cs_begin")
        return state

    return _prove_collective(lambda: r1cs.n_constraints, start, lambda: bb.prove_end(begin()),
                             params, full_vk_params, r, s, group, split_h)


def _prove_collective(n_constraints, start, partials, params, full_vk_params, r, s, group, split_h):
    """The collective of one sharded proof.  A rank starts its proof one of two ways:
    start(bufs, own, lap) -> the bb_prove state: polynomial i's coset evaluations launched into bufs[i] for every bit i
    of `own` (the polynomials this rank owns), then the witness MSMs queued (lap(name) records a host phase);
    partials() -> the 960 bytes of the whole proof on this rank (replicated H pipeline).
    n_constraints() -> the rows of a, b, c."""
    import torch
    import torch.distributed as dist

    import threading

    from . import BackendError, _ERRORS, finalize, finalize_static, h_coset_evals_wait, prove_end

    rank, world = dist.get_rank(group), dist.get_world_size(group)
    backend = dist.get_backend(group)
    device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    # rank 0: the scalar multiplications of the finalisation that need no MSM result run on a host
    # thread while the devices compute the partial sums
    ahead = {}
    worker_thread = None
    if rank == 0:
        def _static():
            try:
                ahead["static"] = finalize_static(full_vk_params, r, s)
            except Exception as e:                       # reported by finalize() below if it matters
                ahead["error"] = e
        worker_thread = threading.Thread(target=_static)
        worker_thread.start()
    import time
    t_ = [time.perf_counter()]
    status, blob, msg = 0, bytes(PARTIALS_BYTES), ""

    def lap(name):
        t_[0] = _mark(name, t_[0])

    def code_of(e):
        return next((code for code, cls in _ERRORS.items() if isinstance(e, cls)), 17 if isinstance(e, BackendError) else 255)

    if split_h and world > 1:
        # 1. the coset evaluations of the polynomials this rank owns are LAUNCHED (asynchronous, high-priority stream):
        #    they head the longest chain of the proof; 2. the witness MSMs are queued underneath (~1 ms of host time,
        #    during which the transforms already run); 3. the evaluations are awaited and broadcast; 4. the last
        #    transform, the h MSM, the waits.  Awaiting the evaluations before the witness MSMs are queued would leave
        #    the GPUs without MSM kernels in flight for that long; launching the transforms first without waiting for
        #    them keeps the critical chain first and the MSMs queued under it.
        # A failure is carried to the all-gather; the broadcasts are entered by every rank whatever happened
        # (nobody may skip a collective).
        state, bufs = None, None
        try:
            n = n_constraints()
            m = 1
            while m < n:
                m *= 2
            key = (str(device), m)
            if key not in _EVAL_BUFFERS:
                _EVAL_BUFFERS[key] = [torch.empty((m, 4), dtype=torch.int64, device=device) for _ in range(3)]
            bufs = _EVAL_BUFFERS[key]
            own = sum(1 << i for i in range(3) if h_owner(i, world) == rank)
            state = start(bufs, own, lap)
        except Exception as e:
            msg, status = str(e), code_of(e)
        if bufs is not None:
            try:
                h_coset_evals_wait(params.worker)
            except Exception as e:
                if status == 0:
                    msg, status = str(e), code_of(e)
        else:                                            # the buffers could not even be made: take part with scratch ones
            bufs = [torch.empty((1, 4), dtype=torch.int64, device=device) for _ in range(3)]
        lap("h_stage1_wait")
        pending = [dist.broadcast(bufs[i], src=h_owner(i, world), group=group, async_op=True) for i in range(3)]
        for p in pending:
            p.wait()
        if backend == "nccl":
            torch.cuda.current_stream().synchronize()
        lap("broadcast_wait")
        if state is not None:
            try:
                if status == 0:
                    blob = prove_end(state, [b.data_ptr() for b in bufs])
                else:
                    prove_end(state, None)               # drain and free what the start queued
            except Exception as e:
                if status == 0:
                    msg, status = str(e), code_of(e)
        lap("h_final_and_msm_waits")
    else:
        try:
            blob = partials()
        except Exception as e:                           # whatever it is, the other ranks must not be left in the all-gather
            msg, status = str(e), code_of(e)
        lap("prove_partials")
    # one collective: partial sums, status and (on failure) the failing rank's own message
    text = msg.encode("utf-8", "replace")[:MSG_BYTES].ljust(MSG_BYTES, b"\0")
    mine = torch.frombuffer(bytearray(blob + bytes([status]) + text), dtype=torch.uint8).to(device)
    out = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(out, mine, group=group)
    gathered = bytes(torch.stack(out).cpu().numpy().tobytes())       # one device->host copy for all ranks' blobs
    gathered = [gathered[i * len(mine):(i + 1) * len(mine)] for i in range(world)]
    lap("all_gather")
    if worker_thread is not None:
        worker_thread.join()
    for rk, g in enumerate(gathered):
        if g[PARTIALS_BYTES]:
            code = g[PARTIALS_BYTES]
            what = g[PARTIALS_BYTES + 1:].rstrip(b"\0").decode("utf-8", "replace")
            raise _ERRORS.get(code, BackendError)(f"rank {rk} failed with status {code}" + (f": {what}" if what else ""))
    if rank == 0:
        proof = finalize(full_vk_params, [g[:PARTIALS_BYTES] for g in gathered], r, s, static=ahead.get("static"))
        lap("finalize")
        return proof
    return None
