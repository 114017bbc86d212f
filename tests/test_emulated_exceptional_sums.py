"""The exceptional additions of test_gpu_exceptional_sums.py -- doublings, cancellations and identities at every MSM
stage, on keys of known multiples of the generator -- executed on host threads (tests/native/) at the sizes a CPU
reaches: G1 jobs of 128 points and G2 jobs of 32, every MSM configuration with two or three of the (key, scalar) family
pairs, the targeted fold and reduction collisions at full size, circuits of 24 aux values, batches of at most 5, and
forced halving rounds and small windows so that the deep stages still run."""
import pytest

import bellman_b200 as bb
import test_gpu_exceptional_sums as G
from emulated import worker  # noqa: F401  (the emulated-library fixture)

PAIRS = [(kf, sf) for kf in G.KEY_FAMILIES for sf in G.SCALAR_FAMILIES]
SHAPE = dict(n_inputs=2, n_aux=24, n_constraints=20)


@pytest.mark.parametrize("config", list(G.MSM_CONFIGS))
@pytest.mark.parametrize("group", [bb.G1, bb.G2], ids=["G1", "G2"])
def test_emulated_msm_special_sums(worker, group, config):
    """two or three (key, scalar) pairs per configuration and group: the 22 cells together take each of the 45 pairs once"""
    cell = 2 * list(G.MSM_CONFIGS).index(config) + group - 1
    combos = [p for j, p in enumerate(PAIRS) if j % (2 * len(G.MSM_CONFIGS)) == cell]
    G.test_msm_special_sums(worker, group, config, n_g1=128, n_g2=32, combos=combos)


def test_emulated_msm_cancels_with_nonzero_scalars(worker):
    G.test_msm_cancels_with_nonzero_scalars(worker, n=16)


def test_emulated_msm_fold_collisions(worker):
    G.test_msm_fold_collisions(worker)


def test_emulated_bucket_reduction_collisions(worker):
    G.test_bucket_reduction_collisions(worker)


def test_emulated_batch_horner_fold(worker):
    G.test_batch_horner_fold(worker, shape=SHAPE)


def test_emulated_single_proofs(worker):
    combos = [("ones", "one"), ("alternating", "plus_minus")]
    G.test_single_proofs(worker, shape=SHAPE, combos=combos, opts=G.DEEP, create_all=False)


def test_emulated_sharded_proofs(worker):
    G.test_sharded_proofs(worker, shape=SHAPE, counts=(3,), key_families=("small",), witness_families=("carry",), by_range=2,
                          opts=G.DEEP)


def test_emulated_batches(worker):
    """the one-bucket-set form, host and device witnesses, whole and in sub-batches of 3 and 1 (the per-window form's
    batched job, with its device Horner fold, runs in test_emulated_batch_horner_fold)"""
    G.test_batches(worker, shape=SHAPE, key_families=("alternating",), count=4, batch_max=3, opts=G.DEEP, forms=(2,))


def test_emulated_identity_results(worker):
    """every identity case alone and in batches of five, in the one-bucket-set form"""
    with G.options(worker, prove_batch_max=5):
        G.test_identity_results(worker, shape=SHAPE, opts=G.DEEP, forms=(2,), single_forms=(2,))
