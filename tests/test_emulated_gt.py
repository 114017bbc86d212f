"""The G_T values of test_gpu_gt.py -- Fp2 and Fp12 operations lane by lane, the multi-pairing, the batch verifier's
value and verify_each's values against exponents of g = e(G1, G2)^k -- executed on host threads (tests/native/) at the
sizes a CPU reaches: every Fp2 edge combination, the Fp12 ops at 65 lanes with two final-exponentiation lanes, up to 5
pairs and 65, batches of at most 5 proofs with one input, and every identity edge of the batch verifier."""
import test_gpu_gt as G
from emulated import worker  # noqa: F401  (the emulated-library fixture)


def test_emulated_fp2_operations(worker):
    G.test_fp2_operations(worker, n_random=200)


def test_emulated_fp12_operations(worker):
    G.test_fp12_operations(worker, sizes=(65,), n_final_exp=2)


def test_emulated_multi_pairing_values(worker):
    """up to 5 pairs, and 65: the Miller loops of a second CTA and an odd tail in the product tree"""
    G.test_multi_pairing_values(worker, sizes=(1, 2, 3, 4, 5, 65))


def test_emulated_batch_exponent_matches_pairs(worker):
    G.test_batch_exponent_matches_pairs(worker)


def test_emulated_batch_values(worker):
    G.test_batch_values(worker, sizes=(1, 2, 5), inputs=(1,))


def test_emulated_batch_identity_edges(worker):
    G.test_batch_identity_edges(worker, n=5, L=1)


def test_emulated_batch_soundness_sweep(worker):
    G.test_batch_soundness_sweep(worker, n=5, L=1)


def test_emulated_each_values(worker):
    G.test_each_values(worker, n=5, L=1)
