/*
 * bellman_b200 -- bench generators and parity-test diagnostics.
 *
 * NOT part of the drop-in boundary (that is bellman_b200.h): nothing here stands for a bellman
 * item.  bb_synth_* manufacture benchmark-size inputs in HBM, bb_selftest_* / bb_diag_* expose
 * single device routines to tests/ so that each can be compared with the CPU oracle.
 */
#ifndef BELLMAN_B200_DIAG_H
#define BELLMAN_B200_DIAG_H

#include "bellman_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- synthetic workload (bench only): the MiMC chain of groth16/tests/common/mod.rs:48-129
 *      through ProvingAssignment's bookkeeping (groth16/src/prover.rs:73-145,193-215) -------- */
/* pseudorandom canonical scalars (< 2^254) generated in HBM */
int bb_synth_scalars_device(bb_ctx* ctx, uint64_t seed, size_t n, void* d_out);
/* base vector [k_i]G with counter-based pseudorandom k_i, made on the device straight into a
 * bb_bases / bb_crs (shard-consistent across ranks) */
int bb_synth_bases(bb_ctx* ctx, int group, uint64_t seed, size_t n, size_t global_offset, size_t global_len, bb_bases** out);
int bb_synth_crs(bb_ctx* ctx, uint64_t seed, size_t h_len, size_t l_len, size_t a_len, size_t b_len,
                 uint32_t shard_index, uint32_t shard_count, bb_crs** out);
int bb_synth_mimc_shape(size_t rounds, uint64_t shape[7]);
int bb_synth_mimc_witness(size_t rounds, uint64_t seed, uint64_t* a, uint64_t* b, uint64_t* c,
                          uint64_t* inputs, uint64_t* aux, uint64_t* a_aux_density,
                          uint64_t* b_input_density, uint64_t* b_aux_density);
/* the constraints bb_synth_mimc_witness's circuit enforces (same constants for the same seed), in bb_r1cs_matrix form
 * without the input rows (bb_r1cs_create appends them): 2 rounds rows; variables ONE = 0, the image = 1, then aux j = 2 + j.
 * a_off, b_off, c_off: 2 rounds + 1 offsets each; A holds 3 rounds terms, B 4 rounds, C 3 rounds (vars uint32, coeffs
 * Montgomery Fr).  Host code. */
int bb_synth_mimc_r1cs(size_t rounds, uint64_t seed, uint64_t* a_off, uint32_t* a_vars, uint64_t* a_coeffs,
                       uint64_t* b_off, uint32_t* b_vars, uint64_t* b_coeffs, uint64_t* c_off, uint32_t* c_vars, uint64_t* c_coeffs);

/* ---- diagnostics (used by the parity tests; not part of the bellman-facing surface) ------ */
/* element-wise on the device: field 0 = Fr, 1 = Fp (Montgomery); op 0 mul, 1 add, 2 sub, 3 sqr;
 * Fp only: 4 = inverse by the binary Euclidean algorithm (fp_inv_gcd), 5 = inverse as a^(p-2); 0 -> 0.
 * field 2 = Fp2, elements 24 u64 (c0 then c1, Montgomery): op 0 mul (the out-of-line operator*), 1 add, 2 sub,
 * 3 sqr (the out-of-line sqr()), 4 inverse (fp2_inv; 0 -> 0), 5 mul_inl, 6 sqr_inl (the inlined forms) */
int bb_selftest_field(bb_ctx* ctx, int field, int op, const void* a, const void* b, void* out, size_t n);
/* element-wise on affine points: op 0: a + b (mixed add); 1: 2a + b; 2: a + (2b - b) */
int bb_selftest_point(bb_ctx* ctx, int group, int op, const void* a, const void* b, void* out, size_t n);
/* out = sum_{i<D} (i+1) * P_i through the bucket-reduction kernels, K buckets per thread (G1) */
int bb_selftest_bucket_reduce(bb_ctx* ctx, const void* affine_pts, uint32_t D, uint32_t K, void* out_affine);

/* out = sum_i a[i] * b[i] mod r over two device arrays of canonical Fr (result canonical, host).
 * With bases [k_i]G from bb_synth_bases(seed) -- k = bb_synth_scalars_device(seed) -- and scalars e_i, [sum k_i e_i]G is what an MSM must return
 * (the naive == fast property of src/multiexp.rs:334-378 at any size). */
int bb_diag_fr_dot(bb_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* out_fr);

/* ---- pairing (verify.cu) ---------------------------------------------------------------------- */
/* prod_i e(P_i, Q_i) after the final exponentiation, P_i / Q_i affine host arrays (identity allowed); gt_out: 12 canonical
 * Fp (6 x u64 each) in tower order c0.c0.c0, c0.c0.c1, c0.c1.c0, ..., c1.c2.c1 of Fp12 = Fp6[w]/(w^2 - v),
 * Fp6 = Fp2[v]/(v^3 - (u + 1)). */
int bb_diag_multi_pairing(bb_ctx* ctx, size_t n, const void* g1, const void* g2, void* gt_out);
/* k of the G_T convention: bb_diag_multi_pairing returns e(P, Q)^k for the pairing e = f_{|x|,Q}(P)^((p^12 - 1) / r) */
int bb_diag_gt_exponent(void);
/* element-wise on n Fp12 values (12 Montgomery Fp each, tower order): op 0 a*b, 1 a^2, 2 1/a, 3 cyclotomic squaring of a,
 * 4 a^p, 5 a^(p^2), 6 the final exponentiation a^(3 (p^12 - 1) / r), 7 a times the sparse line (b.c0.c0 + b.c0.c1 v) + (b.c1.c1 v) w;
 * ops 2 and 6 map zero to zero */
int bb_diag_fp12(bb_ctx* ctx, int op, const void* a, const void* b, void* out, size_t n);
/* bb_groth16_verify_batch, also writing the G_T value its verdict was taken from (format of bb_diag_multi_pairing) */
int bb_diag_verify_batch_gt(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, const void* z, void* gt_out);
/* bb_groth16_verify_each, writing n + 1 G_T values (format of bb_diag_multi_pairing): for each proof the final-exponentiated
 * ML(A_i, B_i) ML(Psi_i, -gamma) ML(C_i, -delta), then the key's e(alpha, beta)^3 they are compared with */
int bb_diag_verify_each_gt(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, void* gt_out);
/* a synthetic verifying key and n valid proofs from trapdoor scalars drawn from `seed`:
 * alpha, beta, gamma, delta, ic_j = [t_j] G1 (j <= n_inputs); proof i: A = [a_i] G1, B = [b_i] G2,
 * C = [(a_i b_i - alpha beta - gamma sum_j x_ij t_j) / delta] G1 (x_i0 = 1), all by fixed-base multiplication on the device.
 * Key parts to host buffers (ic: n_inputs + 1 points); d_a, d_b, d_c, d_inputs (Montgomery Fr, n x n_inputs): device. */
int bb_synth_proof_batch(bb_ctx* ctx, uint64_t seed, size_t n, size_t n_inputs, void* alpha_g1, void* beta_g2, void* gamma_g2,
                         void* delta_g2, void* ic, void* d_a, void* d_b, void* d_c, void* d_inputs);

/* ---- decoding (decode.cu) ------------------------------------------------------------------------------------- */
/* from_compressed (check_subgroup != 0) or from_compressed_unchecked (check_subgroup = 0) of n packed points of `group`
 * (48 or 96 B each, host memory) on the device.  out: n affine points in the ABI format (zeros unless why = 0); why: n
 * bytes, the codes of bb_proofs_read (5 = the identity, a valid encoding that Proof::read rejects). */
int bb_diag_points_decompress(bb_ctx* ctx, int group, const void* bytes, size_t n, int check_subgroup, void* out, uint8_t* why);

/* ---- resident keys (prover.cu, capi.cu) ------------------------------------------------------------------------ */
/* the points a bb_crs holds, ABI format, to host memory: which 0..4 = h, l, a, b_g1, b_g2 (the points this key holds of
 * that vector: all of them on a single GPU); which 5 = alpha_g1, beta_g1, delta_g1 (96 B each) then beta_g2, delta_g2
 * (192 B each) */
int bb_diag_crs_download(const bb_crs* crs, int which, void* out);
/* The owner stage of bb_groth16_prove_r1cs_begin for polynomial `poly` (0 = a, 1 = b, 2 = c) alone, with no MSM in flight:
 * the witness uploaded (on_device = 0) or read in place, matrix poly evaluated into d_out (m Fr, device, 16-byte aligned),
 * zeros to m, ifft + coset_fft there; on the main stream, blocking.  Profile mode records the stages r1cs_owner.upload,
 * r1cs_owner.eval (units: the matrix's terms) and r1cs_owner.transforms (units: m), as the split mode does. */
int bb_diag_r1cs_owner_stage(bb_ctx* ctx, const bb_r1cs* r1cs, const void* input, size_t n_inputs, const void* aux, size_t n_aux,
                             int on_device, int poly, void* d_out);
/* bytes of device memory the context has handed out and not yet taken back (its cache of free blocks excluded) */
uint64_t bb_diag_ctx_live_bytes(const bb_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* BELLMAN_B200_DIAG_H */
