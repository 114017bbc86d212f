/*
 * bellman_b200 -- C ABI of the H100-native Groth16 proving back-end for bellman.
 *
 * This is the drop-in boundary for the two hot paths behind groth16::create_proof
 * (SURVEY.md 8b).  bellman has no FFI seam of its own; each entry point below
 * cites the Rust item a thin shim would forward to it (paths relative to the
 * bellman source tree), and INTEGRATION.md shows that shim.
 *
 * Plain pointers and sizes only.  All functions return a bb_status; no exception
 * or abort crosses the boundary.  bb_last_error() gives a thread-local message.
 *
 * Data formats
 *   Fr element   32 bytes, 4 x u64 little-endian limbs.
 *                BB_FORM_MONTGOMERY: value * 2^256 mod r (bls12_381::Scalar's in-memory
 *                form, what EvaluationDomain's Vec<Scalar<Fr>> holds);
 *                BB_FORM_CANONICAL: the integer itself (PrimeField::to_repr /
 *                PrimeFieldBits::to_le_bits, what Exponent::Bits holds,
 *                src/multiexp.rs:166-182).
 *   G1 affine    96 bytes: x | y, each 6 x u64 LE limbs, Montgomery (value * 2^384 mod p).
 *   G2 affine    192 bytes: x.c0 | x.c1 | y.c0 | y.c1.
 *                The identity is encoded as all-zero bytes ((0,0) is on neither curve).
 *   density      bit i of word i/64 (LSB first) = "variable i appears in this query"
 *                (bitvec::BitVec<usize, Lsb0> raw storage of DensityTracker,
 *                src/multiexp.rs:118-157).  NULL = FullDensity (:97-116).
 */
#ifndef BELLMAN_B200_H
#define BELLMAN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum bb_status {
    BB_OK = 0,
    /* SynthesisError values that can originate on this path (src/lib.rs:304-319) */
    BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE = 1, /* domain.rs:57-59 */
    BB_ERR_UNEXPECTED_IDENTITY = 2,         /* multiexp.rs:63-65, prover.rs:320-324 */
    BB_ERR_IO_UNEXPECTED_EOF = 3,           /* multiexp.rs:55-61,74-80 */
    BB_ERR_UNCONSTRAINED_VARIABLE = 4,      /* generator.rs:464-470 */
    BB_ERR_DENSITY_MISMATCH = 5,            /* the assert! at multiexp.rs:324-329 (a panic upstream) */
    /* VerificationError (src/lib.rs:353-358) */
    BB_ERR_INVALID_VERIFYING_KEY = 6,       /* inputs.len() + 1 != ic.len(): verifier.rs:28-30, batch.rs:105-111 */
    BB_ERR_INVALID_PROOF = 7,               /* the pairing equation does not hold */
    BB_ERR_IO_INVALID_DATA = 8,             /* io::ErrorKind::InvalidData of Parameters::read / VerifyingKey::read */
    /* back-end errors */
    BB_ERR_ARG = 16,
    BB_ERR_CUDA = 17,
    BB_ERR_NO_DEVICE = 18,
    BB_ERR_OOM = 19
} bb_status;

typedef enum bb_form { BB_FORM_CANONICAL = 0, BB_FORM_MONTGOMERY = 1 } bb_form;

/* EvaluationDomain methods, src/domain.rs:81-125 */
typedef enum bb_ntt_mode { BB_NTT_FFT = 0, BB_NTT_IFFT = 1, BB_NTT_COSET_FFT = 2, BB_NTT_ICOSET_FFT = 3 } bb_ntt_mode;

typedef enum bb_group { BB_G1 = 1, BB_G2 = 2 } bb_group;

typedef struct bb_ctx bb_ctx;         /* one CUDA device; stands where multicore::Worker stands (src/multicore.rs:21-92) */
typedef struct bb_bases bb_bases;     /* device-resident Arc<Vec<G::Affine>> (groth16/src/lib.rs:227-243) */
typedef struct bb_msm_job bb_msm_job; /* Waiter<Result<G, SynthesisError>> (src/multicore.rs:94-118) */
typedef struct bb_crs bb_crs;         /* device-resident groth16::Parameters (groth16/src/lib.rs:222-244) */
typedef struct bb_prove bb_prove;     /* one create_proof in flight between bb_groth16_prove_begin and _end */
typedef struct bb_vk bb_vk;           /* device-resident PreparedVerifyingKey (groth16/src/lib.rs:400-409), see bb_vk_prepare */

const char* bb_last_error(void);
int bb_version(void);

/* ---- context ------------------------------------------------------------------------ */
/* Worker::new() (src/multicore.rs:24-27).  `device` is a CUDA ordinal.  Fails with
 * BB_ERR_NO_DEVICE when no CUDA device is usable: there is no CPU fallback. */
int bb_ctx_create(int device, bb_ctx** out);
void bb_ctx_destroy(bb_ctx* ctx);
/* tuning knobs; results never depend on them.  Keys:
 *   msm_window_bits    window size c of the signed-digit Pippenger (0 = by size)
 *   msm_affine_rounds  batched-affine halving rounds before the XYZZ stage (-1 = by mean bucket fill, 0 = none)
 *   msm_affine_batch   pairs per thread in those rounds (default 16)
 *   msm_reduce_k, msm_reduce_k1   entries per thread of the serial recursion (powers of two, default 4)
 *   msm_big_cap        bucket size above which a bucket is cut into tasks (0 = by mean fill)
 *   msm_precompute     keep window multiples of every base vector resident (see bb_bases_precompute): 1 = one bucket
 *                      array per window, added slot-wise; 2 = ONE bucket array for all windows and halving rounds by its fill
 *   msm_unified_rows_log   msm_precompute = 2: the rounds stop at about 2^this rows per bucket (default 3)
 *   msm_precompute_groups  which vectors use the tables: mask of 1 (G1) and 2 (G2), default 3
 *   shard_windows      multi-GPU: window groups per base range (default 4; 1 = base ranges only)
 *   prove_batch_max    bb_groth16_prove_batch: at most this many proofs per sub-batch (0 = as many as memory allows)
 *   params_read_chunk  bb_params_read / bb_vk_read from host memory: staging bytes per chunk (default 64 MiB; rounded
 *                      down to whole points, at least one point)
 *   ntt_tile_log, ntt_col_bits   shape of the NTT tiles
 *   profile            1 = CUDA-event timing of the MSM stages, and of the verify.*, decode.*, r1cs.*, params.* and
 *                      generate.* stages (bb_profile_read)
 *   msm_acc_variant, msm_affine_tma, msm_reduce_2d, ntt_radix8   retired: accepted for compatibility, no effect */
int bb_ctx_set_option(bb_ctx* ctx, const char* key, long value);
int bb_ctx_synchronize(bb_ctx* ctx);
/* counters for the harness: number of kernels this context has launched */
uint64_t bb_ctx_kernel_launches(const bb_ctx* ctx);

/* device buffers, so a caller can keep inputs resident across calls (bench "value" leg) */
int bb_device_alloc(bb_ctx* ctx, size_t bytes, void** d_out);
int bb_device_free(bb_ctx* ctx, void* d_ptr);
int bb_device_upload(bb_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
int bb_device_download(bb_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);

/* ---- NTT: EvaluationDomain::{fft, ifft, coset_fft, icoset_fft} (src/domain.rs:81-125),
 *      i.e. best_fft (:261-269) plus the fused scale / distribute_powers passes --------- */
/* In place on a host buffer of 2^log_n Fr elements.  log_n >= 32 (= Fr::S) returns
 * BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE like from_coeffs (:55-59). */
int bb_ntt(bb_ctx* ctx, void* fr_inout, uint32_t log_n, int mode, int form);
/* same, on a device buffer (Montgomery form) */
int bb_ntt_device(bb_ctx* ctx, void* d_fr_inout, uint32_t log_n, int mode);

/* EvaluationDomain's O(n) methods as stand-alone calls on host buffers (Montgomery Fr); inside
 * bb_h_poly / bb_groth16_prove they are fused into the transforms instead.
 *   op 0  mul_assign   a[i] *= b[i]          (src/domain.rs:154-170)
 *   op 1  sub_assign   a[i] -= b[i]          (:173-189)
 *   op 2  scale        a[i] *= k             (divide_by_z_on_coset with k = 1/z(g), :139-151)
 *   op 3  distribute_powers  a[i] *= k^i     (:101-113) */
int bb_domain_pointwise(bb_ctx* ctx, int op, void* fr_a_inout, const void* fr_b, size_t n, const void* fr_k);

/* The H-polynomial block of create_proof (groth16/src/prover.rs:221-240): from_coeffs on
 * a,b,c (pads to m = 2^k >= n), 3x ifft, 3x coset_fft, mul_assign, sub_assign,
 * divide_by_z_on_coset, icoset_fft, truncate to m-1 coefficients.
 * a,b,c: n_constraints Fr each (Montgomery, host).  h_out: room for m-1 Fr, canonical
 * integers (the Exponent::Bits form multiexp consumes, prover.rs:242).  *m_out = m. */
int bb_h_poly(bb_ctx* ctx, const void* a, const void* b, const void* c, size_t n_constraints,
              void* h_out, size_t* m_out);

/* ---- bases ---------------------------------------------------------------------------- */
/* Uploads n affine points.  `global_offset`/`global_len` describe a shard of a larger base
 * vector for multi-GPU runs (the shard holds indices [global_offset, global_offset+n) of a
 * vector of global_len points); single-GPU callers pass 0 and n. */
int bb_bases_upload(bb_ctx* ctx, int group, const void* affine, size_t n, size_t global_offset,
                    size_t global_len, bb_bases** out);
void bb_bases_free(bb_bases* b);
/* Builds the table of window multiples 2^(c w) P_i of a resident base vector (c chosen from its
 * length).  MSMs over these bases then accumulate every window into one bucket set: one summation
 * by parts and no Horner fold instead of one per window (multiexp.rs:271-300), at (windows x) the
 * base storage.  Results are unchanged.  With bb_ctx_set_option(ctx, "msm_precompute", 1 or 2) the table
 * is built on first use instead; 2 also sorts the digits of all windows into ONE bucket array (deeper halving
 * rounds, a sixteenth of the bucket reduction) -- the form bb_groth16_autotune measures against the default. */
int bb_bases_precompute(bb_ctx* ctx, bb_bases* bases);
/* Frees that table again.  No MSM over these bases may be in flight. */
int bb_bases_drop_table(bb_bases* bases);

/* ---- MSM: multiexp() (src/multiexp.rs:305-332) ---------------------------------------- */
/* Sum over i with density bit set of scalars[i] * bases[base_offset + rank(i)], where rank(i)
 * counts set density bits below i (bases are compacted to set bits, App. C.3).
 * Semantics preserved from multiexp_inner (:242-265): a zero scalar skips its base even if
 * that base is the identity; an identity base under a non-zero scalar is
 * BB_ERR_UNEXPECTED_IDENTITY; running out of bases is BB_ERR_IO_UNEXPECTED_EOF; a density of
 * the wrong length is BB_ERR_DENSITY_MISMATCH.  Returns immediately; the job runs on its own
 * CUDA stream (prover.rs:244-318 starts 8 of these before the first wait()).
 * Host buffers must stay valid until bb_msm_wait returns. */
int bb_msm_async(bb_ctx* ctx, const bb_bases* bases, size_t base_offset,
                 const uint64_t* density_bits, size_t density_len,
                 const void* scalars, size_t n_scalars, int form, bb_msm_job** out);
/* scalars already in HBM (canonical or Montgomery per `form`) */
int bb_msm_async_device(bb_ctx* ctx, const bb_bases* bases, size_t base_offset,
                        const uint64_t* density_bits, size_t density_len,
                        const void* d_scalars, size_t n_scalars, int form, bb_msm_job** out);
/* Waiter::wait() (src/multicore.rs:98-108).  Writes the result as an affine point in the
 * format above (G1 96 B / G2 192 B), frees the job.  With a sharded `bases` the result is
 * this shard's partial sum. */
int bb_msm_wait(bb_msm_job* job, void* out_affine);

/* small group helpers for the host side of a multi-GPU reduction (affine in/out) */
int bb_point_add(int group, const void* a_affine, const void* b_affine, void* out_affine);
int bb_point_mul(int group, const void* a_affine, const void* fr_scalar, int form, void* out_affine);
/* GroupEncoding::to_bytes: G1 48 B / G2 96 B compressed ZCash encoding */
int bb_point_compress(int group, const void* affine, uint8_t* out);
/* in-place canonical <-> Montgomery conversion of n Fp coordinates (host; parameter files) */
int bb_fp_convert(void* fp_inout, size_t n, int to_montgomery);
/* The checks G1Affine/G2Affine::from_uncompressed applies after decoding -- what Parameters::read does
 * with checked = true and VerifyingKey::read always (groth16/src/lib.rs:158-183,289-330): every point on
 * the curve and, with check_subgroup != 0, of order r.  n affine points in the ABI format, host memory;
 * computed on the device.  *first_bad = index of the first offending point (SIZE_MAX if none), *why = 1
 * off the curve, 2 outside the subgroup.  The identity passes (callers decide where it is allowed). */
int bb_points_validate(bb_ctx* ctx, int group, const void* affine, size_t n, int check_subgroup, size_t* first_bad, int* why);
/* out[i] = [k_i] * generator, computed on the device (fixed-base); used to manufacture
 * synthetic CRS material of benchmark size (generator.rs:271-296,398-415 equivalent). */
int bb_fixed_base_mul(bb_ctx* ctx, int group, const void* fr_scalars, size_t n, int form, void* out_affine);

/* ---- whole prover: create_proof after synthesis (groth16/src/prover.rs:217-360) -------- */
typedef struct bb_crs_desc {
    /* VerifyingKey parts the prover reads (prover.rs:219,320-337) */
    const void* alpha_g1; const void* beta_g1; const void* delta_g1;   /* 96 B each  */
    const void* beta_g2;  const void* delta_g2;                        /* 192 B each */
    /* Parameters vectors (groth16/src/lib.rs:227-243) */
    const void* h;    size_t h_len;
    const void* l;    size_t l_len;
    const void* a;    size_t a_len;
    const void* b_g1; size_t b_g1_len;
    const void* b_g2; size_t b_g2_len;
    /* multi-GPU: this process is shard `shard_index` of `shard_count`.  A shard is a contiguous
     * base range of every vector above, crossed with a subset of the MSM windows (any partition
     * of the (base, window) pairs folds to the same point): the library splits the windows into
     * up to 4 groups first and the base vectors second -- 8 shards = 2 base ranges x 4 window
     * groups; bb_ctx_set_option(ctx, "shard_windows", 1) gives base ranges alone.  The arrays
     * passed are the full vectors; only this shard's base range is uploaded.  Single GPU: 0 / 1. */
    uint32_t shard_index; uint32_t shard_count;
} bb_crs_desc;

int bb_crs_create(bb_ctx* ctx, const bb_crs_desc* desc, bb_crs** out);
void bb_crs_destroy(bb_crs* crs);
/* bb_bases_precompute / bb_bases_drop_table over the five vectors of a resident key */
int bb_crs_precompute(bb_ctx* ctx, bb_crs* crs);
int bb_crs_drop_tables(bb_crs* crs);

/* What ProvingAssignment holds when synthesis is done (prover.rs:57-71,193-215), i.e.
 * including the trailing "input * 0 = 0" constraints. */
typedef struct bb_witness {
    const void* a; const void* b; const void* c; size_t n_constraints;   /* Fr, Montgomery */
    const void* input_assignment; size_t n_inputs;                        /* Fr, Montgomery */
    const void* aux_assignment;   size_t n_aux;                           /* Fr, Montgomery */
    const uint64_t* a_aux_density;   /* n_aux bits   */
    const uint64_t* b_input_density; /* n_inputs bits */
    const uint64_t* b_aux_density;   /* n_aux bits   */
    /* non-zero: a, b, c, input_assignment and aux_assignment are DEVICE pointers (inputs already
     * resident in HBM; a, b, c are left untouched).  The density maps are always host memory. */
    int on_device;
} bb_witness;

/* Eight partial MSM results of one proof, in the order prover.rs starts them:
 * h, l, a_inputs, a_aux, b_g1_inputs, b_g1_aux (G1, 96 B each) then b_g2_inputs, b_g2_aux
 * (G2, 192 B each): 6*96 + 2*192 = 960 bytes. */
#define BB_PARTIALS_BYTES 960
/* NTT pipeline + the 8 MSMs over this context's CRS shard. */
int bb_groth16_prove_partials(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, uint8_t partials[BB_PARTIALS_BYTES]);
/* The same in two steps, for multi-GPU provers that split the H pipeline by polynomial.  _begin uploads the
 * assignments and queues the seven witness MSMs (prover.rs:263-318) -- they need nothing from the H pipeline
 * -- and returns at once.  Each of a, b, c is taken through from_coeffs / ifft / coset_fft
 * (prover.rs:225-230) by ONE rank with bb_h_coset_evals and the three result vectors (m Fr each, device
 * memory) are broadcast (NCCL).  _end(state, evals_a, evals_b, evals_c, partials) then runs mul_assign /
 * sub_assign / divide_by_z_on_coset / icoset_fft (:232-237) and the h MSM (:238-244), waits for all eight MSMs
 * and frees the state; with three NULL pointers it runs the whole H pipeline from w->a, w->b, w->c itself.
 * evals_a is clobbered.  The witness arrays must stay valid until _end returns. */
int bb_groth16_prove_begin(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, bb_prove** out);
int bb_groth16_prove_end(bb_prove* state, const void* d_evals_a, const void* d_evals_b, const void* d_evals_c,
                         uint8_t partials[BB_PARTIALS_BYTES]);
/* d_out[0..m) = coset_fft(ifft(from_coeffs(poly))) for one polynomial of n_constraints Fr (Montgomery; host
 * memory, or device memory with on_device != 0); m = next power of two >= n_constraints.  Blocking. */
int bb_h_coset_evals(bb_ctx* ctx, const void* poly, size_t n_constraints, int on_device, void* d_out);
/* The same without blocking: _async queues the copy and the two transforms on the context's high-priority stream
 * and returns at once (poly and d_out must stay valid); _wait blocks until every evaluation queued so far is
 * complete.  Lets a rank launch its transforms FIRST and queue the witness MSMs (bb_groth16_prove_begin, ~1 ms of
 * host time) while they run. */
int bb_h_coset_evals_async(bb_ctx* ctx, const void* poly, size_t n_constraints, int on_device, void* d_out);
int bb_h_coset_evals_wait(bb_ctx* ctx);
/* Sums `count` partial sets (one per shard) and applies prover.rs:320-360 + Proof::write
 * (groth16/src/lib.rs:39-45).  r, s: 32-byte canonical little-endian scalars. */
int bb_groth16_finalize(const bb_crs* crs, const uint8_t* partials, size_t count,
                        const uint8_t r[32], const uint8_t s[32], uint8_t proof[192]);
/* The same in two steps, so that the five scalar multiplications that need no MSM result
 * (delta*r, delta*s, delta*rs, alpha*s, beta*r -- prover.rs:326-337) can run on a host thread while
 * the devices compute the partial sums: finalize_static fills BB_PROOF_STATIC_BYTES opaque bytes,
 * finalize_with consumes them.  bb_groth16_finalize == finalize_static + finalize_with;
 * bb_groth16_prove overlaps them internally.
 * Side channels: the host-side scalar multiplications by r, s and r s run a REGULAR ladder -- signed odd digits
 * (none zero, none skipped), the table read in full under a mask, even scalars as (k + 1) P - P -- so neither the
 * sequence of operations nor any address depends on the scalar.  Not covered: the field products end with a
 * data-dependent final subtraction (the reference uses bls12_381's constant-time arithmetic throughout). */
#define BB_PROOF_STATIC_BYTES 768
int bb_groth16_finalize_static(const bb_crs* crs, const uint8_t r[32], const uint8_t s[32], uint8_t* static_out);
int bb_groth16_finalize_with(const bb_crs* crs, const uint8_t* partials, size_t count, const uint8_t r[32],
                             const uint8_t s[32], const uint8_t* static_in, uint8_t* proof);
/* single-GPU create_proof after synthesis (groth16/src/prover.rs:217-360): partials + finalize.
 * When several errors apply the one the reference would return is reported: the density assert
 * of multiexp() first (call order), then delta = identity (prover.rs:320-324, checked before any
 * wait), then the MSM errors in the order of the reference's waits: a_inputs, a_aux,
 * b_g1_inputs, b_g1_aux, b_g2_inputs, b_g2_aux, h, l (:339-354). */
int bb_groth16_prove(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w,
                     const uint8_t r[32], const uint8_t s[32], uint8_t proof[192]);
/* create_proof (groth16/src/prover.rs:217-360) for `count` witnesses of ONE circuit against one key: w[i], r + 32 i and
 * s + 32 i are what bb_groth16_prove takes, proof i goes to proofs + 192 i.  status[i] (written for every item whenever the call returns BB_OK) is exactly what
 * bb_groth16_prove returns for item i alone -- the same codes in the same precedence -- and the proof bytes are its bytes;
 * a failed item's 192 bytes are zero.  Returns BB_OK whenever the call ran, even if items failed (as bb_proofs_read).
 * Every item must have item 0's n_constraints, n_inputs, n_aux and on_device and density words equal to item 0's (the
 * circuit's structure decides them; the arrays may be distinct); otherwise BB_ERR_ARG naming the first differing item.
 * BB_ERR_ARG also for NULL pointers with count > 0 and for a sharded key (shard_count > 1), before any device work.
 * count = 0 is BB_OK and writes nothing.
 * The call splits the batch into sub-batches by device memory and by the 2^32 bucket entries of one MSM job, at most
 * bb_ctx_set_option(ctx, "prove_batch_max", k) proofs each (0 = no cap); the results never depend on the split.  A
 * sub-batch whose buffers cannot be allocated gives its items BB_ERR_OOM; items of other sub-batches keep their proofs.
 * A sub-batch runs one H pipeline per item and eight MSM jobs over all its items; r and s stay on the host (the ladder
 * documented at bb_groth16_finalize_static), the scalar multiplications of the items run on a pool of host threads. */
int bb_groth16_prove_batch(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, size_t count,
                           const uint8_t* r, const uint8_t* s, uint8_t* proofs, int* status);
/* The message bb_last_error() holds after bb_groth16_prove returned `status` with this key: the text of a batch item's
 * status.  NULL for back-end statuses (BB_ERR_ARG, _CUDA, _OOM), whose text depends on the failure. */
const char* bb_groth16_prove_message(const bb_crs* crs, int status);

/* ---- the constraint system on the device: ProvingAssignment::enforce (groth16/src/prover.rs:19-55,105-145) ---------
 * The A, B, C matrices of a circuit -- what KeypairAssembly records for generate_parameters (generator.rs:43-155) -- kept
 * in HBM beside the key, so that a proof needs only the witness: a = A z, b = B z, c = C z with
 * z = input_assignment || aux_assignment are computed on the device and the enforce closures are never called. */
typedef struct bb_r1cs bb_r1cs;
/* one matrix in CSR by constraint: row k holds the terms row_offsets[k] .. row_offsets[k+1] - 1 of vars / coeffs.
 * vars: input i = i, aux j = n_inputs + j.  coeffs: Fr, Montgomery.  Terms are taken as given, unmerged
 * (LinearCombination + (coeff, var) pushes, src/lib.rs:204-208). */
typedef struct bb_r1cs_matrix {
    const uint64_t* row_offsets;   /* n_constraints + 1 entries, row_offsets[0] = 0, non-decreasing */
    const uint32_t* vars;
    const void* coeffs;
} bb_r1cs_matrix;
typedef struct bb_r1cs_desc {
    bb_r1cs_matrix a, b, c;
    size_t n_constraints;          /* the rows the circuit enforced after alloc_input(ONE) (prover.rs:204-206) */
    size_t n_inputs;               /* including ONE, input 0 */
    size_t n_aux;
} bb_r1cs_desc;
/* Validates the matrices, appends one row per input (A = input_i with coefficient 1, B = C = 0; prover.rs:208-215,
 * generator.rs:193-202), computes the three densities as eval does (prover.rs:31-44: a term counts only with a non-zero
 * coefficient; a_aux_density from A, b_input_density and b_aux_density from B; inputs in A and all of C do not count) and
 * uploads the matrices.  Where bellman would panic on an index, BB_ERR_ARG with a message: n_inputs = 0, row offsets
 * not starting at 0 or decreasing, a variable >= n_inputs + n_aux, a coefficient >= r, more than 2^32 - 1 terms. */
int bb_r1cs_create(bb_ctx* ctx, const bb_r1cs_desc* desc, bb_r1cs** out);
void bb_r1cs_destroy(bb_r1cs* r1cs);
/* shape[BB_R1CS_SHAPE_WORDS] = n_constraints (incl. the input rows, = bb_witness.n_constraints), n_inputs, n_aux, then
 * per matrix A, B, C the terms the evaluation reads (non-zero coefficients, incl. the input rows), then per matrix how
 * many of those have coefficient one.  The densities (any may be NULL) in bb_witness's LSB-first word format. */
#define BB_R1CS_SHAPE_WORDS 9
int bb_r1cs_info(const bb_r1cs* r1cs, uint64_t* shape, uint64_t* a_aux_density, uint64_t* b_input_density, uint64_t* b_aux_density);
/* a, b, c (n_constraints Fr each, Montgomery) = the three products for the witness input (n_inputs Fr) and aux (n_aux
 * Fr): what ProvingAssignment holds after synthesis.  in_on_device / out_on_device: the witness / the results are device
 * pointers (16-byte aligned).  Blocking.  BB_ERR_ARG when n_inputs or n_aux differ from the constraint system's. */
int bb_r1cs_eval(bb_ctx* ctx, const bb_r1cs* r1cs, const void* input, size_t n_inputs, const void* aux, size_t n_aux,
                 int in_on_device, void* a, void* b, void* c, int out_on_device);
/* create_proof from the witness alone: the same 192 bytes as bb_groth16_prove for the bb_witness that ProvingAssignment
 * would have built.  The evaluation runs on the device ahead of the H pipeline; the witness MSMs do not wait for it.  Only
 * input and aux cross the bus (on_device = 0) or none (on_device != 0).  Argument errors as bb_r1cs_eval, before any
 * device work; then exactly bb_groth16_prove's errors and their precedence. */
int bb_groth16_prove_r1cs(bb_ctx* ctx, const bb_crs* crs, const bb_r1cs* r1cs, const void* input, size_t n_inputs,
                          const void* aux, size_t n_aux, int on_device, const uint8_t r[32], const uint8_t s[32], uint8_t proof[192]);
/* bb_groth16_prove_batch from witnesses alone: inputs = count x n_inputs Fr and aux = count x n_aux Fr, row-major (host, or
 * device memory with on_device != 0).  status[i] and proof i are bb_groth16_prove_r1cs's for item i alone.  Argument errors
 * as bb_r1cs_eval's and bb_groth16_prove_batch's, before any device work. */
int bb_groth16_prove_r1cs_batch(bb_ctx* ctx, const bb_crs* crs, const bb_r1cs* r1cs, const void* inputs, size_t n_inputs,
                                const void* aux, size_t n_aux, size_t count, int on_device, const uint8_t* r, const uint8_t* s,
                                uint8_t* proofs, int* status);

/* ---- generating keys: generate_parameters / generate_random_parameters (groth16/src/generator.rs:21-40,159-507) ----------
 * The key of a resident constraint system, computed on the device, element for element the reference's: the rows are the
 * bb_r1cs rows including its input rows (generator.rs:193-202), m = the next power of two >= rows; h[i] = [tau^i t(tau) /
 * delta] g1 for i < m - 1 with t(tau) = tau^m - 1; L = ifft of the m powers of tau; per variable j at_j, bt_j, ct_j = the sums
 * of coeff * L_row over its terms in A, B, C; ic (inputs, inv = 1/gamma) and l (aux, inv = 1/delta) = [(beta at + alpha bt +
 * ct) inv] g1; a, b_g1, b_g2 = [at] g1, [bt] g1, [bt] g2 with the zero scalars dropped in variable order (the evaluated
 * scalar decides, not the prover's density: cancelling terms give a dropped element); the verifying key [alpha] g1,
 * [beta] g1, [delta] g1, [beta] g2, [gamma] g2, [delta] g2.
 * Errors, in this order, all before any device work but the last:
 *   BB_ERR_ARG                     NULL ctx, r1cs or crs_out; an r1cs of another context; a scalar >= r; g1 or g2 the
 *                                  identity, off the curve or outside the subgroup (the reference's types cannot hold such
 *                                  a point; with non-identity generators "scalar zero" and "point is the identity" agree)
 *   BB_ERR_UNEXPECTED_IDENTITY     gamma = 0, then delta = 0 (generator.rs:228-243)
 *   BB_ERR_UNCONSTRAINED_VARIABLE  an l scalar is zero (found after the evaluation); report->unconstrained and
 *                                  bb_last_error() name the first such aux index
 * alpha = 0, beta = 0, tau = 0 and tau a root of unity of the domain (every h element the identity) are accepted.  On
 * failure *crs_out and *vk_out are NULL and every block is back in the context's cache.  The key is a single-GPU key
 * (shard 0 of 1).  toxic == NULL: generate_random_parameters -- alpha, beta, gamma, delta, tau and the two generators (as
 * random multiples of the standard ones) drawn with getrandom, zeros redrawn; none of them leaves the call.
 * Toxic waste: every device block that held a scalar derived from it (powers of tau, Lagrange coefficients, QAP values,
 * compacted scalars) is zeroed before it returns to the context's cache, and the host copies are wiped.  The fixed-base
 * multiplications run in variable time, as the reference's wNAF does. */
typedef struct bb_toxic {
    const void* g1; const void* g2;    /* 96 / 192 B affine in the format above; NULL = the standard generator */
    uint8_t alpha[32], beta[32], gamma[32], delta[32], tau[32];   /* canonical little-endian, < r */
} bb_toxic;
typedef struct bb_generate_report {
    size_t len[6];          /* ic, h, l, a, b_g1, b_g2 */
    size_t m;               /* the domain size */
    size_t unconstrained;   /* BB_ERR_UNCONSTRAINED_VARIABLE: the first aux index whose l scalar is zero (SIZE_MAX if none) */
} bb_generate_report;
/* vk_out (the PreparedVerifyingKey) and report may be NULL */
int bb_groth16_generate(bb_ctx* ctx, const bb_r1cs* r1cs, const bb_toxic* toxic, bb_crs** crs_out, bb_vk** vk_out,
                        bb_generate_report* report);

/* ---- verification: groth16/src/verifier.rs and groth16/src/verifier/batch.rs ------------------
 * Points are taken as valid curve and subgroup elements, as the reference's Proof / VerifyingKey types guarantee
 * through read(); bb_points_validate applies those checks.  The identity is allowed anywhere: a pair with an identity
 * on either side contributes one to the Miller product, as in bls12_381's multi_miller_loop. */
/* PreparedVerifyingKey (groth16/src/lib.rs:400-409, verifier.rs:11-21): the verifying key resident on the device */
typedef struct bb_vk_desc {
    const void* alpha_g1;                                             /* 96 B */
    const void* beta_g2; const void* gamma_g2; const void* delta_g2;  /* 192 B each */
    const void* ic; size_t ic_len;                                    /* 96 B each */
} bb_vk_desc;
int bb_vk_prepare(bb_ctx* ctx, const bb_vk_desc* desc, bb_vk** out);
void bb_vk_destroy(bb_vk* vk);

/* batch::Item x n (batch.rs:40-43): proofs as affine points in the format above (a, c: G1; b: G2), inputs n x n_inputs
 * Fr (Montgomery, row-major).  on_device != 0: a, b, c and inputs are device pointers. */
typedef struct bb_proof_batch {
    const void* a; const void* b; const void* c; size_t n;
    const void* inputs; size_t n_inputs;
    int on_device;
} bb_proof_batch;

/* verify_proof (verifier.rs:23-58): host buffers, one proof.  BB_OK = valid, BB_ERR_INVALID_PROOF = the equation fails,
 * BB_ERR_INVALID_VERIFYING_KEY = n_inputs + 1 != ic_len.  Computed as the batch of one with z = 1. */
int bb_groth16_verify(bb_ctx* ctx, const bb_vk* vk, const void* a, const void* b, const void* c,
                      const void* inputs, size_t n_inputs);
/* batch::Verifier::verify (batch.rs:100-173): one multi-Miller loop over the n + 3 pairs
 * (z_i A_i, -B_i), (sum z_i C_i, delta), (Psi, gamma), ([sum z_i] alpha, beta) and one final exponentiation.
 * z: n canonical 32-byte scalars in [1, r) (zero or >= r: BB_ERR_ARG), or NULL = drawn from the operating system
 * (getrandom, zeros redrawn).  The key check comes first, before any device work.  An empty batch is accepted. */
int bb_groth16_verify_batch(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, const void* z);
/* Item::verify_single (batch.rs:57-65), i.e. verify_proof (verifier.rs:23-58), for each of the n proofs of `batch`
 * (bb_proof_batch as for bb_groth16_verify_batch; host or device buffers): the fallback that finds the invalid proofs of
 * a rejected batch, in one call.  Deterministic (no z).  verdicts: n bytes, host, always written: 0 = valid, 1 = the
 * equation fails.  *n_invalid = number of non-zero verdicts.  BB_OK whenever the call ran, even if some proofs are invalid
 * (as bb_proofs_read).  BB_ERR_INVALID_VERIFYING_KEY: n > 0 and n_inputs + 1 != ic_len, before any device work.
 * BB_ERR_ARG: NULL pointers with n > 0, n >= 2^31.  An empty batch is BB_OK.  The first call for a key builds and keeps
 * with it the prepared lines of -gamma and -delta, e(alpha, beta) and a 784 KB table of byte multiples per non-identity
 * ic[j], j >= 1 (freed by bb_vk_destroy). */
int bb_groth16_verify_each(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, uint8_t* verdicts, size_t* n_invalid);

/* ---- reading and writing proofs: Proof::read / Proof::write (groth16/src/lib.rs:39-99) -------------------------
 * A proof is 192 bytes: compressed A (48 B), B (96 B), C (48 B), the ZCash encoding of bls12_381 0.8.  Decoding runs
 * on the device, one thread per point, in variable time (proof bytes are public).  For each proof A, then B, then C
 * is read; the first element that fails decides the status byte:
 *     status = 0 (valid) or (which << 4) | why,   which: 1 = A, 2 = B, 3 = C
 *     why  check, in this priority                                                 bellman's io::Error (InvalidData)
 *      1   compression bit (0x80 of byte 0) clear; or infinity bit (0x40) set       "invalid G1" / "invalid G2"
 *          with the sort bit (0x20) or any bit of x set
 *      2   x >= p (G2: x.c1 in bytes 0-47 below the flags, or x.c0 in bytes 48-95)  "invalid G1" / "invalid G2"
 *      3   x^3 + b has no square root (not on the curve)                            "invalid G1" / "invalid G2"
 *      4   the point is not in the order-r subgroup                                 "invalid G1" / "invalid G2"
 *      5   a valid encoding of the identity (0xC0, then zeros)                      "point at infinity"
 * y is the square root whose "lexicographically largest" flag (G1: y > (p-1)/2; G2: y.c1 decides, y.c0 if y.c1 = 0)
 * equals the sort bit.  All three points of an invalid proof are written as the identity (zeros). */
#define BB_PROOF_BYTES 192
#define BB_PROOF_WHICH(status) ((status) >> 4)
#define BB_PROOF_WHY(status) ((status) & 15)
enum { BB_READ_OK = 0, BB_READ_BAD_FLAGS = 1, BB_READ_NON_CANONICAL = 2, BB_READ_NOT_ON_CURVE = 3, BB_READ_NOT_IN_SUBGROUP = 4,
       BB_READ_IDENTITY = 5 };
/* Proof::read (groth16/src/lib.rs:47-99) over n proofs; proof i at bytes + i*stride (stride 0 = 192); no alignment is
 * assumed.  on_device != 0: bytes is a device pointer; otherwise only the 192 proof bytes of each record are copied. */
typedef struct bb_proof_bytes { const void* bytes; size_t n; size_t stride; int on_device; } bb_proof_bytes;
/* a, c: n x 96 B, b: n x 192 B, device pointers if out_on_device else host; status: n bytes, host, always written;
 * *n_invalid = number of non-zero statuses.  BB_OK whenever the call ran, even if some proofs are invalid.
 * BB_ERR_ARG: a NULL pointer with n > 0, or 0 < stride < 192. */
int bb_proofs_read(bb_ctx* ctx, const bb_proof_bytes* in, void* a, void* b, void* c, int out_on_device,
                   uint8_t* status, size_t* n_invalid);
/* Proof::write (lib.rs:39-45) over n proofs: out = n x 192 B (a, b, c and out are device pointers if on_device).
 * Byte for byte what bb_point_compress gives for each point. */
int bb_proofs_write(bb_ctx* ctx, const void* a, const void* b, const void* c, size_t n, int on_device, void* out);

/* ---- reading keys: Parameters::read / VerifyingKey::read (groth16/src/lib.rs:158-218, 289-398) -----------------------
 * A key file is read once and decoded on the device, straight into a resident bb_crs (and bb_vk).  File order, all
 * integers big-endian u32: alpha_g1, beta_g1, beta_g2, gamma_g2, delta_g1, delta_g2, |ic|, ic, then (Parameters only)
 * |h|, h, |l|, l, |a|, a, |b_g1|, b_g1, |b_g2|, b_g2.  Points are uncompressed ZCash encodings (G1 96 B: x | y; G2
 * 192 B: x.c1 | x.c0 | y.c1 | y.c0).  Each point is checked in this order; the first failing check gives its why code
 * (the BB_READ_* values of bb_proofs_read):
 *     1  compression (0x80) or sort (0x20) bit set, or the infinity bit (0x40) with any other bit of the point set
 *     2  a coordinate >= p
 *     3  not on the curve                  } only in checked sections: the six VerifyingKey points and ic always,
 *     4  not in the order-r subgroup       } h, l, a, b_g1, b_g2 when checked != 0
 *     5  the identity where it is not allowed: in ic and the five vectors (both modes); the six VerifyingKey points may be
 *        the identity (the prover reports delta = identity itself)
 * The first failing point in file order decides, as the reference reads point by point: BB_ERR_IO_INVALID_DATA, with
 * bb_last_error() = "<section>[<index>]: invalid G1 (<reason>)" / "... invalid G2 ..." / "...: point at infinity".
 * Only when every complete point before the end of the buffer is valid does a short buffer (a truncated point, a
 * truncated prefix, a prefix claiming more points than the buffer holds) give BB_ERR_IO_UNEXPECTED_EOF.  Nothing is
 * allocated beyond what the buffer can hold.  Bytes after the key are not read.  On failure *crs_out and *vk_out are
 * NULL and everything the call allocated is back in the context's cache.
 * bytes: host memory (pageable or pinned; streamed through two pinned staging blocks, copies overlapping the decode) or,
 * with on_device != 0, device memory (decoded in place).  The result is what bb_crs_create / bb_vk_prepare build from the
 * same points.  Single GPU keys only (shard 0 of 1).  BB_ERR_ARG, before any device work: a NULL ctx or out pointer, a
 * NULL bytes with len > 0. */
enum { BB_PARAMS_ALPHA_G1 = 0, BB_PARAMS_BETA_G1, BB_PARAMS_BETA_G2, BB_PARAMS_GAMMA_G2, BB_PARAMS_DELTA_G1,
       BB_PARAMS_DELTA_G2, BB_PARAMS_IC, BB_PARAMS_H, BB_PARAMS_L, BB_PARAMS_A, BB_PARAMS_B_G1, BB_PARAMS_B_G2 };
typedef struct bb_params_report {
    size_t len[6];      /* ic, h, l, a, b_g1, b_g2 as their prefixes declared them (0 for prefixes not reached) */
    size_t consumed;    /* bytes read: the key's length on success; on EOF the offset of the incomplete element */
    int section;        /* first failing element (BB_PARAMS_*), -1 if none */
    size_t index;       /* its index within the section; on EOF the number of complete points of that section */
    int why;            /* BB_READ_* 1..5 for invalid data; 0 otherwise */
} bb_params_report;
/* Parameters::read(reader, checked): *crs_out = the proving key; vk_out (may be NULL) = its PreparedVerifyingKey too;
 * report may be NULL */
int bb_params_read(bb_ctx* ctx, const void* bytes, size_t len, int on_device, int checked,
                   bb_crs** crs_out, bb_vk** vk_out, bb_params_report* report);
/* VerifyingKey::read + prepare_verifying_key: the first 868 + 96 |ic| bytes of a VerifyingKey or Parameters file */
int bb_vk_read(bb_ctx* ctx, const void* bytes, size_t len, int on_device, bb_vk** vk_out, bb_params_report* report);
/* Parameters::write / VerifyingKey::write (groth16/src/lib.rs:258-287, 143-156) of a resident key: byte for byte the format
 * bb_params_read reads (canonical big-endian coordinates, G2 as x.c1 | x.c0 | y.c1 | y.c0, the identity as 0x40 then
 * zeros), encoded on the device.  vk holds gamma_g2 and ic, crs the rest (beta_g1 and delta_g1 live only there, so crs is
 * required with vk_only too).  vk_only: the VerifyingKey alone, the first 868 + 96 |ic| bytes.  out: host memory, or
 * device memory with out_on_device != 0; out == NULL only sets *len_out.  BB_ERR_ARG, before any device work: NULL ctx,
 * crs, vk or len_out; a key of another context; a sharded crs; a vk whose alpha_g1, beta_g2 and delta_g2 are not the
 * crs's ("not this key's verifying key"); cap < the length (with *len_out = the length needed). */
int bb_params_write(bb_ctx* ctx, const bb_crs* crs, const bb_vk* vk, int vk_only, void* out, size_t cap, int out_on_device,
                    size_t* len_out);

/* ---- tuning per key ------------------------------------------------------------------------
 * The MSM has several forms with identical results (per-window bucket sets; one bucket set over resident window
 * multiples with deeper halving rounds, which costs (windows x) the base storage).  Which is fastest depends on
 * the device, the key size and the shard count, and a key serves many proofs, so the choice is MEASURED once per
 * key: bb_groth16_autotune proves the given witness with every form (one checked proof, then `reps` timed ones,
 * fastest taken), admits a form only if its 960 bytes of partial sums equal the default form's, leaves the context
 * and the key configured for the fastest one and frees the tables if they lost.  ms_out (bb_tuning_count()
 * doubles, may be NULL): milliseconds per form; -1 = not available (no room for the tables), -2 = failed,
 * -3 = different partial sums.  *chosen = index of the fastest eligible form, which is now active.
 * Sharded keys: all shards MUST run the same form (the forms cut the scalars into windows of different sizes, so a
 * shard's (base, window) pairs -- and its partial sums -- depend on the form; only the sum over all shards does not).
 * For a key with shard_count > 1 this call therefore only measures (no comparison, *chosen = the fastest form here)
 * and leaves the DEFAULT form active; the shards agree on one index -- time the whole sharded proof, compare the
 * final proof bytes -- and each selects it with bb_crs_apply_tuning.  Form 0 is the default. */
int bb_tuning_count(void);
const char* bb_tuning_name(int index);
int bb_crs_apply_tuning(bb_ctx* ctx, bb_crs* crs, int index);
int bb_groth16_autotune(bb_ctx* ctx, bb_crs* crs, const bb_witness* w, int reps, int* chosen, double* ms_out);

/* ---- profiling: CUDA-event timing of the dominant kernels, on the stream they run on ------ */
/* bb_ctx_set_option(ctx, "profile", 1) makes every MSM job bracket its bucket-accumulation
 * kernel with cudaEvents.  bb_profile_read returns, for `what` = "msm_accumulate_g1" |
 * "msm_accumulate_g2" | "msm_total_g1" | "msm_total_g2" | "ntt_pass", the summed device
 * milliseconds, the number of launches (or jobs) and the number of units they processed
 * ((base, scalar) pairs; NTT points) since the last bb_profile_reset. */
int bb_profile_read(bb_ctx* ctx, const char* what, double* ms, uint64_t* launches, uint64_t* units);
int bb_profile_reset(bb_ctx* ctx);
/* bytes the MSM / prover entry points have copied host->device and device->host so far */
int bb_ctx_bytes_copied(const bb_ctx* ctx, uint64_t* h2d, uint64_t* d2h);

/* Bench generators (bb_synth_*) and parity-test diagnostics (bb_selftest_*, bb_diag_*) are not part
 * of the bellman-facing surface: they are declared in bellman_b200_diag.h. */

#ifdef __cplusplus
}
#endif
#endif /* BELLMAN_B200_H */
