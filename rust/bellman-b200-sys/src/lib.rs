//! Raw bindings to `include/bellman_b200.h` (the C ABI of the CUDA back-end).  One declaration per
//! function of the header, same order.  Formats: Fr = 32 bytes (4 x u64 LE limbs), G1 affine = 96 bytes
//! (x | y, Montgomery limbs), G2 affine = 192 bytes (x.c0 | x.c1 | y.c0 | y.c1), identity = all zero.
#![allow(non_camel_case_types)]

use std::os::raw::{c_char, c_int, c_long, c_uint, c_void};

#[repr(C)] pub struct bb_ctx { _private: [u8; 0] }
#[repr(C)] pub struct bb_bases { _private: [u8; 0] }
#[repr(C)] pub struct bb_msm_job { _private: [u8; 0] }
#[repr(C)] pub struct bb_crs { _private: [u8; 0] }
#[repr(C)] pub struct bb_prove { _private: [u8; 0] }
#[repr(C)] pub struct bb_vk { _private: [u8; 0] }
#[repr(C)] pub struct bb_r1cs { _private: [u8; 0] }

// bb_status
pub const BB_OK: c_int = 0;
pub const BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE: c_int = 1;
pub const BB_ERR_UNEXPECTED_IDENTITY: c_int = 2;
pub const BB_ERR_IO_UNEXPECTED_EOF: c_int = 3;
pub const BB_ERR_UNCONSTRAINED_VARIABLE: c_int = 4;
pub const BB_ERR_DENSITY_MISMATCH: c_int = 5;
pub const BB_ERR_INVALID_VERIFYING_KEY: c_int = 6;
pub const BB_ERR_INVALID_PROOF: c_int = 7;
pub const BB_ERR_IO_INVALID_DATA: c_int = 8;
pub const BB_ERR_ARG: c_int = 16;
pub const BB_ERR_CUDA: c_int = 17;
pub const BB_ERR_NO_DEVICE: c_int = 18;
pub const BB_ERR_OOM: c_int = 19;
// bb_form
pub const BB_FORM_CANONICAL: c_int = 0;
pub const BB_FORM_MONTGOMERY: c_int = 1;
// bb_ntt_mode
pub const BB_NTT_FFT: c_int = 0;
pub const BB_NTT_IFFT: c_int = 1;
pub const BB_NTT_COSET_FFT: c_int = 2;
pub const BB_NTT_ICOSET_FFT: c_int = 3;
// bb_group
pub const BB_G1: c_int = 1;
pub const BB_G2: c_int = 2;

pub const BB_PARTIALS_BYTES: usize = 960;
pub const BB_PROOF_STATIC_BYTES: usize = 768;

#[repr(C)]
pub struct bb_crs_desc {
    pub alpha_g1: *const c_void, pub beta_g1: *const c_void, pub delta_g1: *const c_void,
    pub beta_g2: *const c_void, pub delta_g2: *const c_void,
    pub h: *const c_void, pub h_len: usize,
    pub l: *const c_void, pub l_len: usize,
    pub a: *const c_void, pub a_len: usize,
    pub b_g1: *const c_void, pub b_g1_len: usize,
    pub b_g2: *const c_void, pub b_g2_len: usize,
    pub shard_index: u32, pub shard_count: u32,
}

#[repr(C)]
pub struct bb_witness {
    pub a: *const c_void, pub b: *const c_void, pub c: *const c_void, pub n_constraints: usize,
    pub input_assignment: *const c_void, pub n_inputs: usize,
    pub aux_assignment: *const c_void, pub n_aux: usize,
    pub a_aux_density: *const u64, pub b_input_density: *const u64, pub b_aux_density: *const u64,
    pub on_device: c_int,
}

#[repr(C)]
pub struct bb_vk_desc {
    pub alpha_g1: *const c_void,
    pub beta_g2: *const c_void, pub gamma_g2: *const c_void, pub delta_g2: *const c_void,
    pub ic: *const c_void, pub ic_len: usize,
}

#[repr(C)]
pub struct bb_proof_batch {
    pub a: *const c_void, pub b: *const c_void, pub c: *const c_void, pub n: usize,
    pub inputs: *const c_void, pub n_inputs: usize,
    pub on_device: c_int,
}

#[repr(C)]
pub struct bb_r1cs_matrix {
    pub row_offsets: *const u64, pub vars: *const u32, pub coeffs: *const c_void,
}

#[repr(C)]
pub struct bb_r1cs_desc {
    pub a: bb_r1cs_matrix, pub b: bb_r1cs_matrix, pub c: bb_r1cs_matrix,
    pub n_constraints: usize, pub n_inputs: usize, pub n_aux: usize,
}

pub const BB_R1CS_SHAPE_WORDS: usize = 9;

// Proof::read status byte: (which << 4) | why, which 1 = A, 2 = B, 3 = C
pub const BB_PROOF_BYTES: usize = 192;
pub const BB_READ_OK: u8 = 0;
pub const BB_READ_BAD_FLAGS: u8 = 1;
pub const BB_READ_NON_CANONICAL: u8 = 2;
pub const BB_READ_NOT_ON_CURVE: u8 = 3;
pub const BB_READ_NOT_IN_SUBGROUP: u8 = 4;
pub const BB_READ_IDENTITY: u8 = 5;

#[repr(C)]
pub struct bb_proof_bytes {
    pub bytes: *const c_void, pub n: usize, pub stride: usize, pub on_device: c_int,
}

// key files: the sections of Parameters::read in file order, and what bb_params_read / bb_vk_read report
pub const BB_PARAMS_ALPHA_G1: c_int = 0;
pub const BB_PARAMS_BETA_G1: c_int = 1;
pub const BB_PARAMS_BETA_G2: c_int = 2;
pub const BB_PARAMS_GAMMA_G2: c_int = 3;
pub const BB_PARAMS_DELTA_G1: c_int = 4;
pub const BB_PARAMS_DELTA_G2: c_int = 5;
pub const BB_PARAMS_IC: c_int = 6;
pub const BB_PARAMS_H: c_int = 7;
pub const BB_PARAMS_L: c_int = 8;
pub const BB_PARAMS_A: c_int = 9;
pub const BB_PARAMS_B_G1: c_int = 10;
pub const BB_PARAMS_B_G2: c_int = 11;

#[repr(C)]
#[derive(Default)]
pub struct bb_params_report {
    pub len: [usize; 6], pub consumed: usize, pub section: c_int, pub index: usize, pub why: c_int,
}

// generate_parameters on the device: the toxic waste (canonical little-endian scalars; NULL generators = the standard ones)
#[repr(C)]
pub struct bb_toxic {
    pub g1: *const c_void, pub g2: *const c_void,
    pub alpha: [u8; 32], pub beta: [u8; 32], pub gamma: [u8; 32], pub delta: [u8; 32], pub tau: [u8; 32],
}

#[repr(C)]
#[derive(Default)]
pub struct bb_generate_report {
    pub len: [usize; 6], pub m: usize, pub unconstrained: usize,
}

extern "C" {
    pub fn bb_last_error() -> *const c_char;
    pub fn bb_version() -> c_int;

    pub fn bb_ctx_create(device: c_int, out: *mut *mut bb_ctx) -> c_int;
    pub fn bb_ctx_destroy(ctx: *mut bb_ctx);
    pub fn bb_ctx_set_option(ctx: *mut bb_ctx, key: *const c_char, value: c_long) -> c_int;
    pub fn bb_ctx_synchronize(ctx: *mut bb_ctx) -> c_int;
    pub fn bb_ctx_kernel_launches(ctx: *const bb_ctx) -> u64;

    pub fn bb_device_alloc(ctx: *mut bb_ctx, bytes: usize, d_out: *mut *mut c_void) -> c_int;
    pub fn bb_device_free(ctx: *mut bb_ctx, d_ptr: *mut c_void) -> c_int;
    pub fn bb_device_upload(ctx: *mut bb_ctx, d_dst: *mut c_void, h_src: *const c_void, bytes: usize) -> c_int;
    pub fn bb_device_download(ctx: *mut bb_ctx, h_dst: *mut c_void, d_src: *const c_void, bytes: usize) -> c_int;

    pub fn bb_ntt(ctx: *mut bb_ctx, fr_inout: *mut c_void, log_n: u32, mode: c_int, form: c_int) -> c_int;
    pub fn bb_ntt_device(ctx: *mut bb_ctx, d_fr_inout: *mut c_void, log_n: u32, mode: c_int) -> c_int;
    pub fn bb_domain_pointwise(ctx: *mut bb_ctx, op: c_int, fr_a_inout: *mut c_void, fr_b: *const c_void, n: usize,
                               fr_k: *const c_void) -> c_int;
    pub fn bb_h_poly(ctx: *mut bb_ctx, a: *const c_void, b: *const c_void, c: *const c_void, n_constraints: usize,
                     h_out: *mut c_void, m_out: *mut usize) -> c_int;

    pub fn bb_bases_upload(ctx: *mut bb_ctx, group: c_int, affine: *const c_void, n: usize, global_offset: usize,
                           global_len: usize, out: *mut *mut bb_bases) -> c_int;
    pub fn bb_bases_free(b: *mut bb_bases);
    pub fn bb_bases_precompute(ctx: *mut bb_ctx, bases: *mut bb_bases) -> c_int;
    pub fn bb_bases_drop_table(bases: *mut bb_bases) -> c_int;

    pub fn bb_msm_async(ctx: *mut bb_ctx, bases: *const bb_bases, base_offset: usize, density_bits: *const u64,
                        density_len: usize, scalars: *const c_void, n_scalars: usize, form: c_int,
                        out: *mut *mut bb_msm_job) -> c_int;
    pub fn bb_msm_async_device(ctx: *mut bb_ctx, bases: *const bb_bases, base_offset: usize, density_bits: *const u64,
                               density_len: usize, d_scalars: *const c_void, n_scalars: usize, form: c_int,
                               out: *mut *mut bb_msm_job) -> c_int;
    pub fn bb_msm_wait(job: *mut bb_msm_job, out_affine: *mut c_void) -> c_int;

    pub fn bb_point_add(group: c_int, a_affine: *const c_void, b_affine: *const c_void, out_affine: *mut c_void) -> c_int;
    pub fn bb_point_mul(group: c_int, a_affine: *const c_void, fr_scalar: *const c_void, form: c_int,
                        out_affine: *mut c_void) -> c_int;
    pub fn bb_point_compress(group: c_int, affine: *const c_void, out: *mut u8) -> c_int;
    pub fn bb_fp_convert(fp_inout: *mut c_void, n: usize, to_montgomery: c_int) -> c_int;
    pub fn bb_points_validate(ctx: *mut bb_ctx, group: c_int, affine: *const c_void, n: usize, check_subgroup: c_int,
                              first_bad: *mut usize, why: *mut c_int) -> c_int;
    pub fn bb_fixed_base_mul(ctx: *mut bb_ctx, group: c_int, fr_scalars: *const c_void, n: usize, form: c_int,
                             out_affine: *mut c_void) -> c_int;

    pub fn bb_crs_create(ctx: *mut bb_ctx, desc: *const bb_crs_desc, out: *mut *mut bb_crs) -> c_int;
    pub fn bb_crs_destroy(crs: *mut bb_crs);
    pub fn bb_crs_precompute(ctx: *mut bb_ctx, crs: *mut bb_crs) -> c_int;
    pub fn bb_crs_drop_tables(crs: *mut bb_crs) -> c_int;

    pub fn bb_groth16_prove_partials(ctx: *mut bb_ctx, crs: *const bb_crs, w: *const bb_witness, partials: *mut u8) -> c_int;
    pub fn bb_groth16_prove_begin(ctx: *mut bb_ctx, crs: *const bb_crs, w: *const bb_witness, out: *mut *mut bb_prove) -> c_int;
    pub fn bb_groth16_prove_end(state: *mut bb_prove, d_evals_a: *const c_void, d_evals_b: *const c_void, d_evals_c: *const c_void,
                                partials: *mut u8) -> c_int;
    pub fn bb_h_coset_evals(ctx: *mut bb_ctx, poly: *const c_void, n_constraints: usize, on_device: c_int, d_out: *mut c_void) -> c_int;
    pub fn bb_h_coset_evals_async(ctx: *mut bb_ctx, poly: *const c_void, n_constraints: usize, on_device: c_int, d_out: *mut c_void) -> c_int;
    pub fn bb_h_coset_evals_wait(ctx: *mut bb_ctx) -> c_int;
    pub fn bb_groth16_finalize(crs: *const bb_crs, partials: *const u8, count: usize, r: *const u8, s: *const u8,
                               proof: *mut u8) -> c_int;
    pub fn bb_groth16_finalize_static(crs: *const bb_crs, r: *const u8, s: *const u8, static_out: *mut u8) -> c_int;
    pub fn bb_groth16_finalize_with(crs: *const bb_crs, partials: *const u8, count: usize, r: *const u8, s: *const u8,
                                    static_in: *const u8, proof: *mut u8) -> c_int;
    pub fn bb_groth16_prove(ctx: *mut bb_ctx, crs: *const bb_crs, w: *const bb_witness, r: *const u8, s: *const u8,
                            proof: *mut u8) -> c_int;
    pub fn bb_groth16_prove_message(crs: *const bb_crs, status: c_int) -> *const c_char;
    pub fn bb_groth16_prove_batch(ctx: *mut bb_ctx, crs: *const bb_crs, w: *const bb_witness, count: usize, r: *const u8,
                                  s: *const u8, proofs: *mut u8, status: *mut c_int) -> c_int;
    pub fn bb_r1cs_create(ctx: *mut bb_ctx, desc: *const bb_r1cs_desc, out: *mut *mut bb_r1cs) -> c_int;
    pub fn bb_r1cs_destroy(r1cs: *mut bb_r1cs);
    pub fn bb_r1cs_info(r1cs: *const bb_r1cs, shape: *mut u64, a_aux_density: *mut u64, b_input_density: *mut u64,
                        b_aux_density: *mut u64) -> c_int;
    pub fn bb_r1cs_eval(ctx: *mut bb_ctx, r1cs: *const bb_r1cs, input: *const c_void, n_inputs: usize, aux: *const c_void,
                        n_aux: usize, in_on_device: c_int, a: *mut c_void, b: *mut c_void, c: *mut c_void, out_on_device: c_int) -> c_int;
    pub fn bb_groth16_prove_r1cs(ctx: *mut bb_ctx, crs: *const bb_crs, r1cs: *const bb_r1cs, input: *const c_void, n_inputs: usize,
                                 aux: *const c_void, n_aux: usize, on_device: c_int, r: *const u8, s: *const u8, proof: *mut u8) -> c_int;
    pub fn bb_groth16_prove_r1cs_begin(ctx: *mut bb_ctx, crs: *const bb_crs, r1cs: *const bb_r1cs, input: *const c_void, n_inputs: usize,
                                       aux: *const c_void, n_aux: usize, on_device: c_int, own: c_uint, d_evals: *const *mut c_void,
                                       out: *mut *mut bb_prove) -> c_int;
    pub fn bb_groth16_prove_r1cs_batch(ctx: *mut bb_ctx, crs: *const bb_crs, r1cs: *const bb_r1cs, inputs: *const c_void,
                                       n_inputs: usize, aux: *const c_void, n_aux: usize, count: usize, on_device: c_int,
                                       r: *const u8, s: *const u8, proofs: *mut u8, status: *mut c_int) -> c_int;
    pub fn bb_r1cs_check(ctx: *mut bb_ctx, r1cs: *const bb_r1cs, input: *const c_void, n_inputs: usize, aux: *const c_void,
                         n_aux: usize, on_device: c_int, first: *mut usize, count: *mut usize, unsat_bits: *mut u64) -> c_int;
    pub fn bb_r1cs_check_batch(ctx: *mut bb_ctx, r1cs: *const bb_r1cs, inputs: *const c_void, n_inputs: usize, aux: *const c_void,
                               n_aux: usize, count: usize, on_device: c_int, first: *mut usize, n_unsat: *mut usize) -> c_int;

    pub fn bb_vk_prepare(ctx: *mut bb_ctx, desc: *const bb_vk_desc, out: *mut *mut bb_vk) -> c_int;
    pub fn bb_vk_destroy(vk: *mut bb_vk);
    pub fn bb_groth16_verify(ctx: *mut bb_ctx, vk: *const bb_vk, a: *const c_void, b: *const c_void, c: *const c_void,
                             inputs: *const c_void, n_inputs: usize) -> c_int;
    pub fn bb_groth16_verify_batch(ctx: *mut bb_ctx, vk: *const bb_vk, batch: *const bb_proof_batch, z: *const c_void) -> c_int;
    pub fn bb_groth16_verify_each(ctx: *mut bb_ctx, vk: *const bb_vk, batch: *const bb_proof_batch, verdicts: *mut u8,
                                  n_invalid: *mut usize) -> c_int;
    pub fn bb_proofs_read(ctx: *mut bb_ctx, input: *const bb_proof_bytes, a: *mut c_void, b: *mut c_void, c: *mut c_void,
                          out_on_device: c_int, status: *mut u8, n_invalid: *mut usize) -> c_int;
    pub fn bb_proofs_write(ctx: *mut bb_ctx, a: *const c_void, b: *const c_void, c: *const c_void, n: usize, on_device: c_int,
                           out: *mut c_void) -> c_int;
    pub fn bb_params_read(ctx: *mut bb_ctx, bytes: *const c_void, len: usize, on_device: c_int, checked: c_int,
                          crs_out: *mut *mut bb_crs, vk_out: *mut *mut bb_vk, report: *mut bb_params_report) -> c_int;
    pub fn bb_vk_read(ctx: *mut bb_ctx, bytes: *const c_void, len: usize, on_device: c_int, vk_out: *mut *mut bb_vk,
                      report: *mut bb_params_report) -> c_int;
    pub fn bb_params_write(ctx: *mut bb_ctx, crs: *const bb_crs, vk: *const bb_vk, vk_only: c_int, out: *mut c_void, cap: usize,
                           out_on_device: c_int, len_out: *mut usize) -> c_int;
    pub fn bb_groth16_generate(ctx: *mut bb_ctx, r1cs: *const bb_r1cs, toxic: *const bb_toxic, crs_out: *mut *mut bb_crs,
                               vk_out: *mut *mut bb_vk, report: *mut bb_generate_report) -> c_int;

    pub fn bb_tuning_count() -> c_int;
    pub fn bb_tuning_name(index: c_int) -> *const c_char;
    pub fn bb_crs_apply_tuning(ctx: *mut bb_ctx, crs: *mut bb_crs, index: c_int) -> c_int;
    pub fn bb_groth16_autotune(ctx: *mut bb_ctx, crs: *mut bb_crs, w: *const bb_witness, reps: c_int, chosen: *mut c_int,
                               ms_out: *mut f64) -> c_int;

    pub fn bb_profile_read(ctx: *mut bb_ctx, what: *const c_char, ms: *mut f64, launches: *mut u64, units: *mut u64) -> c_int;
    pub fn bb_profile_reset(ctx: *mut bb_ctx) -> c_int;
    pub fn bb_ctx_bytes_copied(ctx: *const bb_ctx, h2d: *mut u64, d2h: *mut u64) -> c_int;
}
