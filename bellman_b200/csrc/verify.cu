// bellman_b200: Groth16 verification on the device -- PreparedVerifyingKey, verify_proof and the batch
// verifier (groth16/src/verifier.rs:11-58, groth16/src/verifier/batch.rs:72-173).
//
// A batch of n proofs (A_i, B_i, C_i; public inputs x_i) with random non-zero z_i is accepted iff
//     prod_i e(z_i A_i, -B_i) * e(sum_i z_i C_i, delta) * e(Psi, gamma) * e([sum_i z_i] alpha, beta) = 1,
//     Psi = sum_j acc_Gamma[j] ic[j],  acc_Gamma[0] = sum_i z_i,  acc_Gamma[j] = sum_i z_i x_ij.
// Stages (main stream unless noted):
//   k_verify_scalars     z_i to Montgomery form; the scalars of the sum over C (zero where C_i is the identity)
//   k_colsum_*           acc_Gamma: an Fr column reduction over the n x L input matrix
//   MSM jobs             sum z_i C_i and Psi (msm.cu, own streams; their window folds run on the host)
//   k_proof_pairs        [z_i] A_i by a variable-base double-and-add, one thread per proof; -B_i
//   k_alpha_pair         [acc_Y] alpha
//   k_miller             one Miller loop per pair, one thread per pair (tower.cuh)
//   k_fp12_pair_product  the tree product of the n + 3 Miller values, one level per launch
//   k_final_exp          final exponentiation and the comparison with one, one thread
//
// verify_proof for each proof of a batch (bb_groth16_verify_each; Item::verify_single, batch.rs:57-65): proof i is valid iff
//     FE( ML(A_i, B_i) * ML(Psi_i, -gamma) * ML(C_i, -delta) ) == e(alpha, beta)^3,  Psi_i = ic[0] + sum_j x_ij ic[j+1],
// in the device's G_T convention (tower.cuh).  Stages, one thread per proof each:
//   k_each_psi           Psi_i by mixed additions from the byte tables of the ic points (fixed_table.cuh)
//   k_each_miller        one multi-Miller loop over the three pairs sharing f; the two key pairs evaluate stored lines
//   k_each_final_exp     final exponentiation, comparison with the cached target, verdict byte
// The key data they need (EachKey) is built by the first call and cached in the bb_vk.
#include <sys/random.h>

#include "bb_internal.cuh"
#include "fixed_table.cuh"
#include "tower.cuh"

using namespace bb;

namespace {
constexpr int MILLER_STEPS = 68;                 // 63 doubling and 5 addition steps over |x| = 0xd201000000010000
}  // namespace

// What bb_groth16_verify_each adds to bb_vk_prepare's data, built on its first call for the key
struct EachKey {
    Fp2* d_lines = nullptr;             // G2Prepared (lib.rs:400-409) of -gamma, then of -delta: MILLER_STEPS x (A, B, C) each
    Fp12* d_target = nullptr;           // e(alpha, beta)^3
    bool gamma_live = false, delta_live = false;      // false: that G2 point is the identity and its pair contributes one
    std::vector<FixedTable<Fp>> tabs;   // tabs[j]: byte multiples of ic[j] for j >= 1; none for an identity ic[j]
    const G1Affine** d_tabs = nullptr;  // the tables' device addresses by j (nullptr: no table)
};

struct bb_vk {
    bb_ctx* ctx = nullptr;
    G1Affine* d_alpha = nullptr;        // alpha_g1
    G2Affine* d_g2 = nullptr;           // delta_g2, gamma_g2, beta_g2: the G2 sides of the batch's last three pairs
    bb_bases* ic = nullptr;             // ic, resident for the Psi MSM
    size_t ic_len = 0;
    mutable std::mutex each_mu;         // guards `each`
    mutable EachKey* each = nullptr;
};

namespace {

constexpr unsigned MILLER_THREADS = 64;
constexpr size_t COLSUM_CHUNK = 256;

__global__ void __launch_bounds__(256) k_verify_scalars(const Fr* __restrict__ z, const G1Affine* __restrict__ c, size_t n,
                                                        Fr* z_mont, Fr* sc_c) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr zi = z[i];
    z_mont[i] = fr_from_canonical(zi);
    sc_c[i] = c[i].is_identity() ? Fr::zero() : zi;     // an identity base must not meet a non-zero scalar in the MSM
}

// partial[ch * (L + 1) + j] = sum over rows [ch * CHUNK, (ch + 1) * CHUNK) of z_i * x_ij  (x_i0 = 1), Montgomery
__global__ void __launch_bounds__(256) k_colsum_partial(const Fr* __restrict__ z_mont, const Fr* __restrict__ x, size_t n, size_t L,
                                                        size_t chunks, Fr* partial) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= chunks * (L + 1)) return;
    size_t j = t % (L + 1), ch = t / (L + 1);
    size_t lo = ch * COLSUM_CHUNK, hi = lo + COLSUM_CHUNK < n ? lo + COLSUM_CHUNK : n;
    Fr acc = Fr::zero();
    for (size_t i = lo; i < hi; i++) acc = acc + (j == 0 ? z_mont[i] : z_mont[i] * x[i * L + j - 1]);
    partial[t] = acc;
}
// acc_ic[j] = acc_Gamma[j], or zero where ic[j] is the identity; acc_y = acc_Gamma[0] = sum z_i
__global__ void __launch_bounds__(128) k_colsum_final(const Fr* __restrict__ partial, size_t chunks, size_t L,
                                                      const G1Affine* __restrict__ ic, Fr* acc_ic, Fr* acc_y) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j > L) return;
    Fr acc = Fr::zero();
    for (size_t ch = 0; ch < chunks; ch++) acc = acc + partial[ch * (L + 1) + j];
    acc_ic[j] = ic[j].is_identity() ? Fr::zero() : acc;
    if (j == 0) *acc_y = acc;
}

// pair i: ([z_i] A_i, -B_i)
__global__ void __launch_bounds__(128) k_proof_pairs(const G1Affine* __restrict__ a, const G2Affine* __restrict__ b, const Fr* __restrict__ z,
                                                     size_t n, G1Eval* pe, G2Affine* q) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr zi = z[i];
    pe[i] = g1_eval_from_xyzz(G1X::from_affine(a[i]).mul_bits(zi.l));
    q[i] = b[i].neg();
}
__global__ void k_alpha_pair(const G1Affine* __restrict__ alpha, const Fr* __restrict__ acc_y, G1Eval* pe) {
    Fr k = fr_to_canonical(*acc_y);
    *pe = g1_eval_from_xyzz(G1X::from_affine(*alpha).mul_bits(k.l));
}
__global__ void __launch_bounds__(128) k_affine_pairs(const G1Affine* __restrict__ p, size_t n, G1Eval* pe) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pe[i] = g1_eval_from_affine(p[i]);
}

__global__ void __launch_bounds__(MILLER_THREADS) k_miller(const G1Eval* __restrict__ pe, const G2Affine* __restrict__ q, size_t n, Fp12* f) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f[i] = miller_loop(pe[i], q[i]);
}

// out[i] = in[2i] * in[2i + 1] (the last one alone when n is odd)
__global__ void __launch_bounds__(MILLER_THREADS) k_fp12_pair_product(const Fp12* __restrict__ in, size_t n, Fp12* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (2 * i >= n) return;
    out[i] = 2 * i + 1 < n ? fp12_mul(in[2 * i], in[2 * i + 1]) : in[2 * i];
}

// gt = f^(3 (p^12 - 1) / r); verdict = (gt == 1)
__global__ void k_final_exp(const Fp12* __restrict__ f, Fp12* gt, uint32_t* verdict) {
    Fp12 x = *f;
    Fp12 r = x.is_zero() ? x : fp12_final_exp(x);
    *gt = r;
    *verdict = r.is_one() ? 1u : 0u;
}

// diagnostics: element-wise tower operations (bb_diag_fp12).  The inverse and the final exponentiation map zero to zero,
// as k_final_exp does: both invert, and the binary Euclidean inversion does not terminate on zero.
__global__ void __launch_bounds__(64) k_diag_fp12(const Fp12* __restrict__ a, const Fp12* __restrict__ b, size_t n, int op, Fp12* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp12 x = a[i], y = b[i];
    Fp12 r;
    switch (op) {
        case 0: r = fp12_mul(x, y); break;
        case 1: r = fp12_sqr(x); break;
        case 2: r = x.is_zero() ? x : fp12_inv(x); break;
        case 3: r = fp12_cyclotomic_sqr(x); break;
        case 4: r = fp12_frob1(x); break;
        case 5: r = fp12_frob2(x); break;
        case 6: r = x.is_zero() ? x : fp12_final_exp(x); break;
        default: r = fp12_mul_line(x, y.c0.c0, y.c0.c1, y.c1.c1); break;
    }
    out[i] = r;
}

// Root of the batch: miller values of all pairs in d_f[0, m) -> verdict (and the G_T value, host, if asked)
int product_and_final_exp(bb_ctx* ctx, cudaStream_t st, Fp12* d_f, size_t m, StageTimer& tm, bool* accepted, Fp12* gt_host) {
    DevBuf d_tmp, d_out;
    BB_TRY(d_tmp.alloc(ctx, ((m + 1) / 2 + 1) * sizeof(Fp12)));
    BB_TRY(d_out.alloc(ctx, sizeof(Fp12) + 16));
    Fp12* cur = d_f;
    Fp12* nxt = d_tmp.as<Fp12>();
    while (m > 1) {
        size_t h = (m + 1) / 2;
        k_fp12_pair_product<<<cdiv(h, MILLER_THREADS), MILLER_THREADS, 0, st>>>(cur, m, nxt);
        ctx->count_launch();
        Fp12* t = cur;
        cur = nxt;
        nxt = t;
        m = h;
    }
    tm.mark("verify.product");
    Fp12* d_gt = d_out.as<Fp12>();
    uint32_t* d_verdict = (uint32_t*)(d_gt + 1);
    k_final_exp<<<1, 1, 0, st>>>(cur, d_gt, d_verdict);
    ctx->count_launch();
    tm.mark("verify.final_exp");
    BB_CUDA(cudaGetLastError());
    uint32_t verdict = 0;
    BB_CUDA(cudaMemcpyAsync(&verdict, d_verdict, 4, cudaMemcpyDeviceToHost, st));
    if (gt_host) BB_CUDA(cudaMemcpyAsync(gt_host, d_gt, sizeof(Fp12), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    *accepted = verdict == 1;
    return BB_OK;
}

bool fr_is_canonical_nonzero(const Fr& v) {
    if (v.is_zero()) return false;
    for (int i = 7; i >= 0; i--) {
        if (v.l[i] < bbc::FR_MOD[i]) return true;
        if (v.l[i] > bbc::FR_MOD[i]) return false;
    }
    return false;
}

// z_i uniform in [1, r) from the operating system (batch.rs:124-129 loops until z != 0)
int draw_z(std::vector<Fr>& z) {
    for (Fr& v : z) {
        do {
            uint8_t buf[32];
            size_t got = 0;
            while (got < sizeof buf) {
                ssize_t k = getrandom(buf + got, sizeof buf - got, 0);
                if (k < 0) { set_error("getrandom failed"); return BB_ERR_ARG; }
                got += (size_t)k;
            }
            buf[31] &= 0x7f;                                     // 255-bit draws, rejection sampled below r
            std::memcpy(v.l, buf, 32);
        } while (!fr_is_canonical_nonzero(v));
    }
    return BB_OK;
}

// Fp12 of the device -> 12 canonical Fp in tower order
void gt_to_canonical(const Fp12& g, void* out) {
    const Fp* c = (const Fp*)&g;
    Fp* o = (Fp*)out;
    for (int k = 0; k < 12; k++) o[k] = fp_to_canonical(c[k]);
}

// The argument checks of verify_batch and verify_each, before any device work.  outputs: the caller's output arrays
// are present (checked with the proof arrays).
int check_proof_batch(const char* fn, const bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* b, bool outputs) {
    if (!ctx || !vk || !b) { set_error("%s: null argument", fn); return BB_ERR_ARG; }
    const size_t n = b->n, L = b->n_inputs;
    if (n && (!outputs || !b->a || !b->b || !b->c || (L && !b->inputs))) { set_error("%s: null array", fn); return BB_ERR_ARG; }
    if (n && L + 1 != vk->ic_len) {                              // batch.rs:105-111
        set_error("InvalidVerifyingKey: %zu public inputs for a key with %zu ic entries", L, vk->ic_len);
        return BB_ERR_INVALID_VERIFYING_KEY;
    }
    if (n >= (1ull << 31)) { set_error("%s: more than 2^31 proofs", fn); return BB_ERR_ARG; }
    return BB_OK;
}

// The batch verifier.  gt_host: optional, receives the G_T value the verdict was taken from.
int verify_batch(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* b, const void* z_in, Fp12* gt_host) {
    BB_TRY(check_proof_batch("bb_groth16_verify_batch", ctx, vk, b, true));
    const size_t n = b->n, L = b->n_inputs;
    std::vector<Fr> z(n);
    if (z_in) {
        std::memcpy(z.data(), z_in, n * 32);
        for (size_t i = 0; i < n; i++)
            if (!fr_is_canonical_nonzero(z[i])) { set_error("z[%zu] is zero or not below r", i); return BB_ERR_ARG; }
    } else {
        BB_TRY(draw_z(z));
    }
    if (n == 0) {                                                // every accumulator is the identity: the product is one
        if (gt_host) *gt_host = Fp12::one();
        return BB_OK;
    }
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("groth16_verify_batch");
    cudaStream_t st = ctx->main_stream;
    StageTimer tm(ctx, st);
    tm.mark("verify.begin");
    const G1Affine *d_a, *d_c;
    const G2Affine* d_b;
    const Fr* d_x;
    DevBuf up_a, up_b, up_c, up_x, d_z, d_zm, d_scc, d_part, d_acc, d_pe, d_q, d_f;
    BB_TRY(device_input(ctx, st, b->a, n * sizeof(G1Affine), b->on_device, up_a, &d_a));
    BB_TRY(device_input(ctx, st, b->b, n * sizeof(G2Affine), b->on_device, up_b, &d_b));
    BB_TRY(device_input(ctx, st, b->c, n * sizeof(G1Affine), b->on_device, up_c, &d_c));
    BB_TRY(device_input(ctx, st, b->inputs, n * L * 32, b->on_device, up_x, &d_x));
    const size_t pairs = n + 3, chunks = (n + COLSUM_CHUNK - 1) / COLSUM_CHUNK;
    BB_TRY(d_z.alloc(ctx, n * 32));
    BB_TRY(d_zm.alloc(ctx, n * 32));
    BB_TRY(d_scc.alloc(ctx, n * 32));
    BB_TRY(d_part.alloc(ctx, chunks * (L + 1) * 32));
    BB_TRY(d_acc.alloc(ctx, (L + 2) * 32));
    BB_TRY(d_pe.alloc(ctx, pairs * sizeof(G1Eval)));
    BB_TRY(d_q.alloc(ctx, pairs * sizeof(G2Affine)));
    BB_TRY(d_f.alloc(ctx, pairs * sizeof(Fp12)));
    BB_CUDA(cudaMemcpyAsync(d_z.p, z.data(), n * 32, cudaMemcpyHostToDevice, st));
    ctx->h2d_bytes += n * 32;
    Fr* d_acc_ic = d_acc.as<Fr>();
    Fr* d_acc_y = d_acc_ic + L + 1;

    k_verify_scalars<<<cdiv(n, 256), 256, 0, st>>>(d_z.as<Fr>(), d_c, n, d_zm.as<Fr>(), d_scc.as<Fr>());
    k_colsum_partial<<<cdiv(chunks * (L + 1), 256), 256, 0, st>>>(d_zm.as<Fr>(), d_x, n, L, chunks, d_part.as<Fr>());
    k_colsum_final<<<cdiv(L + 1, 128), 128, 0, st>>>(d_part.as<Fr>(), chunks, L, (const G1Affine*)vk->ic->d_points, d_acc_ic, d_acc_y);
    ctx->count_launch(3);
    BB_CUDA(cudaGetLastError());
    tm.mark("verify.accumulators");

    // sum z_i C_i and Psi on the MSM streams, while this stream runs the proofs' scalar multiplications and Miller loops
    cudaEvent_t ev_scalars = nullptr;
    BB_CUDA(cudaEventCreateWithFlags(&ev_scalars, cudaEventDisableTiming));
    bb_bases c_bases;
    c_bases.ctx = ctx; c_bases.group = BB_G1; c_bases.d_points = (void*)d_c; c_bases.n = n; c_bases.global_offset = 0; c_bases.global_len = n;
    bb_msm_job* jobs[2] = {nullptr, nullptr};
    auto drain = [&]() {                                         // every exit waits for the jobs that use this call's buffers
        for (auto& j : jobs) if (j) { int sj; G1X pj; msm_wait(j, &sj, &pj); j = nullptr; }
        if (c_bases.d_table) { ctx->release(c_bases.d_table); c_bases.d_table = nullptr; }
        if (ev_scalars) { cudaEventDestroy(ev_scalars); ev_scalars = nullptr; }
    };
    int s = cudaEventRecord(ev_scalars, st) == cudaSuccess ? BB_OK : BB_ERR_CUDA;
    if (s == BB_OK) s = msm_start(ctx, &c_bases, 0, nullptr, 0, d_scc.p, true, n, BB_FORM_CANONICAL, ev_scalars, &jobs[0], "verify_c");
    if (s == BB_OK) s = msm_start(ctx, vk->ic, 0, nullptr, 0, d_acc_ic, true, L + 1, BB_FORM_MONTGOMERY, ev_scalars, &jobs[1], "verify_psi");
    if (s != BB_OK) { drain(); return s; }

    G1Eval* d_pev = d_pe.as<G1Eval>();
    G2Affine* d_qv = d_q.as<G2Affine>();
    k_proof_pairs<<<cdiv(n, 128), 128, 0, st>>>(d_a, d_b, d_z.as<Fr>(), n, d_pev, d_qv);
    k_alpha_pair<<<1, 1, 0, st>>>(vk->d_alpha, d_acc_y, d_pev + n + 2);
    ctx->count_launch(2);
    tm.mark("verify.scalar_mul");
    if (cudaMemcpyAsync(d_qv + n, vk->d_g2, 3 * sizeof(G2Affine), cudaMemcpyDeviceToDevice, st) != cudaSuccess) { drain(); set_error("vk copy failed"); return BB_ERR_CUDA; }
    k_miller<<<cdiv(n, MILLER_THREADS), MILLER_THREADS, 0, st>>>(d_pev, d_qv, n, d_f.as<Fp12>());
    ctx->count_launch();
    tm.mark("verify.miller");

    G1X res[2];
    int status = BB_OK;
    for (int k = 0; k < 2; k++) {
        int sk;
        msm_wait(jobs[k], &sk, &res[k]);
        jobs[k] = nullptr;
        if (status == BB_OK) status = sk;
    }
    drain();
    if (status != BB_OK) { cudaStreamSynchronize(st); return status; }
    tm.mark("verify.msm_wait");
    G1Eval h_pe[2] = {g1_eval_from_xyzz(res[0]), g1_eval_from_xyzz(res[1])};      // (acc_Delta, delta), (Psi, gamma)
    BB_CUDA(cudaMemcpyAsync(d_pev + n, h_pe, sizeof h_pe, cudaMemcpyHostToDevice, st));
    k_miller<<<1, 3, 0, st>>>(d_pev + n, d_qv + n, 3, d_f.as<Fp12>() + n);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    tm.mark("verify.miller_tail");
    bool accepted = false;
    BB_TRY(product_and_final_exp(ctx, st, d_f.as<Fp12>(), pairs, tm, &accepted, gt_host));
    tm.report(n);
    if (!accepted) { set_error("InvalidProof: the batch does not verify"); return BB_ERR_INVALID_PROOF; }
    return BB_OK;
}

// ---- verify_proof per proof (bb_groth16_verify_each) -----------------------------------------------------------------
// Thread 0: the lines of -gamma (d_g2[1]), thread 1: those of -delta (d_g2[0]).  The ordinary Miller steps evaluated at
// the unit point {x = 1, y = 1, s = 1} return the raw coefficients: they multiply A, B, C by s, x, y.
__global__ void k_each_lines(const G2Affine* __restrict__ g2, Fp2* lines) {
    const int t = threadIdx.x;
    if (t > 1) return;
    const G2Affine q = g2[t == 0 ? 1 : 0].neg();
    if (q.is_identity()) return;
    const Fp one = fp_one();
    const G1Eval unit{one, one, one};
    Fp2* out = lines + (size_t)t * MILLER_STEPS * 3;
    G2Proj T{q.x, q.y, fp2_one()};
    int k = 0;
    for (int i = 62; i >= 0; i--) {
        MillerStep d = miller_dbl_step(T, unit);
        T = d.T;
        out[3 * k] = d.A; out[3 * k + 1] = d.B; out[3 * k + 2] = d.C;
        k++;
        if ((bbc::BLS_X_ABS >> i) & 1) {
            MillerStep a = miller_add_step(T, q, unit);
            T = a.T;
            out[3 * k] = a.A; out[3 * k + 1] = a.B; out[3 * k + 2] = a.C;
            k++;
        }
    }
}

// e(alpha, beta)^3 with the same Miller loop and final exponentiation as every proof's value
__global__ void k_each_target(const G1Affine* __restrict__ alpha, const G2Affine* __restrict__ g2, Fp12* target) {
    *target = fp12_final_exp(miller_loop(g1_eval_from_affine(*alpha), g2[2]));
}

// Psi_i = ic[0] + sum_j x_ij ic[j+1] (verifier.rs:34-41): the digits of x_ij select byte multiples of ic[j+1]
__global__ void __launch_bounds__(128) k_each_psi(const G1Affine* __restrict__ ic, const G1Affine* const* __restrict__ tabs,
                                                  const Fr* __restrict__ x, size_t n, size_t L, G1Eval* pe) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    G1X acc = G1X::from_affine(ic[0]);
    for (size_t j = 0; j < L; j++) {
        const G1Affine* tab = tabs[j + 1];
        if (!tab) continue;                                      // an identity ic[j + 1] contributes nothing
        Fr s = fr_to_canonical(x[i * L + j]);
        for (int w = 0; w < 32; w++) {
            uint32_t d = (s.l[w >> 2] >> (8 * (w & 3))) & 0xffu;
            if (d) acc.add_mixed(tab[w * 255 + d - 1]);
        }
    }
    pe[i] = g1_eval_from_xyzz(acc);
}

// f * (a stored line evaluated at P): 3 Fp2 x Fp products, then the sparse product
BB_HD Fp12 mul_stored_line(const Fp12& f, const Fp2* __restrict__ l, const G1Eval& p) {
    return fp12_mul_line(f, fp2_mul_fp(l[0], p.s), fp2_mul_fp(l[1], p.x), fp2_mul_fp(l[2], p.y));
}

// ML(A_i, B_i) ML(Psi_i, -gamma) ML(C_i, -delta) with one f: 63 squarings in all.  f is shared, so a pair with an
// identity on either side is skipped explicitly (its line would multiply f by zero), which gives the one that
// multi_miller_loop gives it.
__global__ void __launch_bounds__(MILLER_THREADS) k_each_miller(const G1Affine* __restrict__ a, const G2Affine* __restrict__ b,
                                                                const G1Affine* __restrict__ c, const G1Eval* __restrict__ psi, size_t n,
                                                                const Fp2* __restrict__ lines, int gamma_live, int delta_live, Fp12* f_out) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const G1Eval pa = g1_eval_from_affine(a[idx]), pc = g1_eval_from_affine(c[idx]), pp = psi[idx];
    const G2Affine q = b[idx];
    const bool ab = !pa.s.is_zero() && !q.is_identity();
    const bool pg = gamma_live && !pp.s.is_zero();
    const bool cd = delta_live && !pc.s.is_zero();
    const Fp2* lg = lines;
    const Fp2* ld = lines + MILLER_STEPS * 3;
    G2Proj T{q.x, q.y, fp2_one()};
    Fp12 f = Fp12::one();
    int k = 0;
    for (int i = 62; i >= 0; i--) {
        f = fp12_sqr(f);
        if (ab) {
            MillerStep d = miller_dbl_step(T, pa);
            T = d.T;
            f = fp12_mul_line(f, d.A, d.B, d.C);
        }
        if (pg) f = mul_stored_line(f, lg + 3 * k, pp);
        if (cd) f = mul_stored_line(f, ld + 3 * k, pc);
        k++;
        if ((bbc::BLS_X_ABS >> i) & 1) {
            if (ab) {
                MillerStep s = miller_add_step(T, q, pa);
                T = s.T;
                f = fp12_mul_line(f, s.A, s.B, s.C);
            }
            if (pg) f = mul_stored_line(f, lg + 3 * k, pp);
            if (cd) f = mul_stored_line(f, ld + 3 * k, pc);
            k++;
        }
    }
    f_out[idx] = f;
}

// Fp2 equality of the canonical values (limbs of Montgomery forms need not be unique)
BB_HD bool fp2_equal(const Fp2& x, const Fp2& y) {
    return fp_to_canonical(x.c0) == fp_to_canonical(y.c0) && fp_to_canonical(x.c1) == fp_to_canonical(y.c1);
}
BB_HD bool fp12_equal(const Fp12& x, const Fp12& y) {
    return fp2_equal(x.c0.c0, y.c0.c0) && fp2_equal(x.c0.c1, y.c0.c1) && fp2_equal(x.c0.c2, y.c0.c2) &&
           fp2_equal(x.c1.c0, y.c1.c0) && fp2_equal(x.c1.c1, y.c1.c1) && fp2_equal(x.c1.c2, y.c1.c2);
}

// verdict[i] = 0 if FE(f_i) == target, else 1; gt (optional) receives FE(f_i)
__global__ void k_each_final_exp(const Fp12* __restrict__ f, size_t n, const Fp12* __restrict__ target,
                                                                   uint8_t* verdict, Fp12* gt) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp12 x = f[i];
    Fp12 r = x.is_zero() ? x : fp12_final_exp(x);
    if (gt) gt[i] = r;
    verdict[i] = fp12_equal(r, *target) ? 0 : 1;
}

void each_key_free(bb_ctx* ctx, EachKey* e) {
    for (auto& t : e->tabs)
        if (t.d_table) cudaFree(t.d_table);
    if (e->d_lines) ctx->release(e->d_lines);
    if (e->d_target) ctx->release(e->d_target);
    if (e->d_tabs) ctx->release(e->d_tabs);
    delete e;
}

int each_key_build(bb_ctx* ctx, const bb_vk* vk, EachKey* e) {
    const size_t m = vk->ic_len;
    std::vector<G1Affine> ic(m);
    G2Affine g2[3];
    if (m) BB_CUDA(cudaMemcpy(ic.data(), vk->ic->d_points, m * sizeof(G1Affine), cudaMemcpyDeviceToHost));
    BB_CUDA(cudaMemcpy(g2, vk->d_g2, sizeof g2, cudaMemcpyDeviceToHost));
    e->delta_live = !g2[0].is_identity();
    e->gamma_live = !g2[1].is_identity();
    e->tabs.resize(m);
    std::vector<const G1Affine*> ptrs(m > 0 ? m : 1, nullptr);
    for (size_t j = 1; j < m; j++) {                             // ic[0] is added as it is
        if (ic[j].is_identity()) continue;
        BB_TRY(build_fixed_table(e->tabs[j], ic[j]));
        ptrs[j] = e->tabs[j].d_table;
    }
    BB_TRY(ctx->alloc(2 * MILLER_STEPS * 3 * sizeof(Fp2), (void**)&e->d_lines));
    BB_TRY(ctx->alloc(sizeof(Fp12), (void**)&e->d_target));
    BB_TRY(ctx->alloc(ptrs.size() * sizeof(G1Affine*), (void**)&e->d_tabs));
    BB_CUDA(cudaMemcpy(e->d_tabs, ptrs.data(), ptrs.size() * sizeof(G1Affine*), cudaMemcpyHostToDevice));
    cudaStream_t st = ctx->main_stream;
    k_each_lines<<<1, 2, 0, st>>>(vk->d_g2, e->d_lines);
    k_each_target<<<1, 1, 0, st>>>(vk->d_alpha, vk->d_g2, e->d_target);
    ctx->count_launch(2);
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

int each_key(bb_ctx* ctx, const bb_vk* vk, const EachKey** out) {
    std::lock_guard<std::mutex> g(vk->each_mu);
    if (!vk->each) {
        EachKey* e = new EachKey();
        int s = each_key_build(ctx, vk, e);
        if (s != BB_OK) { each_key_free(ctx, e); return s; }
        vk->each = e;
    }
    *out = vk->each;
    return BB_OK;
}

// verify_proof per proof.  gt_host: optional, n + 1 values: every proof's FE(f_i), then the target.
int verify_each(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* b, uint8_t* verdicts, size_t* n_invalid, Fp12* gt_host) {
    BB_TRY(check_proof_batch("bb_groth16_verify_each", ctx, vk, b, verdicts && n_invalid));
    const size_t n = b->n, L = b->n_inputs;
    if (n_invalid) *n_invalid = 0;
    if (n == 0 && !gt_host) return BB_OK;
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("groth16_verify_each");
    const EachKey* ek = nullptr;
    BB_TRY(each_key(vk->ctx, vk, &ek));                         // owned by the key, like its other device buffers
    cudaStream_t st = ctx->main_stream;
    if (n == 0) {
        BB_CUDA(cudaMemcpyAsync(gt_host, ek->d_target, sizeof(Fp12), cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaStreamSynchronize(st));
        return BB_OK;
    }
    StageTimer tm(ctx, st);
    tm.mark("verify_each.begin");
    const G1Affine *d_a, *d_c;
    const G2Affine* d_b;
    const Fr* d_x;
    DevBuf up_a, up_b, up_c, up_x, d_pe, d_f, d_v, d_gt;
    BB_TRY(device_input(ctx, st, b->a, n * sizeof(G1Affine), b->on_device, up_a, &d_a));
    BB_TRY(device_input(ctx, st, b->b, n * sizeof(G2Affine), b->on_device, up_b, &d_b));
    BB_TRY(device_input(ctx, st, b->c, n * sizeof(G1Affine), b->on_device, up_c, &d_c));
    BB_TRY(device_input(ctx, st, b->inputs, n * L * 32, b->on_device, up_x, &d_x));
    BB_TRY(d_pe.alloc(ctx, n * sizeof(G1Eval)));
    BB_TRY(d_f.alloc(ctx, n * sizeof(Fp12)));
    BB_TRY(d_v.alloc(ctx, n));
    if (gt_host) BB_TRY(d_gt.alloc(ctx, n * sizeof(Fp12)));
    tm.mark("verify_each.upload");
    k_each_psi<<<cdiv(n, 128), 128, 0, st>>>((const G1Affine*)vk->ic->d_points, ek->d_tabs, d_x, n, L, d_pe.as<G1Eval>());
    ctx->count_launch();
    tm.mark("verify_each.psi");
    k_each_miller<<<cdiv(n, MILLER_THREADS), MILLER_THREADS, 0, st>>>(d_a, d_b, d_c, d_pe.as<G1Eval>(), n, ek->d_lines, ek->gamma_live ? 1 : 0,
                                                                      ek->delta_live ? 1 : 0, d_f.as<Fp12>());
    ctx->count_launch();
    tm.mark("verify_each.miller");
    k_each_final_exp<<<cdiv(n, MILLER_THREADS), MILLER_THREADS, 0, st>>>(d_f.as<Fp12>(), n, ek->d_target, d_v.as<uint8_t>(),
                                                                         gt_host ? d_gt.as<Fp12>() : nullptr);
    ctx->count_launch();
    tm.mark("verify_each.final_exp");
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaMemcpyAsync(verdicts, d_v.p, n, cudaMemcpyDeviceToHost, st));
    ctx->d2h_bytes += n;
    if (gt_host) {
        BB_CUDA(cudaMemcpyAsync(gt_host, d_gt.p, n * sizeof(Fp12), cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(gt_host + n, ek->d_target, sizeof(Fp12), cudaMemcpyDeviceToHost, st));
    }
    tm.mark("verify_each.download");
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(n);
    size_t bad = 0;
    for (size_t i = 0; i < n; i++) bad += verdicts[i] != 0;
    *n_invalid = bad;
    return BB_OK;
}

struct SplitMix {
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
    Fr fr_nonzero() {                                            // uniform in [1, r), Montgomery
        for (;;) {
            uint64_t c[4] = {next(), next(), next(), next() & 0x7fffffffffffffffull};
            Fr v;
            std::memcpy(v.l, c, 32);
            if (fr_is_canonical_nonzero(v)) return fr_from_canonical(v);
        }
    }
};

// c_i = (a_i b_i - alpha beta - sum_{j <= L} x_ij gamma t_j) / delta with x_i0 = 1; a, b, x canonical in, x also out (Montgomery)
__global__ void __launch_bounds__(128) k_synth_c(const Fr* __restrict__ a, const Fr* __restrict__ b, Fr* x, size_t n, size_t L,
                                                 const Fr* __restrict__ gt_j, Fr alpha_beta, Fr delta_inv, Fr* c) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr acc = fr_from_canonical(a[i]) * fr_from_canonical(b[i]) - alpha_beta - gt_j[0];
    for (size_t j = 0; j < L; j++) {
        Fr xv = fr_from_canonical(x[i * L + j]);
        x[i * L + j] = xv;
        acc = acc - xv * gt_j[j + 1];
    }
    c[i] = acc * delta_inv;
}

}  // namespace

extern "C" {

int bb_vk_prepare(bb_ctx* ctx, const bb_vk_desc* d, bb_vk** out) {
    if (!ctx || !d || !out || !d->alpha_g1 || !d->beta_g2 || !d->gamma_g2 || !d->delta_g2 || (d->ic_len && !d->ic)) {
        set_error("bb_vk_prepare: null argument");
        return BB_ERR_ARG;
    }
    BB_CUDA(cudaSetDevice(ctx->device));
    bb_vk* vk = new bb_vk();
    vk->ctx = ctx;
    vk->ic_len = d->ic_len;
    auto fail = [&](int s) { bb_vk_destroy(vk); return s; };
    int s;
    if ((s = ctx->alloc(sizeof(G1Affine), (void**)&vk->d_alpha)) != BB_OK) return fail(s);
    if ((s = ctx->alloc(3 * sizeof(G2Affine), (void**)&vk->d_g2)) != BB_OK) return fail(s);
    G2Affine g2[3];
    std::memcpy(&g2[0], d->delta_g2, sizeof(G2Affine));
    std::memcpy(&g2[1], d->gamma_g2, sizeof(G2Affine));
    std::memcpy(&g2[2], d->beta_g2, sizeof(G2Affine));
    if (cudaMemcpy(vk->d_alpha, d->alpha_g1, sizeof(G1Affine), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(vk->d_g2, g2, sizeof g2, cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("bb_vk_prepare: upload failed");
        return fail(BB_ERR_CUDA);
    }
    if ((s = bb_bases_upload(ctx, BB_G1, d->ic, d->ic_len, 0, d->ic_len, &vk->ic)) != BB_OK) return fail(s);
    *out = vk;
    return BB_OK;
}

}  // extern "C"

namespace bb {
bb_vk* vk_adopt(bb_ctx* ctx, G1Affine* d_alpha, G2Affine* d_g2, bb_bases* ic) {
    bb_vk* vk = new bb_vk();
    vk->ctx = ctx;
    vk->d_alpha = d_alpha;
    vk->d_g2 = d_g2;
    vk->ic = ic;
    vk->ic_len = ic->n;
    return vk;
}
VkView vk_view(const bb_vk* vk) { return VkView{vk->ctx, vk->d_alpha, vk->d_g2, vk->ic}; }
}  // namespace bb

extern "C" {

void bb_vk_destroy(bb_vk* vk) {
    if (!vk) return;
    if (vk->d_alpha) vk->ctx->release(vk->d_alpha);
    if (vk->d_g2) vk->ctx->release(vk->d_g2);
    if (vk->ic) bb_bases_free(vk->ic);
    if (vk->each) each_key_free(vk->ctx, vk->each);
    delete vk;
}

int bb_groth16_verify(bb_ctx* ctx, const bb_vk* vk, const void* a, const void* b, const void* c, const void* inputs, size_t n_inputs) {
    bb_proof_batch batch{a, b, c, 1, inputs, n_inputs, 0};
    Fr one = Fr::zero();
    one.l[0] = 1;                                                // verify_proof = the batch of one with z = 1
    return verify_batch(ctx, vk, &batch, one.l, nullptr);
}

int bb_groth16_verify_batch(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, const void* z) {
    return verify_batch(ctx, vk, batch, z, nullptr);
}

int bb_diag_verify_batch_gt(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, const void* z, void* gt_out) {
    if (!gt_out) { set_error("bb_diag_verify_batch_gt: null output"); return BB_ERR_ARG; }
    Fp12 g = Fp12::one();
    int s = verify_batch(ctx, vk, batch, z, &g);
    if (s == BB_OK || s == BB_ERR_INVALID_PROOF) gt_to_canonical(g, gt_out);
    return s;
}

int bb_groth16_verify_each(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, uint8_t* verdicts, size_t* n_invalid) {
    return verify_each(ctx, vk, batch, verdicts, n_invalid, nullptr);
}

int bb_diag_verify_each_gt(bb_ctx* ctx, const bb_vk* vk, const bb_proof_batch* batch, void* gt_out) {
    if (!batch || !gt_out) { set_error("bb_diag_verify_each_gt: null argument"); return BB_ERR_ARG; }
    const size_t n = batch->n;
    std::vector<uint8_t> verdicts(n);
    std::vector<Fp12> g(n + 1);
    size_t bad = 0;
    int s = verify_each(ctx, vk, batch, verdicts.data(), &bad, g.data());
    if (s != BB_OK) return s;
    for (size_t k = 0; k <= n; k++) gt_to_canonical(g[k], (uint8_t*)gt_out + k * sizeof(Fp12));
    return BB_OK;
}

int bb_diag_multi_pairing(bb_ctx* ctx, size_t n, const void* g1, const void* g2, void* gt_out) {
    if (!ctx || !gt_out || (n && (!g1 || !g2))) { set_error("bb_diag_multi_pairing: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    if (n == 0) { gt_to_canonical(Fp12::one(), gt_out); return BB_OK; }
    cudaStream_t st = ctx->main_stream;
    DevBuf d_p, d_pe, d_q, d_f;
    BB_TRY(d_p.alloc(ctx, n * sizeof(G1Affine)));
    BB_TRY(d_pe.alloc(ctx, n * sizeof(G1Eval)));
    BB_TRY(d_q.alloc(ctx, n * sizeof(G2Affine)));
    BB_TRY(d_f.alloc(ctx, n * sizeof(Fp12)));
    BB_CUDA(cudaMemcpyAsync(d_p.p, g1, n * sizeof(G1Affine), cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaMemcpyAsync(d_q.p, g2, n * sizeof(G2Affine), cudaMemcpyHostToDevice, st));
    k_affine_pairs<<<cdiv(n, 128), 128, 0, st>>>(d_p.as<G1Affine>(), n, d_pe.as<G1Eval>());
    k_miller<<<cdiv(n, MILLER_THREADS), MILLER_THREADS, 0, st>>>(d_pe.as<G1Eval>(), d_q.as<G2Affine>(), n, d_f.as<Fp12>());
    ctx->count_launch(2);
    BB_CUDA(cudaGetLastError());
    StageTimer tm(ctx, st);
    bool accepted = false;
    Fp12 g;
    BB_TRY(product_and_final_exp(ctx, st, d_f.as<Fp12>(), n, tm, &accepted, &g));
    gt_to_canonical(g, gt_out);
    return BB_OK;
}

int bb_diag_gt_exponent(void) { return 3; }

int bb_diag_fp12(bb_ctx* ctx, int op, const void* a, const void* b, void* out, size_t n) {
    if (!ctx || op < 0 || op > 7 || (n && (!a || !b || !out))) { set_error("bb_diag_fp12: bad argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    if (!n) return BB_OK;
    cudaStream_t st = ctx->main_stream;
    DevBuf da, db, d_o;
    BB_TRY(da.alloc(ctx, n * sizeof(Fp12)));
    BB_TRY(db.alloc(ctx, n * sizeof(Fp12)));
    BB_TRY(d_o.alloc(ctx, n * sizeof(Fp12)));
    BB_CUDA(cudaMemcpyAsync(da.p, a, n * sizeof(Fp12), cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaMemcpyAsync(db.p, b, n * sizeof(Fp12), cudaMemcpyHostToDevice, st));
    k_diag_fp12<<<cdiv(n, 64), 64, 0, st>>>(da.as<Fp12>(), db.as<Fp12>(), n, op, d_o.as<Fp12>());
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaMemcpyAsync(out, d_o.p, n * sizeof(Fp12), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

int bb_synth_proof_batch(bb_ctx* ctx, uint64_t seed, size_t n, size_t L, void* alpha_g1, void* beta_g2, void* gamma_g2, void* delta_g2,
                         void* ic, void* d_a, void* d_b, void* d_c, void* d_inputs) {
    if (!ctx || !alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || !ic || (n && (!d_a || !d_b || !d_c || (L && !d_inputs)))) {
        set_error("bb_synth_proof_batch: null argument");
        return BB_ERR_ARG;
    }
    BB_CUDA(cudaSetDevice(ctx->device));
    SplitMix g{seed ^ 0x5eed0f0f5eed0f0full};
    const Fr alpha = g.fr_nonzero(), beta = g.fr_nonzero(), gamma = g.fr_nonzero(), delta = g.fr_nonzero();
    std::vector<Fr> t(L + 1), gt(L + 1);
    for (size_t j = 0; j <= L; j++) { t[j] = g.fr_nonzero(); gt[j] = gamma * t[j]; }
    BB_TRY(bb_fixed_base_mul(ctx, BB_G1, &alpha, 1, BB_FORM_MONTGOMERY, alpha_g1));
    BB_TRY(bb_fixed_base_mul(ctx, BB_G1, t.data(), L + 1, BB_FORM_MONTGOMERY, ic));
    Fr g2s[3] = {beta, gamma, delta};
    G2Affine g2[3];
    BB_TRY(bb_fixed_base_mul(ctx, BB_G2, g2s, 3, BB_FORM_MONTGOMERY, g2));
    std::memcpy(beta_g2, &g2[0], sizeof(G2Affine));
    std::memcpy(gamma_g2, &g2[1], sizeof(G2Affine));
    std::memcpy(delta_g2, &g2[2], sizeof(G2Affine));
    if (!n) return BB_OK;
    // a_i, b_i, x_ij: the counter-based streams of bb_synth_scalars_device (canonical, < 2^254)
    DevBuf d_sa, d_sb, d_sc, d_gt;
    BB_TRY(d_sa.alloc(ctx, n * 32));
    BB_TRY(d_sb.alloc(ctx, n * 32));
    BB_TRY(d_sc.alloc(ctx, n * 32));
    BB_TRY(d_gt.alloc(ctx, (L + 1) * 32));
    BB_TRY(bb_synth_scalars_device(ctx, seed * 3 + 1, n, d_sa.p));
    BB_TRY(bb_synth_scalars_device(ctx, seed * 3 + 2, n, d_sb.p));
    if (L) BB_TRY(bb_synth_scalars_device(ctx, seed * 3 + 3, n * L, d_inputs));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d_gt.p, gt.data(), (L + 1) * 32, cudaMemcpyHostToDevice, st));
    k_synth_c<<<cdiv(n, 128), 128, 0, st>>>(d_sa.as<Fr>(), d_sb.as<Fr>(), (Fr*)d_inputs, n, L, d_gt.as<Fr>(), alpha * beta, fr_inv(delta),
                                             d_sc.as<Fr>());
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_sa.as<Fr>(), n, false, d_a, st));
    BB_TRY(fixed_base_mul_device(ctx, BB_G2, d_sb.as<Fr>(), n, false, d_b, st));
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_sc.as<Fr>(), n, true, d_c, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

}  // extern "C"
