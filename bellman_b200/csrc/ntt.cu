// bellman_b200: radix-2 NTT over BLS12-381 Fr for sm_90a.
//
// Replaces best_fft / serial_fft / parallel_fft (bellman/src/domain.rs:261-372)
// and the O(n) passes EvaluationDomain wraps around them: the m^-1 scaling of ifft
// (:88-98), distribute_powers (:101-113), divide_by_z_on_coset (:139-151), mul_assign
// (:154-170) and sub_assign (:173-189).
//
// Same transform as the reference (natural order in, natural order out,
// out[k] = sum_j a[j] w^{jk}; decimation in time over bit-reversed input), but staged for
// the GPU: the log n butterfly stages are grouped into passes of up to 8 stages; one CTA
// owns a tile of 2^k rows x 2^cbits adjacent columns, gathers it into shared memory
// (structure-of-arrays so the 8 limbs of consecutive elements sit in consecutive banks),
// runs its k stages there and writes the tile back.  Every element is one 32-byte DRAM
// sector, so even the strided passes move only algorithmic bytes: 64 B per point per pass.
// The bit reversal is folded into the first pass's gather, and all the O(n) passes of the
// reference are folded into the first-pass load or the last-pass store:
//   ifft          -> last pass multiplies by m^-1
//   coset_fft     -> first pass multiplies by g^i
//   icoset_fft    -> last pass multiplies by g^-i m^-1
//   H pipeline    -> ifft+distribute fused (g^i m^-1), a*b-c fused into the gather of the
//                    final inverse transform, 1/Z(g) folded into its g^-i m^-1 table.
// Field arithmetic is exact, so re-association does not change a single bit.
#include "bb_internal.cuh"

namespace bb {

struct NttTables {
    uint32_t log_n = 0;
    Fr* tw_fwd = nullptr;            // w^e, e < max(n/2,1)
    Fr* tw_inv = nullptr;            // w^-e
    Fr* pow_g = nullptr;             // g^i
    Fr* pow_ginv_minv = nullptr;     // g^-i m^-1
    Fr* pow_g_minv = nullptr;        // g^i m^-1
    Fr* pow_ginv_minv_zinv = nullptr;  // g^-i m^-1 / (g^m - 1)
    Fr minv;
};

__device__ __forceinline__ Fr ld_fr(const Fr* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    Fr r;
    r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w;
    r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
    return r;
}
__device__ __forceinline__ void st_fr(Fr* p, const Fr& v) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}

// out[i] = scale * base^i
__global__ void __launch_bounds__(256) k_powers(Fr* out, size_t n, Fr base, Fr scale) {
    constexpr size_t CH = 32;
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t start = t * CH;
    if (start >= n) return;
    Fr cur = scale * base.pow_u64((uint64_t)start, fr_one());
    size_t end = start + CH < n ? start + CH : n;
    for (size_t i = start; i < end; i++) {
        st_fr(out + i, cur);
        cur = cur * base;
    }
}

__global__ void __launch_bounds__(256) k_fr_convert(Fr* data, size_t n, int to_mont) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = ld_fr(data + i);
    st_fr(data + i, to_mont ? fr_from_canonical(v) : fr_to_canonical(v));
}

// EvaluationDomain's O(n) methods as stand-alone operations (inside create_proof they are fused
// into the transforms, see h_poly_device): op 0 mul_assign a*=b (domain.rs:154-170), 1 sub_assign
// a-=b (:173-189), 2 scale a*=k (divide_by_z_on_coset :139-151, ifft's m^-1 :88-98),
// 3 distribute_powers a[i]*=k^i (:101-113)
__global__ void __launch_bounds__(256) k_domain_pointwise(Fr* a, const Fr* b, size_t n, int op, Fr k) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr x = ld_fr(a + i);
    if (op == 0) x = x * ld_fr(b + i);
    else if (op == 1) x = x - ld_fr(b + i);
    else if (op == 2) x = x * k;
    else x = x * k.pow_u64((uint64_t)i, fr_one());
    st_fr(a + i, x);
}

struct PassArgs {
    const Fr* src;
    Fr* dst;
    const Fr* src_b;       // fused a*b-c at the gather (first pass of the H transform)
    const Fr* src_c;
    const Fr* tw;
    const Fr* pre;         // indexed by source (natural) index, first pass
    const Fr* post;        // indexed by output index, last pass
    Fr post_const;
    int use_post_const;
    int bitrev;
    uint32_t log_n, s0, k, cbits, lowbits;
    size_t poly_stride;    // grid y = polynomial: src, dst, src_b and src_c of polynomial y start y * poly_stride further
};

__global__ void __launch_bounds__(256) k_ntt_pass(PassArgs A) {
    extern __shared__ uint32_t sm[];
    const size_t poff = (size_t)blockIdx.y * A.poly_stride;
    const Fr* const src = A.src + poff;
    Fr* const dst = A.dst + poff;
    const Fr* const src_b = A.src_b ? A.src_b + poff : nullptr;
    const Fr* const src_c = A.src_b ? A.src_c + poff : nullptr;
    const uint32_t T = 1u << (A.k + A.cbits);
    const uint32_t C = 1u << A.cbits;
    const uint32_t hibits = A.cbits - A.lowbits;
    const uint32_t blo_bits = A.s0 - A.lowbits;
    const uint32_t B_lo = blockIdx.x & ((1u << blo_bits) - 1u);
    const uint32_t B_hi = blockIdx.x >> blo_bits;
    const uint32_t base_addr = (B_lo << A.lowbits) | (B_hi << (A.s0 + A.k + hibits));
    const uint32_t lowmask = (1u << A.lowbits) - 1u;
    auto addr = [&](uint32_t e) -> uint32_t {
        uint32_t c = e & (C - 1u), r = e >> A.cbits;
        return base_addr | (c & lowmask) | (r << A.s0) | ((c >> A.lowbits) << (A.s0 + A.k));
    };
    for (uint32_t e = threadIdx.x; e < T; e += blockDim.x) {
        uint32_t p = addr(e);
        uint32_t i = A.bitrev ? (__brev(p) >> (32u - A.log_n)) : p;
        Fr v = ld_fr(src + i);
        if (src_b) v = v * ld_fr(src_b + i) - ld_fr(src_c + i);
        if (A.pre) v = v * ld_fr(A.pre + i);
#pragma unroll
        for (int w = 0; w < 8; w++) sm[w * T + e] = v.l[w];
    }
    __syncthreads();
    for (uint32_t t = 0; t < A.k; t++) {
        const uint32_t s = A.s0 + t;
        for (uint32_t q = threadIdx.x; q < T / 2; q += blockDim.x) {
            uint32_t c = q & (C - 1u), rr = q >> A.cbits;
            uint32_t r0 = ((rr >> t) << (t + 1)) | (rr & ((1u << t) - 1u));
            uint32_t e0 = r0 * C + c, e1 = e0 + (C << t);
            Fr x, y;
#pragma unroll
            for (int w = 0; w < 8; w++) { x.l[w] = sm[w * T + e0]; y.l[w] = sm[w * T + e1]; }
            if (s != 0) {
                uint32_t j = addr(e0) & ((1u << s) - 1u);
                Fr wv = ld_fr(A.tw + ((size_t)j << (A.log_n - s - 1u)));
                y = y * wv;
            }
            Fr u = x + y, d = x - y;
#pragma unroll
            for (int w = 0; w < 8; w++) { sm[w * T + e0] = u.l[w]; sm[w * T + e1] = d.l[w]; }
        }
        __syncthreads();
    }
    for (uint32_t e = threadIdx.x; e < T; e += blockDim.x) {
        uint32_t p = addr(e);
        Fr v;
#pragma unroll
        for (int w = 0; w < 8; w++) v.l[w] = sm[w * T + e];
        if (A.post) v = v * ld_fr(A.post + p);
        if (A.use_post_const) v = v * A.post_const;
        st_fr(dst + p, v);
    }
}

static Fr h_pow(const Fr& b, uint64_t e) { return b.pow_u64(e, fr_one()); }

struct DomainConsts { Fr omega, omegainv, g, ginv, minv, zinv; };

static DomainConsts domain_consts(uint32_t log_n) {
    DomainConsts d;
    Fr omega = fr_root_of_unity();                  // domain.rs:63-66
    for (uint32_t i = log_n; i < (uint32_t)bbc::FR_S; i++) omega = omega.sqr();
    d.omega = omega;
    d.omegainv = fr_inv(omega);                     // :75
    d.g = fr_generator();
    d.ginv = fr_inv(d.g);                           // :76
    d.minv = fr_inv(fr_from_u64(1ull << log_n));    // :77
    Fr z = h_pow(d.g, 1ull << log_n) - fr_one();    // z(g) = g^m - 1, :129-134
    d.zinv = fr_inv(z);                             // :140
    return d;
}

enum TableKind { T_TW_FWD, T_TW_INV, T_POW_G, T_POW_GINV_MINV, T_POW_G_MINV, T_POW_GINV_MINV_ZINV };

static int get_table(bb_ctx* ctx, cudaStream_t st, uint32_t log_n, TableKind kind, NttTables** tabs, const Fr** out) {
    std::lock_guard<std::mutex> g(ctx->mu);
    NttTables*& t = ctx->ntt_tables[log_n];
    if (!t) { t = new NttTables(); t->log_n = log_n; t->minv = domain_consts(log_n).minv; }
    *tabs = t;
    size_t n = (size_t)1 << log_n;
    size_t half = n / 2 ? n / 2 : 1;
    Fr** slot = nullptr;
    switch (kind) {
        case T_TW_FWD: slot = &t->tw_fwd; break;
        case T_TW_INV: slot = &t->tw_inv; break;
        case T_POW_G: slot = &t->pow_g; break;
        case T_POW_GINV_MINV: slot = &t->pow_ginv_minv; break;
        case T_POW_G_MINV: slot = &t->pow_g_minv; break;
        case T_POW_GINV_MINV_ZINV: slot = &t->pow_ginv_minv_zinv; break;
    }
    if (!*slot) {
        DomainConsts d = domain_consts(log_n);
        // allocation must not take ctx->mu again: use raw cudaMalloc for long-lived tables
        size_t cnt = (kind == T_TW_FWD || kind == T_TW_INV) ? half : n;
        Fr* p = nullptr;
        BB_CUDA(cudaMalloc(&p, cnt * sizeof(Fr)));
        Fr base, scale = fr_one();
        switch (kind) {
            case T_TW_FWD: base = d.omega; break;
            case T_TW_INV: base = d.omegainv; break;
            case T_POW_G: base = d.g; break;
            case T_POW_GINV_MINV: base = d.ginv; scale = d.minv; break;
            case T_POW_G_MINV: base = d.g; scale = d.minv; break;
            case T_POW_GINV_MINV_ZINV: base = d.ginv; scale = d.minv * d.zinv; break;
        }
        size_t threads = (cnt + 31) / 32;
        k_powers<<<cdiv(threads, 256), 256, 0, st>>>(p, cnt, base, scale);
        ctx->count_launch();
        BB_CUDA(cudaGetLastError());
        // tables are shared by later calls on other streams: make them visible first
        BB_CUDA(cudaStreamSynchronize(st));
        *slot = p;
    }
    *out = *slot;
    return BB_OK;
}

struct Fusion {
    const Fr* src_b = nullptr;
    const Fr* src_c = nullptr;
    const Fr* pre = nullptr;
    const Fr* post = nullptr;
    bool post_const = false;
    Fr post_const_v;
};

// One transform: data (natural order) -> data, scratch tmp of the same size.  polys > 1: the same transform of `polys`
// polynomials at src, data, tmp (and the fused src_b, src_c) + j * stride, j < polys, in the same launches (grid y).
static int run_passes(bb_ctx* ctx, cudaStream_t st, const Fr* src, Fr* data, Fr* tmp, uint32_t log_n,
                      const Fr* tw, const Fusion& fu, uint32_t polys = 1, size_t stride = 0) {
    if (log_n == 0) {
        // single point: only the fused multiplications apply
        PassArgs A{};
        A.src = src; A.dst = data; A.src_b = fu.src_b; A.src_c = fu.src_c; A.tw = tw; A.pre = fu.pre; A.post = fu.post;
        A.use_post_const = fu.post_const; A.post_const = fu.post_const_v; A.bitrev = 0;
        A.log_n = 0; A.s0 = 0; A.k = 0; A.cbits = 0; A.lowbits = 0;
        A.poly_stride = stride;
        k_ntt_pass<<<dim3(1, polys), 32, 32, st>>>(A);
        ctx->count_launch();
        BB_CUDA(cudaGetLastError());
        return BB_OK;
    }
    uint32_t tile_log = (uint32_t)ctx->opt_ntt_tile_log, col_bits = (uint32_t)ctx->opt_ntt_col_bits;
    if (tile_log < 2 || tile_log > 12 || col_bits >= tile_log) { tile_log = 11; col_bits = 3; }
    uint32_t kmax = tile_log - col_bits;
    uint32_t npass = (log_n + kmax - 1) / kmax;
    uint32_t s0 = 0;
    for (uint32_t pi = 0; pi < npass; pi++) {
        // spread the stages evenly over the passes
        uint32_t k = (log_n - s0 + (npass - pi) - 1) / (npass - pi);
        uint32_t cbits = col_bits < log_n - k ? col_bits : log_n - k;
        PassArgs A{};
        bool first = pi == 0, last = pi + 1 == npass;
        A.src = first ? src : (const Fr*)tmp;
        A.dst = last ? data : tmp;
        if (first && last) A.dst = tmp;          // a gather cannot run in place
        A.src_b = first ? fu.src_b : nullptr;
        A.src_c = first ? fu.src_c : nullptr;
        A.pre = first ? fu.pre : nullptr;
        A.post = last ? fu.post : nullptr;
        A.use_post_const = last && fu.post_const;
        A.post_const = fu.post_const_v;
        A.tw = tw;
        A.bitrev = first;
        A.log_n = log_n; A.s0 = s0; A.k = k; A.cbits = cbits;
        A.lowbits = s0 < cbits ? s0 : cbits;
        A.poly_stride = stride;
        size_t smem = ((size_t)32) << (k + cbits);
        if (smem > 48 * 1024) BB_CUDA(cudaFuncSetAttribute(k_ntt_pass, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const dim3 grid(1u << (log_n - k - cbits), polys);
        unsigned threads = (1u << (k + cbits)) / 2 < 256 ? ((1u << (k + cbits)) / 2 < 32 ? 32 : (1u << (k + cbits)) / 2) : 256;
        k_ntt_pass<<<grid, threads, smem, st>>>(A);
        ctx->count_launch();
        BB_CUDA(cudaGetLastError());
        s0 += k;
    }
    if (npass == 1) {
        if (polys == 1) BB_CUDA(cudaMemcpyAsync(data, tmp, sizeof(Fr) << log_n, cudaMemcpyDeviceToDevice, st));
        else BB_CUDA(cudaMemcpy2DAsync(data, stride * sizeof(Fr), tmp, stride * sizeof(Fr), sizeof(Fr) << log_n, polys, cudaMemcpyDeviceToDevice, st));
    }
    return BB_OK;
}

int ntt_run_device(bb_ctx* ctx, cudaStream_t st, Fr* d_data, Fr* d_tmp, uint32_t log_n, int mode) {
    if (log_n >= (uint32_t)bbc::FR_S) { set_error("2^%u-point domain: PolynomialDegreeTooLarge", log_n); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    NttTables* t = nullptr;
    const Fr* tw = nullptr;
    Fusion fu;
    switch (mode) {
        case BB_NTT_FFT:
            BB_TRY(get_table(ctx, st, log_n, T_TW_FWD, &t, &tw));
            break;
        case BB_NTT_IFFT:
            BB_TRY(get_table(ctx, st, log_n, T_TW_INV, &t, &tw));
            fu.post_const = true; fu.post_const_v = t->minv;
            break;
        case BB_NTT_COSET_FFT:
            BB_TRY(get_table(ctx, st, log_n, T_TW_FWD, &t, &tw));
            BB_TRY(get_table(ctx, st, log_n, T_POW_G, &t, &fu.pre));
            break;
        case BB_NTT_ICOSET_FFT:
            BB_TRY(get_table(ctx, st, log_n, T_TW_INV, &t, &tw));
            BB_TRY(get_table(ctx, st, log_n, T_POW_GINV_MINV, &t, &fu.post));
            break;
        default:
            set_error("bad ntt mode %d", mode);
            return BB_ERR_ARG;
    }
    return run_passes(ctx, st, d_data, d_data, d_tmp, log_n, tw, fu);
}

// prover.rs:225-237 on device buffers of m = 2^log_m elements (already zero padded).
// Result (m coefficients, Montgomery) is left in d_a; d_b, d_c are clobbered.
int h_poly_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, Fr* d_b, Fr* d_c, Fr* d_tmp, uint32_t log_m) {
    if (log_m >= (uint32_t)bbc::FR_S) { set_error("2^%u-point domain: PolynomialDegreeTooLarge", log_m); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    NttTables* t = nullptr;
    const Fr *tw_f = nullptr, *tw_i = nullptr, *gm = nullptr, *gz = nullptr;
    BB_TRY(get_table(ctx, st, log_m, T_TW_FWD, &t, &tw_f));
    BB_TRY(get_table(ctx, st, log_m, T_TW_INV, &t, &tw_i));
    BB_TRY(get_table(ctx, st, log_m, T_POW_G_MINV, &t, &gm));
    BB_TRY(get_table(ctx, st, log_m, T_POW_GINV_MINV_ZINV, &t, &gz));
    Fr* polys[3] = {d_a, d_b, d_c};
    for (Fr* p : polys) {
        Fusion inv;                     // ifft (:225,227,229) with the coset shift of :226,228,230 fused in
        inv.post = gm;
        BB_TRY(run_passes(ctx, st, p, p, d_tmp, log_m, tw_i, inv));
        Fusion fwd;                     // the fft half of coset_fft
        BB_TRY(run_passes(ctx, st, p, p, d_tmp, log_m, tw_f, fwd));
    }
    Fusion fin;                         // mul_assign, sub_assign, divide_by_z_on_coset, icoset_fft (:232-237)
    fin.src_b = d_b; fin.src_c = d_c; fin.post = gz;
    return run_passes(ctx, st, d_a, d_a, d_tmp, log_m, tw_i, fin);
}

// h_poly_device for B proofs in the same launches: d_abc holds a_0 .. a_{B-1}, b_0 .. b_{B-1}, c_0 .. c_{B-1}, m = 2^log_m
// elements each (zero padded); d_tmp the same 3 B m.  The 3 B inverse and forward transforms run as one pass sequence
// each, the final transform as one over the B products: 3 pass sequences per sub-batch.  h_j is left in a_j.
int h_poly_batch_device(bb_ctx* ctx, cudaStream_t st, Fr* d_abc, Fr* d_tmp, uint32_t log_m, uint32_t B) {
    if (log_m >= (uint32_t)bbc::FR_S) { set_error("2^%u-point domain: PolynomialDegreeTooLarge", log_m); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    NttTables* t = nullptr;
    const Fr *tw_f = nullptr, *tw_i = nullptr, *gm = nullptr, *gz = nullptr;
    BB_TRY(get_table(ctx, st, log_m, T_TW_FWD, &t, &tw_f));
    BB_TRY(get_table(ctx, st, log_m, T_TW_INV, &t, &tw_i));
    BB_TRY(get_table(ctx, st, log_m, T_POW_G_MINV, &t, &gm));
    BB_TRY(get_table(ctx, st, log_m, T_POW_GINV_MINV_ZINV, &t, &gz));
    const size_t m = (size_t)1 << log_m;
    Fusion inv;                         // ifft with the coset shift fused (:225-230), all 3 B polynomials
    inv.post = gm;
    BB_TRY(run_passes(ctx, st, d_abc, d_abc, d_tmp, log_m, tw_i, inv, 3 * B, m));
    Fusion fwd;                         // the fft half of coset_fft
    BB_TRY(run_passes(ctx, st, d_abc, d_abc, d_tmp, log_m, tw_f, fwd, 3 * B, m));
    Fusion fin;                         // a*b - c, divide_by_z_on_coset, icoset_fft (:232-237), B polynomials
    fin.src_b = d_abc + (size_t)B * m; fin.src_c = d_abc + 2 * (size_t)B * m; fin.post = gz;
    return run_passes(ctx, st, d_abc, d_abc, d_tmp, log_m, tw_i, fin, B, m);
}

// The two halves of h_poly_device for the multi-GPU split by polynomial: the coset evaluations of one
// polynomial (ifft with the coset shift fused, then fft) ...
int h_poly_evals_device(bb_ctx* ctx, cudaStream_t st, Fr* d_p, Fr* d_tmp, uint32_t log_m) {
    if (log_m >= (uint32_t)bbc::FR_S) { set_error("2^%u-point domain: PolynomialDegreeTooLarge", log_m); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    NttTables* t = nullptr;
    const Fr *tw_f = nullptr, *tw_i = nullptr, *gm = nullptr;
    BB_TRY(get_table(ctx, st, log_m, T_TW_FWD, &t, &tw_f));
    BB_TRY(get_table(ctx, st, log_m, T_TW_INV, &t, &tw_i));
    BB_TRY(get_table(ctx, st, log_m, T_POW_G_MINV, &t, &gm));
    Fusion inv;
    inv.post = gm;
    BB_TRY(run_passes(ctx, st, d_p, d_p, d_tmp, log_m, tw_i, inv));
    Fusion fwd;
    return run_passes(ctx, st, d_p, d_p, d_tmp, log_m, tw_f, fwd);
}
// ... and the last transform over three evaluation vectors (result in d_a)
int h_poly_final_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, const Fr* d_b, const Fr* d_c, Fr* d_tmp, uint32_t log_m) {
    if (log_m >= (uint32_t)bbc::FR_S) { set_error("2^%u-point domain: PolynomialDegreeTooLarge", log_m); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    NttTables* t = nullptr;
    const Fr *tw_i = nullptr, *gz = nullptr;
    BB_TRY(get_table(ctx, st, log_m, T_TW_INV, &t, &tw_i));
    BB_TRY(get_table(ctx, st, log_m, T_POW_GINV_MINV_ZINV, &t, &gz));
    Fusion fin;
    fin.src_b = d_b; fin.src_c = d_c; fin.post = gz;
    return run_passes(ctx, st, d_a, d_a, d_tmp, log_m, tw_i, fin);
}

int domain_pointwise_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, const Fr* d_b, size_t n, int op, const Fr& k) {
    if (!n) return BB_OK;
    k_domain_pointwise<<<cdiv(n, 256), 256, 0, st>>>(d_a, d_b, n, op, k);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

int powers_device(bb_ctx* ctx, cudaStream_t st, Fr* d_out, size_t n, const Fr& base, const Fr& scale) {
    if (!n) return BB_OK;
    const size_t threads = (n + 31) / 32;
    k_powers<<<cdiv(threads, 256), 256, 0, st>>>(d_out, n, base, scale);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

void ntt_free_tables(bb_ctx* ctx) {
    for (auto& kv : ctx->ntt_tables) {
        NttTables* t = kv.second;
        if (!t) continue;
        Fr* ptrs[] = {t->tw_fwd, t->tw_inv, t->pow_g, t->pow_ginv_minv, t->pow_g_minv, t->pow_ginv_minv_zinv};
        for (Fr* p : ptrs) if (p) cudaFree(p);
        delete t;
    }
    ctx->ntt_tables.clear();
}

int fr_convert_device(bb_ctx* ctx, cudaStream_t st, Fr* d_data, size_t n, bool to_montgomery) {
    if (!n) return BB_OK;
    k_fr_convert<<<cdiv(n, 256), 256, 0, st>>>(d_data, n, to_montgomery ? 1 : 0);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

}  // namespace bb
