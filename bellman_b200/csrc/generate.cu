// bellman_b200: groth16::generate_parameters / generate_random_parameters on the device (bellman/groth16/src/generator.rs:
// 21-40, 159-507) from a resident constraint system.  The per-variable (coefficient, constraint) lists KeypairAssembly
// records (generator.rs:43-155) are the columns of the bb_r1cs matrices (r1cs.cu), so the key comes from what is already
// in HBM; only the toxic waste crosses the bus, and only the key's points stay behind.
//
// Pipeline, on the main stream (DESIGN.md 4.11):
//   transpose  the CSR of 3 n rows by constraint becomes 3 nv columns by variable (nv = n_inputs + n_aux): the terms per
//              column (k_gen_col_count), an exclusive scan (k_scan_tiles / k_scan_add), a scatter keeping the one-flag and
//              the coefficient (k_gen_col_scatter), the columns binned by length (k_gen_bin_count / k_gen_bin_scatter).
//              Built per call and freed after it: bb_r1cs_create and the resident constraint system are unchanged.
//   lagrange   the m powers of tau (k_powers), the h scalars tau^i t(tau) / delta (the domain's scale), L = ifft(powers)
//   qap        at, bt, ct = the transposed matrix times L: r1cs.cu's row kernels run it unchanged (a column is their row,
//              L their witness); k_gen_combine gives the ic / l scalars, the unconstrained check and the non-zero flags of at
//              and bt, which an order-preserving compaction (scan, k_gen_compact) turns into the a and b scalars
//   g1, g2     fixed-base multiplications written straight into the buffers the resident key adopts
// Field additions are exact, so the order in which the scatter's atomics lay out a column's terms changes nothing: the key
// does not depend on grid shapes.
#include <sys/random.h>

#include <cstring>
#include <deque>

#include "bb_internal.cuh"
#include "encoding.cuh"

using namespace bb;

namespace {

constexpr uint32_t ONE_FLAG = R1CS_ONE_FLAG;
constexpr unsigned SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// the row holding term t: off[row] <= t < off[row + 1] (off non-decreasing from 0, t < off[rows])
__device__ __forceinline__ uint32_t term_row(const uint32_t* off, uint32_t rows, uint32_t t) {
    uint32_t lo = 0, hi = rows;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (off[mid] <= t) lo = mid;
        else hi = mid;
    }
    return lo;
}

// column of a term in row g: matrix (g / n) times nv, plus its variable
__device__ __forceinline__ uint32_t term_col(uint32_t g, uint32_t v, uint32_t n, uint32_t nv) { return (g / n) * nv + (v & ~ONE_FLAG); }

__global__ void __launch_bounds__(256) k_gen_col_count(const uint32_t* __restrict__ off, const uint32_t* __restrict__ idx, uint32_t rows,
                                                       uint32_t terms, uint32_t n, uint32_t nv, uint32_t* cnt) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= terms) return;
    atomicAdd(&cnt[term_col(term_row(off, rows, (uint32_t)t), idx[t], n, nv)], 1u);
}

// term t goes to the next free slot of its column; its row becomes the column's index into L
__global__ void __launch_bounds__(256) k_gen_col_scatter(const uint32_t* __restrict__ off, const uint32_t* __restrict__ idx,
                                                         const Fr* __restrict__ coef, uint32_t rows, uint32_t terms, uint32_t n, uint32_t nv,
                                                         uint32_t* cursor, uint32_t* t_idx, Fr* t_coef) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= terms) return;
    const uint32_t g = term_row(off, rows, (uint32_t)t), v = idx[t];
    const uint32_t pos = atomicAdd(&cursor[term_col(g, v, n, nv)], 1u);
    t_idx[pos] = (g % n) | (v & ONE_FLAG);
    t_coef[pos] = coef[t];
}

// exclusive scan of data[0 .. n) in place, one tile of SCAN_TILE words per block: each thread sums SCAN_ITEMS consecutive
// words, a block-wide scan of those sums in shared memory, then every word gets its prefix; sums[block] = the tile total
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(uint32_t* data, size_t n, uint32_t* sums) {
    __shared__ uint32_t sh[SCAN_THREADS];
    const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], s = 0;
    for (unsigned k = 0; k < SCAN_ITEMS; k++) {
        v[k] = base + k < n ? data[base + k] : 0u;
        s += v[k];
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (unsigned d = 1; d < SCAN_THREADS; d <<= 1) {
        const uint32_t x = threadIdx.x >= d ? sh[threadIdx.x - d] : 0u;
        __syncthreads();
        sh[threadIdx.x] += x;
        __syncthreads();
    }
    uint32_t run = sh[threadIdx.x] - s;
    for (unsigned k = 0; k < SCAN_ITEMS; k++) {
        if (base + k < n) data[base + k] = run;
        run += v[k];
    }
    if (threadIdx.x == SCAN_THREADS - 1) sums[blockIdx.x] = sh[threadIdx.x];
}

__global__ void __launch_bounds__(256) k_scan_add(uint32_t* data, size_t n, const uint32_t* __restrict__ tile_prefix) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    data[i] += tile_prefix[i / SCAN_TILE];
}

__device__ __forceinline__ uint32_t col_bin(uint32_t len) { return len <= R1CS_SHORT_MAX ? 0u : len <= R1CS_WARP_MAX ? 1u : 2u; }

__global__ void __launch_bounds__(256) k_gen_bin_count(const uint32_t* __restrict__ col_off, uint32_t cols, uint32_t* bins) {
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    atomicAdd(&bins[col_bin(col_off[c + 1] - col_off[c])], 1u);
}

__global__ void __launch_bounds__(256) k_gen_bin_scatter(const uint32_t* __restrict__ col_off, uint32_t cols, uint32_t* cursor, uint32_t* rows) {
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    rows[atomicAdd(&cursor[col_bin(col_off[c + 1] - col_off[c])], 1u)] = (uint32_t)c;
}

// per variable j (generator.rs:391-415): ext_j = (beta at_j + alpha bt_j + ct_j) inv, inv = 1/gamma for inputs and 1/delta
// for aux; fa_j, fb_j = at_j, bt_j non-zero; the first aux variable whose ext is zero (l's identity, :464-470) in *first_unc
__global__ void __launch_bounds__(256) k_gen_combine(const Fr* __restrict__ at, const Fr* __restrict__ bt, const Fr* __restrict__ ct, uint32_t nv,
                                                     uint32_t ni, Fr alpha, Fr beta, Fr gamma_inv, Fr delta_inv, Fr* ext, uint32_t* fa,
                                                     uint32_t* fb, uint32_t* first_unc) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    const Fr a = at[j], b = bt[j];
    const Fr e = (beta * a + alpha * b + ct[j]) * (j < ni ? gamma_inv : delta_inv);
    ext[j] = e;
    fa[j] = a.is_zero() ? 0u : 1u;
    fb[j] = b.is_zero() ? 0u : 1u;
    if (j >= ni && e.is_zero()) atomicMin(first_unc, (uint32_t)(j - ni));
}

// order-preserving compaction (generator.rs:491-505): pos = the exclusive scan of the non-zero flags
__global__ void __launch_bounds__(256) k_gen_compact(const Fr* __restrict__ v, const uint32_t* __restrict__ pos, uint32_t nv, Fr* out) {
    const size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nv) return;
    if (pos[j + 1] != pos[j]) out[pos[j]] = v[j];
}

// exclusive scan of n words in place; the tile sums live in `keep` until the caller has drained the stream
int scan_exclusive(bb_ctx* ctx, cudaStream_t st, uint32_t* data, size_t n, std::deque<DevBuf>& keep) {
    if (!n) return BB_OK;
    const size_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    DevBuf& sums = keep.emplace_back();
    BB_TRY(sums.alloc(ctx, tiles * 4));
    k_scan_tiles<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(data, n, sums.as<uint32_t>());
    ctx->count_launch();
    if (tiles > 1) {
        BB_TRY(scan_exclusive(ctx, st, sums.as<uint32_t>(), tiles, keep));
        k_scan_add<<<cdiv(n, 256), 256, 0, st>>>(data, n, sums.as<uint32_t>());
        ctx->count_launch();
    }
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

void wipe(void* p, size_t n) {
    volatile uint8_t* q = (volatile uint8_t*)p;
    while (n--) *q++ = 0;
}

// device blocks that hold scalars derived from the toxic waste: zeroed (and the stream drained) before their DevBufs return
// them to the context's cache -- declare after the DevBufs it covers
struct Scrub {
    cudaStream_t st;
    std::vector<std::pair<void*, size_t>> blocks;
    explicit Scrub(cudaStream_t s) : st(s) {}
    void add(const DevBuf& b, size_t bytes) { if (b.p && bytes) blocks.emplace_back(b.p, bytes); }
    ~Scrub() {
        for (auto& b : blocks) cudaMemsetAsync(b.first, 0, b.second, st);
        cudaStreamSynchronize(st);
    }
};

// the toxic waste and what the host derives from it, wiped on every return
struct Secrets {
    Fr alpha, beta, gamma, delta, tau, gamma_inv, delta_inv, h_scale;
    Fr vk[6];                                     // alpha, beta, delta (G1) and delta, gamma, beta (G2), Montgomery
    Fr g1s, g2s;                                  // generate_random_parameters: the generators' multiples
    G1Affine g1;
    G2Affine g2;
    ~Secrets() { wipe(this, sizeof *this); }
};

bool fr_below_r(const Fr& v) {
    for (int i = 7; i >= 0; i--) {
        if (v.l[i] != bbc::FR_MOD[i]) return v.l[i] < bbc::FR_MOD[i];
    }
    return false;
}

// the checks the reference's types guarantee for a generator: a non-identity point of order r on the curve
template <class F>
const char* bad_generator(const Affine<F>& p) {
    if (!is_canonical(p.x) || !is_canonical(p.y)) return "a coordinate is not below p";
    if (p.is_identity()) return "the identity";
    if (!on_curve(p)) return "not on the curve";
    if (!rP_is_identity(p)) return "not in the prime-order subgroup";
    return nullptr;
}

// a uniform non-zero scalar below r (generate_random_parameters' Fr::random, redrawn at zero as the batch verifier's z)
int draw_scalar(Fr* v) {
    do {
        uint8_t buf[32];
        size_t got = 0;
        while (got < sizeof buf) {
            const ssize_t k = getrandom(buf + got, sizeof buf - got, 0);
            if (k < 0) { set_error("bb_groth16_generate: getrandom failed"); return BB_ERR_ARG; }
            got += (size_t)k;
        }
        buf[31] &= 0x7f;
        std::memcpy(v->l, buf, 32);
        wipe(buf, sizeof buf);
    } while (v->is_zero() || !fr_below_r(*v));
    return BB_OK;
}

bb_bases* adopt_bases(bb_ctx* ctx, int group, DevBuf& buf, size_t n) {
    bb_bases* b = new bb_bases();
    b->ctx = ctx; b->group = group; b->n = n; b->global_offset = 0; b->global_len = n;
    b->d_points = buf.take();
    return b;
}

struct TableGuard {                                // a per-call fixed-base table, zeroed and freed with the call
    int group;
    void* d = nullptr;
    explicit TableGuard(int g) : group(g) {}
    ~TableGuard() { fixed_table_free(group, d); }
};

}  // namespace

extern "C" {

int bb_groth16_generate(bb_ctx* ctx, const bb_r1cs* r1cs, const bb_toxic* toxic, bb_crs** crs_out, bb_vk** vk_out,
                        bb_generate_report* report) {
    if (crs_out) *crs_out = nullptr;
    if (vk_out) *vk_out = nullptr;
    bb_generate_report rep{};
    rep.unconstrained = SIZE_MAX;
    if (report) *report = rep;
    if (!ctx || !r1cs || !crs_out) { set_error("bb_groth16_generate: null argument"); return BB_ERR_ARG; }
    const R1csView R = r1cs_view(r1cs);
    if (R.ctx != ctx) { set_error("bb_groth16_generate: the constraint system lives on another context"); return BB_ERR_ARG; }
    const size_t ni = R.n_inputs, nv = R.n_inputs + R.n_aux, n = R.n;
    if (3 * (uint64_t)nv + 1 >= ((uint64_t)1 << 32)) { set_error("bb_groth16_generate: %zu variables: at most (2^32 - 2) / 3", nv); return BB_ERR_ARG; }
    size_t m = 1;
    uint32_t log_m = 0;
    while (m < n) { m <<= 1; log_m++; }                           // EvaluationDomain::from_coeffs (domain.rs:48-70)
    if (log_m >= (uint32_t)bbc::FR_S) { set_error("bb_groth16_generate: PolynomialDegreeTooLarge"); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }

    Secrets S;
    const bool own_g1 = !toxic || toxic->g1, own_g2 = !toxic || toxic->g2;
    if (toxic) {
        Fr* dst[5] = {&S.alpha, &S.beta, &S.gamma, &S.delta, &S.tau};
        const uint8_t* src[5] = {toxic->alpha, toxic->beta, toxic->gamma, toxic->delta, toxic->tau};
        static const char* const name[5] = {"alpha", "beta", "gamma", "delta", "tau"};
        for (int k = 0; k < 5; k++) {
            std::memcpy(dst[k]->l, src[k], 32);
            if (!fr_below_r(*dst[k])) { set_error("bb_groth16_generate: %s is not below r", name[k]); return BB_ERR_ARG; }
        }
        if (toxic->g1) {
            std::memcpy(&S.g1, toxic->g1, sizeof S.g1);
            if (const char* why = bad_generator(S.g1)) { set_error("bb_groth16_generate: g1 is %s", why); return BB_ERR_ARG; }
        }
        if (toxic->g2) {
            std::memcpy(&S.g2, toxic->g2, sizeof S.g2);
            if (const char* why = bad_generator(S.g2)) { set_error("bb_groth16_generate: g2 is %s", why); return BB_ERR_ARG; }
        }
    } else {                                                      // generate_random_parameters (generator.rs:21-40)
        for (Fr* v : {&S.g1s, &S.g2s, &S.alpha, &S.beta, &S.gamma, &S.delta, &S.tau}) BB_TRY(draw_scalar(v));
        S.g1 = XYZZ<Fp>::from_affine(g1_generator()).mul_bits(S.g1s.l).to_affine();
        S.g2 = XYZZ<Fp2>::from_affine(g2_generator()).mul_bits(S.g2s.l).to_affine();
    }
    if (S.gamma.is_zero()) { set_error("bb_groth16_generate: gamma is zero (UnexpectedIdentity)"); return BB_ERR_UNEXPECTED_IDENTITY; }
    if (S.delta.is_zero()) { set_error("bb_groth16_generate: delta is zero (UnexpectedIdentity)"); return BB_ERR_UNEXPECTED_IDENTITY; }
    for (Fr* v : {&S.alpha, &S.beta, &S.gamma, &S.delta, &S.tau}) *v = fr_from_canonical(*v);
    S.gamma_inv = fr_inv(S.gamma);
    S.delta_inv = fr_inv(S.delta);
    S.h_scale = (S.tau.pow_u64(m, fr_one()) - fr_one()) * S.delta_inv;     // t(tau) / delta (generator.rs:266-268)
    S.vk[0] = S.alpha; S.vk[1] = S.beta; S.vk[2] = S.delta;
    S.vk[3] = S.delta; S.vk[4] = S.gamma; S.vk[5] = S.beta;

    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("groth16_generate");
    TableGuard tab1(BB_G1), tab2(BB_G2);
    if (own_g1) BB_TRY(fixed_table_build(BB_G1, &S.g1, &tab1.d));
    if (own_g2) BB_TRY(fixed_table_build(BB_G2, &S.g2, &tab2.d));

    cudaStream_t st = ctx->main_stream;
    const uint32_t rows = (uint32_t)(3 * n), cols = (uint32_t)(3 * nv), terms = (uint32_t)R.terms;
    DevBuf d_col_off, d_cursor, d_tidx, d_tcoef, d_bins, d_order;                  // the transposed matrix (public)
    DevBuf d_pow, d_tmp, d_hq, d_abc, d_ext, d_fa, d_fb, d_unc, d_asc, d_bsc, d_vks;   // scalars derived from the toxic waste
    DevBuf d_h, d_ic, d_l, d_a, d_b1, d_b2, d_vk1, d_g2, d_alpha;                  // the key
    std::deque<DevBuf> keep;
    StageTimer tm(ctx, st);
    tm.mark("generate.begin");

    // transpose: 3 n rows by constraint -> 3 nv columns by variable
    BB_TRY(d_col_off.alloc(ctx, ((size_t)cols + 1) * 4));
    BB_TRY(d_cursor.alloc(ctx, ((size_t)cols + 1) * 4));
    BB_TRY(d_tidx.alloc(ctx, (size_t)terms * 4));
    BB_TRY(d_tcoef.alloc(ctx, (size_t)terms * sizeof(Fr)));
    BB_TRY(d_bins.alloc(ctx, 3 * 4));
    BB_TRY(d_order.alloc(ctx, (size_t)cols * 4));
    uint32_t* col_off = d_col_off.as<uint32_t>();
    BB_CUDA(cudaMemsetAsync(col_off, 0, ((size_t)cols + 1) * 4, st));
    BB_CUDA(cudaMemsetAsync(d_bins.p, 0, 3 * 4, st));
    if (terms) {
        k_gen_col_count<<<cdiv(terms, 256), 256, 0, st>>>(R.off, R.idx, rows, terms, (uint32_t)n, (uint32_t)nv, col_off);
        ctx->count_launch();
    }
    BB_TRY(scan_exclusive(ctx, st, col_off, (size_t)cols + 1, keep));
    BB_CUDA(cudaMemcpyAsync(d_cursor.p, col_off, ((size_t)cols + 1) * 4, cudaMemcpyDeviceToDevice, st));
    if (terms) {
        k_gen_col_scatter<<<cdiv(terms, 256), 256, 0, st>>>(R.off, R.idx, R.coef, rows, terms, (uint32_t)n, (uint32_t)nv, d_cursor.as<uint32_t>(),
                                                            d_tidx.as<uint32_t>(), d_tcoef.as<Fr>());
        ctx->count_launch();
    }
    if (cols) {
        k_gen_bin_count<<<cdiv(cols, 256), 256, 0, st>>>(col_off, cols, d_bins.as<uint32_t>());
        ctx->count_launch();
    }
    uint32_t bins[3] = {0, 0, 0};
    BB_CUDA(cudaMemcpyAsync(bins, d_bins.p, sizeof bins, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    const uint32_t start[3] = {0, bins[0], bins[0] + bins[1]};
    BB_CUDA(cudaMemcpyAsync(d_bins.p, start, sizeof start, cudaMemcpyHostToDevice, st));
    if (cols) {
        k_gen_bin_scatter<<<cdiv(cols, 256), 256, 0, st>>>(col_off, cols, d_bins.as<uint32_t>(), d_order.as<uint32_t>());
        ctx->count_launch();
    }
    BB_CUDA(cudaGetLastError());
    tm.mark("generate.transpose");

    // lagrange: powers of tau (generator.rs:249-264), the h scalars (:266-296), L = ifft (:300)
    Scrub scrub(st);
    BB_TRY(d_pow.alloc(ctx, m * sizeof(Fr)));
    scrub.add(d_pow, m * sizeof(Fr));
    BB_TRY(d_tmp.alloc(ctx, m * sizeof(Fr)));
    scrub.add(d_tmp, m * sizeof(Fr));
    BB_TRY(d_hq.alloc(ctx, (m - 1) * sizeof(Fr)));
    scrub.add(d_hq, (m - 1) * sizeof(Fr));
    Fr* pw = d_pow.as<Fr>();
    BB_TRY(powers_device(ctx, st, pw, m, S.tau, fr_one()));
    if (m > 1) {
        BB_CUDA(cudaMemcpyAsync(d_hq.p, pw, (m - 1) * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
        BB_TRY(domain_pointwise_device(ctx, st, d_hq.as<Fr>(), nullptr, m - 1, 2, S.h_scale));
    }
    BB_TRY(ntt_run_device(ctx, st, pw, d_tmp.as<Fr>(), log_m, BB_NTT_IFFT));
    tm.mark("generate.lagrange");

    // qap: at, bt, ct (generator.rs:376-394), ext and the flags, then the compacted a and b scalars
    BB_TRY(d_abc.alloc(ctx, 3 * nv * sizeof(Fr)));
    scrub.add(d_abc, 3 * nv * sizeof(Fr));
    BB_TRY(d_ext.alloc(ctx, nv * sizeof(Fr)));
    scrub.add(d_ext, nv * sizeof(Fr));
    BB_TRY(d_fa.alloc(ctx, (nv + 1) * 4));
    scrub.add(d_fa, (nv + 1) * 4);
    BB_TRY(d_fb.alloc(ctx, (nv + 1) * 4));
    scrub.add(d_fb, (nv + 1) * 4);
    BB_TRY(d_unc.alloc(ctx, 4));
    Fr* abc = d_abc.as<Fr>();
    const CsrMatrix T{col_off, d_tidx.as<uint32_t>(), d_tcoef.as<Fr>(), d_order.as<uint32_t>(), bins[0], bins[1], bins[2], (uint32_t)nv};
    BB_TRY(csr_eval_queue(ctx, st, T, pw, 0xffffffffu, nullptr, abc, abc + nv, abc + 2 * nv));
    BB_CUDA(cudaMemsetAsync(d_fa.p, 0, (nv + 1) * 4, st));
    BB_CUDA(cudaMemsetAsync(d_fb.p, 0, (nv + 1) * 4, st));
    BB_CUDA(cudaMemsetAsync(d_unc.p, 0xff, 4, st));
    k_gen_combine<<<cdiv(nv, 256), 256, 0, st>>>(abc, abc + nv, abc + 2 * nv, (uint32_t)nv, (uint32_t)ni, S.alpha, S.beta, S.gamma_inv,
                                                 S.delta_inv, d_ext.as<Fr>(), d_fa.as<uint32_t>(), d_fb.as<uint32_t>(), d_unc.as<uint32_t>());
    ctx->count_launch();
    BB_TRY(scan_exclusive(ctx, st, d_fa.as<uint32_t>(), nv + 1, keep));
    BB_TRY(scan_exclusive(ctx, st, d_fb.as<uint32_t>(), nv + 1, keep));
    uint32_t na = 0, nb = 0, unc = ~0u;
    BB_CUDA(cudaMemcpyAsync(&na, d_fa.as<uint32_t>() + nv, 4, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(&nb, d_fb.as<uint32_t>() + nv, 4, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(&unc, d_unc.p, 4, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    rep.m = m;
    rep.len[0] = ni; rep.len[1] = m - 1; rep.len[2] = R.n_aux; rep.len[3] = na; rep.len[4] = nb; rep.len[5] = nb;
    if (unc != ~0u) {                                             // generator.rs:464-470
        rep.unconstrained = unc;
        set_error("bb_groth16_generate: auxiliary variable %u is unconstrained (its l element is the identity)", unc);
        if (report) *report = rep;
        return BB_ERR_UNCONSTRAINED_VARIABLE;
    }
    BB_TRY(d_asc.alloc(ctx, (size_t)na * sizeof(Fr)));
    scrub.add(d_asc, (size_t)na * sizeof(Fr));
    BB_TRY(d_bsc.alloc(ctx, (size_t)nb * sizeof(Fr)));
    scrub.add(d_bsc, (size_t)nb * sizeof(Fr));
    k_gen_compact<<<cdiv(nv, 256), 256, 0, st>>>(abc, d_fa.as<uint32_t>(), (uint32_t)nv, d_asc.as<Fr>());
    k_gen_compact<<<cdiv(nv, 256), 256, 0, st>>>(abc + nv, d_fb.as<uint32_t>(), (uint32_t)nv, d_bsc.as<Fr>());
    ctx->count_launch(2);
    BB_TRY(d_vks.alloc(ctx, sizeof S.vk));
    scrub.add(d_vks, sizeof S.vk);
    BB_CUDA(cudaMemcpyAsync(d_vks.p, S.vk, sizeof S.vk, cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaStreamSynchronize(st));                           // S.vk is wiped on return
    BB_CUDA(cudaGetLastError());
    tm.mark("generate.qap");

    // g1, g2: straight into the buffers the key adopts
    const Fr* vks = d_vks.as<Fr>();
    BB_TRY(d_h.alloc(ctx, (m - 1) * sizeof(G1Affine)));
    BB_TRY(d_l.alloc(ctx, R.n_aux * sizeof(G1Affine)));
    BB_TRY(d_a.alloc(ctx, (size_t)na * sizeof(G1Affine)));
    BB_TRY(d_b1.alloc(ctx, (size_t)nb * sizeof(G1Affine)));
    BB_TRY(d_b2.alloc(ctx, (size_t)nb * sizeof(G2Affine)));
    BB_TRY(d_vk1.alloc(ctx, 3 * sizeof(G1Affine)));
    BB_TRY(d_g2.alloc(ctx, 3 * sizeof(G2Affine)));
    if (vk_out) {
        BB_TRY(d_ic.alloc(ctx, ni * sizeof(G1Affine)));
        BB_TRY(d_alpha.alloc(ctx, sizeof(G1Affine)));
    }
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_hq.as<Fr>(), m - 1, true, d_h.p, st, tab1.d));
    if (vk_out) BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_ext.as<Fr>(), ni, true, d_ic.p, st, tab1.d));
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_ext.as<Fr>() + ni, R.n_aux, true, d_l.p, st, tab1.d));
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_asc.as<Fr>(), na, true, d_a.p, st, tab1.d));
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, d_bsc.as<Fr>(), nb, true, d_b1.p, st, tab1.d));
    BB_TRY(fixed_base_mul_device(ctx, BB_G1, vks, 3, true, d_vk1.p, st, tab1.d));
    tm.mark("generate.g1");
    BB_TRY(fixed_base_mul_device(ctx, BB_G2, d_bsc.as<Fr>(), nb, true, d_b2.p, st, tab2.d));
    BB_TRY(fixed_base_mul_device(ctx, BB_G2, vks + 3, 3, true, d_g2.p, st, tab2.d));
    tm.mark("generate.g2");
    G1Affine g1[3];                                               // alpha, beta, delta
    G2Affine g2[3];                                               // delta, gamma, beta
    BB_CUDA(cudaMemcpyAsync(g1, d_vk1.p, sizeof g1, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(g2, d_g2.p, sizeof g2, cudaMemcpyDeviceToHost, st));
    if (vk_out) BB_CUDA(cudaMemcpyAsync(d_alpha.p, d_vk1.p, sizeof(G1Affine), cudaMemcpyDeviceToDevice, st));
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(R.terms);

    bb_bases* vec[5] = {adopt_bases(ctx, BB_G1, d_h, m - 1), adopt_bases(ctx, BB_G1, d_l, R.n_aux), adopt_bases(ctx, BB_G1, d_a, na),
                        adopt_bases(ctx, BB_G1, d_b1, nb), adopt_bases(ctx, BB_G2, d_b2, nb)};
    const G2Affine crs_g2[2] = {g2[2], g2[0]};
    *crs_out = crs_adopt(ctx, vec, g1, crs_g2);
    if (vk_out) *vk_out = vk_adopt(ctx, (G1Affine*)d_alpha.take(), (G2Affine*)d_g2.take(), adopt_bases(ctx, BB_G1, d_ic, ni));
    if (report) *report = rep;
    return BB_OK;
}

}  // extern "C"
