// bellman_b200: C-ABI entry points that are not MSM / prover specific (include/bellman_b200.h).
#include "bb_internal.cuh"
#include "encoding.cuh"
#include "fixed_table.cuh"

using namespace bb;

namespace bb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}
G1X g1_host_mul(const G1X& p, const uint32_t* k);
G2X g2_host_mul(const G2X& p, const uint32_t* k);
}  // namespace bb

int bb_ctx::alloc(size_t bytes, void** out) {
    // round up so that slightly different sizes share cached blocks
    size_t want = (bytes + 255) & ~(size_t)255;
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = free_blocks.lower_bound(want);
        if (it != free_blocks.end() && it->first <= want + want / 4 + 4096) {
            *out = it->second;
            live_blocks[it->second] = it->first;
            free_blocks.erase(it);
            return BB_OK;
        }
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        // drop the cache and retry once
        {
            std::lock_guard<std::mutex> g(mu);
            for (auto& kv : free_blocks) cudaFree(kv.second);
            free_blocks.clear();
        }
        cudaGetLastError();
        e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu): %s", want, cudaGetErrorString(e)); cudaGetLastError(); return BB_ERR_OOM; }
    }
    std::lock_guard<std::mutex> g(mu);
    live_blocks[p] = want;
    *out = p;
    return BB_OK;
}
void bb_ctx::release(void* p) {
    std::lock_guard<std::mutex> g(mu);
    auto it = live_blocks.find(p);
    if (it == live_blocks.end()) return;
    free_blocks.emplace(it->second, p);
    live_blocks.erase(it);
}
int bb_ctx::pinned_acquire(size_t bytes, void** out) {
    if (bytes > PINNED_BLOCK) { set_error("pinned staging block too small for %zu bytes", bytes); return BB_ERR_ARG; }
    {
        std::lock_guard<std::mutex> g(mu);
        if (!pinned_free.empty()) { *out = pinned_free.back(); pinned_free.pop_back(); return BB_OK; }
    }
    BB_CUDA(cudaMallocHost(out, PINNED_BLOCK));
    return BB_OK;
}
void bb_ctx::pinned_release(void* p) {
    std::lock_guard<std::mutex> g(mu);
    pinned_free.push_back(p);
}
cudaStream_t bb_ctx::pick_stream() {
    std::lock_guard<std::mutex> g(mu);
    cudaStream_t s = streams[next_stream % streams.size()];
    next_stream++;
    return s;
}

namespace {

// fixed-base tables of the two generators for bb_fixed_base_mul (fixed_table.cuh)
constexpr int MAX_DEVICES = 64;
FixedTable<Fp> g_tab1[MAX_DEVICES];      // one table per device (a process may open several contexts)
FixedTable<Fp2> g_tab2[MAX_DEVICES];
std::mutex g_tab_mu;

// [k_i]G through the 32 x 255 table of byte multiples: at most 32 mixed additions per point, result left in
// XYZZ form; zzz[i] = its ZZZ coordinate (one for the identity) for the shared inversion below
template <class F>
__global__ void __launch_bounds__(128) k_fixed_base_mul(const Affine<F>* __restrict__ table, const Fr* scalars, size_t n, int montgomery,
                                                        XYZZ<F>* out, F* zzz) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = scalars[i];
    if (montgomery) s = fr_to_canonical(s);
    XYZZ<F> acc = XYZZ<F>::identity();
    for (int w = 0; w < 32; w++) {
        uint32_t d = (s.l[w >> 2] >> (8 * (w & 3))) & 0xffu;
        if (d) acc.add_mixed(table[w * 255 + d - 1]);
    }
    out[i] = acc;
    zzz[i] = acc.is_identity() ? FieldOps<F>::one() : acc.ZZZ;
}
// batch normalisation (generator.rs:271-296 normalises its batches the same way): zinv[i] = 1 / ZZZ_i
template <class F>
__global__ void __launch_bounds__(128) k_xyzz_normalize(const XYZZ<F>* __restrict__ in, const F* __restrict__ zinv, size_t n, Affine<F>* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    XYZZ<F> P = in[i];
    if (P.is_identity()) { out[i] = Affine<F>::identity(); return; }
    F zi3 = zinv[i];
    F zi2 = (zi3 * P.ZZ).sqr();                          // (z^-3 z^2)^2 = z^-2
    out[i] = {P.X * zi2, P.Y * zi3};
}

inline int batch_invert_any(bb_ctx* ctx, cudaStream_t st, Fp* v, size_t n, Fp* scratch) { return batch_invert_fp(ctx, st, v, n, scratch); }
inline int batch_invert_any(bb_ctx* ctx, cudaStream_t st, Fp2* v, size_t n, Fp2* scratch) { return batch_invert_fp2(ctx, st, v, n, scratch); }

template <class F>
int fixed_base_mul_dev(bb_ctx* ctx, FixedTable<F>& tab, const Affine<F>& gen, const Fr* d_scalars, size_t n, bool montgomery,
                       Affine<F>* d_out, cudaStream_t st) {
    {
        std::lock_guard<std::mutex> g(g_tab_mu);
        BB_TRY(build_fixed_table(tab, gen));
    }
    if (!n) return BB_OK;
    // chunks of at most 2^22 points keep the XYZZ scratch below 1.6 GB
    const size_t CH = size_t(1) << 22;
    const size_t ch = n < CH ? n : CH;
    DevBuf d_x, d_z;
    BB_TRY(d_x.alloc(ctx, ch * sizeof(XYZZ<F>)));
    BB_TRY(d_z.alloc(ctx, (ch + batch_invert_scratch(ch)) * sizeof(F)));
    for (size_t lo = 0; lo < n; lo += ch) {
        const size_t len = n - lo < ch ? n - lo : ch;
        k_fixed_base_mul<F><<<cdiv(len, 128), 128, 0, st>>>(tab.d_table, d_scalars + lo, len, montgomery, d_x.as<XYZZ<F>>(), d_z.as<F>());
        ctx->count_launch();
        BB_TRY(batch_invert_any(ctx, st, d_z.as<F>(), len, d_z.as<F>() + len));
        k_xyzz_normalize<F><<<cdiv(len, 128), 128, 0, st>>>(d_x.as<XYZZ<F>>(), d_z.as<F>(), len, d_out + lo);
        ctx->count_launch();
    }
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaStreamSynchronize(st));                   // the scratch buffers go back to the cache on return
    return BB_OK;
}

template <class F>
int fixed_base_mul(bb_ctx* ctx, FixedTable<F>& tab, const Affine<F>& gen, const void* scalars, size_t n, int form, void* out) {
    DevBuf d_s, d_o;
    BB_TRY(d_s.alloc(ctx, n * 32));
    BB_TRY(d_o.alloc(ctx, n * sizeof(Affine<F>)));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d_s.p, scalars, n * 32, cudaMemcpyHostToDevice, st));
    BB_TRY(fixed_base_mul_dev<F>(ctx, tab, gen, d_s.as<Fr>(), n, form == BB_FORM_MONTGOMERY, d_o.as<Affine<F>>(), st));
    BB_CUDA(cudaMemcpyAsync(out, d_o.p, n * sizeof(Affine<F>), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}


// ---- curve and subgroup membership of a vector of affine points -----------------------------------
// What G1Affine/G2Affine::from_uncompressed (bls12_381 crate; called by Parameters::read with
// checked = true and always by VerifyingKey::read, groth16/src/lib.rs:158-183,289-330) verifies
// beyond the encoding: y^2 = x^3 + b and [r]P = identity.  One thread per point; the first offending
// index is reported through atomicMin (bad[0]: off the curve, bad[1]: outside the subgroup).  The
// identity itself passes here: the callers decide where it is allowed.
template <class F>
__global__ void __launch_bounds__(128) k_points_validate(const Affine<F>* __restrict__ pts, size_t n, int check_subgroup, uint32_t* bad) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine<F> p = pts[i];
    if (p.is_identity()) return;
    if (!on_curve(p)) { atomicMin(&bad[0], (uint32_t)i); return; }
    if (!check_subgroup) return;
    if (!rP_is_identity(p)) atomicMin(&bad[1], (uint32_t)i);
}

// ---- diagnostics: element-wise field / point operations on the device ------------------------
template <class FE>
__global__ void k_selftest_field(const FE* a, const FE* b, FE* o, size_t n, int op) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FE x = a[i], y = b[i];
    o[i] = op == 0 ? x * y : op == 1 ? x + y : op == 2 ? x - y : x.sqr();
}
// Fp only: op 4 = inverse by the binary Euclidean algorithm (what FieldOps<Fp>::inv runs), 5 = a^(p-2); zero -> zero
__global__ void k_selftest_fp_inv(const Fp* a, Fp* o, size_t n, int op) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp x = a[i];
    o[i] = x.is_zero() ? x : (op == 4 ? fp_inv_gcd(x) : fp_inv(x));
}
// Fp2: op 0 operator* and 3 sqr() (the out-of-line calls of the tower and the verifier), 1 +, 2 -, 4 fp2_inv (zero -> zero),
// 5 mul_inl and 6 sqr_inl (the inlined forms of the halving rounds)
__global__ void k_selftest_fp2(const Fp2* a, const Fp2* b, Fp2* o, size_t n, int op) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fp2 x = a[i], y = b[i];
    Fp2 r;
    switch (op) {
        case 0: r = x * y; break;
        case 1: r = x + y; break;
        case 2: r = x - y; break;
        case 3: r = x.sqr(); break;
        case 4: r = x.is_zero() ? x : fp2_inv(x); break;
        case 5: r = x.mul_inl(y); break;
        default: r = x.sqr_inl(); break;
    }
    o[i] = r;
}
template <class F>
__global__ void k_selftest_point(const Affine<F>* a, const Affine<F>* b, Affine<F>* o, size_t n, int op) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    XYZZ<F> x = XYZZ<F>::from_affine(a[i]);
    if (op == 0) x.add_mixed(b[i]);
    else if (op == 1) { x = x.dbl(); x.add(XYZZ<F>::from_affine(b[i])); }   // 2a + b through the projective paths
    else if (op == 2) { XYZZ<F> y = XYZZ<F>::from_affine(b[i]); y = y.dbl(); y.add_mixed(b[i].neg()); x.add(y); }  // a + (2b - b)
    o[i] = x.to_affine();
}
template <class T, class K>
int selftest_run(bb_ctx* ctx, K kernel, const void* a, const void* b, void* o, size_t n, int op) {
    DevBuf da, db, d_o2;
    BB_TRY(da.alloc(ctx, n * sizeof(T))); BB_TRY(db.alloc(ctx, n * sizeof(T))); BB_TRY(d_o2.alloc(ctx, n * sizeof(T)));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(da.p, a, n * sizeof(T), cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaMemcpyAsync(db.p, b, n * sizeof(T), cudaMemcpyHostToDevice, st));
    if (n) { kernel<<<cdiv(n, 64), 64, 0, st>>>(da.as<T>(), db.as<T>(), d_o2.as<T>(), n, op); ctx->count_launch(); }
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaMemcpyAsync(o, d_o2.p, n * sizeof(T), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

}  // namespace

namespace bb {
int fixed_base_mul_device(bb_ctx* ctx, int group, const Fr* d_scalars, size_t n, bool montgomery, void* d_out, cudaStream_t st,
                          const void* d_table) {
    if (ctx->device < 0 || ctx->device >= MAX_DEVICES) { set_error("device ordinal out of range"); return BB_ERR_ARG; }
    if (d_table) {                                        // a caller's table: already built, the generator is not needed
        if (group == BB_G1) {
            FixedTable<Fp> t{(G1Affine*)d_table};
            return fixed_base_mul_dev<Fp>(ctx, t, G1Affine::identity(), d_scalars, n, montgomery, (G1Affine*)d_out, st);
        }
        FixedTable<Fp2> t{(G2Affine*)d_table};
        return fixed_base_mul_dev<Fp2>(ctx, t, G2Affine::identity(), d_scalars, n, montgomery, (G2Affine*)d_out, st);
    }
    if (group == BB_G1) return fixed_base_mul_dev<Fp>(ctx, g_tab1[ctx->device], g1_generator(), d_scalars, n, montgomery, (G1Affine*)d_out, st);
    return fixed_base_mul_dev<Fp2>(ctx, g_tab2[ctx->device], g2_generator(), d_scalars, n, montgomery, (G2Affine*)d_out, st);
}

int fixed_table_build(int group, const void* gen, void** d_table) {
    *d_table = nullptr;
    if (group == BB_G1) {
        FixedTable<Fp> t;
        G1Affine g;
        std::memcpy(&g, gen, sizeof g);
        BB_TRY(build_fixed_table(t, g));
        *d_table = t.d_table;
    } else {
        FixedTable<Fp2> t;
        G2Affine g;
        std::memcpy(&g, gen, sizeof g);
        BB_TRY(build_fixed_table(t, g));
        *d_table = t.d_table;
    }
    return BB_OK;
}

void fixed_table_free(int group, void* d_table) {
    if (!d_table) return;
    cudaMemsetAsync(d_table, 0, (size_t)32 * 255 * (group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine)));
    cudaDeviceSynchronize();
    cudaFree(d_table);
}
}  // namespace bb

extern "C" {

const char* bb_last_error(void) { return g_err; }
int bb_version(void) { return 100; }

int bb_ctx_create(int device, bb_ctx** out) {
    if (!out) { set_error("bb_ctx_create: null out"); return BB_ERR_ARG; }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("no usable CUDA device (%s); bellman_b200 has no CPU fallback", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
        cudaGetLastError();
        return BB_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= count) { set_error("device %d out of range (%d devices)", device, count); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(device));
    bb_ctx* ctx = new bb_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    BB_CUDA(cudaGetDeviceProperties(&prop, device));
    ctx->num_sms = prop.multiProcessorCount;
    // The H pipeline (7 NTTs) and the h MSM that waits for it are the critical path of a proof: their
    // streams outrank the seven witness MSMs, so their CTAs are placed first whenever an SM has room.
    int prio_lo = 0, prio_hi = 0;
    BB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    BB_CUDA(cudaStreamCreateWithPriority(&ctx->main_stream, cudaStreamNonBlocking, prio_hi));
    for (auto& cs : ctx->crit_stream) BB_CUDA(cudaStreamCreateWithPriority(&cs, cudaStreamNonBlocking, prio_hi));
    for (int i = 0; i < 8; i++) {
        cudaStream_t s;
        BB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
        ctx->streams.push_back(s);
    }
    *out = ctx;
    return BB_OK;
}

void bb_ctx_destroy(bb_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (auto& kv : ctx->free_blocks) cudaFree(kv.second);
    for (auto& kv : ctx->live_blocks) cudaFree(kv.first);
    for (auto p : ctx->pinned_free) cudaFreeHost(p);
    for (auto p : ctx->read_stage) if (p) cudaFreeHost(p);
    for (auto s : ctx->streams) cudaStreamDestroy(s);
    if (ctx->main_stream) cudaStreamDestroy(ctx->main_stream);
    for (auto& cs : ctx->crit_stream) if (cs) cudaStreamDestroy(cs);
    if (ctx->epoch_ev) cudaEventDestroy(ctx->epoch_ev);
    ntt_free_tables(ctx);
    delete ctx;
}

// Options whose second implementation was measured slower than (or level with) the default path and then removed.
// The keys stay accepted and have no effect, so that callers which still set them keep working.
static bool retired_option(const std::string& k) {
    for (const char* r : {"msm_acc_variant", "msm_affine_tma", "msm_reduce_2d", "ntt_radix8"})
        if (k == r) return true;
    return false;
}

int bb_ctx_set_option(bb_ctx* ctx, const char* key, long value) {
    if (!ctx || !key) { set_error("bb_ctx_set_option: null argument"); return BB_ERR_ARG; }
    std::string k(key);
    if (k == "msm_window_bits") ctx->opt_msm_window_bits = value;
    else if (k == "ntt_tile_log") ctx->opt_ntt_tile_log = value;
    else if (k == "ntt_col_bits") ctx->opt_ntt_col_bits = value;
    else if (k == "profile") ctx->opt_profile = value;
    else if (k == "msm_big_cap") ctx->opt_msm_big_cap = value;
    else if (k == "msm_precompute") { if (value < 0 || value > 2) { set_error("msm_precompute is 0, 1 or 2"); return BB_ERR_ARG; } ctx->opt_msm_precompute = value; }
    else if (k == "msm_precompute_groups") { if (value < 0 || value > 3) { set_error("msm_precompute_groups is a mask of 1 (G1) and 2 (G2)"); return BB_ERR_ARG; } ctx->opt_msm_precompute_groups = value; }
    else if (k == "msm_unified_rows_log") { if (value < 0 || value > 12) { set_error("msm_unified_rows_log is 0..12"); return BB_ERR_ARG; } ctx->opt_msm_unified_rows_log = value; }
    else if (k == "prove_batch_max") { if (value < 0) { set_error("prove_batch_max >= 0"); return BB_ERR_ARG; } ctx->opt_prove_batch_max = value; }
    else if (k == "params_read_chunk") { if (value < 1) { set_error("params_read_chunk >= 1"); return BB_ERR_ARG; } ctx->opt_params_read_chunk = value; }
    else if (k == "msm_affine_rounds") ctx->opt_msm_affine_rounds = value;
    else if (k == "msm_affine_batch") ctx->opt_msm_affine_batch = value;
    else if (k == "shard_windows") { if (value < 1) { set_error("shard_windows >= 1"); return BB_ERR_ARG; } ctx->opt_shard_windows = value; }
    else if (k == "msm_reduce_k1") { if (value < 2 || (value & (value - 1))) { set_error("msm_reduce_k1 must be a power of two >= 2"); return BB_ERR_ARG; } ctx->opt_msm_reduce_k1 = value; }
    else if (k == "msm_reduce_k") { if (value < 2 || (value & (value - 1))) { set_error("msm_reduce_k must be a power of two >= 2"); return BB_ERR_ARG; } ctx->opt_msm_reduce_k = value; }
    else if (retired_option(k)) {}
    else { set_error("unknown option %s", key); return BB_ERR_ARG; }
    return BB_OK;
}

int bb_ctx_synchronize(bb_ctx* ctx) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    BB_CUDA(cudaDeviceSynchronize());
    return BB_OK;
}

uint64_t bb_ctx_kernel_launches(const bb_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }

int bb_profile_read(bb_ctx* ctx, const char* what, double* ms, uint64_t* launches, uint64_t* units) {
    if (!ctx || !what) return BB_ERR_ARG;
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = ctx->prof.find(what);
    bb_ctx::ProfEntry e;
    if (it != ctx->prof.end()) e = it->second;
    if (ms) *ms = e.ms;
    if (launches) *launches = e.launches;
    if (units) *units = e.units;
    return BB_OK;
}
int bb_ctx_bytes_copied(const bb_ctx* ctx, uint64_t* h2d, uint64_t* d2h) {
    if (!ctx) return BB_ERR_ARG;
    if (h2d) *h2d = ctx->h2d_bytes.load();
    if (d2h) *d2h = ctx->d2h_bytes.load();
    return BB_OK;
}
uint64_t bb_diag_ctx_live_bytes(const bb_ctx* ctx) {
    if (!ctx) return 0;
    std::lock_guard<std::mutex> g(const_cast<bb_ctx*>(ctx)->mu);
    uint64_t s = 0;
    for (auto& kv : ctx->live_blocks) s += kv.second;
    return s;
}
int bb_profile_reset(bb_ctx* ctx) {
    if (!ctx) return BB_ERR_ARG;
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->prof.clear();
    return BB_OK;
}

int bb_device_alloc(bb_ctx* ctx, size_t bytes, void** d_out) {
    if (!ctx || !d_out) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    return ctx->alloc(bytes, d_out);
}
int bb_device_free(bb_ctx* ctx, void* d_ptr) {
    if (!ctx) return BB_ERR_ARG;
    if (d_ptr) ctx->release(d_ptr);
    return BB_OK;
}
int bb_device_upload(bb_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    BB_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->main_stream));
    BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    return BB_OK;
}
int bb_device_download(bb_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    BB_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->main_stream));
    BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    return BB_OK;
}

int bb_ntt_device(bb_ctx* ctx, void* d_fr_inout, uint32_t log_n, int mode) {
    if (!ctx || !d_fr_inout) { set_error("bb_ntt_device: null argument"); return BB_ERR_ARG; }
    if (log_n >= (uint32_t)bbc::FR_S) { set_error("PolynomialDegreeTooLarge"); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    BB_CUDA(cudaSetDevice(ctx->device));
    DevBuf tmp;
    BB_TRY(tmp.alloc(ctx, (size_t)32 << log_n));
    BB_TRY(ntt_run_device(ctx, ctx->main_stream, (Fr*)d_fr_inout, tmp.as<Fr>(), log_n, mode));
    BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    return BB_OK;
}

int bb_ntt(bb_ctx* ctx, void* fr_inout, uint32_t log_n, int mode, int form) {
    if (!ctx || !fr_inout) { set_error("bb_ntt: null argument"); return BB_ERR_ARG; }
    if (log_n >= (uint32_t)bbc::FR_S) { set_error("PolynomialDegreeTooLarge"); return BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE; }
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t n = (size_t)1 << log_n;
    DevBuf d, tmp;
    BB_TRY(d.alloc(ctx, n * 32));
    BB_TRY(tmp.alloc(ctx, n * 32));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d.p, fr_inout, n * 32, cudaMemcpyHostToDevice, st));
    // the transform is linear, so canonical inputs can be transformed as they are (the
    // twiddles carry the Montgomery factor); only the fused multiplications by table entries
    // are Montgomery products, which is exactly what keeps a canonical vector canonical.
    (void)form;
    BB_TRY(ntt_run_device(ctx, st, d.as<Fr>(), tmp.as<Fr>(), log_n, mode));
    BB_CUDA(cudaMemcpyAsync(fr_inout, d.p, n * 32, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

int bb_domain_pointwise(bb_ctx* ctx, int op, void* fr_a_inout, const void* fr_b, size_t n, const void* fr_k) {
    if (!ctx || (n && !fr_a_inout) || op < 0 || op > 3) { set_error("bb_domain_pointwise: bad argument"); return BB_ERR_ARG; }
    if (op <= 1 && n && !fr_b) { set_error("bb_domain_pointwise: op %d needs a second vector", op); return BB_ERR_ARG; }
    if (op >= 2 && !fr_k) { set_error("bb_domain_pointwise: op %d needs a scalar", op); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    DevBuf d_a, d_b;
    BB_TRY(d_a.alloc(ctx, n * 32));
    BB_TRY(d_b.alloc(ctx, n * 32));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d_a.p, fr_a_inout, n * 32, cudaMemcpyHostToDevice, st));
    if (op <= 1) BB_CUDA(cudaMemcpyAsync(d_b.p, fr_b, n * 32, cudaMemcpyHostToDevice, st));
    Fr k = Fr::zero();
    if (fr_k) std::memcpy(k.l, fr_k, 32);
    BB_TRY(domain_pointwise_device(ctx, st, d_a.as<Fr>(), d_b.as<Fr>(), n, op, k));
    BB_CUDA(cudaMemcpyAsync(fr_a_inout, d_a.p, n * 32, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

int bb_h_poly(bb_ctx* ctx, const void* a, const void* b, const void* c, size_t n, void* h_out, size_t* m_out) {
    if (!ctx || !h_out || (n && (!a || !b || !c))) { set_error("bb_h_poly: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t m;
    uint32_t log_m;
    BB_TRY(domain_size(n, &m, &log_m));
    DevBuf d_a, d_b, d_c, d_t;
    BB_TRY(d_a.alloc(ctx, m * 32)); BB_TRY(d_b.alloc(ctx, m * 32)); BB_TRY(d_c.alloc(ctx, m * 32)); BB_TRY(d_t.alloc(ctx, m * 32));
    cudaStream_t st = ctx->main_stream;
    const void* srcs[3] = {a, b, c};
    DevBuf* dst[3] = {&d_a, &d_b, &d_c};
    for (int k = 0; k < 3; k++) {
        if (m > n) BB_CUDA(cudaMemsetAsync((char*)dst[k]->p + n * 32, 0, (m - n) * 32, st));
        if (n) BB_CUDA(cudaMemcpyAsync(dst[k]->p, srcs[k], n * 32, cudaMemcpyHostToDevice, st));
    }
    BB_TRY(h_poly_device(ctx, st, d_a.as<Fr>(), d_b.as<Fr>(), d_c.as<Fr>(), d_t.as<Fr>(), log_m));
    BB_TRY(fr_convert_device(ctx, st, d_a.as<Fr>(), m - 1, false));
    if (m > 1) BB_CUDA(cudaMemcpyAsync(h_out, d_a.p, (m - 1) * 32, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    if (m_out) *m_out = m;
    return BB_OK;
}

int bb_bases_upload(bb_ctx* ctx, int group, const void* affine, size_t n, size_t global_offset, size_t global_len, bb_bases** out) {
    if (!ctx || !out || (n && !affine) || (group != BB_G1 && group != BB_G2)) { set_error("bb_bases_upload: bad argument"); return BB_ERR_ARG; }
    if (global_offset + n > global_len) { set_error("bb_bases_upload: shard [%zu,%zu) exceeds %zu", global_offset, global_offset + n, global_len); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t stride = group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine);
    void* d = nullptr;
    BB_TRY(ctx->alloc((n ? n : 1) * stride, &d));
    if (n) {
        BB_CUDA(cudaMemcpyAsync(d, affine, n * stride, cudaMemcpyHostToDevice, ctx->main_stream));
        BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    }
    bb_bases* b = new bb_bases();
    b->ctx = ctx; b->group = group; b->d_points = d; b->n = n; b->global_offset = global_offset; b->global_len = global_len;
    *out = b;
    return BB_OK;
}
void bb_bases_free(bb_bases* b) {
    if (!b) return;
    if (b->d_points) b->ctx->release(b->d_points);
    if (b->d_table) b->ctx->release(b->d_table);
    delete b;
}

int bb_point_add(int group, const void* a, const void* b, void* out) {
    if (!a || !b || !out) return BB_ERR_ARG;
    if (group == BB_G1) {
        G1Affine pa, pb; std::memcpy(&pa, a, 96); std::memcpy(&pb, b, 96);
        G1X x = G1X::from_affine(pa); x.add_mixed(pb);
        G1Affine r = x.to_affine(); std::memcpy(out, &r, 96);
    } else if (group == BB_G2) {
        G2Affine pa, pb; std::memcpy(&pa, a, 192); std::memcpy(&pb, b, 192);
        G2X x = G2X::from_affine(pa); x.add_mixed(pb);
        G2Affine r = x.to_affine(); std::memcpy(out, &r, 192);
    } else return BB_ERR_ARG;
    return BB_OK;
}
int bb_point_mul(int group, const void* a, const void* k, int form, void* out) {
    if (!a || !k || !out) return BB_ERR_ARG;
    Fr s; std::memcpy(s.l, k, 32);
    if (form == BB_FORM_MONTGOMERY) s = fr_to_canonical(s);
    if (group == BB_G1) {
        G1Affine pa; std::memcpy(&pa, a, 96);
        G1Affine r = g1_host_mul(G1X::from_affine(pa), s.l).to_affine(); std::memcpy(out, &r, 96);
    } else if (group == BB_G2) {
        G2Affine pa; std::memcpy(&pa, a, 192);
        G2Affine r = g2_host_mul(G2X::from_affine(pa), s.l).to_affine(); std::memcpy(out, &r, 192);
    } else return BB_ERR_ARG;
    return BB_OK;
}
int bb_point_compress(int group, const void* a, uint8_t* out) {
    if (!a || !out) return BB_ERR_ARG;
    if (group == BB_G1) { G1Affine p; std::memcpy(&p, a, 96); encode_compressed(p, out); }
    else if (group == BB_G2) { G2Affine p; std::memcpy(&p, a, 192); encode_compressed(p, out); }
    else return BB_ERR_ARG;
    return BB_OK;
}
// In-place conversion of n Fp coordinates (6 x u64 each) between canonical integers and the
// Montgomery form the ABI uses; host code (parameter files: groth16/src/lib.rs:258-398 stores
// canonical big-endian coordinates).
int bb_fp_convert(void* fp_inout, size_t n, int to_montgomery) {
    if (n && !fp_inout) return BB_ERR_ARG;
    Fp* v = (Fp*)fp_inout;
    for (size_t i = 0; i < n; i++) {
        Fp x;
        std::memcpy(&x, v + i, sizeof x);
        if (to_montgomery) {
            if (!is_canonical(x)) { set_error("coordinate %zu is not a canonical field element", i); return BB_ERR_ARG; }
            x = fp_from_canonical(x);
        } else {
            x = fp_to_canonical(x);
        }
        std::memcpy(v + i, &x, sizeof x);
    }
    return BB_OK;
}
// Checks n affine points (ABI format, host memory) the way from_uncompressed does after decoding:
// on the curve, and (check_subgroup != 0) in the prime-order subgroup.  *first_bad = index of the
// first offending point (SIZE_MAX if none), *why = 1 off the curve, 2 outside the subgroup.
int bb_points_validate(bb_ctx* ctx, int group, const void* affine, size_t n, int check_subgroup, size_t* first_bad, int* why) {
    if (!ctx || (n && !affine) || !first_bad || !why || (group != BB_G1 && group != BB_G2)) { set_error("bb_points_validate: bad argument"); return BB_ERR_ARG; }
    if (n >= (1ull << 32)) { set_error("bb_points_validate: more than 2^32 points"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    *first_bad = (size_t)-1; *why = 0;
    if (!n) return BB_OK;
    const size_t stride = group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine);
    DevBuf d_p, d_bad;
    BB_TRY(d_p.alloc(ctx, n * stride));
    BB_TRY(d_bad.alloc(ctx, 8));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d_p.p, affine, n * stride, cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaMemsetAsync(d_bad.p, 0xff, 8, st));
    if (group == BB_G1) k_points_validate<Fp><<<cdiv(n, 128), 128, 0, st>>>(d_p.as<G1Affine>(), n, check_subgroup, d_bad.as<uint32_t>());
    else k_points_validate<Fp2><<<cdiv(n, 128), 128, 0, st>>>(d_p.as<G2Affine>(), n, check_subgroup, d_bad.as<uint32_t>());
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    uint32_t bad[2] = {0xffffffffu, 0xffffffffu};
    BB_CUDA(cudaMemcpyAsync(bad, d_bad.p, 8, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    if (bad[0] != 0xffffffffu && bad[0] <= bad[1]) { *first_bad = bad[0]; *why = 1; }
    else if (bad[1] != 0xffffffffu) { *first_bad = bad[1]; *why = 2; }
    return BB_OK;
}
int bb_fixed_base_mul(bb_ctx* ctx, int group, const void* scalars, size_t n, int form, void* out) {
    if (!ctx || (n && (!scalars || !out))) { set_error("bb_fixed_base_mul: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    if (ctx->device < 0 || ctx->device >= MAX_DEVICES) { set_error("device ordinal out of range"); return BB_ERR_ARG; }
    if (group == BB_G1) return fixed_base_mul<Fp>(ctx, g_tab1[ctx->device], g1_generator(), scalars, n, form, out);
    if (group == BB_G2) return fixed_base_mul<Fp2>(ctx, g_tab2[ctx->device], g2_generator(), scalars, n, form, out);
    set_error("bad group");
    return BB_ERR_ARG;
}

int bb_selftest_field(bb_ctx* ctx, int field, int op, const void* a, const void* b, void* out, size_t n) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    if (field == 0) return selftest_run<Fr>(ctx, k_selftest_field<Fr>, a, b, out, n, op);
    if (field == 1 && (op == 4 || op == 5)) {
        DevBuf da, d_o;
        BB_TRY(da.alloc(ctx, n * sizeof(Fp))); BB_TRY(d_o.alloc(ctx, n * sizeof(Fp)));
        cudaStream_t st = ctx->main_stream;
        BB_CUDA(cudaMemcpyAsync(da.p, a, n * sizeof(Fp), cudaMemcpyHostToDevice, st));
        if (n) { k_selftest_fp_inv<<<cdiv(n, 64), 64, 0, st>>>(da.as<Fp>(), d_o.as<Fp>(), n, op); ctx->count_launch(); }
        BB_CUDA(cudaGetLastError());
        BB_CUDA(cudaMemcpyAsync(out, d_o.p, n * sizeof(Fp), cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaStreamSynchronize(st));
        return BB_OK;
    }
    if (field == 1) return selftest_run<Fp>(ctx, k_selftest_field<Fp>, a, b, out, n, op);
    if (field == 2 && op >= 0 && op <= 6) return selftest_run<Fp2>(ctx, k_selftest_fp2, a, b, out, n, op);
    return BB_ERR_ARG;
}
int bb_selftest_point(bb_ctx* ctx, int group, int op, const void* a, const void* b, void* out, size_t n) {
    if (!ctx) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    if (group == BB_G1) return selftest_run<G1Affine>(ctx, k_selftest_point<Fp>, a, b, out, n, op);
    if (group == BB_G2) return selftest_run<G2Affine>(ctx, k_selftest_point<Fp2>, a, b, out, n, op);
    return BB_ERR_ARG;
}

}  // extern "C"
