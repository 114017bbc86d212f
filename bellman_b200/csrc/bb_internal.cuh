// bellman_b200 internal: context, device memory cache, error plumbing.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bellman_b200_diag.h"
#include "curve.cuh"

// NVTX ranges (header-only nvtx3, no link dependency; a no-op unless a tool such as nsys is attached):
// one range per prove, per MSM job launch sequence and per H pipeline, so that a timeline shows the job graph.
#if defined(__CUDACC__)
#include <nvtx3/nvToolsExt.h>
namespace bb {
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
}  // namespace bb
#else
namespace bb {
struct NvtxRange { explicit NvtxRange(const char*) {} };
}  // namespace bb
#endif

namespace bb {

void set_error(const char* fmt, ...);

#define BB_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess) {                                                             \
            bb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return BB_ERR_CUDA;                                                               \
        }                                                                                     \
    } while (0)

#define BB_TRY(call)                       \
    do {                                   \
        int s__ = (call);                  \
        if (s__ != BB_OK) return s__;      \
    } while (0)

struct NttTables;

}  // namespace bb

// Context = one device.  Device allocations are cached by size so that the steady state of a
// prover issues no cudaMalloc/cudaFree (both synchronise the device).
struct bb_ctx {
    int device = 0;
    int num_sms = 0;
    std::mutex mu;
    std::multimap<size_t, void*> free_blocks;
    std::map<void*, size_t> live_blocks;
    std::vector<cudaStream_t> streams;       // round-robin pool for async jobs
    size_t next_stream = 0;
    cudaStream_t main_stream = nullptr;      // high priority: NTTs / the H pipeline
    cudaStream_t crit_stream[2] = {nullptr, nullptr};   // high priority: the MSMs on a proof's critical path (h, and the G2 job)
    std::atomic<uint64_t> launches{0};
    std::atomic<uint64_t> h2d_bytes{0}, d2h_bytes{0};   // host<->device traffic of the hot-path calls
    long opt_msm_window_bits = 0;
    long opt_ntt_tile_log = 11;
    long opt_ntt_col_bits = 3;
    long opt_profile = 0;
    long opt_msm_reduce_k = 4;       // entries per thread and level of the bucket reduction: 4 halves the length of the
    long opt_msm_reduce_k1 = 4;      // dependent-addition chain of 16 (2K per level, log_K D levels) for 1.25x its additions
    long opt_msm_big_cap = 0;
    long opt_shard_windows = 4;      // multi-GPU: up to this many window shards per base range (1 = base ranges only)
    long opt_msm_affine_rounds = -1;  // batched-affine halving rounds per MSM: -1 = by size, 0 = none (XYZZ accumulation only)
    long opt_msm_affine_batch = 16;   // pairs per thread sharing one link of the inversion chain
    long opt_msm_precompute = 0;     // resident window multiples 2^(c w) P of every base vector (msm.cu: bases_build_table):
                                     // 1 = one bucket array per window slot, 2 = ONE bucket array for all windows
    long opt_msm_precompute_groups = 3;  // which groups use the tables: bit 0 = G1 vectors, bit 1 = G2 vectors
    long opt_msm_unified_rows_log = 3;   // msm_precompute = 2: halving rounds until about 2^this rows per bucket are left
    long opt_prove_batch_max = 0;        // bb_groth16_prove_batch: at most this many proofs per sub-batch (0 = by memory)
    long opt_params_read_chunk = 64l << 20;   // bb_params_read from host memory: staging bytes per chunk
    // bb_params_read's two page-locked staging blocks (read_stage_bytes each), kept for the next read; read_mu serialises
    // the reads that use them
    std::mutex read_mu;
    void* read_stage[2] = {nullptr, nullptr};
    size_t read_stage_bytes = 0;
    struct ProfEntry { double ms = 0; uint64_t launches = 0, units = 0; };
    std::map<std::string, ProfEntry> prof;
    void prof_add(const char* what, double ms, uint64_t launches, uint64_t units) {
        std::lock_guard<std::mutex> g(mu);
        ProfEntry& e = prof[what];
        e.ms += ms; e.launches += launches; e.units += units;
    }
    std::map<uint32_t, bb::NttTables*> ntt_tables;   // by log_n
    std::vector<void*> h_evals_scratch;              // transform scratch of bb_h_coset_evals_async calls not yet waited for
    cudaEvent_t epoch_ev = nullptr;                  // profile mode: start of the current prove (device timeline origin)

    // small page-locked staging blocks for results (cudaMallocHost/cudaFreeHost synchronise the
    // device and are slow; jobs borrow fixed-size blocks instead)
    static constexpr size_t PINNED_BLOCK = 64 * 1024;
    std::vector<void*> pinned_free;
    int pinned_acquire(size_t bytes, void** out);
    void pinned_release(void* p);
    int alloc(size_t bytes, void** out);
    void release(void* p);
    cudaStream_t pick_stream();
    void count_launch(uint64_t k = 1) { launches.fetch_add(k, std::memory_order_relaxed); }
};

struct bb_bases {
    bb_ctx* ctx;
    int group;
    void* d_points;          // Affine<Fp> or Affine<Fp2>
    size_t n;                // points held here
    size_t global_offset;    // first global index held
    size_t global_len;       // length of the whole (unsharded) vector
    uint32_t win_index = 0;  // window shard: this device accumulates windows w % win_count == win_index
    uint32_t win_count = 1;
    // Optional table of window multiples: slot s = w / win_count of every owned window w holds
    // 2^(tab_c * w) * P_i at d_table[s * n + i] (affine).  With it all windows share one bucket set.
    void* d_table = nullptr;
    uint32_t tab_c = 0, tab_W = 0, tab_slots = 0;
    std::mutex tab_mu;
};

namespace bb {

// RAII device buffer from the context cache
struct DevBuf {
    bb_ctx* ctx = nullptr;
    void* p = nullptr;
    DevBuf() {}
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { reset(); }
    int alloc(bb_ctx* c, size_t bytes) { reset(); ctx = c; return c->alloc(bytes ? bytes : 16, &p); }
    void reset() { if (p && ctx) ctx->release(p); p = nullptr; }
    void* take() { void* q = p; p = nullptr; return q; }      // the block now belongs to the caller
    template <class T> T* as() const { return (T*)p; }
};

// The caller's array on the device: `p` itself when it is in device memory, else a copy queued on `st` into `buf`
// (counted in h2d_bytes)
template <class T>
int device_input(bb_ctx* ctx, cudaStream_t st, const void* p, size_t bytes, bool on_device, DevBuf& buf, const T** out) {
    if (on_device) { *out = (const T*)p; return BB_OK; }
    BB_TRY(buf.alloc(ctx, bytes));
    if (bytes) BB_CUDA(cudaMemcpyAsync(buf.p, p, bytes, cudaMemcpyHostToDevice, st));
    ctx->h2d_bytes += bytes;
    *out = buf.as<T>();
    return BB_OK;
}

// CUDA-event brackets of a call's stages (profile mode only)
struct StageTimer {
    static constexpr uint64_t REPORT_UNITS = ~0ull;          // a mark without units of its own: report()'s
    bb_ctx* ctx;
    cudaStream_t st;
    std::vector<std::pair<const char*, cudaEvent_t>> marks;
    std::vector<uint64_t> mark_units;
    StageTimer(bb_ctx* c, cudaStream_t s) : ctx(c), st(s) {}
    ~StageTimer() { for (auto& m : marks) cudaEventDestroy(m.second); }
    void mark(const char* stage_ending_here, uint64_t units = REPORT_UNITS) {
        if (!ctx->opt_profile) return;
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        cudaEventRecord(e, st);
        marks.emplace_back(stage_ending_here, e);
        mark_units.push_back(units);
    }
    // after the stream has drained: stage k = the interval between marks k-1 and k
    void report(uint64_t units) {
        for (size_t k = 1; k < marks.size(); k++) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, marks[k - 1].second, marks[k].second) == cudaSuccess)
                ctx->prof_add(marks[k].first, ms, 1, mark_units[k] == REPORT_UNITS ? units : mark_units[k]);
        }
    }
};

inline unsigned cdiv(size_t a, size_t b) { return (unsigned)((a + b - 1) / b); }

// ---- ntt.cu ----
// The evaluation domain of n coefficients: m = 2^log_m >= n, or PolynomialDegreeTooLarge
int domain_size(size_t n, size_t* m, uint32_t* log_m);
int ntt_run_device(bb_ctx* ctx, cudaStream_t st, Fr* d_data, Fr* d_tmp, uint32_t log_n, int mode);
int h_poly_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, Fr* d_b, Fr* d_c, Fr* d_tmp, uint32_t log_m);
int h_poly_batch_device(bb_ctx* ctx, cudaStream_t st, Fr* d_abc, Fr* d_tmp, uint32_t log_m, uint32_t B);
int h_poly_evals_device(bb_ctx* ctx, cudaStream_t st, Fr* d_p, Fr* d_tmp, uint32_t log_m);
int h_poly_final_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, const Fr* d_b, const Fr* d_c, Fr* d_tmp, uint32_t log_m);
int fr_convert_device(bb_ctx* ctx, cudaStream_t st, Fr* d_data, size_t n, bool to_montgomery);
void ntt_free_tables(bb_ctx* ctx);
int domain_pointwise_device(bb_ctx* ctx, cudaStream_t st, Fr* d_a, const Fr* d_b, size_t n, int op, const Fr& k);
// d_out[i] = scale * base^i for i < n (k_powers)
int powers_device(bb_ctx* ctx, cudaStream_t st, Fr* d_out, size_t n, const Fr& base, const Fr& scale);

// ---- prover.cu ----
// Queues on `st` the evaluation of a sub-batch's a, b, c into abc (rows a_0 .. a_{B-1}, b_0 .., c_0 .. of m Fr; the first
// n_constraints of each) from its uploaded witnesses d_in (B x n_inputs) and d_aux (B x n_aux)
using BatchAbcFill = std::function<int(cudaStream_t st, uint32_t B, Fr* abc, size_t m, const Fr* d_in, const Fr* d_aux)>;
// bb_groth16_prove_batch (with `fill`, the witnesses' a, b, c are not read: fill computes them) and its argument checks
int prove_batch_impl(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, size_t count, const uint8_t* r, const uint8_t* s,
                     uint8_t* proofs, int* status, const BatchAbcFill* fill = nullptr);
int prove_batch_check(const char* fn, const bb_ctx* ctx, const bb_crs* crs, size_t count, const void* r, const void* s, const void* proofs,
                      const int* status);
// Queues on the main stream, after the witness upload and ahead of the witness MSMs, the owner stage of a proof from a
// resident constraint system: d_in / d_aux the witness on the device, tmp m Fr of scratch, tm its profile-mode stages
using ProveHead = std::function<int(cudaStream_t st, const Fr* d_in, const Fr* d_aux, Fr* tmp, StageTimer& tm)>;
// How bb_groth16_prove_r1cs_begin starts a proof (its witness, device or host, is read in place or uploaded once).  split:
// `head` (empty: nothing is owned) runs ahead of the witness MSMs and bb_groth16_prove_end takes the three vectors.
// Otherwise `fill` (B = 1) evaluates a, b, c into the H pipeline's rows, and the H pipeline and the h MSM are queued ahead
// of the witness MSMs; bb_groth16_prove_end takes no vectors.  units: the terms of the three matrices, the profile-mode
// units of the replicated mode's r1cs.upload and r1cs.eval stages.
struct R1csStart {
    bool split;
    ProveHead head;
    BatchAbcFill fill;
    uint64_t units;
};
int prove_begin_r1cs(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, const R1csStart& start, bb_prove** out);
// bb_groth16_prove after its argument checks: `begin` queues the proof on an unsharded key, the scalar multiplications
// that need no MSM result run on the host meanwhile, then the waits and the finalisation
int prove_single(bb_ctx* ctx, const bb_crs* crs, const std::function<int(bb_prove**)>& begin, const uint8_t* r, const uint8_t* s,
                 uint8_t* proof);
// A single-GPU bb_crs that adopts the five resident vectors h, l, a, b_g1, b_g2 (freed with it); g1 = alpha, beta, delta,
// g2 = beta, delta (bb_params_read)
bb_crs* crs_adopt(bb_ctx* ctx, bb_bases* const vec[5], const G1Affine g1[3], const G2Affine g2[2]);
// What a bb_crs holds (bb_params_write): its context, shard count, the vectors h, l, a, b_g1, b_g2 and g1 = alpha, beta,
// delta, g2 = beta, delta
struct CrsView {
    bb_ctx* ctx;
    uint32_t shard_count;
    const bb_bases* vec[5];
    G1Affine g1[3];
    G2Affine g2[2];
};
CrsView crs_view(const bb_crs* crs);

// ---- verify.cu ----
// A bb_vk that adopts its device parts (context allocations): alpha_g1, the G2 points in the order delta, gamma, beta, and
// the resident ic (bb_params_read, bb_vk_read)
bb_vk* vk_adopt(bb_ctx* ctx, G1Affine* d_alpha, G2Affine* d_g2, bb_bases* ic);
// The device parts of a bb_vk, as vk_adopt takes them (bb_params_write)
struct VkView {
    bb_ctx* ctx;
    const G1Affine* d_alpha;
    const G2Affine* d_g2;
    const bb_bases* ic;
};
VkView vk_view(const bb_vk* vk);

// ---- r1cs.cu ----
// A sparse matrix over Fr as the evaluation kernels read it: row g holds the terms off[g] .. off[g + 1] - 1, each a column
// index (bit 31 set: coefficient one, the product is skipped) and its coefficient (Montgomery).  rows: the row ids binned
// by length, n_short rows of at most R1CS_SHORT_MAX terms (one thread each), then n_warp of at most R1CS_WARP_MAX (one
// warp each), then n_cta longer ones (one CTA each).  Row g of the 3 n goes to out_a[g], out_b[g - n] or out_c[g - 2 n].
constexpr uint32_t R1CS_ONE_FLAG = 0x80000000u, R1CS_SHORT_MAX = 32, R1CS_WARP_MAX = 2048;
struct CsrMatrix {
    const uint32_t* off;
    const uint32_t* idx;
    const Fr* coef;
    const uint32_t* rows;
    uint32_t n_short, n_warp, n_cta;
    uint32_t n;                      // rows per output
};
// out = M x, with x = input (columns < n_inputs) || aux, queued on `st`
int csr_eval_queue(bb_ctx* ctx, cudaStream_t st, const CsrMatrix& M, const Fr* input, uint32_t n_inputs, const Fr* aux, Fr* out_a, Fr* out_b,
                   Fr* out_c);
// A bb_r1cs as it lies in HBM: the one CSR of its 3 n rows (n constraints incl. the input rows, columns = variables)
struct R1csView {
    bb_ctx* ctx;
    size_t n, n_inputs, n_aux;
    uint64_t terms;
    const uint32_t* off;
    const uint32_t* idx;
    const Fr* coef;
};
R1csView r1cs_view(const bb_r1cs* r1cs);

// ---- capi.cu ----
// d_table: NULL = the standard generator's cached table, or a table of fixed_table_build
int fixed_base_mul_device(bb_ctx* ctx, int group, const Fr* d_scalars, size_t n, bool montgomery, void* d_out, cudaStream_t st,
                          const void* d_table = nullptr);
// The byte-multiple table of another generator (96 / 192 B affine, not the identity), built on the host and uploaded;
// the caller zeroes and frees it with fixed_table_free
int fixed_table_build(int group, const void* gen_affine, void** d_table);
void fixed_table_free(int group, void* d_table);

// ---- msm.cu ----
// batch != 0: one job over `batch` scalar vectors (device memory, vector p at scalars + p * scalar_stride) sharing the
// bases, the offset and the density map
int msm_start(bb_ctx* ctx, const bb_bases* bases, size_t base_offset, const uint64_t* density_bits, size_t density_len,
              const void* scalars, bool scalars_on_device, size_t n, int form, cudaEvent_t wait_for, bb_msm_job** out,
              const char* tag = nullptr, int critical = 0, uint32_t batch = 0, size_t scalar_stride = 0);
// Waits for a job and frees it.  For each scalar vector p (one for an unbatched job), status[p] is what bb_msm_wait would
// report for that vector alone, and points[p] (G1X or G2X) its sum where status[p] is BB_OK.  Returns the job-level status
// (a failure before or during the launch, or of the stream), which then stands for every vector.
int msm_wait(bb_msm_job* job, int* status, void* points);
size_t msm_batch_bytes(bb_ctx* ctx, const bb_bases* bases, size_t n, size_t n_dense, uint32_t batch, uint64_t* slots);
int bases_build_table(bb_ctx* ctx, bb_bases* bases);
// vals[i] <- 1 / vals[i] for n NON-ZERO field elements in HBM (Montgomery's trick, fan-in 32, one Fermat inversion);
// scratch: batch_invert_scratch(n) elements
int batch_invert_fp(bb_ctx* ctx, cudaStream_t st, Fp* vals, size_t n, Fp* scratch);
int batch_invert_fp2(bb_ctx* ctx, cudaStream_t st, Fp2* vals, size_t n, Fp2* scratch);
size_t batch_invert_scratch(size_t n);

}  // namespace bb
