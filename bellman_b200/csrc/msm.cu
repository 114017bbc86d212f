// bellman_b200: Pippenger multi-scalar multiplication over BLS12-381 G1/G2 for sm_90a.
//
// Replaces multiexp() / multiexp_inner() (bellman/src/multiexp.rs:210-332).  The
// reference runs one CPU task per c-bit window, each scanning all n scalars and doing a
// projective += affine per non-zero digit (:242-265), then a serial summation by parts
// (:271-275) and a serial Horner fold (:295-300).  Here:
//   1. k_msm_digits   one thread per scalar: canonicalise (Exponent::from, :172-182),
//                     resolve the base index through the density map (:242-243, bases are
//                     compacted to set bits), signed-digit recode into W windows (halves the
//                     bucket count) and histogram the (window, |digit|) keys;
//   2. scan           exclusive prefix sum of the histogram, every count rounded up to a multiple
//                     of 2^R -> padded bucket segments;
//   3. k_msm_digits   again in scatter mode: counting sort of base indices by bucket;
//   4. halving rounds (batch_affine.cuh) x R: inside every bucket entries 0+1, 2+3, ... are added as
//                     AFFINE points; all additions of a round share one inversion (Montgomery's
//                     trick), 6 instead of 10 field multiplications each; R follows the mean fill;
//   5. k_msm_accumulate  one thread per bucket sums what is left (all entries when R = 0) with
//                     XYZZ mixed additions; oversized buckets are cut into tasks;
//   6. bucket reduction  summation by parts (:271-275) in two dimensions (k_bucket_fold: row and
//                     column sums as full-grid trees), then the serial running-sum recursion
//                     (k_msm_reduce_level) only over 2 sqrt(D) entries per window;
//   7. host           Horner fold of the W window sums (255 doublings), to_affine.
// Scalars equal to one (Exponent::One, :246-252) bypass the buckets through a list that is
// summed by a tree, zero scalars (Exponent::Zero, :245) are dropped -- exactly the
// reference's fast paths, kept because real witnesses are dominated by 0/1.
// Error semantics (Source::next / skip, :53-86) are reproduced, see bb_msm_wait.
#include <cmath>
#include <cstdlib>
#include <ctime>

#include "bb_internal.cuh"
#include "batch_affine.cuh"

namespace bb {

struct DigitArgs {
    const Fr* scalars;
    size_t n;
    int montgomery;
    const uint64_t* density;        // NULL = FullDensity
    const uint32_t* density_rank;   // set bits before word j
    uint64_t base_offset;           // Source start position (global)
    uint64_t shard_lo, shard_n;     // this device holds global base indices [shard_lo, shard_lo+shard_n)
    uint64_t global_len;
    uint32_t c, W;
    uint32_t win_index, win_count;  // this device owns windows w with w % win_count == win_index
    uint32_t table_stride;          // precomputed window multiples: entry of window slot s is base index + s * stride; 0 = none
    uint32_t key_stride;            // buckets of window slot s start at s * key_stride: D, or 0 when all windows share ONE bucket set
    uint32_t* counts;               // mode 0: histogram; mode 1: cursors
    uint32_t* sorted;               // mode 1
    uint32_t* ones_list;            // base indices with scalar == 1
    uint32_t* ones_count;
    uint32_t* err;                  // [0] = min scalar index hitting EOF (0xffffffff none), [1] identity base hit,
                                    // [4] scalars that enter the buckets here, [5] bucket entries (digits) -- profile counters
    int mode;
    // a job over B scalar vectors (grid y = proof; one base vector, offset and density map for all of them): vector p
    // starts at scalars + p * scalar_stride and owns the buckets [p * proof_keys, (p + 1) * proof_keys).  With proof_err
    // set, a scalar equal to one is digit 1 of window 0 (no ones list) and an identity base under a non-zero scalar is
    // flagged in proof_err[p] (points: the base vector, point_u4 16-byte words per point).  B = 1 without proof_err is
    // the single job.
    size_t scalar_stride;
    uint32_t proof_keys;
    uint32_t* proof_err;
    const uint4* points;
    uint32_t point_u4;
};

__device__ __forceinline__ uint32_t extract_bits(const uint32_t* l, uint32_t pos, uint32_t c) {
    uint32_t word = pos >> 5, off = pos & 31;
    if (word >= 8) return 0;
    uint64_t v = l[word];
    if (word + 1 < 8) v |= (uint64_t)l[word + 1] << 32;
    return (uint32_t)(v >> off) & ((1u << c) - 1u);
}

__global__ void __launch_bounds__(256) k_msm_digits(DigitArgs A) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t proof = blockIdx.y;
    if (i >= A.n) return;
    uint64_t rank = i;
    if (A.density) {
        uint64_t word = A.density[i >> 6];
        if (!((word >> (i & 63)) & 1)) return;                       // multiexp.rs:243
        rank = (uint64_t)A.density_rank[i >> 6] + __popcll(word & ((1ull << (i & 63)) - 1ull));
    }
    uint64_t gi = A.base_offset + rank;
    if (gi >= A.global_len) {                                        // Source::next/skip EOF, :55-61,74-80
        atomicMin(&A.err[0], (uint32_t)i);
        return;
    }
    if (gi < A.shard_lo || gi >= A.shard_lo + A.shard_n) return;     // another device's shard: its scalar is never read here
    const uint4* q = reinterpret_cast<const uint4*>(A.scalars + (size_t)proof * A.scalar_stride + i);
    uint4 lo = q[0], hi = q[1];
    Fr s;
    s.l[0] = lo.x; s.l[1] = lo.y; s.l[2] = lo.z; s.l[3] = lo.w;
    s.l[4] = hi.x; s.l[5] = hi.y; s.l[6] = hi.z; s.l[7] = hi.w;
    if (A.montgomery) s = fr_to_canonical(s);                        // to_le_bits, :179
    if (s.is_zero()) return;                                         // Exponent::Zero, :245
    uint32_t local = (uint32_t)(gi - A.shard_lo);
    uint32_t rest = s.l[1] | s.l[2] | s.l[3] | s.l[4] | s.l[5] | s.l[6] | s.l[7];
    if (A.proof_err) {                                               // batch: the base is read under every non-zero scalar
        if (A.mode == 0) {
            const uint4* pt = A.points + (size_t)local * A.point_u4;
            uint32_t any = 0;
            for (uint32_t k = 0; k < A.point_u4; k++) { const uint4 v = pt[k]; any |= v.x | v.y | v.z | v.w; }
            if (!any) atomicOr(&A.proof_err[proof], 1u);             // Source::next, multiexp.rs:63-65
        }
    } else if (rest == 0 && s.l[0] == 1) {                           // Exponent::One, :246-252
        if (A.mode == 1 && A.win_index == 0) A.ones_list[atomicAdd(A.ones_count, 1u)] = local;   // window 0's owner
        return;
    }
    const uint32_t D = 1u << (A.c - 1);
    if (A.mode == 0) {                                               // warp-aggregated count of the pairs consumed
        const unsigned live = __activemask();
        if ((threadIdx.x & 31u) == (unsigned)(__ffs((int)live) - 1)) atomicAdd(&A.err[4], (uint32_t)__popc(live));
    }
    uint32_t carry = 0;
    for (uint32_t w = 0; w < A.W; w++) {
        uint32_t raw = extract_bits(s.l, w * A.c, A.c) + carry;
        uint32_t mag, neg;
        if (raw > D) { mag = (1u << A.c) - raw; neg = 1; carry = 1; }
        else { mag = raw; neg = 0; carry = 0; }
        if (mag == 0 || w % A.win_count != A.win_index) continue;   // the carry chain runs over all windows
        const uint32_t slot = w / A.win_count;
        uint32_t key = proof * A.proof_keys + slot * A.key_stride + (mag - 1);
        if (A.mode == 0) atomicAdd(&A.counts[key], 1u);
        else A.sorted[atomicAdd(&A.counts[key], 1u)] = (local + slot * A.table_stride) | (neg << 31);
    }
}

// ---- exclusive scan over the histogram (NB+1 outputs) ---------------------------------
constexpr int SCAN_ITEMS = 8, SCAN_THREADS = 256, SCAN_TILE = SCAN_ITEMS * SCAN_THREADS;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t ws = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, ws, d);
            if (lane >= d) ws += t;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = ws;
    }
    __syncthreads();
    uint32_t prefix = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[SCAN_THREADS / 32 - 1];
    uint32_t res = prefix + inc - v;
    __syncthreads();
    return res;
}

// counts are rounded up to a multiple of pad_mask + 1 on the fly (segments of the batched-affine rounds)
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(const uint32_t* in, uint32_t* out, size_t n, uint32_t* tile_sums, uint32_t pad_mask, uint32_t* raw_total) {
    size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], sum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { v[k] = base + k < n ? ((in[base + k] + pad_mask) & ~pad_mask) : 0; sum += v[k]; }
    if (raw_total) {                                                 // profile counter: entries before padding
        uint32_t raw = 0;
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; k++) raw += base + k < n ? in[base + k] : 0;
        if (raw) atomicAdd(raw_total, raw);
    }
    uint32_t total, ex = block_exclusive_scan(sum, &total);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = ex; ex += v[k]; }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_sums(uint32_t* tile_sums, size_t ntiles) {
    uint32_t running = 0;
    for (size_t base = 0; base < ntiles; base += SCAN_THREADS) {
        size_t i = base + threadIdx.x;
        uint32_t v = i < ntiles ? tile_sums[i] : 0;
        uint32_t total, ex = block_exclusive_scan(v, &total);
        if (i < ntiles) tile_sums[i] = running + ex;
        running += total;
    }
}
// out[i] += tile offset; also writes the grand total at out[n] and copies to cursor
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_finish(uint32_t* out, uint32_t* cursor, size_t n, const uint32_t* tile_sums,
                                                              const uint32_t* in, uint32_t pad_mask) {
    size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t off = tile_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) {
        size_t i = base + k;
        if (i < n) {
            uint32_t cnt = (in[i] + pad_mask) & ~pad_mask;   // `in` aliases `cursor`: read before the overwrite
            uint32_t v = out[i] + off;
            out[i] = v;
            cursor[i] = v;
            if (i == n - 1) out[n] = v + cnt;
        }
    }
}

// ---- bucket order: heaviest first, equal sizes adjacent --------------------------------------
// One thread owns one bucket, so a warp runs as long as its largest bucket: with Poisson-sized
// buckets only ~72% of the lanes do useful work (measured).  Handing the threads buckets in
// order of size (a counting sort over the sizes, three tiny kernels) makes the 32 buckets of a
// warp equally long and schedules the long ones first.
constexpr uint32_t SIZE_BINS = 4096;      // sizes >= SIZE_BINS-1 share the last bin

__global__ void __launch_bounds__(256) k_size_hist(const uint32_t* __restrict__ offsets, size_t nb, uint32_t* size_hist) {
    size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    uint32_t sz = offsets[b + 1] - offsets[b];
    atomicAdd(&size_hist[sz < SIZE_BINS - 1 ? sz : SIZE_BINS - 1], 1u);
}
// size_hist[s] <- first position of size class s in the descending order
__global__ void __launch_bounds__(1024) k_size_scan(uint32_t* size_hist) {
    __shared__ uint32_t sh[SIZE_BINS];
    for (uint32_t i = threadIdx.x; i < SIZE_BINS; i += blockDim.x) sh[i] = size_hist[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t run = 0;
        for (int s = SIZE_BINS - 1; s >= 0; s--) { uint32_t c = sh[s]; sh[s] = run; run += c; }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < SIZE_BINS; i += blockDim.x) size_hist[i] = sh[i];
}
// Oversized buckets (skewed scalars: a witness full of equal small values) are cut into tasks of
// at most `cap` entries so that no single thread owns a long serial chain; big[0] counts tasks,
// big[1] counts oversized buckets.
struct BigTask { uint32_t bucket, begin, end; };
struct BigBucket { uint32_t bucket, first_task, num_tasks; };

__global__ void __launch_bounds__(256) k_size_order(const uint32_t* __restrict__ offsets, size_t nb, uint32_t* size_cursor, uint32_t* order,
                                                     uint32_t cap, uint32_t task_len, uint32_t* big, BigTask* tasks, BigBucket* big_list) {
    size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    uint32_t start = offsets[b], end = offsets[b + 1];
    uint32_t sz = end - start;
    order[atomicAdd(&size_cursor[sz < SIZE_BINS - 1 ? sz : SIZE_BINS - 1], 1u)] = (uint32_t)b;
    if (sz > cap) {
        uint32_t nt = (sz + task_len - 1) / task_len;
        uint32_t first = atomicAdd(&big[0], nt);
        big_list[atomicAdd(&big[1], 1u)] = {(uint32_t)b, first, nt};
        for (uint32_t i = 0; i < nt; i++) {
            uint32_t lo = start + i * task_len, hi = lo + task_len < end ? lo + task_len : end;
            tasks[first + i] = {(uint32_t)b, lo, hi};
        }
    }
}

// ---- bucket accumulation ------------------------------------------------------------------
// DENSE = false: entries k of the sorted index array select rows of the base table (bit 31 = negate).
// DENSE = true:  rows k of the dense array the batched-affine rounds left behind (identity = padding).
template <class F, bool DENSE>
__device__ __forceinline__ XYZZ<F> accumulate_range(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ sorted,
                                                    uint32_t start, uint32_t end, uint32_t* err) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t k = start; k < end; k++) {
        if (DENSE) {
            Affine<F> p = ld_affine(bases + k);
            if (p.is_identity()) continue;
            acc.add_mixed(p);
        } else {
            uint32_t v = sorted[k];
            Affine<F> p = ld_affine(bases + (v & 0x7fffffffu));
            if (p.is_identity()) { atomicOr(&err[1], 1u); continue; }           // Source::next, multiexp.rs:63-65
            if (v >> 31) p.y = p.y.neg();
            acc.add_mixed(p);
        }
    }
    return acc;
}

template <class F, bool DENSE>
__global__ void __launch_bounds__(128) k_msm_accumulate(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ offsets,
                                                        const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ order,
                                                        XYZZ<F>* buckets, size_t nb, uint32_t cap, uint32_t* err) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nb) return;
    const uint32_t b = order[t];
    uint32_t start = offsets[b], end = offsets[b + 1];
    if (end - start > cap) return;                                   // cut into tasks, see k_msm_accumulate_tasks
    XYZZ<F> acc = accumulate_range<F, DENSE>(bases, sorted, start, end, err);
    st_words(buckets + b, acc);
}

// bucket b's rows of the dense array after R halvings of its padded segment
__global__ void __launch_bounds__(256) k_dense_offsets(const uint32_t* __restrict__ offsets, size_t nb1, uint32_t shift, uint32_t* out) {
    size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < nb1) out[b] = offsets[b] >> shift;
}

// one thread per task of an oversized bucket (grid-stride: the task count lives on the device)
template <class F, bool DENSE>
__global__ void __launch_bounds__(128) k_msm_accumulate_tasks(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ sorted,
                                                              const uint32_t* __restrict__ big, const BigTask* __restrict__ tasks,
                                                              XYZZ<F>* task_sums, uint32_t* err) {
    const uint32_t ntasks = big[0];
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < ntasks; t += gridDim.x * blockDim.x) {
        BigTask tk = tasks[t];
        XYZZ<F> acc = accumulate_range<F, DENSE>(bases, sorted, tk.begin, tk.end, err);
        st_words(task_sums + t, acc);
    }
}

// sum of listed bases (scalar == 1): thread-strided partials then CTA tree
template <class F>
__device__ __forceinline__ void block_tree_reduce(XYZZ<F>& acc, XYZZ<F>* sh) {
    // explicit 16-byte word copies (st_words / ld_words) rather than struct assignment: nvcc
    // 12.9 drops the first 16-byte store of `sh[tid] = acc` in k_msm_reduce (seen in SASS)
    st_words(sh + threadIdx.x, acc);
    __syncthreads();
    for (uint32_t stride = blockDim.x / 2; stride > 0; stride >>= 1) {
        if (threadIdx.x < stride) {
            XYZZ<F> a = ld_words(sh + threadIdx.x);
            XYZZ<F> b = ld_words(sh + threadIdx.x + stride);
            a.add(b);
            st_words(sh + threadIdx.x, a);
        }
        __syncthreads();
    }
    acc = ld_words(sh);
}

// bucket = sum of its task sums; one CTA per oversized bucket (grid-stride)
template <class F>
__global__ void __launch_bounds__(128) k_msm_merge_big(const uint32_t* __restrict__ big, const BigBucket* __restrict__ big_list,
                                                       const XYZZ<F>* task_sums, XYZZ<F>* buckets) {
    extern __shared__ uint4 shraw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(shraw);
    const uint32_t nbig = big[1];
    for (uint32_t i = blockIdx.x; i < nbig; i += gridDim.x) {
        BigBucket bb_ = big_list[i];
        XYZZ<F> acc = XYZZ<F>::identity();
        for (uint32_t k = threadIdx.x; k < bb_.num_tasks; k += blockDim.x) acc.add(ld_words(task_sums + bb_.first_task + k));
        block_tree_reduce(acc, sh);
        if (threadIdx.x == 0) st_words(buckets + bb_.bucket, acc);
        __syncthreads();
    }
}

template <class F>
__global__ void __launch_bounds__(128) k_msm_sum_list(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ list,
                                                      const uint32_t* __restrict__ count, XYZZ<F>* partials, uint32_t* err) {
    extern __shared__ uint4 shraw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(shraw);
    uint32_t n = *count;
    XYZZ<F> acc = XYZZ<F>::identity();
    for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
        Affine<F> p = ld_affine(bases + list[k]);
        if (p.is_identity()) { atomicOr(&err[1], 1u); continue; }
        acc.add_mixed(p);
    }
    block_tree_reduce(acc, sh);
    if (threadIdx.x == 0) st_words(partials + blockIdx.x, acc);
}

// out[g] = sum_{k < cnt} in[g*cnt + k]
template <class F>
__global__ void __launch_bounds__(128) k_point_tree_sum(const XYZZ<F>* in, uint32_t cnt, XYZZ<F>* out) {
    extern __shared__ uint4 shraw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(shraw);
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) acc.add(ld_words(in + (size_t)blockIdx.x * cnt + k));
    block_tree_reduce(acc, sh);
    if (threadIdx.x == 0) st_words(out + blockIdx.x, acc);
}

// Summation by parts (multiexp.rs:271-275) in parallel and without scalar multiplications.
// A window's D buckets carry weights 1..D.  Thread j owns K adjacent entries and produces
//   acc_j = sum_t (t + base) * in[jK+t]   (base = 1 on the first level, 0 afterwards)
//   run_j = sum_t in[jK+t]
// so that  sum_d w(d) in[d] = sum_j acc_j + K * sum_j j * run_j : the second term is the same
// problem on the D/K run sums with 0-based weights.  Recursing until one run is left gives
//   S = A_1 + K_1 (A_2 + K_2 (A_3 + ...)),   A_l = sum_j acc_j at level l,
// two additions per bucket in total, every level fully parallel.
template <class F>
__global__ void __launch_bounds__(128) k_msm_reduce_level(const XYZZ<F>* in, uint32_t D_in, uint32_t K, uint32_t one_based_windows,
                                                          XYZZ<F>* run_out, XYZZ<F>* acc_partials) {
    extern __shared__ uint4 shraw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(shraw);
    const uint32_t w = blockIdx.y;
    const uint32_t runs = D_in / K;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    XYZZ<F> acc = XYZZ<F>::identity();
    if (j < runs) {
        const XYZZ<F>* B = in + (size_t)w * D_in + (size_t)j * K;
        XYZZ<F> running = XYZZ<F>::identity();
        for (int t = (int)K - 1; t >= 1; t--) {
            running.add(ld_words(B + t));
            acc.add(running);
        }
        running.add(ld_words(B));
        if (w < one_based_windows) acc.add(running);      // weights t + 1 instead of t
        st_words(run_out + (size_t)w * runs + j, running);
    }
    block_tree_reduce(acc, sh);
    if (threadIdx.x == 0) st_words(acc_partials + (size_t)w * gridDim.x + blockIdx.x, acc);
}

// ---- two-dimensional bucket reduction ---------------------------------------------------------------
// The weights of a window's D buckets are 1..D.  Write the bucket index as d = hi * Lo + lo: then
//   sum_d (d + 1) B_d = sum_lo (lo + 1) C_lo + Lo * sum_hi hi R_hi,
// with the column sums C_lo = sum_hi B[hi][lo] and the row sums R_hi = sum_lo B[hi][lo].  Row and column sums
// are plain sums -- trees of independent additions over the whole array, D additions each, every level a full
// grid -- and only the two short weighted sums (Lo and D / Lo entries per window) are left for the serial
// recursion below.  Same two additions per bucket as the running-sum form (multiexp.rs:271-275), but the long
// dependent chains (2K additions per thread and level over D / K threads) shrink to chains over sqrt(D) entries.
//
// out[w][o] = sum_{k < folds} in[w][a * inner_in + b + k * kstride],  o = a * inner_out + b, b < inner_out
template <class F>
__global__ void __launch_bounds__(128) k_bucket_fold(const XYZZ<F>* in, XYZZ<F>* out, uint32_t n_out, uint32_t in_window, uint32_t out_window,
                                                     uint32_t inner_out, uint32_t inner_in, uint32_t kstride, uint32_t folds) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x, w = blockIdx.y;
    if (o >= n_out) return;
    const uint32_t a = o / inner_out, b = o - a * inner_out;
    const XYZZ<F>* src = in + (size_t)w * in_window + (size_t)a * inner_in + b;
    XYZZ<F> acc = ld_words(src);
    for (uint32_t k = 1; k < folds; k++) acc.add(ld_words(src + (size_t)k * kstride));
    st_words(out + (size_t)w * out_window + o, acc);
}
// out[w] = sc[w] + 2^shift * sr[w]
template <class F>
__global__ void __launch_bounds__(32) k_bucket_fold_combine(const XYZZ<F>* sums, uint32_t W, uint32_t shift, XYZZ<F>* out) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    XYZZ<F> r = ld_words(sums + W + w);
    for (uint32_t k = 0; k < shift; k++) r = r.dbl();
    r.add(ld_words(sums + w));
    st_words(out + w, r);
}

// S_w = A_1[w] + K_1 (A_2[w] + K_2 (A_3[w] + ...)); level sums are stored level-major: A[l*W + w]
struct ReduceLevels { uint32_t n; uint32_t logk[12]; uint32_t nblk[12]; uint32_t part_off[12]; };

// level_sums[l*W + w] = sum of the nblk[l] CTA partials of window w at level l; grid (W, levels)
template <class F>
__global__ void __launch_bounds__(128) k_msm_level_sums(const XYZZ<F>* partials, uint32_t W, ReduceLevels L, XYZZ<F>* level_sums) {
    extern __shared__ uint4 shraw[];
    XYZZ<F>* sh = reinterpret_cast<XYZZ<F>*>(shraw);
    const uint32_t w = blockIdx.x, l = blockIdx.y, cnt = L.nblk[l];
    const XYZZ<F>* in = partials + L.part_off[l] + (size_t)w * cnt;
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t k = threadIdx.x; k < cnt; k += blockDim.x) acc.add(ld_words(in + k));
    block_tree_reduce(acc, sh);
    if (threadIdx.x == 0) st_words(level_sums + (size_t)l * W + w, acc);
}
template <class F>
__global__ void __launch_bounds__(32) k_msm_reduce_combine(const XYZZ<F>* level_sums, uint32_t W, ReduceLevels L, XYZZ<F>* out) {
    uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    XYZZ<F> s = ld_words(level_sums + (size_t)(L.n - 1) * W + w);
    for (int l = (int)L.n - 2; l >= 0; l--) {
        for (uint32_t k = 0; k < L.logk[l]; k++) s = s.dbl();
        s.add(ld_words(level_sums + (size_t)l * W + w));
    }
    st_words(out + w, s);
}

// ---- precomputed window multiples ---------------------------------------------------------------
// The CRS is fixed and fills a small part of the 80 GB of HBM (430 MB at 2^20 constraints), so every base vector can keep
// T[s][i] = 2^(c w_s) P_i for each window it owns.  A digit of window w then selects T[w][i] and all
// windows accumulate into buckets of the SAME weights, so the summation by parts and the Horner fold run
// once instead of W times.  Two forms:
//   msm_precompute = 1  one bucket array per window slot, added slot-wise afterwards (k_msm_fold_slots);
//   msm_precompute = 2  ONE bucket array: the digits of every window are sorted into the same D buckets
//                       (key = |digit| - 1).  A bucket then holds W times as many entries, which is what the
//                       batched-affine halving rounds want: R follows the fill (6 rounds at 2^20 scalars and
//                       c = 16), the XYZZ stage is left with a handful of rows per bucket and the bucket
//                       reduction with D instead of W D buckets.
template <class F>
__global__ void __launch_bounds__(128) k_table_multiples(const Affine<F>* __restrict__ pts, size_t n, uint32_t c, uint32_t W,
                                                         uint32_t wi, uint32_t wc, XYZZ<F>* scratch) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    XYZZ<F> cur = XYZZ<F>::from_affine(ld_affine(pts + i));
    for (uint32_t w = 0; w < W; w++) {
        if (w % wc == wi) st_words(scratch + (size_t)(w / wc) * n + i, cur);
        if (w + 1 < W)
            for (uint32_t k = 0; k < c; k++) cur = cur.dbl();
    }
}
// scratch (XYZZ) -> table (affine): one inversion per thread shared by its `slots` points
// (Montgomery's trick; the prefix products are parked in the x slot of the output)
template <class F>
__global__ void __launch_bounds__(128) k_table_normalize(const XYZZ<F>* __restrict__ scratch, size_t n, uint32_t slots, Affine<F>* table,
                                                         size_t table_n, size_t table_off) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F acc = FieldOps<F>::one();
    for (uint32_t s = 0; s < slots; s++) {
        F z = ld_words(&scratch[(size_t)s * n + i].ZZZ);
        st_words(&table[(size_t)s * table_n + table_off + i].x, acc);
        if (!z.is_zero()) acc = acc * z;
    }
    F inv = FieldOps<F>::inv(acc);
    for (int s = (int)slots - 1; s >= 0; s--) {
        XYZZ<F> P = ld_words(scratch + (size_t)s * n + i);
        Affine<F>* dst = table + (size_t)s * table_n + table_off + i;
        if (P.is_identity()) { st_words(dst, Affine<F>::identity()); continue; }
        F pre = ld_words(&dst->x);
        F zi3 = inv * pre;
        inv = inv * P.ZZZ;
        F zi2 = (zi3 * P.ZZ).sqr();
        Affine<F> a{P.X * zi2, P.Y * zi3};
        st_words(dst, a);
    }
}
// out[p][d] = buckets[p][0][d] + buckets[p][1][d] + ... + buckets[p][slots-1][d]  (p = blockIdx.y; out may be buckets
// itself when there is one proof)
template <class F>
__global__ void __launch_bounds__(128) k_msm_fold_slots(const XYZZ<F>* buckets, uint32_t slots, uint32_t D, XYZZ<F>* out) {
    uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    const XYZZ<F>* in = buckets + (size_t)blockIdx.y * slots * D;
    XYZZ<F> acc = ld_words(in + d);
    for (uint32_t s = 1; s < slots; s++) acc.add(ld_words(in + (size_t)s * D + d));
    st_words(out + (size_t)blockIdx.y * D + d, acc);
}

// Horner fold of each proof's W window sums (multiexp.rs:295-300) on the device: out[p] = sum_w 2^(c w) win[p * W + w].
// One thread per proof vector of a batched job; only these B points cross the bus.
template <class F>
__global__ void __launch_bounds__(32) k_msm_fold_windows(const XYZZ<F>* win, uint32_t B, uint32_t W, uint32_t c, XYZZ<F>* out) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= B) return;
    const XYZZ<F>* w = win + (size_t)p * W;
    XYZZ<F> acc = ld_words(w + W - 1);
    for (int k = (int)W - 2; k >= 0; k--) {
        for (uint32_t d = 0; d < c; d++) acc = acc.dbl();
        acc.add(ld_words(w + k));
    }
    st_words(out + p, acc);
}

// Error classification when BOTH an EOF and an identity base were seen: the reference folds
// window results from the top window down (multiexp.rs:295-300), so the error reported is the
// top window's, and that window raises UnexpectedIdentity only for an identity base whose
// digit *in that window* (window size c_ref = ceil(ln n), :318-322) is non-zero and that is
// consumed before the bases run out.  Finds the first such scalar index.
template <class F>
__global__ void __launch_bounds__(256) k_msm_classify(DigitArgs A, const Affine<F>* bases, uint32_t c_ref, uint32_t top_chunk,
                                                      uint32_t* first_top_identity) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    uint64_t rank = i;
    if (A.density) {
        uint64_t word = A.density[i >> 6];
        if (!((word >> (i & 63)) & 1)) return;
        rank = (uint64_t)A.density_rank[i >> 6] + __popcll(word & ((1ull << (i & 63)) - 1ull));
    }
    uint64_t gi = A.base_offset + rank;
    if (gi >= A.global_len || gi < A.shard_lo || gi >= A.shard_lo + A.shard_n) return;
    Fr s = *(A.scalars + i);
    if (A.montgomery) s = fr_to_canonical(s);
    if (s.is_zero()) return;
    uint32_t rest = s.l[1] | s.l[2] | s.l[3] | s.l[4] | s.l[5] | s.l[6] | s.l[7];
    bool one = rest == 0 && s.l[0] == 1;
    bool hit = one ? (top_chunk == 0) : (extract_bits(s.l, top_chunk * c_ref, c_ref) != 0);
    if (!hit) return;
    Affine<F> p = ld_affine(bases + (gi - A.shard_lo));
    if (p.is_identity()) atomicMin(first_top_identity, (uint32_t)i);
}

}  // namespace bb

using namespace bb;

// ----------------------------------------------------------------------------------------------
struct bb_msm_job {
    bb_ctx* ctx = nullptr;
    const bb_bases* bases = nullptr;
    cudaStream_t st = nullptr;
    int group = BB_G1;
    uint32_t c = 0, W = 0, D = 0;   // W = windows of the whole scalar
    uint32_t W_local = 0;            // windows this device owns (all of them unless window-sharded)
    uint32_t W_out = 0;              // window sums copied back: W_local, or 1 with precomputed window multiples
    bool precomp = false;
    bool unified = false;            // precomp and every window's digits go to ONE set of D buckets (msm_precompute = 2)
    uint32_t affine_rounds = 0;      // batched-affine halving rounds before the XYZZ stage
    size_t n = 0;
    size_t n_dense = 0;              // scalars the density map selects (= n for FullDensity): what can reach the buckets
    uint32_t B = 1;                  // scalar vectors (proofs) of a batched job
    bool batched = false;            // per-proof error words and a device fold: h_out = [B points][err 8 words][B words]
    int status = BB_OK;              // pre-launch failure, reported at wait()
    const char* tag = nullptr;       // profile mode: name of this job in the prover's timeline
    DigitArgs dargs{};
    DevBuf d_scalars, d_density, d_rank, d_counts, d_offsets, d_tiles, d_sorted, d_order, d_buckets, d_partials, d_runs, d_levels, d_onesp, d_final, d_ones, d_err, d_big, d_tasks, d_biglist, d_tasksums, d_aff0, d_aff1, d_pre, d_tp, d_doffsets, d_fold, d_slotsum, d_perr, d_folded;
    std::vector<uint32_t> h_rank;
    void* h_out = nullptr;           // pinned: [W window sums][1 ones sum] then err[4]
    size_t h_out_bytes = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // profile: job start, accumulate start/end, job end
    cudaEvent_t ev_done = nullptr;   // blocking-sync event behind the result copy: the waiting host thread sleeps instead of spinning
};

namespace {

uint32_t choose_window(bb_ctx* ctx, size_t n) {
    if (ctx->opt_msm_window_bits >= 2 && ctx->opt_msm_window_bits <= 24) return (uint32_t)ctx->opt_msm_window_bits;
    // Signed-digit windows of c bits: W = floor(255/c)+1 windows, the top one holding only
    // tb = 255 - (W-1)c scalar bits.  Window sizes whose top window has only a few live buckets
    // (c = 13, 14, 18, 19, 21: tb = 8, 3, 3, 8, 3) do badly even with the oversized-bucket path, so
    // the choice is restricted to 8 (tb 7), 15 and 17 (tb 0: the top window is the carry alone, a
    // single bucket that the task path sums as a tree) and 16 (tb 15).  Measured on an H100 SXM
    // (80 GB HBM3, 700 W; bench.py --workload msm --autotune 0 --window-bits):
    // 2^20: c=15 10.4 ms, c=16 10.8, c=17 11.2 (the whole 2^20 prove: c=15 and c=16 both 59.2 ms);
    // 2^24: c=16 117.5, c=17 115.5, c=20 128.0.
    if (n < 32) return 4;
    if (n < (1u << 13)) return 8;
    if (n < (1u << 19)) return 15;
    if (n < (1u << 23)) return 16;
    return 17;
}

// Runs the multi-level bucket reduction for W windows of D buckets; window sums -> out[0..W)
template <class F>
int reduce_buckets(bb_ctx* ctx, cudaStream_t st, const XYZZ<F>* buckets, uint32_t W, uint32_t D, uint32_t K0, uint32_t K1,
                   DevBuf& d_runs, DevBuf& d_partials, DevBuf& d_levels, XYZZ<F>* out, uint32_t one_based_windows = 0xffffffffu) {
    struct Level { uint32_t D_in, K, runs, nblk; };
    std::vector<Level> lv;
    for (uint32_t d = D;;) {
        uint32_t Kl = lv.empty() ? K1 : K0;
        uint32_t K = Kl < d ? Kl : d;
        uint32_t runs = d / K;
        lv.push_back({d, K, runs, (runs + 127) / 128});
        if (runs == 1) break;
        d = runs;
    }
    if (lv.size() > 12) { set_error("bucket reduction: too many levels"); return BB_ERR_ARG; }
    size_t run_total = 0, part_total = 0;
    for (auto& l : lv) { run_total += (size_t)W * l.runs; part_total += (size_t)W * l.nblk; }
    BB_TRY(d_runs.alloc(ctx, run_total * sizeof(XYZZ<F>)));
    BB_TRY(d_partials.alloc(ctx, part_total * sizeof(XYZZ<F>)));
    BB_TRY(d_levels.alloc(ctx, lv.size() * W * sizeof(XYZZ<F>)));
    const size_t sh = 128 * sizeof(XYZZ<F>);
    if (sh > 48 * 1024) {
        BB_CUDA(cudaFuncSetAttribute(k_msm_reduce_level<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
        BB_CUDA(cudaFuncSetAttribute(k_msm_level_sums<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
        BB_CUDA(cudaFuncSetAttribute(k_point_tree_sum<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    }
    const XYZZ<F>* in = buckets;
    XYZZ<F>* runs = d_runs.as<XYZZ<F>>();
    XYZZ<F>* parts = d_partials.as<XYZZ<F>>();
    XYZZ<F>* levels = d_levels.as<XYZZ<F>>();
    ReduceLevels RL{};
    RL.n = (uint32_t)lv.size();
    size_t part_off = 0;
    for (size_t l = 0; l < lv.size(); l++) {
        const Level& L = lv[l];
        k_msm_reduce_level<F><<<dim3(L.nblk, W), 128, sh, st>>>(in, L.D_in, L.K, l == 0 ? one_based_windows : 0u, runs, parts + part_off);
        ctx->count_launch();
        uint32_t lg = 0;
        while ((1u << lg) < L.K) lg++;
        RL.logk[l] = lg;
        RL.nblk[l] = L.nblk;
        RL.part_off[l] = (uint32_t)part_off;
        in = runs;
        runs += (size_t)W * L.runs;
        part_off += (size_t)W * L.nblk;
    }
    k_msm_level_sums<F><<<dim3(W, RL.n), 128, sh, st>>>(parts, W, RL, levels);
    ctx->count_launch();
    k_msm_reduce_combine<F><<<cdiv(W, 32), 32, 0, st>>>(levels, W, RL, out);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

// Window sums of W windows of D buckets each (XYZZ, CLOBBERED).  Large windows go through the two-dimensional
// form: row sums into `fold`, column sums in place, then one run of the serial recursion over 2 W short arrays.
template <class F>
int reduce_buckets_2d(bb_ctx* ctx, cudaStream_t st, XYZZ<F>* buckets, uint32_t W, uint32_t D, uint32_t K0, uint32_t K1,
                      DevBuf& d_fold, DevBuf& d_runs, DevBuf& d_partials, DevBuf& d_levels, XYZZ<F>* out) {
    uint32_t lg = 0;
    while ((1u << lg) < D) lg++;
    if (D < 1024 || (1u << lg) != D) return reduce_buckets<F>(ctx, st, buckets, W, D, K0, K1, d_runs, d_partials, d_levels, out);
    const uint32_t lo_bits = (lg + 1) / 2, Lo = 1u << lo_bits, H = D >> lo_bits;       // Lo >= H
    // small[0..W) = column sums (Lo each, weights lo + 1), small[W..2W) = row sums (H each, padded to Lo, weights hi)
    BB_TRY(d_fold.alloc(ctx, ((size_t)W * D / 2 + (size_t)W * D / 4 + (size_t)2 * W * Lo + 2 * (size_t)W) * sizeof(XYZZ<F>)));
    XYZZ<F>* rowbuf[2] = {d_fold.as<XYZZ<F>>(), d_fold.as<XYZZ<F>>() + (size_t)W * D / 2};
    XYZZ<F>* small = rowbuf[1] + (size_t)W * D / 4;
    XYZZ<F>* sums = small + (size_t)2 * W * Lo;
    auto folds_of = [](uint32_t len) { return len % 4 == 0 && len >= 4 ? 4u : 2u; };
    // rows first (they read the untouched buckets): [H][Lo] -> [H][Lo / f] -> ... -> [H][1]; a row fold
    // compacts the rows, so it cannot run in place: two scratch buffers take turns
    {
        const XYZZ<F>* in = buckets;
        uint32_t in_window = D, len = Lo, turn = 0;
        while (len > 1) {
            const uint32_t f = folds_of(len), nl = len / f, n_out = H * nl;
            const bool last = nl == 1;
            XYZZ<F>* dst = last ? small + (size_t)W * Lo : rowbuf[turn];
            const uint32_t out_window = last ? Lo : n_out;
            k_bucket_fold<F><<<dim3(cdiv(n_out, 128), W), 128, 0, st>>>(in, dst, n_out, in_window, out_window, nl, len, nl, f);
            ctx->count_launch();
            in = dst; in_window = out_window; len = nl; turn ^= 1u;
        }
        if (H < Lo) BB_CUDA(cudaMemset2DAsync(small + (size_t)W * Lo + H, (size_t)Lo * sizeof(XYZZ<F>), 0, (size_t)(Lo - H) * sizeof(XYZZ<F>), W, st));   // identity padding
    }
    // columns in place: [H][Lo] -> [H / f][Lo] -> ... -> [1][Lo]
    {
        uint32_t rows = H;
        XYZZ<F>* cur = buckets;
        uint32_t in_window = D;
        while (rows > 1) {
            const uint32_t f = folds_of(rows), nr = rows / f, n_out = nr * Lo;
            const bool last = nr == 1;
            XYZZ<F>* dst = last ? small : cur;
            const uint32_t out_window = last ? Lo : in_window;
            k_bucket_fold<F><<<dim3(cdiv(n_out, 128), W), 128, 0, st>>>(cur, dst, n_out, in_window, out_window, n_out, n_out, n_out, f);
            ctx->count_launch();
            cur = dst; in_window = out_window; rows = nr;
        }
        if (H == 1) BB_CUDA(cudaMemcpy2DAsync(small, (size_t)Lo * sizeof(XYZZ<F>), buckets, (size_t)D * sizeof(XYZZ<F>), (size_t)Lo * sizeof(XYZZ<F>), W, cudaMemcpyDeviceToDevice, st));
    }
    BB_TRY(reduce_buckets<F>(ctx, st, small, 2 * W, Lo, K0, K1, d_runs, d_partials, d_levels, sums, W));
    k_bucket_fold_combine<F><<<cdiv(W, 32), 32, 0, st>>>(sums, W, lo_bits, out);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

// BB_TRACE=1: synchronise after every stage and report it (debugging aid, off the hot path)
static bool trace_on() { static int v = -1; if (v < 0) v = getenv("BB_TRACE") ? 1 : 0; return v == 1; }
#define BB_STAGE(name)                                                                            \
    do {                                                                                          \
        if (trace_on()) {                                                                         \
            cudaError_t e_ = cudaStreamSynchronize(st);                                           \
            struct timespec ts_; clock_gettime(CLOCK_MONOTONIC, &ts_);                            \
            fprintf(stderr, "[bb trace %8.3f] msm n=%zu c=%u W=%u %-12s %s\n", ts_.tv_sec % 1000 + ts_.tv_nsec * 1e-9, job->n, job->c, job->W, name, cudaGetErrorString(e_)); \
            fflush(stderr);                                                                       \
        }                                                                                         \
    } while (0)

// ---- upper levels of the batch inversion (batch_affine.cuh) ------------------------------------------
template <class F>
__device__ __forceinline__ void tile_scans(F v, uint32_t cnt, F* sh, F* pre_out, F* suf_out, F* total) {
    const uint32_t t = threadIdx.x;
    // inclusive prefix products
    st_words(sh + t, v);
    __syncthreads();
    F acc = v;
    for (uint32_t d = 1; d < BINV_TILE; d <<= 1) {
        F other = acc;
        const bool take = t >= d && t < cnt;
        if (take) other = ld_words(sh + t - d);
        __syncthreads();
        if (take) { acc = other * acc; st_words(sh + t, acc); }
        __syncthreads();
    }
    *total = ld_words(sh + cnt - 1);
    *pre_out = t == 0 ? FieldOps<F>::one() : ld_words(sh + (t < cnt ? t : cnt) - 1);
    __syncthreads();
    // inclusive suffix products
    st_words(sh + t, v);
    __syncthreads();
    acc = v;
    for (uint32_t d = 1; d < BINV_TILE; d <<= 1) {
        F other = acc;
        const bool take = t + d < cnt;
        if (take) other = ld_words(sh + t + d);
        __syncthreads();
        if (take) { acc = acc * other; st_words(sh + t, acc); }
        __syncthreads();
    }
    *suf_out = t + 1 < cnt ? ld_words(sh + t + 1) : FieldOps<F>::one();
    __syncthreads();
}

template <class F>
__global__ void __launch_bounds__(BINV_TILE) k_binv_scan_up(const F* __restrict__ vals, size_t n, F* __restrict__ pre, F* __restrict__ suf,
                                                            F* __restrict__ up) {
    extern __shared__ uint4 shraw[];
    F* sh = reinterpret_cast<F*>(shraw);
    const size_t base = (size_t)blockIdx.x * BINV_TILE;
    const uint32_t cnt = n - base < BINV_TILE ? (uint32_t)(n - base) : BINV_TILE;
    const size_t i = base + threadIdx.x;
    F v = threadIdx.x < cnt ? ld_words(vals + i) : FieldOps<F>::one();
    F p, q, tot;
    tile_scans<F>(v, cnt, sh, &p, &q, &tot);
    if (threadIdx.x < cnt) { st_words(pre + i, p); st_words(suf + i, q); }
    if (threadIdx.x == 0) st_words(up + blockIdx.x, tot);
}
// up[tile] now holds 1 / (product of the tile): vals[i] <- up * pre[i] * suf[i] = 1 / vals[i]
template <class F>
__global__ void __launch_bounds__(BINV_TILE) k_binv_scan_down(F* __restrict__ vals, size_t n, const F* __restrict__ pre, const F* __restrict__ suf,
                                                              const F* __restrict__ up) {
    const size_t i = (size_t)blockIdx.x * BINV_TILE + threadIdx.x;
    if (i >= n) return;
    st_words(vals + i, ld_words(up + blockIdx.x) * (ld_words(pre + i) * ld_words(suf + i)));
}
// top: at most BINV_TILE elements left, one CTA: scans, ONE inversion (Fermat, thread 0), back-substitution
template <class F>
__global__ void __launch_bounds__(BINV_TILE) k_binv_top(F* vals, uint32_t n) {
    extern __shared__ uint4 shraw[];
    F* sh = reinterpret_cast<F*>(shraw);
    __shared__ F inv_total;
    F v = threadIdx.x < n ? ld_words(vals + threadIdx.x) : FieldOps<F>::one();
    F p, q, tot;
    tile_scans<F>(v, n, sh, &p, &q, &tot);
    if (threadIdx.x == 0) inv_total = FieldOps<F>::inv(tot);
    __syncthreads();
    if (threadIdx.x < n) st_words(vals + threadIdx.x, inv_total * (p * q));
}

// vals[i] <- 1 / vals[i] for n non-zero field elements (batch_affine.cuh); scratch: batch_invert_scratch_elems(n)
template <class F>
int batch_invert_device(bb_ctx* ctx, cudaStream_t st, F* vals, size_t n, F* scratch) {
    if (!n) return BB_OK;
    const size_t sh = BINV_TILE * sizeof(F);
    // level 0 -> 1: serial fan-in 32 per thread (work-efficient: this is the big level); above: tile scans
    struct Lv { F* vals; F* pre; F* suf; size_t n; };
    std::vector<Lv> lv;
    F* p = scratch;
    lv.push_back({vals, p, nullptr, n});
    p += n;
    if (n > BINV_TILE) {
        size_t m = (n + BINV_FAN - 1) / BINV_FAN;
        lv.push_back({p, p + m, p + 2 * m, m});
        p += 3 * m;
        while (m > BINV_TILE) {
            m = (m + BINV_TILE - 1) / BINV_TILE;
            lv.push_back({p, p + m, p + 2 * m, m});
            p += 3 * m;
        }
        k_binv_up<F><<<cdiv(lv[1].n, 128), 128, 0, st>>>(lv[0].vals, lv[0].n, lv[0].pre, lv[1].vals);
        ctx->count_launch();
        for (size_t l = 1; l + 1 < lv.size(); l++) {
            k_binv_scan_up<F><<<(unsigned)lv[l + 1].n, BINV_TILE, sh, st>>>(lv[l].vals, lv[l].n, lv[l].pre, lv[l].suf, lv[l + 1].vals);
            ctx->count_launch();
        }
    }
    k_binv_top<F><<<1, BINV_TILE, sh, st>>>(lv.back().vals, (uint32_t)lv.back().n);
    ctx->count_launch();
    if (lv.size() > 1) {
        for (size_t l = lv.size() - 2; l >= 1; l--) {
            k_binv_scan_down<F><<<(unsigned)lv[l + 1].n, BINV_TILE, 0, st>>>(lv[l].vals, lv[l].n, lv[l].pre, lv[l].suf, lv[l + 1].vals);
            ctx->count_launch();
        }
        k_binv_down<F><<<cdiv(lv[1].n, 128), 128, 0, st>>>(lv[0].vals, lv[0].n, lv[0].pre, lv[1].vals);
        ctx->count_launch();
    }
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

// How many batched-affine halving rounds an MSM gets: each round needs its own inversion chain
// (~0.5 ms of latency), so small jobs and thinly filled buckets keep the plain XYZZ path.
// Padding a bucket to 2^R entries costs (2^R - 1) / 2 null entries on average, so R follows the mean fill
// (measured on the 2^20 prove: R = 2 beats R = 3 at 16 entries per bucket, R = 3 wins from 32).
uint32_t choose_affine_rounds(const bb_ctx* ctx, size_t pairs, uint64_t entries, size_t NB, bool unified) {
    if (ctx->opt_msm_affine_rounds >= 0) return (uint32_t)(ctx->opt_msm_affine_rounds > 8 ? 8 : ctx->opt_msm_affine_rounds);
    if (unified) {
        // one bucket set for all windows: there is one thread per bucket in the XYZZ stage and only D of them, so
        // the rounds go on until about eight rows per bucket are left (round(log2 fill) - msm_unified_rows_log, at most 8)
        if (pairs < (1u << 13)) return 0;
        const uint64_t fill = entries / (NB ? NB : 1);
        uint32_t lg = 0;                                 // log2 of the fill, rounded to the nearest power of two
        while (((fill + fill / 2) >> (lg + 1)) != 0) lg++;
        const uint32_t keep = ctx->opt_msm_unified_rows_log < 0 ? 0u : (uint32_t)ctx->opt_msm_unified_rows_log;
        return lg <= keep ? 0u : (lg - keep > 8 ? 8u : lg - keep);
    }
    // every round puts an inversion chain (~0.3 ms of dependent latency) on the job's critical path: a job
    // whose whole accumulation is shorter than that (a small shard of a multi-GPU prove) keeps the XYZZ kernel
    if (pairs < (1u << 15) || entries < (3u << 20)) return 0;
    const uint64_t avg = entries / (NB ? NB : 1);
    if (avg >= 24) return 3;
    if (avg >= 10) return 2;
    if (avg >= 5) return 1;
    return 0;
}

// The form, window and bucket layout of a job over B vectors of n scalars (n_dense selected by the density map): what
// msm_start and launch_msm run, and what msm_batch_bytes estimates.  table_on_use: count a table that msm_start would
// build on first use as present.
struct MsmPlan { bool precomp, unified; uint32_t c, W, W_local, D, Wb, R; uint64_t NB, slots; };
MsmPlan msm_plan(bb_ctx* ctx, const bb_bases* bases, bool table_on_use, size_t n, size_t n_dense, uint32_t B) {
    MsmPlan p{};
    const bool tables_wanted = ctx->opt_msm_precompute && (ctx->opt_msm_precompute_groups & (bases->group == BB_G1 ? 1 : 2));
    const bool table = bases->d_table != nullptr || (table_on_use && tables_wanted && bases->n);
    p.precomp = table && (tables_wanted || !ctx->opt_msm_precompute);   // a table built by hand (bb_bases_precompute) is used as it is
    p.unified = p.precomp && ctx->opt_msm_precompute >= 2;
    p.c = p.precomp ? (bases->d_table ? bases->tab_c : choose_window(ctx, bases->n)) : choose_window(ctx, n < bases->n + 1 ? n : bases->n + 1);
    p.W = 255 / p.c + 1;
    p.D = 1u << (p.c - 1);
    const uint32_t wc = bases->win_count ? bases->win_count : 1;
    for (uint32_t w = 0; w < p.W; w++) p.W_local += (w % wc == bases->win_index);
    if (p.W_local == 0) p.W_local = 1;          // degenerate: more shards than windows; slot stays empty
    p.Wb = p.unified ? 1u : p.W_local;
    p.NB = (uint64_t)B * p.Wb * p.D;
    p.R = p.precomp && !p.unified ? 0u : choose_affine_rounds(ctx, n_dense * B, (uint64_t)n_dense * p.W_local * B, p.NB, p.unified);
    p.slots = (uint64_t)n * p.W_local * B + p.NB * ((1u << p.R) - 1u);
    return p;
}

template <class F>
int launch_msm(bb_msm_job* job) {
    NvtxRange range(job->tag ? job->tag : "bb: msm job");
    bb_ctx* ctx = job->ctx;
    cudaStream_t st = job->st;
    const MsmPlan plan = msm_plan(ctx, job->bases, false, job->n, job->n_dense, job->B);
    const uint32_t W = job->W_local, D = job->D;   // everything below works on the owned windows only
    const uint32_t Wb = plan.Wb;                    // bucket sets: one per window, or one for all of them
    const uint32_t B = job->B;                      // proofs: B consecutive groups of Wb bucket sets
    const size_t NB = plan.NB;
    const size_t n = job->n;
    const uint32_t R = plan.R;                      // halving rounds; every bucket is padded to 2^R entries
    const uint32_t pad_mask = (1u << R) - 1u;
    const uint64_t slots = plan.slots;              // one entry per non-zero digit at most, plus the padding
    if (slots >= (1ull << 32)) { set_error("bb_msm: %u x %zu scalars x %u windows exceed 2^32 bucket entries; split the job", B, n, W); return BB_ERR_ARG; }
    job->affine_rounds = R;
    BB_TRY(job->d_counts.alloc(ctx, (NB + 1) * 4));
    BB_TRY(job->d_offsets.alloc(ctx, (NB + 1) * 4));
    size_t ntiles = (NB + SCAN_TILE - 1) / SCAN_TILE;
    BB_TRY(job->d_tiles.alloc(ctx, ntiles * 4));
    BB_TRY(job->d_sorted.alloc(ctx, (slots ? slots : 1) * 4));
    BB_TRY(job->d_ones.alloc(ctx, (n + 4) * 4));
    BB_TRY(job->d_err.alloc(ctx, 32));
    BB_TRY(job->d_buckets.alloc(ctx, NB * sizeof(XYZZ<F>)));
    BB_TRY(job->d_order.alloc(ctx, (NB + SIZE_BINS) * 4));
    const uint32_t ONES_BLOCKS = 64;
    BB_TRY(job->d_final.alloc(ctx, ((size_t)B * Wb + 1) * sizeof(XYZZ<F>) + 16));
    if (job->batched) BB_TRY(job->d_perr.alloc(ctx, (size_t)B * 4));

    BB_CUDA(cudaMemsetAsync(job->d_counts.p, 0, (NB + 1) * 4, st));
    BB_CUDA(cudaMemsetAsync(job->d_err.p, 0xff, 4, st));
    BB_CUDA(cudaMemsetAsync((char*)job->d_err.p + 4, 0, 28, st));
    BB_CUDA(cudaMemsetAsync(job->d_ones.p, 0, 4, st));
    if (R) BB_CUDA(cudaMemsetAsync(job->d_sorted.p, 0xff, slots * 4, st));      // AFF_NULL padding
    if (job->batched) BB_CUDA(cudaMemsetAsync(job->d_perr.p, 0, (size_t)B * 4, st));

    const bool prof = ctx->opt_profile != 0;
    if (prof) {
        for (auto& e : job->ev) BB_CUDA(cudaEventCreate(&e));
        BB_CUDA(cudaEventRecord(job->ev[0], st));
    }
    DigitArgs& A = job->dargs;
    A.counts = job->d_counts.as<uint32_t>();
    A.sorted = job->d_sorted.as<uint32_t>();
    A.ones_count = job->d_ones.as<uint32_t>();
    A.ones_list = job->d_ones.as<uint32_t>() + 4;
    A.err = job->d_err.as<uint32_t>();
    A.proof_keys = (uint32_t)((size_t)Wb * D);
    A.proof_err = job->batched ? job->d_perr.as<uint32_t>() : nullptr;
    A.points = (const uint4*)job->bases->d_points;
    A.point_u4 = (uint32_t)(sizeof(Affine<F>) / 16);
    BB_STAGE("setup");
    if (n) {
        A.mode = 0;
        k_msm_digits<<<dim3(cdiv(n, 256), B), 256, 0, st>>>(A);
        ctx->count_launch();
    }
    BB_STAGE("histogram");
    uint32_t* offsets = job->d_offsets.as<uint32_t>();
    k_scan_tiles<<<(unsigned)ntiles, SCAN_THREADS, 0, st>>>(A.counts, offsets, NB, job->d_tiles.as<uint32_t>(), pad_mask, A.err + 5);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(job->d_tiles.as<uint32_t>(), ntiles);
    // cursors live in the histogram buffer: after this kernel counts[] holds bucket starts
    k_scan_finish<<<(unsigned)ntiles, SCAN_THREADS, 0, st>>>(offsets, A.counts, NB, job->d_tiles.as<uint32_t>(), A.counts, pad_mask);
    ctx->count_launch(3);
    BB_STAGE("scan");
    if (n) {
        A.mode = 1;
        k_msm_digits<<<dim3(cdiv(n, 256), B), 256, 0, st>>>(A);
        ctx->count_launch();
    }
    BB_STAGE("scatter");
    const Affine<F>* bases = (const Affine<F>*)(job->precomp ? job->bases->d_table : job->bases->d_points);
    if (prof) BB_CUDA(cudaEventRecord(job->ev[1], st));

    // ---- batched-affine halving rounds: offsets[NB] padded entries -> offsets[NB] >> R dense rows
    const Affine<F>* dense = nullptr;
    if (R) {
        const uint32_t L = ctx->opt_msm_affine_batch >= 1 && ctx->opt_msm_affine_batch <= 1024 ? (uint32_t)ctx->opt_msm_affine_batch : 16u;
        const size_t max_pairs = (size_t)(slots / 2);
        BB_TRY(job->d_aff0.alloc(ctx, (max_pairs ? max_pairs : 1) * sizeof(Affine<F>)));
        if (R > 1) BB_TRY(job->d_aff1.alloc(ctx, (max_pairs / 2 + 1) * sizeof(Affine<F>)));
        BB_TRY(job->d_pre.alloc(ctx, (max_pairs ? max_pairs : 1) * sizeof(F)));
        const size_t T0 = (max_pairs + L - 1) / L;
        BB_TRY(job->d_tp.alloc(ctx, (T0 + batch_invert_scratch_elems(T0) + 1) * sizeof(F)));
        F* pre = job->d_pre.as<F>();
        F* tp = job->d_tp.as<F>();
        const uint32_t* d_entries = offsets + NB;
        Affine<F>* bufs[2] = {job->d_aff0.as<Affine<F>>(), job->d_aff1.as<Affine<F>>()};
        for (uint32_t r = 0; r < R; r++) {
            const size_t pairs = max_pairs >> r;
            const size_t T = (pairs + L - 1) / L;
            if (!T) break;
            Affine<F>* out = bufs[r & 1];
            if (r == 0) {
                PairLoader<F, true> ld{bases, A.sorted};
                k_aff_phase1<F, true><<<cdiv(T, 128), 128, 0, st>>>(ld, d_entries, r + 1, T, L, pre, tp);
                BB_TRY(batch_invert_device<F>(ctx, st, tp, T, tp + T));
                k_aff_phase3<F, true><<<cdiv(T, 128), 128, 0, st>>>(ld, d_entries, r + 1, T, L, pre, tp, out, A.err);
            } else {
                PairLoader<F, false> ld{bufs[(r - 1) & 1], nullptr};
                k_aff_phase1<F, false><<<cdiv(T, 128), 128, 0, st>>>(ld, d_entries, r + 1, T, L, pre, tp);
                BB_TRY(batch_invert_device<F>(ctx, st, tp, T, tp + T));
                k_aff_phase3<F, false><<<cdiv(T, 128), 128, 0, st>>>(ld, d_entries, r + 1, T, L, pre, tp, out, A.err);
            }
            ctx->count_launch(2);
            dense = out;
            BB_STAGE("affine round");
        }
        // the buckets' rows of the dense array
        BB_TRY(job->d_doffsets.alloc(ctx, (NB + 1) * 4));
        k_dense_offsets<<<cdiv(NB + 1, 256), 256, 0, st>>>(offsets, NB + 1, R, job->d_doffsets.as<uint32_t>());
        ctx->count_launch();
        offsets = job->d_doffsets.as<uint32_t>();
    }

    XYZZ<F>* buckets = job->d_buckets.as<XYZZ<F>>();
    uint32_t* order = job->d_order.as<uint32_t>();
    uint32_t* size_hist = order + NB;
    // A bucket is oversized above 4x the mean load (at least 64 entries); it is cut into tasks of
    // about the mean load (at least 32 entries, and few enough that <= ~1M tasks can exist), so
    // the serial chain any thread owns stays short and the task sums are merged by a tree.
    const uint64_t rows = slots >> R;                 // what the XYZZ stage walks
    // deep buckets without halving rounds (few buckets: a small window, or one bucket set under a short job) must not
    // become one long serial chain per thread either: above 64 rows per bucket every bucket is cut into tasks of 64
    const uint64_t avg_raw = (rows + NB - 1) / NB;
    const uint64_t avg = avg_raw > 64 ? 64 : avg_raw;
    uint64_t cap64 = 4 * avg < 64 ? 64 : 4 * avg;
    uint64_t len64 = avg < 32 ? 32 : avg;
    if (len64 < (rows + 1048575) / 1048576) len64 = (rows + 1048575) / 1048576;
    if (ctx->opt_msm_big_cap > 0) { cap64 = (uint64_t)ctx->opt_msm_big_cap; len64 = cap64; }
    if (cap64 < len64) cap64 = len64;
    const uint32_t cap = (uint32_t)cap64, task_len = (uint32_t)len64;
    const size_t max_big = (size_t)(rows / cap) + 16, max_tasks = (size_t)(rows / task_len) + max_big + 16;
    BB_TRY(job->d_big.alloc(ctx, 16));
    BB_TRY(job->d_tasks.alloc(ctx, max_tasks * sizeof(BigTask)));
    BB_TRY(job->d_biglist.alloc(ctx, max_big * sizeof(BigBucket)));
    BB_TRY(job->d_tasksums.alloc(ctx, max_tasks * sizeof(XYZZ<F>)));
    uint32_t* big = job->d_big.as<uint32_t>();
    BB_CUDA(cudaMemsetAsync(big, 0, 16, st));
    BB_CUDA(cudaMemsetAsync(size_hist, 0, SIZE_BINS * 4, st));
    k_size_hist<<<cdiv(NB, 256), 256, 0, st>>>(offsets, NB, size_hist);
    k_size_scan<<<1, 1024, 0, st>>>(size_hist);
    k_size_order<<<cdiv(NB, 256), 256, 0, st>>>(offsets, NB, size_hist, order, cap, task_len, big, job->d_tasks.as<BigTask>(), job->d_biglist.as<BigBucket>());
    ctx->count_launch(3);
    BB_STAGE("order");
    const size_t sh_pt = 128 * sizeof(XYZZ<F>);
    if (sh_pt > 48 * 1024) BB_CUDA(cudaFuncSetAttribute(k_msm_merge_big<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh_pt));
    {
        unsigned tgrid = (unsigned)((max_tasks + 127) / 128);
        if (tgrid > (unsigned)ctx->num_sms * 4) tgrid = (unsigned)ctx->num_sms * 4;
        if (dense) {
            k_msm_accumulate<F, true><<<cdiv(NB, 128), 128, 0, st>>>(dense, offsets, nullptr, order, buckets, NB, cap, A.err);
            k_msm_accumulate_tasks<F, true><<<tgrid, 128, 0, st>>>(dense, nullptr, big, job->d_tasks.as<BigTask>(), job->d_tasksums.as<XYZZ<F>>(), A.err);
        } else {
            k_msm_accumulate<F, false><<<cdiv(NB, 128), 128, 0, st>>>(bases, offsets, A.sorted, order, buckets, NB, cap, A.err);
            k_msm_accumulate_tasks<F, false><<<tgrid, 128, 0, st>>>(bases, A.sorted, big, job->d_tasks.as<BigTask>(), job->d_tasksums.as<XYZZ<F>>(), A.err);
        }
        unsigned mgrid = max_big < 1024 ? (unsigned)max_big : 1024u;
        k_msm_merge_big<F><<<mgrid, 128, sh_pt, st>>>(big, job->d_biglist.as<BigBucket>(), job->d_tasksums.as<XYZZ<F>>(), buckets);
    }
    ctx->count_launch(3);
    if (prof) BB_CUDA(cudaEventRecord(job->ev[2], st));
    BB_STAGE("accumulate");
    XYZZ<F>* fin = job->d_final.as<XYZZ<F>>();
    uint32_t Wr = Wb;                                  // window sums the reduction produces (per proof)
    if (job->precomp && !job->unified) {
        if (W > 1) {
            XYZZ<F>* folded = buckets;                 // one proof: in place; several: each proof's D sums side by side
            if (B > 1) { BB_TRY(job->d_slotsum.alloc(ctx, (size_t)B * D * sizeof(XYZZ<F>))); folded = job->d_slotsum.as<XYZZ<F>>(); }
            k_msm_fold_slots<F><<<dim3(cdiv(D, 128), B), 128, 0, st>>>(buckets, W, D, folded);
            ctx->count_launch();
            buckets = folded;
        }
        Wr = 1;
        BB_STAGE("fold slots");
    }
    job->W_out = Wr;
    BB_TRY(reduce_buckets_2d<F>(ctx, st, buckets, B * Wr, D, (uint32_t)ctx->opt_msm_reduce_k, (uint32_t)ctx->opt_msm_reduce_k1, job->d_fold, job->d_runs, job->d_partials, job->d_levels, fin));
    size_t sh = 128 * sizeof(XYZZ<F>);
    if (sh > 48 * 1024) BB_CUDA(cudaFuncSetAttribute(k_msm_sum_list<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    BB_TRY(job->d_onesp.alloc(ctx, ONES_BLOCKS * sizeof(XYZZ<F>)));
    XYZZ<F>* ones_partials = job->d_onesp.as<XYZZ<F>>();
    k_msm_sum_list<F><<<ONES_BLOCKS, 128, sh, st>>>(bases, A.ones_list, A.ones_count, ones_partials, A.err);
    k_point_tree_sum<F><<<1, 128, sh, st>>>(ones_partials, ONES_BLOCKS, fin + (size_t)B * Wr);
    ctx->count_launch(2);
    BB_STAGE("reduce");
    const XYZZ<F>* result = fin;
    size_t pts = (size_t)(Wr + 1) * sizeof(XYZZ<F>);
    if (job->batched) {                                // the ones are in the buckets: one folded point per proof
        BB_TRY(job->d_folded.alloc(ctx, (size_t)B * sizeof(XYZZ<F>)));
        k_msm_fold_windows<F><<<cdiv(B, 32), 32, 0, st>>>(fin, B, Wr, job->c, job->d_folded.as<XYZZ<F>>());
        ctx->count_launch();
        result = job->d_folded.as<XYZZ<F>>();
        pts = (size_t)B * sizeof(XYZZ<F>);
        BB_STAGE("fold windows");
    }
    BB_CUDA(cudaGetLastError());
    const size_t perr = job->batched ? (size_t)B * 4 : 0;
    job->h_out_bytes = pts + 32 + perr;
    BB_TRY(ctx->pinned_acquire(job->h_out_bytes, &job->h_out));
    BB_CUDA(cudaMemcpyAsync(job->h_out, result, pts, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync((char*)job->h_out + pts, job->d_err.p, 32, cudaMemcpyDeviceToHost, st));
    if (perr) BB_CUDA(cudaMemcpyAsync((char*)job->h_out + pts + 32, job->d_perr.p, perr, cudaMemcpyDeviceToHost, st));
    ctx->d2h_bytes += pts + 32 + perr;
    if (prof) BB_CUDA(cudaEventRecord(job->ev[3], st));
    // a proof has eight of these waits on eight host threads, and a multi-GPU box one process per GPU: the waiters
    // must not burn a core each (cudaStreamSynchronize spins by default)
    if (cudaEventCreateWithFlags(&job->ev_done, cudaEventBlockingSync | cudaEventDisableTiming) == cudaSuccess) {
        if (cudaEventRecord(job->ev_done, st) != cudaSuccess) { cudaEventDestroy(job->ev_done); job->ev_done = nullptr; }
    } else job->ev_done = nullptr;
    cudaGetLastError();
    return BB_OK;
}

}  // namespace

namespace {
template <class F>
int build_table_t(bb_ctx* ctx, bb_bases* b, uint32_t c, uint32_t W, uint32_t slots) {
    const size_t n = b->n;
    void* table = nullptr;
    BB_TRY(ctx->alloc((size_t)slots * n * sizeof(Affine<F>), &table));
    // scratch in chunks of bases: slots * chunk XYZZ points (<= ~1 GB)
    size_t chunk = (size_t(1) << 30) / ((size_t)slots * sizeof(XYZZ<F>));
    if (chunk > n) chunk = n;
    if (chunk < 128) chunk = 128;
    DevBuf scratch;
    int s = scratch.alloc(ctx, (size_t)slots * chunk * sizeof(XYZZ<F>));
    cudaStream_t st = ctx->main_stream;
    for (size_t lo = 0; s == BB_OK && lo < n; lo += chunk) {
        size_t len = n - lo < chunk ? n - lo : chunk;
        k_table_multiples<F><<<cdiv(len, 128), 128, 0, st>>>((const Affine<F>*)b->d_points + lo, len, c, W, b->win_index, b->win_count, scratch.as<XYZZ<F>>());
        k_table_normalize<F><<<cdiv(len, 128), 128, 0, st>>>(scratch.as<XYZZ<F>>(), len, slots, (Affine<F>*)table, n, lo);
        ctx->count_launch(2);
        if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) { set_error("window-multiple table: kernel failed"); s = BB_ERR_CUDA; }
    }
    if (s != BB_OK) { ctx->release(table); return s; }
    b->d_table = table; b->tab_c = c; b->tab_W = W; b->tab_slots = slots;
    return BB_OK;
}
}  // namespace

namespace bb {
int batch_invert_fp(bb_ctx* ctx, cudaStream_t st, Fp* vals, size_t n, Fp* scratch) { return batch_invert_device<Fp>(ctx, st, vals, n, scratch); }
int batch_invert_fp2(bb_ctx* ctx, cudaStream_t st, Fp2* vals, size_t n, Fp2* scratch) { return batch_invert_device<Fp2>(ctx, st, vals, n, scratch); }
size_t batch_invert_scratch(size_t n) { return batch_invert_scratch_elems(n); }
}  // namespace bb
namespace bb {
// Builds the window-multiple table of a base vector for the window size its length selects (the
// window of an MSM over these bases is then fixed, whatever the density of the query).
int bases_build_table(bb_ctx* ctx, bb_bases* b) {
    std::lock_guard<std::mutex> g(b->tab_mu);
    if (b->d_table || !b->n) return BB_OK;
    BB_CUDA(cudaSetDevice(ctx->device));
    const uint32_t c = choose_window(ctx, b->n);
    const uint32_t W = 255 / c + 1, wc = b->win_count ? b->win_count : 1;
    uint32_t slots = 0;
    for (uint32_t w = 0; w < W; w++) slots += (w % wc == b->win_index);
    if (slots == 0) slots = 1;
    if ((uint64_t)slots * b->n >= (1ull << 31)) { set_error("window-multiple table: %u slots x %zu bases exceed 2^31 entries", slots, b->n); return BB_ERR_ARG; }
    return b->group == BB_G1 ? build_table_t<Fp>(ctx, b, c, W, slots) : build_table_t<Fp2>(ctx, b, c, W, slots);
}
}  // namespace bb
namespace bb {
int msm_start(bb_ctx* ctx, const bb_bases* bases, size_t base_offset, const uint64_t* density_bits, size_t density_len,
              const void* scalars, bool scalars_on_device, size_t n, int form, cudaEvent_t wait_for, bb_msm_job** out,
              const char* tag, int critical, uint32_t batch, size_t scalar_stride) {
    if (!ctx || !bases || !out || (n && !scalars)) { set_error("bb_msm: null argument"); return BB_ERR_ARG; }
    if (batch && (!scalars_on_device || bases->win_count > 1 || batch > 65535)) { set_error("bb_msm: a batched job takes device scalars, an unsharded vector and at most 65535 proofs"); return BB_ERR_ARG; }
    if (n >= (1ull << 31) || bases->n >= (1ull << 31)) { set_error("bb_msm: more than 2^31 terms"); return BB_ERR_ARG; }
    if (form != BB_FORM_CANONICAL && form != BB_FORM_MONTGOMERY) { set_error("bb_msm: bad form"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    bb_msm_job* job = new bb_msm_job();
    *out = job;
    job->ctx = ctx; job->bases = bases; job->group = bases->group; job->n = n; job->n_dense = n;
    job->tag = tag;
    job->B = batch ? batch : 1; job->batched = batch != 0;
    job->st = critical ? ctx->crit_stream[(critical - 1) & 1] : ctx->pick_stream();
    if (wait_for) BB_CUDA(cudaStreamWaitEvent(job->st, wait_for, 0));
    if (density_bits && density_len != n) {                 // the assert! at multiexp.rs:324-329
        set_error("density map has %zu entries for %zu exponents", density_len, n);
        job->status = BB_ERR_DENSITY_MISMATCH;
        return BB_OK;
    }
    // the pairs this device accumulates: all scalars on one GPU, about one shard's worth when sharded
    const bool tables_wanted = ctx->opt_msm_precompute && (ctx->opt_msm_precompute_groups & (bases->group == BB_G1 ? 1 : 2));
    if (tables_wanted && bases->n && !bases->d_table) {
        int ts = bases_build_table(ctx, const_cast<bb_bases*>(bases));     // first use; bb_bases_precompute does it up front
        // no room for the table: the per-window path needs none -- but only a whole key may fall back by itself: the shards
        // of a window-sharded key must all cut the scalars into the same windows
        if (ts != BB_OK && !(ts == BB_ERR_OOM && bases->win_count <= 1)) { job->status = ts; return BB_OK; }
    }
    const MsmPlan plan = msm_plan(ctx, bases, false, n, n, job->B);
    job->precomp = plan.precomp;
    job->unified = plan.unified;
    job->c = plan.c;
    job->W = plan.W;
    job->D = plan.D;
    auto fail = [&](int s) { job->status = s; return BB_OK; };
    DigitArgs& A = job->dargs;
    A.n = n; A.montgomery = form == BB_FORM_MONTGOMERY;
    A.scalar_stride = scalar_stride;
    A.base_offset = base_offset;
    A.shard_lo = bases->global_offset; A.shard_n = bases->n; A.global_len = bases->global_len;
    A.c = job->c; A.W = job->W;
    A.win_index = bases->win_index; A.win_count = bases->win_count ? bases->win_count : 1;
    A.table_stride = job->precomp ? (uint32_t)bases->n : 0u;
    A.key_stride = job->unified ? 0u : job->D;
    if (A.win_index >= A.win_count) { set_error("bb_msm: window shard %u of %u", A.win_index, A.win_count); return fail(BB_ERR_ARG); }
    job->W_local = plan.W_local;
    int s;
    if (scalars_on_device) A.scalars = (const Fr*)scalars;
    else {
        if ((s = job->d_scalars.alloc(ctx, n * 32)) != BB_OK) return fail(s);
        ctx->h2d_bytes += n * 32;
        if (n && cudaMemcpyAsync(job->d_scalars.p, scalars, n * 32, cudaMemcpyHostToDevice, job->st) != cudaSuccess) {
            set_error("scalar upload failed");
            return fail(BB_ERR_CUDA);
        }
        A.scalars = job->d_scalars.as<Fr>();
    }
    if (density_bits) {
        size_t words = (n + 63) / 64;
        job->h_rank.resize(words ? words : 1);
        uint32_t acc = 0;
        for (size_t j = 0; j < words; j++) {
            job->h_rank[j] = acc;
            uint64_t wv = density_bits[j];
            if (j == words - 1 && (n & 63)) wv &= (1ull << (n & 63)) - 1ull;
            acc += (uint32_t)__builtin_popcountll(wv);
        }
        job->n_dense = acc;
        if ((s = job->d_density.alloc(ctx, words * 8)) != BB_OK) return fail(s);
        if ((s = job->d_rank.alloc(ctx, words * 4)) != BB_OK) return fail(s);
        if (words) {
            if (cudaMemcpyAsync(job->d_density.p, density_bits, words * 8, cudaMemcpyHostToDevice, job->st) != cudaSuccess ||
                cudaMemcpyAsync(job->d_rank.p, job->h_rank.data(), words * 4, cudaMemcpyHostToDevice, job->st) != cudaSuccess) {
                set_error("density map upload failed");
                return fail(BB_ERR_CUDA);
            }
            ctx->h2d_bytes += words * 12;
        }
        A.density = job->d_density.as<uint64_t>();
        A.density_rank = job->d_rank.as<uint32_t>();
    }
    s = job->group == BB_G1 ? launch_msm<Fp>(job) : launch_msm<Fp2>(job);
    if (s != BB_OK) return fail(s);
    return BB_OK;
}

}  // namespace bb
namespace {
// Horner fold over the window sums (multiexp.rs:295-300) plus the Exponent::One sum.  `win` holds
// the W_local windows this device owns (window w lives in slot w / wc when w % wc == wi), then the
// ones sum; windows owned elsewhere contribute the identity here and are added by their owners'
// partial results (the fold is linear).
template <class F>
XYZZ<F> fold_windows(const XYZZ<F>* win, uint32_t W, uint32_t W_local, uint32_t c, uint32_t wi, uint32_t wc) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (int w = (int)W - 1; w >= 0; w--) {
        for (uint32_t k = 0; k < c; k++) acc = acc.dbl();
        if ((uint32_t)w % wc == wi && (uint32_t)w / wc < W_local) acc.add(win[(uint32_t)w / wc]);
    }
    acc.add(win[W_local]);
    return acc;
}

template <class F>
int classify_both_errors(bb_msm_job* job, uint32_t eof_index, int* status) {
    bb_ctx* ctx = job->ctx;
    size_t n = job->n;
    uint32_t c_ref = n < 32 ? 3u : (uint32_t)std::ceil(std::log((double)(uint32_t)n));   // multiexp.rs:318-322
    uint32_t chunks = (255 + c_ref - 1) / c_ref;                                          // step_by(c) over 0..NUM_BITS
    uint32_t* d_first = job->d_err.as<uint32_t>() + 2;
    BB_CUDA(cudaMemsetAsync(d_first, 0xff, 4, job->st));
    k_msm_classify<F><<<cdiv(n, 256), 256, 0, job->st>>>(job->dargs, (const Affine<F>*)job->bases->d_points, c_ref, chunks - 1, d_first);
    ctx->count_launch();
    uint32_t first = 0xffffffffu;
    BB_CUDA(cudaMemcpyAsync(&first, d_first, 4, cudaMemcpyDeviceToHost, job->st));
    BB_CUDA(cudaStreamSynchronize(job->st));
    *status = first < eof_index ? BB_ERR_UNEXPECTED_IDENTITY : BB_ERR_IO_UNEXPECTED_EOF;
    return BB_OK;
}

}  // namespace

namespace bb {
// profile mode: the job's stage times (accumulation, whole job, prover timeline) from its events, then the events go;
// `cnt` = the job's counter words as copied back (err[4] pairs, err[5] bucket entries)
void record_profile(bb_msm_job* job, int status, const uint32_t* cnt) {
    if (job->ev[3]) {
        float acc_ms = 0, tot_ms = 0;
        if (status == BB_OK && cudaEventElapsedTime(&acc_ms, job->ev[1], job->ev[2]) == cudaSuccess &&
            cudaEventElapsedTime(&tot_ms, job->ev[0], job->ev[3]) == cudaSuccess) {
            bool g2 = job->group == BB_G2;
            // units: the (base, scalar) pairs this job consumed -- density-selected, non-zero, not Exponent::One,
            // in this shard (counted by k_msm_digits); entries = non-zero digits of those scalars
            job->ctx->prof_add(g2 ? "msm_accumulate_g2" : "msm_accumulate_g1", acc_ms, 1, cnt[4]);
            job->ctx->prof_add(g2 ? "msm_total_g2" : "msm_total_g1", tot_ms, 1, cnt[4]);
            job->ctx->prof_add(g2 ? "msm_entries_g2" : "msm_entries_g1", acc_ms, 1, cnt[5]);
            // Fp / Fp2 multiplications of the accumulation stage: halving round r adds entries / 2^(r+1) pairs at 6
            // each (batch_affine.cuh), the XYZZ stage adds what is left at 10 each -- an upper bound, padding rows and
            // first entries of a bucket cost nothing
            uint64_t muls = 0, left = cnt[5];
            for (uint32_t r = 0; r < job->affine_rounds; r++) { muls += 6 * (left / 2); left -= left / 2; }
            muls += 10 * left;
            job->ctx->prof_add(g2 ? "msm_fieldmuls_g2" : "msm_fieldmuls_g1", acc_ms, job->affine_rounds, muls);
            if (job->tag && job->ctx->epoch_ev) {            // device timeline of the prover: ms since the prove started
                static const char* const mark[4] = {"start", "acc_start", "acc_end", "end"};
                for (int i = 0; i < 4; i++) {
                    float t = 0;
                    if (cudaEventElapsedTime(&t, job->ctx->epoch_ev, job->ev[i]) == cudaSuccess)
                        job->ctx->prof_add((std::string("tl.") + job->tag + "." + mark[i]).c_str(), t, 1, 0);
                }
            }
        }
        for (auto& e : job->ev) if (e) { cudaEventDestroy(e); e = nullptr; }
        cudaGetLastError();
    }
}

// used by prover.cu: wait and return the projective result
int msm_wait_result(bb_msm_job* job, MsmResult* res) {
    int status = job->status;
    {   // also on a failed launch: kernels already queued may still use the job's buffers
        if (job->ev_done) { cudaEventSynchronize(job->ev_done); cudaEventDestroy(job->ev_done); job->ev_done = nullptr; }   // sleeps
        cudaError_t e = cudaStreamSynchronize(job->st);                                                                     // returns at once after that
        if (e != cudaSuccess && status == BB_OK) { set_error("msm stream: %s", cudaGetErrorString(e)); status = BB_ERR_CUDA; }
    }
    if (status == BB_OK) {
        bool g2 = job->group == BB_G2;
        size_t pts = (size_t)(job->W_out + 1) * (g2 ? sizeof(G2X) : sizeof(G1X));
        const uint32_t* err = (const uint32_t*)((char*)job->h_out + pts);
        bool eof = err[0] != 0xffffffffu, ident = err[1] != 0;
        if (eof && ident) {
            int s = g2 ? classify_both_errors<Fp2>(job, err[0], &status) : classify_both_errors<Fp>(job, err[0], &status);
            if (s != BB_OK) status = s;
        } else if (eof) {
            status = BB_ERR_IO_UNEXPECTED_EOF;
        } else if (ident) {
            status = BB_ERR_UNEXPECTED_IDENTITY;
        }
        if (status == BB_ERR_IO_UNEXPECTED_EOF) set_error("expected more bases from source");
        if (status == BB_ERR_UNEXPECTED_IDENTITY) set_error("encountered an identity element in the CRS");
        if (status == BB_OK) {
            res->g2 = g2;
            const uint32_t wi = job->dargs.win_index, wc = job->dargs.win_count;
            if (job->precomp) {                       // one window sum (weights already in the table) + the ones sum
                if (g2) { res->x2 = ((const G2X*)job->h_out)[0]; res->x2.add(((const G2X*)job->h_out)[1]); }
                else { res->g1 = ((const G1X*)job->h_out)[0]; res->g1.add(((const G1X*)job->h_out)[1]); }
            } else if (g2) res->x2 = fold_windows<Fp2>((const G2X*)job->h_out, job->W, job->W_local, job->c, wi, wc);
            else res->g1 = fold_windows<Fp>((const G1X*)job->h_out, job->W, job->W_local, job->c, wi, wc);
        }
    }
    res->status = status;
    record_profile(job, status, (const uint32_t*)((const char*)job->h_out + (size_t)(job->W_out + 1) * (job->group == BB_G2 ? sizeof(G2X) : sizeof(G1X))));
    if (job->h_out) job->ctx->pinned_release(job->h_out);
    delete job;
    return status;
}

// A batched job (msm_start with batch = B): for each proof p, status[p] is what msm_wait_result would report for that
// vector alone, and points[p] (G1X or G2X) its folded sum where status[p] is BB_OK.  Returns the job-level status (a
// failure before or during the launch, or of the stream), which then stands for every proof.  Frees the job.
int msm_wait_batch(bb_msm_job* job, int* status, void* points) {
    int st = job->status;
    if (job->ev_done) { cudaEventSynchronize(job->ev_done); cudaEventDestroy(job->ev_done); job->ev_done = nullptr; }
    cudaError_t e = cudaStreamSynchronize(job->st);
    if (e != cudaSuccess && st == BB_OK) { set_error("msm stream: %s", cudaGetErrorString(e)); st = BB_ERR_CUDA; }
    const uint32_t B = job->B;
    const bool g2 = job->group == BB_G2;
    const size_t psz = g2 ? sizeof(G2X) : sizeof(G1X);
    for (uint32_t p = 0; p < B; p++) status[p] = st;
    if (st == BB_OK && job->h_out) {
        const uint32_t* err = (const uint32_t*)((const char*)job->h_out + B * psz);
        const uint32_t* perr = err + 8;
        const bool eof = err[0] != 0xffffffffu;           // the shape alone decides it: the same for every proof
        for (uint32_t p = 0; p < B && st == BB_OK; p++) {
            int s = BB_OK;
            if (eof && perr[p]) {
                const DigitArgs saved = job->dargs;
                job->dargs.scalars += (size_t)p * saved.scalar_stride;
                int c = g2 ? classify_both_errors<Fp2>(job, err[0], &s) : classify_both_errors<Fp>(job, err[0], &s);
                job->dargs = saved;
                if (c != BB_OK) st = c;
            } else if (eof) {
                s = BB_ERR_IO_UNEXPECTED_EOF;
            } else if (perr[p]) {
                s = BB_ERR_UNEXPECTED_IDENTITY;
            }
            status[p] = s;
        }
        if (st != BB_OK) for (uint32_t p = 0; p < B; p++) status[p] = st;
        else std::memcpy(points, job->h_out, B * psz);
    }
    record_profile(job, st, job->h_out ? (const uint32_t*)((const char*)job->h_out + B * psz) : nullptr);
    for (auto& ev : job->ev) if (ev) cudaEventDestroy(ev);      // the events of a job that failed before its last record
    cudaGetLastError();
    if (job->h_out) job->ctx->pinned_release(job->h_out);
    delete job;
    return st;
}

// What a batched job of B vectors of n scalars (n_dense of them selected by the density map) over `bases` needs:
// *slots = its bucket entries (launch_msm refuses 2^32 and more), and an estimate of its device bytes.
size_t msm_batch_bytes(bb_ctx* ctx, const bb_bases* bases, size_t n, size_t n_dense, uint32_t B, uint64_t* slots) {
    const bool g2 = bases->group == BB_G2;
    const MsmPlan p = msm_plan(ctx, bases, true, n, n_dense, B);
    const uint64_t s = p.slots;
    *slots = s;
    const size_t aff = g2 ? sizeof(G2Affine) : sizeof(G1Affine), xyzz = g2 ? sizeof(G2X) : sizeof(G1X), fe = aff / 2;
    double bytes = 4.0 * s + (double)p.NB * (2.0 * xyzz + 20.0) + (double)(s >> p.R) / 32.0 * (12.0 + xyzz);
    if (p.R) bytes += (double)s / 2 * (aff + fe) + (double)s / 4 * aff;
    return (size_t)bytes;
}
}  // namespace bb

extern "C" {

int bb_msm_async(bb_ctx* ctx, const bb_bases* bases, size_t base_offset, const uint64_t* density_bits, size_t density_len,
                 const void* scalars, size_t n_scalars, int form, bb_msm_job** out) {
    return msm_start(ctx, bases, base_offset, density_bits, density_len, scalars, false, n_scalars, form, nullptr, out);
}
int bb_msm_async_device(bb_ctx* ctx, const bb_bases* bases, size_t base_offset, const uint64_t* density_bits, size_t density_len,
                        const void* d_scalars, size_t n_scalars, int form, bb_msm_job** out) {
    return msm_start(ctx, bases, base_offset, density_bits, density_len, d_scalars, true, n_scalars, form, nullptr, out);
}
int bb_bases_precompute(bb_ctx* ctx, bb_bases* bases) {
    if (!ctx || !bases || bases->ctx != ctx) { set_error("bb_bases_precompute: bad argument"); return BB_ERR_ARG; }
    return bases_build_table(ctx, bases);
}
int bb_bases_drop_table(bb_bases* bases) {
    if (!bases) { set_error("bb_bases_drop_table: null argument"); return BB_ERR_ARG; }
    std::lock_guard<std::mutex> g(bases->tab_mu);
    if (bases->d_table) bases->ctx->release(bases->d_table);
    bases->d_table = nullptr; bases->tab_c = bases->tab_W = bases->tab_slots = 0;
    return BB_OK;
}
int bb_msm_wait(bb_msm_job* job, void* out_affine) {
    if (!job || !out_affine) { set_error("bb_msm_wait: null argument"); return BB_ERR_ARG; }
    MsmResult r;
    int s = msm_wait_result(job, &r);
    if (s != BB_OK) return s;
    if (r.g2) { G2Affine a = r.x2.to_affine(); std::memcpy(out_affine, &a, sizeof a); }
    else { G1Affine a = r.g1.to_affine(); std::memcpy(out_affine, &a, sizeof a); }
    return BB_OK;
}

// diagnostics: out = sum_{i<D} (i+1) * P_i through k_msm_reduce + k_point_tree_sum (G1)
int bb_selftest_bucket_reduce(bb_ctx* ctx, const void* affine_pts, uint32_t D, uint32_t K, void* out_affine) {
    if (!ctx || !affine_pts || !out_affine || !D || !K) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    std::vector<G1X> h(D);
    const G1Affine* a = (const G1Affine*)affine_pts;
    for (uint32_t i = 0; i < D; i++) h[i] = G1X::from_affine(a[i]);
    DevBuf d_b, d_p, d_r, d_l, d_f;
    BB_TRY(d_b.alloc(ctx, D * sizeof(G1X))); BB_TRY(d_f.alloc(ctx, sizeof(G1X)));
    cudaStream_t st = ctx->main_stream;
    BB_CUDA(cudaMemcpyAsync(d_b.p, h.data(), D * sizeof(G1X), cudaMemcpyHostToDevice, st));
    DevBuf d_fold;                                       // a power of two D >= 1024 takes the two-dimensional form
    BB_TRY(reduce_buckets_2d<Fp>(ctx, st, d_b.as<G1X>(), 1, D, K, K, d_fold, d_r, d_p, d_l, d_f.as<G1X>()));
    G1X r;
    BB_CUDA(cudaMemcpyAsync(&r, d_f.p, sizeof r, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    G1Affine ra = r.to_affine();
    std::memcpy(out_affine, &ra, sizeof ra);
    return BB_OK;
}

}  // extern "C"
