// bellman_b200: batched-affine pairwise bucket accumulation for sm_90a.
//
// The bucket loop of multiexp_inner (bellman/src/multiexp.rs:253-262) adds every base whose
// digit selects a bucket into that bucket.  One thread per bucket with an XYZZ accumulator costs 10
// field multiplications per addition (madd-2008-s).  An AFFINE addition costs 1 inversion + 3
// multiplications; with Montgomery's trick the inversion is shared by every addition that is
// independent of the others, which leaves 6 multiplications per addition.  Independence is obtained by
// reducing each bucket as a TREE: the counting sort lays the entries of a bucket side by side, so in one
// round every bucket adds its entries 0+1, 2+3, 4+5, ... -- all of them independent -- and halves its
// length.  Buckets are padded to a multiple of 2^R entries (null entries) so that pair j of the whole
// array is always (2j, 2j+1), never straddles two buckets, and its sum lands at position j of the next
// round's array: no per-round scan, no search, pure streaming.  After R rounds the few points left per
// bucket are summed by the XYZZ kernel as before (msm.cu).
//
// One round =
//   k_aff_phase1   thread t walks its pairs j = t, t+T, t+2T, ...: denominator d_j (x2-x1, or 2y for a
//                  doubling, or 1 when the pair needs no inversion), running product, exclusive prefixes
//                  to HBM; the thread's total goes to tp[t]
//   batch_invert   tp[t] <- 1/tp[t] for all T threads: the same trick once more with fan-in 32, then
//                  shared-memory product scans over tiles of 256 until one tile is left, ONE Fermat
//                  inversion per round, then back down
//   k_aff_phase3   the thread walks its pairs backwards: 1/d_j = run * prefix_j, run *= d_j, and finishes
//                  the affine addition; result j to the next array.
// The results are group elements: any evaluation order gives the same bucket sums, hence the same
// window sums and the same proof bytes.
#pragma once
#include "curve.cuh"

namespace bb {

template <class F> struct PointIO;
template <> struct PointIO<Fp> { static constexpr int VEC = 6; };     // uint4 loads per affine point
template <> struct PointIO<Fp2> { static constexpr int VEC = 12; };

template <class T>
__device__ __forceinline__ void st_words(T* dst, const T& v) {
    constexpr int V = sizeof(T) / 16;
    uint4* q = reinterpret_cast<uint4*>(dst);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
    for (int i = 0; i < V; i++) q[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
}
template <class T>
__device__ __forceinline__ T ld_words(const T* src) {
    constexpr int V = sizeof(T) / 16;
    const uint4* q = reinterpret_cast<const uint4*>(src);
    T r;
    uint32_t* w = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int i = 0; i < V; i++) {
        uint4 v = q[i];
        w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
    }
    return r;
}
// read-only path (bases never change while an MSM runs)
template <class T>
__device__ __forceinline__ T ldg_words(const T* src) {
    constexpr int V = sizeof(T) / 16;
    const uint4* q = reinterpret_cast<const uint4*>(src);
    T r;
    uint32_t* w = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int i = 0; i < V; i++) {
        uint4 v = __ldg(q + i);
        w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
    }
    return r;
}
template <class F>
__device__ __forceinline__ Affine<F> ld_affine(const Affine<F>* p) { return ldg_words(p); }

// ---- batch inversion of T non-zero field elements, in place -------------------------------------------
constexpr uint32_t BINV_FAN = 32;

// level up: group g = elements [g*FAN, (g+1)*FAN): pre[i] = product of the group's elements before i,
// up[g] = product of the whole group
template <class F>
__global__ void __launch_bounds__(128) k_binv_up(const F* __restrict__ vals, size_t n, F* __restrict__ pre, F* __restrict__ up) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t lo = g * BINV_FAN;
    if (lo >= n) return;
    size_t hi = lo + BINV_FAN < n ? lo + BINV_FAN : n;
    F run = ld_words(vals + lo);
    for (size_t i = lo + 1; i < hi; i++) {
        st_words(pre + i, run);
        run = run * ld_words(vals + i);
    }
    st_words(up + g, run);
}
// level down: up[g] now holds the inverse of the group product; vals[i] <- 1 / vals[i]
template <class F>
__global__ void __launch_bounds__(128) k_binv_down(F* __restrict__ vals, size_t n, const F* __restrict__ pre, const F* __restrict__ up) {
    size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t lo = g * BINV_FAN;
    if (lo >= n) return;
    size_t hi = lo + BINV_FAN < n ? lo + BINV_FAN : n;
    F run = ld_words(up + g);
    for (size_t i = hi - 1; i > lo; i--) {
        F v = ld_words(vals + i);
        st_words(vals + i, run * ld_words(pre + i));
        run = run * v;
    }
    st_words(vals + lo, run);
}
// Upper levels: one CTA per tile of SCAN_TILE elements, Hillis-Steele product scans in shared memory
// (depth 2 log2(tile) multiplications instead of 3 * fan-in for the serial walk -- these levels are tiny, so
// the extra work is irrelevant and the latency of the chain is what counts: it is paid once per halving round
// on the job's critical path).  pre[i] / suf[i] = products of the tile's elements before / after i,
// up[tile] = product of the tile.
constexpr uint32_t BINV_TILE = 256;

// (the tile-scan kernels k_binv_scan_up / k_binv_scan_down / k_binv_top live in msm.cu next to their launches)

// scratch elements batch_invert needs for n values: prefixes of level 0, then values + prefixes + suffixes of
// every upper level
inline size_t batch_invert_scratch_elems(size_t n) {
    size_t tot = n;                       // pre of level 0
    if (n > BINV_TILE) {
        n = (n + BINV_FAN - 1) / BINV_FAN;
        tot += 3 * n;
        while (n > BINV_TILE) { n = (n + BINV_TILE - 1) / BINV_TILE; tot += 3 * n; }
    }
    return tot + 2 * BINV_TILE;
}

// ---- one pair -----------------------------------------------------------------------------------------
// kinds: 0 ordinary addition (d = x2 - x1), 1 doubling (d = 2 y1), 2 no inversion needed (a null /
// identity operand, or P + (-P))
template <class F>
struct PairClass { int kind; F den; };

constexpr uint32_t AFF_NULL = 0xffffffffu;     // padding entry of the sorted index array

template <class F>
__device__ __forceinline__ bool affine_is_identity(const Affine<F>& p) { return p.x.is_zero() && p.y.is_zero(); }

// Operands of pair j.  GATHER: entries of the sorted index array (bit 31 = negate) select rows of the base
// table; otherwise rows 2j, 2j+1 of the previous round's dense array.  `need_y` false loads x only unless
// the classification needs y (equal x coordinates).
template <class F, bool GATHER>
struct PairLoader {
    const Affine<F>* pts;
    const uint32_t* sorted;
    __device__ __forceinline__ const Affine<F>* row(size_t j, int k, bool* null_entry, bool* negate) const {
        if (GATHER) {
            uint32_t v = sorted[2 * j + k];
            *null_entry = v == AFF_NULL;
            *negate = (v >> 31) != 0;
            return pts + (v & 0x7fffffffu);
        }
        *null_entry = false;
        *negate = false;
        return pts + 2 * j + k;
    }
};

template <class F>
__device__ __forceinline__ F ld_field(const F* p) { return ldg_words(p); }

// minimum resident CTAs of 128 threads per SM for phase 3 (ptxas -v, sm_90a, see DESIGN 4.1).  G1 needs ~176
// registers unbounded (two CTAs); three CTAs cap it at 168, which it fits without spilling.  G2 takes all 255.
template <class F> struct AffBounds { static constexpr int MINB = 3; };
template <> struct AffBounds<Fp2> { static constexpr int MINB = 1; };

// phase 1: denominators and their running products.  The products are inlined (FieldOps): an out-of-line Fp2
// product would keep its operands in a local-memory stack frame.
template <class F, bool GATHER>
__global__ void __launch_bounds__(128) k_aff_phase1(PairLoader<F, GATHER> ld, const uint32_t* __restrict__ d_entries, uint32_t shift,
                                                    size_t T, uint32_t L, F* __restrict__ pre, F* __restrict__ tp) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const size_t npairs = (size_t)(*d_entries) >> shift;
    F run = FieldOps<F>::one();
    for (uint32_t i = 0; i < L; i++) {
        size_t j = (size_t)i * T + t;
        if (j >= npairs) break;
        bool n1, n2, g1, g2;
        const Affine<F>* p1 = ld.row(j, 0, &n1, &g1);
        const Affine<F>* p2 = ld.row(j, 1, &n2, &g2);
        if (n1 || n2) continue;
        F x1 = ld_field(&p1->x), x2 = ld_field(&p2->x);
        F den = x2 - x1;
        if (x1.is_zero() || x2.is_zero() || den.is_zero()) {       // rare: identity operand, doubling or cancellation
            F y1 = ld_field(&p1->y), y2 = ld_field(&p2->y);
            if ((x1.is_zero() && y1.is_zero()) || (x2.is_zero() && y2.is_zero())) continue;
            if (den.is_zero()) {
                if (g1) y1 = y1.neg();
                if (g2) y2 = y2.neg();
                if (y1 != y2 || y1.is_zero()) continue;              // P + (-P) (or a 2-torsion point): identity
                den = y1.dbl();
            }
        }
        st_words(pre + j, run);
        run = FieldOps<F>::mul(run, den);
    }
    st_words(tp + t, run);
}

// Operands of pair j for phase 3.  Returns false when the sum needs no inversion; it has then been written to
// out[j] already: the other operand for a null / identity one, the identity for P + (-P).  Otherwise *den / *num
// are the slope's denominator and numerator, and x1, x2, y1 what the sum needs of the operands.  Each operand is
// stored separately (no `i1 ? P2 : P1`: selecting between two local points by reference put both in a stack frame).
// err[1] is raised for an identity base selected by a digit (Source::next, multiexp.rs:63-65): only gathered rows
// can be CRS bases.
template <class F, bool GATHER>
__device__ __forceinline__ bool pair_operands(const PairLoader<F, GATHER>& ld, size_t j, Affine<F>* __restrict__ out, uint32_t* err,
                                              F* den, F* num, F* x1, F* x2, F* y1) {
    bool n1, n2, g1, g2;
    const Affine<F>* r1 = ld.row(j, 0, &n1, &g1);
    const Affine<F>* r2 = ld.row(j, 1, &n2, &g2);
    Affine<F> P1 = n1 ? Affine<F>::identity() : ld_affine(r1);
    Affine<F> P2 = n2 ? Affine<F>::identity() : ld_affine(r2);
    const bool i1 = affine_is_identity(P1), i2 = affine_is_identity(P2);
    if (GATHER && ((i1 && !n1) || (i2 && !n2))) atomicOr(&err[1], 1u);
    if (g1) P1.y = P1.y.neg();
    if (g2) P2.y = P2.y.neg();
    if (i1) { st_words(out + j, P2); return false; }
    if (i2) { st_words(out + j, P1); return false; }
    *den = P2.x - P1.x;
    if (den->is_zero()) {
        if (P1.y != P2.y || P1.y.is_zero()) { st_words(out + j, Affine<F>::identity()); return false; }
        *den = P1.y.dbl();
        F xx = FieldOps<F>::sqr(P1.x);
        *num = xx.dbl() + xx;
    } else {
        *num = P2.y - P1.y;
    }
    *x1 = P1.x;
    *x2 = P2.x;
    *y1 = P1.y;
    return true;
}

// phase 3: finish the additions, walking the thread's pairs backwards.  tp[t] = 1 / (product of the
// thread's denominators).  Products inlined as in phase 1.
template <class F, bool GATHER>
__global__ void __launch_bounds__(128, AffBounds<F>::MINB) k_aff_phase3(PairLoader<F, GATHER> ld, const uint32_t* __restrict__ d_entries, uint32_t shift,
                                                                        size_t T, uint32_t L, const F* __restrict__ pre, const F* __restrict__ tp,
                                                                        Affine<F>* __restrict__ out, uint32_t* err) {
    typedef FieldOps<F> O;
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const size_t npairs = (size_t)(*d_entries) >> shift;
    if (t >= npairs) return;
    F run = ld_words(tp + t);
    uint32_t cnt = (uint32_t)((npairs - t + T - 1) / T);            // pairs this thread owns: j = t + i T < npairs
    if (cnt > L) cnt = L;
    for (int i = (int)cnt - 1; i >= 0; i--) {
        size_t j = (size_t)i * T + t;
        F den, num, x1, x2, y1;
        if (!pair_operands(ld, j, out, err, &den, &num, &x1, &x2, &y1)) continue;
        F inv = O::mul(run, ld_words(pre + j));
        run = O::mul(run, den);
        F lam = O::mul(num, inv);
        Affine<F> R;
        R.x = O::sqr(lam) - x1 - x2;
        R.y = O::mul(lam, x1 - R.x) - y1;
        st_words(out + j, R);
    }
}

}  // namespace bb
