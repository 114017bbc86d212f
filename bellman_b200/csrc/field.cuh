// bellman_b200: BLS12-381 Fr / Fp / Fp2 on top of mp.cuh.
// Fr is the field EvaluationDomain works over (bellman/src/domain.rs:21-28)
// and the scalar field of multiexp (src/multiexp.rs:305-316); Fp / Fp2 are the
// coordinate fields of G1 / G2.
#pragma once
#include "bls_constants.cuh"
#include "mp.cuh"

namespace bb {

// per-translation-unit copies of the moduli in constant memory: operands of the
// reduction rows come straight from the constant bank, no registers.
#if defined(__CUDACC__)
static __device__ __constant__ uint32_t kFrMod[8] = {BBC_FR_MOD_LIST};
static __device__ __constant__ uint32_t kFpMod[12] = {BBC_FP_MOD_LIST};
static __device__ __constant__ uint32_t kFpModSq[24] = {BBC_FP_MODSQ_LIST};   // p^2
#endif

struct FrCfg {
    static constexpr int N = 8;
    static constexpr uint32_t INV = bbc::FR_INV;
    static constexpr uint64_t INV64 = 0xfffffffeffffffffull;
#if defined(__CUDACC__)
    static __device__ __forceinline__ uint32_t dmod(int k) { return kFrMod[k]; }
#elif defined(BB_EMULATE_PTX)
    static uint32_t dmod(int k) { return bbc::FR_MOD[k]; }
#endif
    static const uint32_t* hmod() { return bbc::FR_MOD; }
};
struct FpCfg {
    static constexpr int N = 12;
    static constexpr uint32_t INV = bbc::FP_INV;
    static constexpr uint64_t INV64 = 0x89f3fffcfffcfffdull;
#if defined(__CUDACC__)
    static __device__ __forceinline__ uint32_t dmod(int k) { return kFpMod[k]; }
#elif defined(BB_EMULATE_PTX)
    static uint32_t dmod(int k) { return bbc::FP_MOD[k]; }
#endif
    static const uint32_t* hmod() { return bbc::FP_MOD; }
};
static_assert((uint32_t)FrCfg::INV64 == FrCfg::INV && (uint32_t)FpCfg::INV64 == FpCfg::INV, "inv");

typedef Fe<FrCfg> Fr;
typedef Fe<FpCfg> Fp;

BB_HD Fr fr_from_limbs(const uint32_t* p) { Fr r; for (int i = 0; i < 8; i++) r.l[i] = p[i]; return r; }
BB_HD Fp fp_from_limbs(const uint32_t* p) { Fp r; for (int i = 0; i < 12; i++) r.l[i] = p[i]; return r; }

// constants as immediates (constexpr arrays are not addressable from device code)
BB_HD Fr fr_one() { return Fr{{BBC_FR_R_LIST}}; }
BB_HD Fr fr_r2() { return Fr{{BBC_FR_R2_LIST}}; }
BB_HD Fr fr_generator() { return Fr{{BBC_FR_GENERATOR_M_LIST}}; }
BB_HD Fr fr_root_of_unity() { return Fr{{BBC_FR_ROOT_OF_UNITY_M_LIST}}; }
BB_HD Fp fp_one() { return Fp{{BBC_FP_R_LIST}}; }
BB_HD Fp fp_r2() { return Fp{{BBC_FP_R2_LIST}}; }

BB_HD Fr fr_raw_one() { Fr r = Fr::zero(); r.l[0] = 1; return r; }
BB_HD Fp fp_raw_one() { Fp r = Fp::zero(); r.l[0] = 1; return r; }
BB_HD Fr fr_to_canonical(const Fr& a) { return a * fr_raw_one(); }
BB_HD Fr fr_from_canonical(const Fr& a) { return a * fr_r2(); }
BB_HD Fp fp_to_canonical(const Fp& a) { return a * fp_raw_one(); }
BB_HD Fp fp_from_canonical(const Fp& a) { return a * fp_r2(); }
BB_HD Fr fr_from_u64(uint64_t v) { Fr r = Fr::zero(); r.l[0] = (uint32_t)v; r.l[1] = (uint32_t)(v >> 32); return fr_from_canonical(r); }

// a^(q-2)
BB_HD Fr fr_inv(const Fr& a) {
    uint32_t e[8];
    uint32_t borrow = 2;                       // r - 2 (the low 32-bit limb of r is 1: borrows)
    for (int i = 0; i < 8; i++) { uint32_t m = Fr::modl(i); e[i] = m - borrow; borrow = m < borrow ? 1u : 0u; }
    return a.pow(e, 8, fr_one());
}
BB_HD Fp fp_inv(const Fp& a) {
    uint32_t e[12];
    uint32_t borrow = 2;
    for (int i = 0; i < 12; i++) { uint32_t m = Fp::modl(i); e[i] = m - borrow; borrow = m < borrow ? 1u : 0u; }
    return a.pow(e, 12, fp_one());
}

// Inversion by the binary extended Euclidean algorithm on the raw limbs: at most 2 * 381 halving /
// subtraction steps of shifts and additions instead of the 570 dependent Montgomery products of a^(p-2).
// It runs where ONE thread inverts while everything else waits on it (the single inversion at the top of
// each batched-affine round, k_binv_top), so it is the latency of one thread that counts: ~5x shorter.
// Variable time (inputs there are products of public x-coordinate differences).  a != 0.
// On raw integers the loop yields (a R)^-1; one Montgomery product with R^3 turns that into a^-1 R.
template <class Cfg>
BB_HD Fe<Cfg> fe_inv_gcd(const Fe<Cfg>& a, const Fe<Cfg>& r2) {
    constexpr int N = Cfg::N;
    typedef Fe<Cfg> FE;
    uint32_t u[N], v[N], x1[N], x2[N], p[N];
    for (int i = 0; i < N; i++) { u[i] = a.l[i]; v[i] = p[i] = FE::modl(i); x1[i] = 0; x2[i] = 0; }
    x1[0] = 1;
    auto is_one = [&](const uint32_t* w) { uint32_t acc = w[0] ^ 1u; for (int i = 1; i < N; i++) acc |= w[i]; return acc == 0; };
    auto shr1 = [&](uint32_t* w) { for (int i = 0; i < N - 1; i++) w[i] = (w[i] >> 1) | (w[i + 1] << 31); w[N - 1] >>= 1; };
    auto add_p = [&](uint32_t* w) { uint64_t c = 0; for (int i = 0; i < N; i++) { c += (uint64_t)w[i] + p[i]; w[i] = (uint32_t)c; c >>= 32; } };   // no carry out: both < 2^(32N-1)
    auto sub = [&](uint32_t* w, const uint32_t* y) { int64_t b = 0; for (int i = 0; i < N; i++) { b += (int64_t)w[i] - y[i]; w[i] = (uint32_t)b; b >>= 32; } return b != 0; };
    auto geq = [&](const uint32_t* w, const uint32_t* y) { for (int i = N - 1; i >= 0; i--) { if (w[i] != y[i]) return w[i] > y[i]; } return true; };
    auto halve_mod = [&](uint32_t* x) { if (x[0] & 1u) add_p(x); shr1(x); };
    auto sub_mod = [&](uint32_t* x, const uint32_t* y) { if (sub(x, y)) add_p(x); };
    for (int guard = 0; guard < 4 * 32 * N && !is_one(u) && !is_one(v); guard++) {
        while (!(u[0] & 1u)) { shr1(u); halve_mod(x1); }
        while (!(v[0] & 1u)) { shr1(v); halve_mod(x2); }
        if (geq(u, v)) { sub(u, v); sub_mod(x1, x2); }
        else { sub(v, u); sub_mod(x2, x1); }
    }
    FE y;
    const uint32_t* res = is_one(u) ? x1 : x2;
    for (int i = 0; i < N; i++) y.l[i] = res[i];
    return y * (r2 * r2);                              // (a R)^-1 * R^3 * R^-1 = a^-1 R
}
BB_HD Fp fp_inv_gcd(const Fp& a) { return fe_inv_gcd<FpCfg>(a, fp_r2()); }

// Fp2 = Fp[u]/(u^2+1)
struct Fp2 {
    Fp c0, c1;
#if defined(__CUDACC__)
    static __device__ __forceinline__ uint32_t modsq(int k) { return kFpModSq[k]; }
#elif defined(BB_EMULATE_PTX)
    static uint32_t modsq(int k) { return bbc::FP_MODSQ[k]; }
#endif
    BB_HD static Fp2 zero() { return {Fp::zero(), Fp::zero()}; }
    BB_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    BB_HD bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
    BB_HD bool operator!=(const Fp2& o) const { return !(*this == o); }
    BB_HD Fp2 operator+(const Fp2& o) const { return {c0 + o.c0, c1 + o.c1}; }
    BB_HD Fp2 operator-(const Fp2& o) const { return {c0 - o.c0, c1 - o.c1}; }
    // Out of line on the device (BB_HD_NOINLINE): the tower, verifier and reduction kernels make hundreds of these
    // calls.  The operands of such a call are passed by address, so the caller keeps them in its local-memory stack
    // frame; the halving-round kernels (batch_affine.cuh) use the inlined forms through FieldOps instead.
    BB_HD_NOINLINE Fp2 operator*(const Fp2& o) const { return mul_inl(o); }
    BB_HD_NOINLINE Fp2 sqr() const { return sqr_inl(); }
    BB_HD Fp2 mul_inl(const Fp2& o) const {              // Karatsuba: 3 Fp products
#if defined(BB_DEVPATH) && BB_FP2_LAZY
        // lazy reduction: three 24-limb integer products, two Montgomery reductions.
        //   c0 = redc(a0 b0 + p^2 - a1 b1)              (< 2 p^2)
        //   c1 = redc((a0+a1)(b0+b1) - a0 b0 - a1 b1)   (= a0 b1 + a1 b0 < 2 p^2; sums < 2p fit 12 limbs)
        uint32_t T0[24], T1[24];
        wide_mul<12>(T0, c0.l, o.c0.l);
        wide_mul<12>(T1, c1.l, o.c1.l);
        uint32_t D[24];
        D[0] = ptx::add_cc(T0[0], modsq(0));
#pragma unroll
        for (int k = 1; k < 24; k++) D[k] = ptx::addc_cc(T0[k], modsq(k));
        D[0] = ptx::sub_cc(D[0], T1[0]);
#pragma unroll
        for (int k = 1; k < 24; k++) D[k] = ptx::subc_cc(D[k], T1[k]);
        T0[0] = ptx::add_cc(T0[0], T1[0]);                 // S = a0 b0 + a1 b1
#pragma unroll
        for (int k = 1; k < 24; k++) T0[k] = ptx::addc_cc(T0[k], T1[k]);
        Fp2 r;
        redc_wide<FpCfg>(r.c0.l, D);
        uint32_t sa[12], sb[12];
        sa[0] = ptx::add_cc(c0.l[0], c1.l[0]);
#pragma unroll
        for (int k = 1; k < 12; k++) sa[k] = ptx::addc_cc(c0.l[k], c1.l[k]);
        sb[0] = ptx::add_cc(o.c0.l[0], o.c1.l[0]);
#pragma unroll
        for (int k = 1; k < 12; k++) sb[k] = ptx::addc_cc(o.c0.l[k], o.c1.l[k]);
        wide_mul<12>(T1, sa, sb);
        T1[0] = ptx::sub_cc(T1[0], T0[0]);
#pragma unroll
        for (int k = 1; k < 24; k++) T1[k] = ptx::subc_cc(T1[k], T0[k]);
        redc_wide<FpCfg>(r.c1.l, T1);
        return r;
#else
        Fp aa = c0 * o.c0, bb_ = c1 * o.c1;
        Fp t = (c0 + c1) * (o.c0 + o.c1);
        return {aa - bb_, t - aa - bb_};
#endif
    }
    BB_HD Fp2 sqr_inl() const {                        // (c0+c1)(c0-c1), 2 c0 c1
        Fp s = c0 + c1, d = c0 - c1, m = c0 * c1;
        return {s * d, m + m};
    }
    BB_HD Fp2 dbl() const { return {c0.dbl(), c1.dbl()}; }
    BB_HD Fp2 neg() const { return {c0.neg(), c1.neg()}; }
    BB_HD Fp2& operator+=(const Fp2& o) { *this = *this + o; return *this; }
    BB_HD Fp2& operator-=(const Fp2& o) { *this = *this - o; return *this; }
    BB_HD Fp2& operator*=(const Fp2& o) { *this = *this * o; return *this; }
};
BB_HD Fp2 fp2_one() { return {fp_one(), Fp::zero()}; }
BB_HD Fp2 fp2_inv(const Fp2& a) {
    Fp n = fp_inv_gcd(a.c0.sqr() + a.c1.sqr());
    return {a.c0 * n, (a.c1 * n).neg()};
}

// uniform field-trait view used by the curve templates; mul / sqr are always inlined
template <class F> struct FieldOps;
template <> struct FieldOps<Fp> {
    BB_HD static Fp one() { return fp_one(); }
    BB_HD static Fp inv(const Fp& a) { return fp_inv_gcd(a); }
    BB_HD static Fp mul(const Fp& a, const Fp& b) { return a * b; }
    BB_HD static Fp sqr(const Fp& a) { return a.sqr(); }
    static constexpr int WORDS = 12;
};
template <> struct FieldOps<Fp2> {
    BB_HD static Fp2 one() { return fp2_one(); }
    BB_HD static Fp2 inv(const Fp2& a) { return fp2_inv(a); }
    BB_HD static Fp2 mul(const Fp2& a, const Fp2& b) { return a.mul_inl(b); }
    BB_HD static Fp2 sqr(const Fp2& a) { return a.sqr_inl(); }
    static constexpr int WORDS = 24;
};

}  // namespace bb
