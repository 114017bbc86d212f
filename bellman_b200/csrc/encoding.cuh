// bellman_b200: the ZCash encoding of BLS12-381 points that bls12_381 0.8 reads and writes (to_compressed /
// from_compressed, to_uncompressed / from_uncompressed), and the rules that go with it: the curve equation, coordinates
// below p and the prime-order subgroup.  Each rule is written once over Fp (G1) and Fp2 (G2).  The device decoders and
// encoders (decode.cu), the host proof bytes (prover.cu), point validation and compression (capi.cu) and the generator
// checks (generate.cu) all call these.
//
// A coordinate is the 48 big-endian bytes of its canonical integer; an Fp2 coordinate is c1, then c0.  The three top bits
// of a point's first byte are flags: 0x80 compressed, 0x40 the point at infinity, 0x20 (compressed only) the sort bit,
// set when y is the lexicographically larger of the two roots.
//
// Algorithms (variable time: the points decoded are public data):
//   Fp square root   a^((p+1)/4) (p = 3 mod 4) by a fixed 4-bit window over the constant exponent, then a squaring check
//   Fp2 square root  Algorithm 9 of eprint 2012/685: a1 = a^((p-3)/4), alpha = a1^2 a, x0 = a1 a; x = u x0 if alpha = -1,
//                    else (1 + alpha)^((p-1)/2) x0; then the squaring check
//   subgroup, G1     phi(P) = -[x^2] P with phi(x, y) = (beta x, y)    (eprint 2021/1130; proof in 2022/352)
//   subgroup, G2     psi(P) = [x] P with psi the untwist-Frobenius-twist map
// x = -0xd201000000010000: [x^2] is two multiplications by |x| (126 doublings, 10 additions), [x] one.  rP_is_identity is
// the plain [r]P = O test.
#pragma once
#include "curve.cuh"

namespace bb {

// why a point does not decode, in the order of the checks (include/bellman_b200.h, BB_READ_*)
constexpr int WHY_OK = 0, WHY_FLAGS = 1, WHY_NONCANONICAL = 2, WHY_NOT_ON_CURVE = 3, WHY_NOT_IN_SUBGROUP = 4, WHY_IDENTITY = 5;

#if defined(__CUDACC__)
static __device__ __constant__ uint32_t kExpSqrt[12] = {BBC_EXP_SQRT_LIST};     // (p + 1) / 4
static __device__ __constant__ uint32_t kExpSqrt2[12] = {BBC_EXP_SQRT2_LIST};   // (p - 3) / 4
static __device__ __constant__ uint32_t kFpHalf[12] = {BBC_FP_HALF_LIST};       // (p - 1) / 2
#else
static const uint32_t kExpSqrt[12] = {BBC_EXP_SQRT_LIST};
static const uint32_t kExpSqrt2[12] = {BBC_EXP_SQRT2_LIST};
static const uint32_t kFpHalf[12] = {BBC_FP_HALF_LIST};
#endif

// limb k of (p - 1) / 2: constant memory on the device, the host table on the host (as Fe::modl)
BB_HD uint32_t fp_half(int k) {
#if defined(BB_DEVPATH)
    return kFpHalf[k];
#else
    return bbc::FP_HALF[k];
#endif
}

// b of y^2 = x^3 + b: 4 on E (G1), 4(u + 1) on E' (G2)
template <class F> BB_HD F curve_b();
template <> BB_HD Fp curve_b<Fp>() { Fp four = Fp::zero(); four.l[0] = 4; return fp_from_canonical(four); }
template <> BB_HD Fp2 curve_b<Fp2>() { Fp b = curve_b<Fp>(); return {b, b}; }

template <class F>
BB_HD bool on_curve(const Affine<F>& p) { return p.y.sqr() == p.x.sqr() * p.x + curve_b<F>(); }

// the limbs are below p (every coordinate of an Fp2)
BB_HD bool is_canonical(const Fp& x) {
    for (int k = 11; k >= 0; k--) {
        uint32_t m = Fp::modl(k);
        if (x.l[k] != m) return x.l[k] < m;
    }
    return false;
}
BB_HD bool is_canonical(const Fp2& x) { return is_canonical(x.c0) && is_canonical(x.c1); }

BB_HD Fp from_canonical(const Fp& x) { return fp_from_canonical(x); }
BB_HD Fp2 from_canonical(const Fp2& x) { return {fp_from_canonical(x.c0), fp_from_canonical(x.c1)}; }

// the sort bit of a Montgomery y: canonical y > (p - 1) / 2; in Fp2 y.c1 decides, y.c0 when y.c1 is zero
BB_HD bool lexi_larger(const Fp& y) {
    Fp c = fp_to_canonical(y);
    for (int k = 11; k >= 0; k--)
        if (c.l[k] != fp_half(k)) return c.l[k] > fp_half(k);
    return false;
}
BB_HD bool lexi_larger(const Fp2& y) { return y.c1.is_zero() ? lexi_larger(y.c0) : lexi_larger(y.c1); }

// big-endian bytes -> canonical limbs, the top byte masked by mask0 (the flag bits); sizeof(F) bytes
BB_HD void load_be(Fp& r, const uint8_t* s, uint32_t mask0) {
    for (int k = 0; k < 12; k++) {
        const uint8_t* q = s + 44 - 4 * k;
        uint32_t b0 = k == 11 ? (q[0] & mask0) : q[0];
        r.l[k] = (b0 << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    }
}
BB_HD void load_be(Fp2& r, const uint8_t* s, uint32_t mask0) { load_be(r.c1, s, mask0); load_be(r.c0, s + 48, 0xff); }
// a Montgomery coordinate -> its canonical big-endian bytes
BB_HD void store_be(const Fp& v, uint8_t* o) {
    Fp c = fp_to_canonical(v);
    for (int k = 0; k < 12; k++) {
        uint8_t* q = o + 44 - 4 * k;
        uint32_t w = c.l[k];
        q[0] = (uint8_t)(w >> 24); q[1] = (uint8_t)(w >> 16); q[2] = (uint8_t)(w >> 8); q[3] = (uint8_t)w;
    }
}
BB_HD void store_be(const Fp2& v, uint8_t* o) { store_be(v.c1, o); store_be(v.c0, o + 48); }
static_assert(sizeof(Fp) == 48 && sizeof(Fp2) == 96, "an encoded coordinate is as long as its limbs");

// ---- square roots --------------------------------------------------------------------------------------------------
// a^e for a constant 384-bit exponent e (12 limbs), fixed 4-bit windows: 15 products for the table, then per window
// four squarings and at most one product
template <class F>
BB_D F pow_fixed(const F& a, const uint32_t* e) {
    F tab[16];
    tab[0] = FieldOps<F>::one();
    tab[1] = a;
    for (int k = 2; k < 16; k++) tab[k] = tab[k - 1] * a;
    int w = 95;
    while (w > 0 && ((e[w >> 3] >> (4 * (w & 7))) & 15u) == 0) w--;
    F r = tab[(e[w >> 3] >> (4 * (w & 7))) & 15u];
    for (w--; w >= 0; w--) {
        r = r.sqr(); r = r.sqr(); r = r.sqr(); r = r.sqr();
        uint32_t d = (e[w >> 3] >> (4 * (w & 7))) & 15u;
        if (d) r = r * tab[d];
    }
    return r;
}

template <class F> struct Root { F v; bool ok; };

BB_D Root<Fp> square_root(const Fp& a) {
    Fp r = pow_fixed(a, kExpSqrt);
    return {r, r.sqr() == a};
}
BB_D Root<Fp2> square_root(const Fp2& a) {
    Fp2 a1 = pow_fixed(a, kExpSqrt2);
    Fp2 alpha = a1.sqr() * a;
    Fp2 x0 = a1 * a;
    Fp2 minus_one{fp_one().neg(), Fp::zero()};
    Fp2 x;
    if (alpha == minus_one) x = Fp2{x0.c1.neg(), x0.c0};                            // u * x0
    else x = pow_fixed(alpha + fp2_one(), kFpHalf) * x0;
    return {x, x.sqr() == a};
}

// ---- the prime-order subgroup --------------------------------------------------------------------------------------
// [|x|] P, |x| = 0xd201000000010000: 63 doublings, 5 additions
template <class F>
BB_D XYZZ<F> mul_by_x_abs(const XYZZ<F>& p) {
    XYZZ<F> acc = p;
    for (int i = 62; i >= 0; i--) {
        acc = acc.dbl();
        if ((bbc::BLS_X_ABS >> i) & 1) acc.add(p);
    }
    return acc;
}
// q == (x, y) for an affine (x, y) that is not the identity
template <class F>
BB_D bool xyzz_equals_affine(const XYZZ<F>& q, const F& x, const F& y) {
    return !q.is_identity() && q.X == x * q.ZZ && q.Y == y * q.ZZZ;
}
BB_D Fp2 fp2_conj(const Fp2& a) { return {a.c0, a.c1.neg()}; }
// phi(P) = -[x^2] P  <=>  [x^2] P = (beta x, -y)
BB_D bool in_subgroup(const G1Affine& p) {
    G1X q = mul_by_x_abs(mul_by_x_abs(G1X::from_affine(p)));
    return xyzz_equals_affine(q, p.x * Fp{{BBC_BETA_M_LIST}}, p.y.neg());
}
// psi(P) = [x] P = -[|x|] P  <=>  [|x|] P = -psi(P)
BB_D bool in_subgroup(const G2Affine& p) {
    const Fp2 psi_x{Fp{{BBC_PSI_X_C0_M_LIST}}, Fp{{BBC_PSI_X_C1_M_LIST}}};
    const Fp2 psi_y{Fp{{BBC_PSI_Y_C0_M_LIST}}, Fp{{BBC_PSI_Y_C1_M_LIST}}};
    G2X q = mul_by_x_abs(G2X::from_affine(p));
    return xyzz_equals_affine(q, fp2_conj(p.x) * psi_x, (fp2_conj(p.y) * psi_y).neg());
}
// [r] P = O, by a 255-bit double-and-add
template <class F>
BB_HD bool rP_is_identity(const Affine<F>& p) {
    const uint32_t r[8] = {BBC_FR_MOD_LIST};
    return XYZZ<F>::from_affine(p).mul_bits(r).is_identity();
}

// ---- compressed points: sizeof(F) bytes ----------------------------------------------------------------------------
// to_compressed
template <class F>
BB_HD void encode_compressed(const Affine<F>& p, uint8_t* o) {
    if (p.is_identity()) { o[0] = 0xc0; for (int k = 1; k < (int)sizeof(F); k++) o[k] = 0; return; }
    store_be(p.x, o);
    o[0] |= 0x80 | (lexi_larger(p.y) ? 0x20 : 0);
}

// from_compressed (check_subgroup) or from_compressed_unchecked; p = the point, or the identity unless why is WHY_OK
template <class F> struct Decoded { Affine<F> p; int why; };

template <class F>
BB_D Decoded<F> decode_compressed(const uint8_t* s, bool check_subgroup) {
    const Affine<F> none = Affine<F>::identity();
    const uint32_t flags = s[0];
    F x;
    load_be(x, s, 0x1f);
    if (!(flags & 0x80)) return {none, WHY_FLAGS};
    if (flags & 0x40) return {none, (flags & 0x20) || !x.is_zero() ? WHY_FLAGS : WHY_IDENTITY};
    if (!is_canonical(x)) return {none, WHY_NONCANONICAL};
    F xm = from_canonical(x);
    Root<F> y = square_root(xm.sqr() * xm + curve_b<F>());
    if (!y.ok) return {none, WHY_NOT_ON_CURVE};
    if (lexi_larger(y.v) != ((flags & 0x20) != 0)) y.v = y.v.neg();
    Affine<F> p{xm, y.v};
    if (check_subgroup && !in_subgroup(p)) return {none, WHY_NOT_IN_SUBGROUP};
    return {p, WHY_OK};
}

// ---- uncompressed points: 2 sizeof(F) bytes, x then y --------------------------------------------------------------
// to_uncompressed; the identity is the infinity flag, then zeros
template <class F>
BB_HD void store_uncompressed(const Affine<F>& p, uint8_t* o) {
    if (p.is_identity()) { o[0] = 0x40; for (int k = 1; k < 2 * (int)sizeof(F); k++) o[k] = 0; return; }
    store_be(p.x, o);
    store_be(p.y, o + sizeof(F));
}

// from_uncompressed (checked) or from_uncompressed_unchecked, then bellman's identity rule (the identity is an error
// unless allow_identity); *out = the Montgomery point when the result is WHY_OK
template <class F>
BB_D int read_uncompressed(const uint8_t* s, bool checked, bool allow_identity, Affine<F>* out) {
    const uint32_t flags = s[0];
    if (flags & 0xa0) return WHY_FLAGS;                                  // compression or sort bit
    F x, y;
    load_be(x, s, 0x1f);
    load_be(y, s + sizeof(F), 0xff);
    if (flags & 0x40) {
        if (!x.is_zero() || !y.is_zero()) return WHY_FLAGS;
        *out = Affine<F>::identity();
        return allow_identity ? WHY_OK : WHY_IDENTITY;
    }
    if (!is_canonical(x) || !is_canonical(y)) return WHY_NONCANONICAL;
    Affine<F> p{from_canonical(x), from_canonical(y)};
    if (checked) {
        if (!on_curve(p)) return WHY_NOT_ON_CURVE;
        if (!in_subgroup(p)) return WHY_NOT_IN_SUBGROUP;
    }
    *out = p;
    return WHY_OK;
}

}  // namespace bb
