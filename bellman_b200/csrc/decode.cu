// bellman_b200: Proof::read and Proof::write over a batch on the device (groth16/src/lib.rs:39-99).
//
// A proof is the 192-byte encoding of Proof::write: compressed A (48 B), B (96 B), C (48 B) in the ZCash format of
// bls12_381 0.8 (to_compressed / from_compressed).  Reading a point follows from_compressed and then bellman's identity
// rule; the first failing check decides its code (bellman_b200.h, bb_proofs_read):
//   1 bad flags       compression bit clear; or the infinity bit with the sort bit or any bit of x set
//   2 non-canonical   x >= p (G2: either coordinate)
//   3 not on curve    x^3 + b has no square root
//   4 not in subgroup the point is not of order r
//   5 identity        a valid encoding of the point at infinity (Proof::read: "point at infinity")
// A proof reads A, then B, then C; its status is (which << 4) | why of the first failing element.
//
// Algorithms (variable time throughout: proof bytes are public data):
//   Fp square root   a^((p+1)/4) (p = 3 mod 4) by a fixed 4-bit window over the constant exponent, then a squaring check
//   Fp2 square root  Algorithm 9 of eprint 2012/685: a1 = a^((p-3)/4), alpha = a1^2 a, x0 = a1 a; x = u x0 if alpha = -1,
//                    else (1 + alpha)^((p-1)/2) x0; then the squaring check
//   subgroup, G1     phi(P) = -[x^2] P with phi(x, y) = (beta x, y)    (eprint 2021/1130; proof in 2022/352)
//   subgroup, G2     psi(P) = [x] P with psi the untwist-Frobenius-twist map
// x = -0xd201000000010000: [x^2] is two multiplications by |x| (126 doublings, 10 additions), [x] one.
// Kernels (one thread per point):
//   k_decode_g1      the 2n A and C points (or n packed points for the diagnostic)
//   k_decode_g2      the n B points
//   k_proof_status   folds the three element codes into the status byte, zeroes all points of an invalid proof
//   k_encode_proofs  the inverse: Proof::write of n affine triples
// Nothing outside this file calls into it.
#include "bb_internal.cuh"

using namespace bb;

namespace {

constexpr unsigned DECODE_THREADS = 64;

#if defined(__CUDACC__)
static __device__ __constant__ uint32_t kExpSqrt[12] = {BBC_EXP_SQRT_LIST};     // (p + 1) / 4
static __device__ __constant__ uint32_t kExpSqrt2[12] = {BBC_EXP_SQRT2_LIST};   // (p - 3) / 4
static __device__ __constant__ uint32_t kFpHalf[12] = {BBC_FP_HALF_LIST};       // (p - 1) / 2
#else
static const uint32_t kExpSqrt[12] = {BBC_EXP_SQRT_LIST};
static const uint32_t kExpSqrt2[12] = {BBC_EXP_SQRT2_LIST};
static const uint32_t kFpHalf[12] = {BBC_FP_HALF_LIST};
#endif

constexpr int WHY_OK = 0, WHY_FLAGS = 1, WHY_NONCANONICAL = 2, WHY_NOT_ON_CURVE = 3, WHY_NOT_IN_SUBGROUP = 4, WHY_IDENTITY = 5;

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

BB_D Root<Fp> fp_sqrt(const Fp& a) {
    Fp r = pow_fixed(a, kExpSqrt);
    return {r, r.sqr() == a};
}

BB_D Root<Fp2> fp2_sqrt(const Fp2& a) {
    Fp2 a1 = pow_fixed(a, kExpSqrt2);
    Fp2 alpha = a1.sqr() * a;
    Fp2 x0 = a1 * a;
    Fp2 minus_one{fp_one().neg(), Fp::zero()};
    Fp2 x;
    if (alpha == minus_one) x = Fp2{x0.c1.neg(), x0.c0};                            // u * x0
    else x = pow_fixed(alpha + fp2_one(), kFpHalf) * x0;
    return {x, x.sqr() == a};
}

BB_D Fp g1_b() { Fp four = Fp::zero(); four.l[0] = 4; return fp_from_canonical(four); }
BB_D Fp2 g2_b() { Fp b = g1_b(); return {b, b}; }

// 48 big-endian bytes -> canonical limbs; the top byte masked by mask0 (the flag bits)
BB_D Fp fp_load_be(const uint8_t* s, uint32_t mask0) {
    Fp r;
    for (int k = 0; k < 12; k++) {
        const uint8_t* q = s + 44 - 4 * k;
        uint32_t b0 = k == 11 ? (q[0] & mask0) : q[0];
        r.l[k] = (b0 << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    }
    return r;
}
BB_D void fp_store_be(const Fp& canonical, uint8_t* o) {
    for (int k = 0; k < 12; k++) {
        uint8_t* q = o + 44 - 4 * k;
        uint32_t v = canonical.l[k];
        q[0] = (uint8_t)(v >> 24); q[1] = (uint8_t)(v >> 16); q[2] = (uint8_t)(v >> 8); q[3] = (uint8_t)v;
    }
}
BB_D bool fp_is_canonical(const Fp& x) {
    for (int k = 11; k >= 0; k--) {
        uint32_t m = Fp::modl(k);
        if (x.l[k] != m) return x.l[k] < m;
    }
    return false;
}
// canonical y > (p - 1) / 2, for a Montgomery y
BB_D bool fp_lexi_larger(const Fp& y) {
    Fp c = fp_to_canonical(y);
    for (int k = 11; k >= 0; k--)
        if (c.l[k] != kFpHalf[k]) return c.l[k] > kFpHalf[k];
    return false;
}
BB_D bool fp2_lexi_larger(const Fp2& y) { return y.c1.is_zero() ? fp_lexi_larger(y.c0) : fp_lexi_larger(y.c1); }
BB_D Fp2 fp2_conj(const Fp2& a) { return {a.c0, a.c1.neg()}; }

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
// phi(P) = -[x^2] P  <=>  [x^2] P = (beta x, -y)
BB_D bool g1_in_subgroup(const G1Affine& p) {
    G1X q = mul_by_x_abs(mul_by_x_abs(G1X::from_affine(p)));
    return xyzz_equals_affine(q, p.x * Fp{{BBC_BETA_M_LIST}}, p.y.neg());
}
// psi(P) = [x] P = -[|x|] P  <=>  [|x|] P = -psi(P)
BB_D bool g2_in_subgroup(const G2Affine& p) {
    const Fp2 psi_x{Fp{{BBC_PSI_X_C0_M_LIST}}, Fp{{BBC_PSI_X_C1_M_LIST}}};
    const Fp2 psi_y{Fp{{BBC_PSI_Y_C0_M_LIST}}, Fp{{BBC_PSI_Y_C1_M_LIST}}};
    G2X q = mul_by_x_abs(G2X::from_affine(p));
    return xyzz_equals_affine(q, fp2_conj(p.x) * psi_x, (fp2_conj(p.y) * psi_y).neg());
}

// from_compressed (check_subgroup != 0) or from_compressed_unchecked of one point; out = the point, or zeros unless 0
template <class F> struct Decoded { Affine<F> p; int why; };

BB_D Decoded<Fp> g1_decode(const uint8_t* s, bool check_subgroup) {
    const G1Affine none = G1Affine::identity();
    const uint32_t flags = s[0];
    Fp x = fp_load_be(s, 0x1f);
    if (!(flags & 0x80)) return {none, WHY_FLAGS};
    if (flags & 0x40) return {none, (flags & 0x20) || !x.is_zero() ? WHY_FLAGS : WHY_IDENTITY};
    if (!fp_is_canonical(x)) return {none, WHY_NONCANONICAL};
    Fp xm = fp_from_canonical(x);
    Root<Fp> y = fp_sqrt(xm.sqr() * xm + g1_b());
    if (!y.ok) return {none, WHY_NOT_ON_CURVE};
    if (fp_lexi_larger(y.v) != ((flags & 0x20) != 0)) y.v = y.v.neg();
    G1Affine p{xm, y.v};
    if (check_subgroup && !g1_in_subgroup(p)) return {none, WHY_NOT_IN_SUBGROUP};
    return {p, WHY_OK};
}

BB_D Decoded<Fp2> g2_decode(const uint8_t* s, bool check_subgroup) {
    const G2Affine none = G2Affine::identity();
    const uint32_t flags = s[0];
    Fp x1 = fp_load_be(s, 0x1f), x0 = fp_load_be(s + 48, 0xff);
    if (!(flags & 0x80)) return {none, WHY_FLAGS};
    if (flags & 0x40) return {none, (flags & 0x20) || !x0.is_zero() || !x1.is_zero() ? WHY_FLAGS : WHY_IDENTITY};
    if (!fp_is_canonical(x0) || !fp_is_canonical(x1)) return {none, WHY_NONCANONICAL};
    Fp2 xm{fp_from_canonical(x0), fp_from_canonical(x1)};
    Root<Fp2> y = fp2_sqrt(xm.sqr() * xm + g2_b());
    if (!y.ok) return {none, WHY_NOT_ON_CURVE};
    if (fp2_lexi_larger(y.v) != ((flags & 0x20) != 0)) y.v = y.v.neg();
    G2Affine p{xm, y.v};
    if (check_subgroup && !g2_in_subgroup(p)) return {none, WHY_NOT_IN_SUBGROUP};
    return {p, WHY_OK};
}

// point j of rows x parts: bytes base + (j % rows) * stride + (j / rows) * part_offset -> out[j / rows][j % rows]
__global__ void __launch_bounds__(DECODE_THREADS) k_decode_g1(const uint8_t* __restrict__ base, size_t stride, size_t rows, size_t parts,
                                                              size_t part_offset, int check_subgroup, G1Affine* out0, G1Affine* out1,
                                                              uint8_t* why) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= rows * parts) return;
    size_t row = j % rows, part = j / rows;
    Decoded<Fp> d = g1_decode(base + row * stride + part * part_offset, check_subgroup != 0);
    (part ? out1 : out0)[row] = d.p;
    why[j] = (uint8_t)d.why;
}
__global__ void __launch_bounds__(DECODE_THREADS) k_decode_g2(const uint8_t* __restrict__ base, size_t stride, size_t rows,
                                                              int check_subgroup, G2Affine* out, uint8_t* why) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= rows) return;
    Decoded<Fp2> d = g2_decode(base + j * stride, check_subgroup != 0);
    out[j] = d.p;
    why[j] = (uint8_t)d.why;
}
// why_ac: n codes of A then n of C; status (which << 4) | why of the first failing element in A, B, C order
__global__ void __launch_bounds__(128) k_proof_status(const uint8_t* __restrict__ why_ac, const uint8_t* __restrict__ why_b, size_t n,
                                                      G1Affine* a, G2Affine* b, G1Affine* c, uint8_t* status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t wa = why_ac[i], wb = why_b[i], wc = why_ac[n + i];
    uint8_t s = wa ? (uint8_t)(0x10 | wa) : wb ? (uint8_t)(0x20 | wb) : wc ? (uint8_t)(0x30 | wc) : (uint8_t)0;
    status[i] = s;
    if (s) {                                                     // nothing half-decoded leaves an invalid proof
        a[i] = G1Affine::identity();
        b[i] = G2Affine::identity();
        c[i] = G1Affine::identity();
    }
}

// Proof::write (lib.rs:39-45): to_compressed of A, B, C
BB_D void g1_encode(const G1Affine& p, uint8_t* o) {
    if (p.is_identity()) { o[0] = 0xc0; for (int k = 1; k < 48; k++) o[k] = 0; return; }
    fp_store_be(fp_to_canonical(p.x), o);
    o[0] |= 0x80 | (fp_lexi_larger(p.y) ? 0x20 : 0);
}
BB_D void g2_encode(const G2Affine& p, uint8_t* o) {
    if (p.is_identity()) { o[0] = 0xc0; for (int k = 1; k < 96; k++) o[k] = 0; return; }
    fp_store_be(fp_to_canonical(p.x.c1), o);
    fp_store_be(fp_to_canonical(p.x.c0), o + 48);
    o[0] |= 0x80 | (fp2_lexi_larger(p.y) ? 0x20 : 0);
}
__global__ void __launch_bounds__(128) k_encode_proofs(const G1Affine* __restrict__ a, const G2Affine* __restrict__ b,
                                                       const G1Affine* __restrict__ c, size_t n, uint8_t* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t* o = out + i * 192;
    g1_encode(a[i], o);
    g2_encode(b[i], o + 48);
    g1_encode(c[i], o + 144);
}

constexpr size_t MAX_PROOFS = (size_t)1 << 31;

}  // namespace

extern "C" {

int bb_proofs_read(bb_ctx* ctx, const bb_proof_bytes* in, void* a, void* b, void* c, int out_on_device, uint8_t* status, size_t* n_invalid) {
    if (!ctx || !in || !n_invalid) { set_error("bb_proofs_read: null argument"); return BB_ERR_ARG; }
    const size_t n = in->n, stride = in->stride ? in->stride : 192;
    if (stride < 192) { set_error("bb_proofs_read: stride %zu is below the 192 bytes of a proof", stride); return BB_ERR_ARG; }
    if (n && (!in->bytes || !a || !b || !c || !status)) { set_error("bb_proofs_read: null pointer with n = %zu", n); return BB_ERR_ARG; }
    if (n >= MAX_PROOFS) { set_error("bb_proofs_read: more than 2^31 proofs"); return BB_ERR_ARG; }
    *n_invalid = 0;
    if (!n) return BB_OK;
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("proofs_read");
    cudaStream_t st = ctx->main_stream;
    StageTimer tm(ctx, st);
    tm.mark("decode.begin");
    const uint8_t* src = (const uint8_t*)in->bytes;
    size_t src_stride = stride;
    DevBuf up, d_a, d_b, d_c, d_why, d_status;
    if (!in->on_device) {                                        // only the 192 proof bytes of each record cross the bus
        BB_TRY(up.alloc(ctx, n * 192));
        BB_CUDA(cudaMemcpy2DAsync(up.p, 192, in->bytes, stride, 192, n, cudaMemcpyHostToDevice, st));
        ctx->h2d_bytes += n * 192;
        src = up.as<uint8_t>();
        src_stride = 192;
    }
    tm.mark("decode.upload");
    G1Affine *oa = (G1Affine*)a, *oc = (G1Affine*)c;
    G2Affine* ob = (G2Affine*)b;
    if (!out_on_device) {
        BB_TRY(d_a.alloc(ctx, n * sizeof(G1Affine)));
        BB_TRY(d_b.alloc(ctx, n * sizeof(G2Affine)));
        BB_TRY(d_c.alloc(ctx, n * sizeof(G1Affine)));
        oa = d_a.as<G1Affine>(); ob = d_b.as<G2Affine>(); oc = d_c.as<G1Affine>();
    }
    BB_TRY(d_why.alloc(ctx, 3 * n));
    BB_TRY(d_status.alloc(ctx, n));
    uint8_t* why_ac = d_why.as<uint8_t>();
    uint8_t* why_b = why_ac + 2 * n;
    k_decode_g1<<<cdiv(2 * n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(src, src_stride, n, 2, 144, 1, oa, oc, why_ac);
    ctx->count_launch();
    tm.mark("decode.g1");
    k_decode_g2<<<cdiv(n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(src + 48, src_stride, n, 1, ob, why_b);
    ctx->count_launch();
    tm.mark("decode.g2");
    k_proof_status<<<cdiv(n, 128), 128, 0, st>>>(why_ac, why_b, n, oa, ob, oc, d_status.as<uint8_t>());
    ctx->count_launch();
    tm.mark("decode.status");
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaMemcpyAsync(status, d_status.p, n, cudaMemcpyDeviceToHost, st));
    if (!out_on_device) {
        BB_CUDA(cudaMemcpyAsync(a, oa, n * sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(b, ob, n * sizeof(G2Affine), cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(c, oc, n * sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
        ctx->d2h_bytes += n * (2 * sizeof(G1Affine) + sizeof(G2Affine));
    }
    ctx->d2h_bytes += n;
    tm.mark("decode.download");
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(n);
    size_t bad = 0;
    for (size_t i = 0; i < n; i++) bad += status[i] != 0;
    *n_invalid = bad;
    return BB_OK;
}

int bb_proofs_write(bb_ctx* ctx, const void* a, const void* b, const void* c, size_t n, int on_device, void* out) {
    if (!ctx || (n && (!a || !b || !c || !out))) { set_error("bb_proofs_write: null argument"); return BB_ERR_ARG; }
    if (n >= MAX_PROOFS) { set_error("bb_proofs_write: more than 2^31 proofs"); return BB_ERR_ARG; }
    if (!n) return BB_OK;
    BB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->main_stream;
    const G1Affine *da = (const G1Affine*)a, *dc = (const G1Affine*)c;
    const G2Affine* db = (const G2Affine*)b;
    uint8_t* dout = (uint8_t*)out;
    DevBuf up_a, up_b, up_c, d_out;
    if (!on_device) {
        BB_TRY(up_a.alloc(ctx, n * sizeof(G1Affine)));
        BB_TRY(up_b.alloc(ctx, n * sizeof(G2Affine)));
        BB_TRY(up_c.alloc(ctx, n * sizeof(G1Affine)));
        BB_TRY(d_out.alloc(ctx, n * 192));
        BB_CUDA(cudaMemcpyAsync(up_a.p, a, n * sizeof(G1Affine), cudaMemcpyHostToDevice, st));
        BB_CUDA(cudaMemcpyAsync(up_b.p, b, n * sizeof(G2Affine), cudaMemcpyHostToDevice, st));
        BB_CUDA(cudaMemcpyAsync(up_c.p, c, n * sizeof(G1Affine), cudaMemcpyHostToDevice, st));
        da = up_a.as<G1Affine>(); db = up_b.as<G2Affine>(); dc = up_c.as<G1Affine>(); dout = d_out.as<uint8_t>();
    }
    k_encode_proofs<<<cdiv(n, 128), 128, 0, st>>>(da, db, dc, n, dout);
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    if (!on_device) BB_CUDA(cudaMemcpyAsync(out, dout, n * 192, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

int bb_diag_points_decompress(bb_ctx* ctx, int group, const void* bytes, size_t n, int check_subgroup, void* out, uint8_t* why) {
    if (!ctx || (group != BB_G1 && group != BB_G2) || (n && (!bytes || !out || !why))) {
        set_error("bb_diag_points_decompress: bad argument");
        return BB_ERR_ARG;
    }
    if (n >= MAX_PROOFS) { set_error("bb_diag_points_decompress: more than 2^31 points"); return BB_ERR_ARG; }
    if (!n) return BB_OK;
    BB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->main_stream;
    const size_t enc = group == BB_G1 ? 48 : 96, pt = group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine);
    DevBuf d_in, d_out, d_why;
    BB_TRY(d_in.alloc(ctx, n * enc));
    BB_TRY(d_out.alloc(ctx, n * pt));
    BB_TRY(d_why.alloc(ctx, n));
    BB_CUDA(cudaMemcpyAsync(d_in.p, bytes, n * enc, cudaMemcpyHostToDevice, st));
    if (group == BB_G1)
        k_decode_g1<<<cdiv(n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(d_in.as<uint8_t>(), enc, n, 1, 0, check_subgroup, d_out.as<G1Affine>(),
                                                                         d_out.as<G1Affine>(), d_why.as<uint8_t>());
    else
        k_decode_g2<<<cdiv(n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(d_in.as<uint8_t>(), enc, n, check_subgroup, d_out.as<G2Affine>(),
                                                                         d_why.as<uint8_t>());
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaMemcpyAsync(out, d_out.p, n * pt, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(why, d_why.p, n, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    return BB_OK;
}

}  // extern "C"
