// bellman_b200: the device side of groth16::create_proof after synthesis
// (bellman/groth16/src/prover.rs:217-360): CRS residency, the H pipeline, the eight
// multiexps in flight, and the host finalisation.
#include <sched.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <functional>
#include <memory>
#include <string>
#include <thread>

#include "bb_internal.cuh"
#include "encoding.cuh"

using namespace bb;

struct bb_crs {
    bb_ctx* ctx = nullptr;
    bb_bases *h = nullptr, *l = nullptr, *a = nullptr, *b_g1 = nullptr, *b_g2 = nullptr;
    G1Affine alpha_g1, beta_g1, delta_g1;
    G2Affine beta_g2, delta_g2;
    uint32_t shard_index = 0, shard_count = 1;
};

namespace {

// Shard `idx` of `cnt` -> (base range b of nb) x (window shard v of nv).  Any partition of the
// (base, window) pairs of an MSM folds to the same point, so the shards split the windows first
// (that also divides the per-window bucket reduction, which base ranges alone do not) and the
// base vector second: nv = the largest divisor of cnt not above ctx->opt_shard_windows (4),
// nb = cnt / nv.  8 GPUs: 2 base ranges x 4 window shards.
void shard_policy(const bb_ctx* ctx, uint32_t idx, uint32_t cnt, uint32_t* b, uint32_t* nb, uint32_t* v, uint32_t* nv) {
    uint32_t lim = (uint32_t)(ctx->opt_shard_windows < 1 ? 1 : ctx->opt_shard_windows), w = 1;
    for (uint32_t d = 1; d <= lim && d <= cnt; d++) if (cnt % d == 0) w = d;
    *nv = w; *nb = cnt / w; *v = idx % w; *b = idx / w;
}

// scalar multiplication on the host (the five Affine * Fr of prover.rs:326-337 and the two
// MulAssign<Fr> of :342,351); k is a canonical little-endian 256-bit integer.  The scalars here are the
// proof's blinding factors r, s (and r s), so the sequence of operations does not depend on them:
//   * regular signed-digit recoding (Joye-Tunstall): with k made odd, k = 16^64 + sum_{i<64} d_i 16^i where
//     d_i = (((k >> 4i) | 1) & 31) - 16 is odd and non-zero -- every digit costs four doublings and ONE
//     addition, none is skipped;
//   * the table of odd multiples P, 3P, ..., 15P is read in full for every digit and the entry (and its sign) is
//     selected under a mask -- no secret-dependent address or branch;
//   * an even k is handled as (k + 1) P - P, both results computed, one selected under a mask.
// What is left: the XYZZ formulas branch on exceptional operands (identity, P = +-Q), which no digit of a
// random scalar produces for a point of prime order, and the host field arithmetic ends its products with a
// data-dependent final subtraction.  (The reference multiplies with the bls12_381 crate's constant-time routine.)
template <class T>
void masked_select(T* dst, const T& a, const T& b, uint32_t take_b) {     // take_b = 0 or 0xffffffff
    static_assert(sizeof(T) % 4 == 0, "whole words");
    uint32_t wa[sizeof(T) / 4], wb[sizeof(T) / 4];
    std::memcpy(wa, &a, sizeof(T));
    std::memcpy(wb, &b, sizeof(T));
    for (size_t i = 0; i < sizeof(T) / 4; i++) wa[i] = (wa[i] & ~take_b) | (wb[i] & take_b);
    std::memcpy(dst, wa, sizeof(T));
}

template <class F>
XYZZ<F> host_mul(const XYZZ<F>& p, const uint32_t* k_in) {
    uint32_t k[9];
    const uint32_t even = (~k_in[0]) & 1u;                  // k -> k + 1 when even (no carry out: the low bit is clear)
    for (int i = 0; i < 8; i++) k[i] = k_in[i];
    k[0] |= 1u;
    k[8] = 0;
    XYZZ<F> tab[8];                                         // (2j + 1) P
    const XYZZ<F> p2 = p.dbl();
    tab[0] = p;
    for (int j = 1; j < 8; j++) { tab[j] = tab[j - 1]; tab[j].add(p2); }
    XYZZ<F> acc = p;                                        // the leading digit is always 1 (bit 256)
    for (int i = 63; i >= 0; i--) {
        for (int d = 0; d < 4; d++) acc = acc.dbl();
        const uint32_t pos = 4u * (uint32_t)i, word = pos >> 5, off = pos & 31u;
        const uint64_t two = (uint64_t)k[word] | ((uint64_t)k[word + 1] << 32);
        const uint32_t v = ((uint32_t)(two >> off) | 1u) & 31u;          // odd, 1..31; digit = v - 16
        const uint32_t negative = 0u - (uint32_t)(v < 16u);               // mask
        const uint32_t mag = ((16u - v) & negative) | ((v - 16u) & ~negative);   // |digit|: odd, 1..15
        const uint32_t idx = mag >> 1;
        XYZZ<F> t = tab[0];
        for (uint32_t j = 1; j < 8; j++) masked_select(&t, t, tab[j], 0u - (uint32_t)(j == idx));
        const XYZZ<F> tn = t.neg();
        masked_select(&t, t, tn, negative);
        acc.add(t);
    }
    XYZZ<F> minus = acc;
    minus.add(p.neg());
    masked_select(&acc, acc, minus, 0u - even);
    return acc;
}

}  // namespace

namespace bb {
G1X g1_host_mul(const G1X& p, const uint32_t* k) { return host_mul<Fp>(p, k); }
G2X g2_host_mul(const G2X& p, const uint32_t* k) { return host_mul<Fp2>(p, k); }
}  // namespace bb

extern "C" {

int bb_synth_bases(bb_ctx* ctx, int group, uint64_t seed, size_t n, size_t global_offset, size_t global_len, bb_bases** out);
void bb_crs_destroy(bb_crs* crs);

int bb_crs_create(bb_ctx* ctx, const bb_crs_desc* d, bb_crs** out) {
    if (!ctx || !d || !out) { set_error("bb_crs_create: null argument"); return BB_ERR_ARG; }
    if (!d->alpha_g1 || !d->beta_g1 || !d->delta_g1 || !d->beta_g2 || !d->delta_g2) { set_error("bb_crs_create: missing vk element"); return BB_ERR_ARG; }
    uint32_t cnt = d->shard_count ? d->shard_count : 1, idx = d->shard_index;
    if (idx >= cnt) { set_error("bb_crs_create: shard %u of %u", idx, cnt); return BB_ERR_ARG; }
    bb_crs* crs = new bb_crs();
    crs->ctx = ctx; crs->shard_index = idx; crs->shard_count = cnt;
    std::memcpy(&crs->alpha_g1, d->alpha_g1, 96); std::memcpy(&crs->beta_g1, d->beta_g1, 96);
    std::memcpy(&crs->delta_g1, d->delta_g1, 96);
    std::memcpy(&crs->beta_g2, d->beta_g2, 192); std::memcpy(&crs->delta_g2, d->delta_g2, 192);
    uint32_t sb, snb, sv, snv;
    shard_policy(ctx, idx, cnt, &sb, &snb, &sv, &snv);
    auto up = [&](int group, const void* pts, size_t len, bb_bases** dst) -> int {
        size_t lo = len * sb / snb, hi = len * (sb + 1) / snb;
        size_t stride = group == BB_G1 ? 96 : 192;
        int rc = bb_bases_upload(ctx, group, (const char*)pts + lo * stride, hi - lo, lo, len, dst);
        if (rc == BB_OK) { (*dst)->win_index = sv; (*dst)->win_count = snv; }
        return rc;
    };
    int s;
    if ((s = up(BB_G1, d->h, d->h_len, &crs->h)) || (s = up(BB_G1, d->l, d->l_len, &crs->l)) ||
        (s = up(BB_G1, d->a, d->a_len, &crs->a)) || (s = up(BB_G1, d->b_g1, d->b_g1_len, &crs->b_g1)) ||
        (s = up(BB_G2, d->b_g2, d->b_g2_len, &crs->b_g2))) {
        bb_crs_destroy(crs);
        return s;
    }
    *out = crs;
    return BB_OK;
}

// Synthetic Parameters for the benchmark: every vector is [k_i]G with counter-based pseudorandom
// k_i, generated on the device directly into this rank's base-range shard.  Same vector lengths a
// real key has; not a trapdoor CRS (parity with a valid CRS at this size lives in tests/).
int bb_synth_crs(bb_ctx* ctx, uint64_t seed, size_t h_len, size_t l_len, size_t a_len, size_t b_len,
                 uint32_t shard_index, uint32_t shard_count, bb_crs** out) {
    if (!ctx || !out || !shard_count || shard_index >= shard_count) return BB_ERR_ARG;
    bb_crs* crs = new bb_crs();
    crs->ctx = ctx; crs->shard_index = shard_index; crs->shard_count = shard_count;
    uint64_t k1[3][4], k2[2][4];
    for (int i = 0; i < 3; i++) { k1[i][0] = seed * 7 + i + 11; k1[i][1] = seed + 3 * i; k1[i][2] = 5 + i; k1[i][3] = 1 + i; }
    for (int i = 0; i < 2; i++) { k2[i][0] = seed * 13 + i + 17; k2[i][1] = seed + 5 * i; k2[i][2] = 9 + i; k2[i][3] = 2 + i; }
    G1Affine v1[3]; G2Affine v2[2];
    int s = bb_fixed_base_mul(ctx, BB_G1, k1, 3, BB_FORM_CANONICAL, v1);
    if (s == BB_OK) s = bb_fixed_base_mul(ctx, BB_G2, k2, 2, BB_FORM_CANONICAL, v2);
    crs->alpha_g1 = v1[0]; crs->beta_g1 = v1[1]; crs->delta_g1 = v1[2];
    crs->beta_g2 = v2[0]; crs->delta_g2 = v2[1];
    uint32_t sb, snb, sv, snv;
    shard_policy(ctx, shard_index, shard_count, &sb, &snb, &sv, &snv);
    auto gen = [&](int group, uint64_t sd, size_t len, bb_bases** dst) -> int {
        size_t lo = len * sb / snb, hi = len * (sb + 1) / snb;
        int rc = bb_synth_bases(ctx, group, sd, hi - lo, lo, len, dst);
        if (rc == BB_OK) { (*dst)->win_index = sv; (*dst)->win_count = snv; }
        return rc;
    };
    if (s == BB_OK) s = gen(BB_G1, seed + 1, h_len, &crs->h);
    if (s == BB_OK) s = gen(BB_G1, seed + 2, l_len, &crs->l);
    if (s == BB_OK) s = gen(BB_G1, seed + 3, a_len, &crs->a);
    if (s == BB_OK) s = gen(BB_G1, seed + 4, b_len, &crs->b_g1);
    if (s == BB_OK) s = gen(BB_G2, seed + 4, b_len, &crs->b_g2);       // same dlogs in G1 and G2, like a real B query
    if (s != BB_OK) { bb_crs_destroy(crs); return s; }
    *out = crs;
    return BB_OK;
}

void bb_crs_destroy(bb_crs* crs) {
    if (!crs) return;
    bb_bases_free(crs->h); bb_bases_free(crs->l); bb_bases_free(crs->a); bb_bases_free(crs->b_g1); bb_bases_free(crs->b_g2);
    delete crs;
}

int bb_diag_crs_download(const bb_crs* crs, int which, void* out) {
    if (!crs || !out || which < 0 || which > 5) { set_error("bb_diag_crs_download: bad argument"); return BB_ERR_ARG; }
    if (which == 5) {
        uint8_t* o = (uint8_t*)out;
        std::memcpy(o, &crs->alpha_g1, 96); std::memcpy(o + 96, &crs->beta_g1, 96); std::memcpy(o + 192, &crs->delta_g1, 96);
        std::memcpy(o + 288, &crs->beta_g2, 192); std::memcpy(o + 480, &crs->delta_g2, 192);
        return BB_OK;
    }
    const bb_bases* b = which == 0 ? crs->h : which == 1 ? crs->l : which == 2 ? crs->a : which == 3 ? crs->b_g1 : crs->b_g2;
    const size_t bytes = b->n * (b->group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine));
    BB_CUDA(cudaSetDevice(crs->ctx->device));
    if (bytes) BB_CUDA(cudaMemcpyAsync(out, b->d_points, bytes, cudaMemcpyDeviceToHost, crs->ctx->main_stream));
    BB_CUDA(cudaStreamSynchronize(crs->ctx->main_stream));
    return BB_OK;
}

}  // extern "C"

namespace bb {
bb_crs* crs_adopt(bb_ctx* ctx, bb_bases* const vec[5], const G1Affine g1[3], const G2Affine g2[2]) {
    bb_crs* crs = new bb_crs();
    crs->ctx = ctx;
    crs->h = vec[0]; crs->l = vec[1]; crs->a = vec[2]; crs->b_g1 = vec[3]; crs->b_g2 = vec[4];
    crs->alpha_g1 = g1[0]; crs->beta_g1 = g1[1]; crs->delta_g1 = g1[2];
    crs->beta_g2 = g2[0]; crs->delta_g2 = g2[1];
    return crs;
}
CrsView crs_view(const bb_crs* crs) {
    return CrsView{crs->ctx, crs->shard_count, {crs->h, crs->l, crs->a, crs->b_g1, crs->b_g2}, {crs->alpha_g1, crs->beta_g1, crs->delta_g1},
                   {crs->beta_g2, crs->delta_g2}};
}
}  // namespace bb

namespace {

// x_i / zz_i, y_i / zzz_i for n points with ONE field inversion (Montgomery's trick)
template <class F>
void batch_to_affine(const XYZZ<F>* in, size_t n, Affine<F>* out) {
    std::vector<F> pre(n);
    F acc = FieldOps<F>::one();
    for (size_t i = 0; i < n; i++) { pre[i] = acc; if (!in[i].is_identity()) acc = acc * in[i].ZZZ; }
    F inv = FieldOps<F>::inv(acc);
    for (size_t i = n; i-- > 0;) {
        if (in[i].is_identity()) { out[i] = Affine<F>::identity(); continue; }
        F zi3 = inv * pre[i];
        inv = inv * in[i].ZZZ;
        F zi2 = (zi3 * in[i].ZZ).sqr();
        out[i] = {in[i].X * zi2, in[i].Y * zi3};
    }
}

bool delta_is_identity(const bb_crs* crs) { return crs->delta_g1.is_identity() || crs->delta_g2.is_identity(); }     // prover.rs:320-324

// The message bb_groth16_prove reports with status s for this key (NULL for the back-end statuses, whose text varies)
const char* prove_status_message(const bb_crs* crs, int s) {
    switch (s) {
        case BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE: return "PolynomialDegreeTooLarge";
        case BB_ERR_UNEXPECTED_IDENTITY:
            return delta_is_identity(crs) ? "delta is the identity: subversion-CRS attack" : "encountered an identity element in the CRS";
        case BB_ERR_IO_UNEXPECTED_EOF: return "expected more bases from source";
        case BB_ERR_DENSITY_MISMATCH: return "density map length differs from the number of exponents";
        default: return nullptr;
    }
}

int prove_error(const bb_crs* crs, int s) {
    if (const char* msg = prove_status_message(crs, s)) set_error("%s", msg);
    return s;
}

// The status of one proof from its eight jobs' statuses st[k * stride] when several errors apply: the density assert fires
// inside the multiexp() call itself (multiexp.rs:324-329; calls are made in slot order), the delta check comes before the
// first wait (prover.rs:320-324), and the waits run a_inputs, a_aux, b_g1_inputs, b_g1_aux, b_g2_inputs, b_g2_aux, h, l
// (:339-354).
int proof_status(const int* st, size_t stride, bool bad_delta) {
    static const int ref_wait_order[8] = {2, 3, 4, 5, 6, 7, 0, 1};
    for (int k = 0; k < 8; k++) if (st[k * stride] == BB_ERR_DENSITY_MISMATCH) return BB_ERR_DENSITY_MISMATCH;
    if (bad_delta) return BB_ERR_UNEXPECTED_IDENTITY;
    for (int k : ref_wait_order) if (st[k * stride] != BB_OK) return st[k * stride];
    return BB_OK;
}

size_t density_count(const uint64_t* bits, size_t n) {        // get_total_density, prover.rs:288-291
    if (!bits) return n;
    size_t c = 0;
    for (size_t j = 0; j < (n + 63) / 64; j++) {
        uint64_t wv = bits[j];
        if (j == (n + 63) / 64 - 1 && (n & 63)) wv &= (1ull << (n & 63)) - 1ull;
        c += (size_t)__builtin_popcountll(wv);
    }
    return c;
}

// The eight jobs of a proof in slot order: bases, base offset, density map, scalars, scalars the density selects, and the
// device scalars of item i at src + i * stride Fr.  Slot 0 (h) takes its scalars from the H pipeline.
struct Slot { const bb_bases* bases; size_t off; const uint64_t* dens; size_t n, n_dense; const void* src; size_t stride; };
static const char* const job_tag[8] = {"h", "l", "a_inputs", "a_aux", "b_g1_inputs", "b_g1_aux", "b_g2_inputs", "b_g2_aux"};
// h and the G2 job have the longest dependency chains: each gets one of the high-priority streams
static const int job_critical[8] = {1, 0, 0, 0, 0, 0, 0, 2};

void slot_table(const bb_crs* crs, const bb_witness& w, size_t m, const void* in, const void* aux, Slot out[8]) {
    const size_t ni = w.n_inputs, na = w.n_aux, b_in = density_count(w.b_input_density, ni), b_aux = density_count(w.b_aux_density, na);
    out[0] = {crs->h, 0, nullptr, m - 1, m - 1, nullptr, m};                                      // prover.rs:238-244
    out[1] = {crs->l, 0, nullptr, na, na, aux, na};                                               // :263-268
    out[2] = {crs->a, 0, nullptr, ni, ni, in, ni};                                                // :275-280
    out[3] = {crs->a, ni, w.a_aux_density, na, density_count(w.a_aux_density, na), aux, na};      // :281-286
    out[4] = {crs->b_g1, 0, w.b_input_density, ni, b_in, in, ni};                                 // :296-301
    out[5] = {crs->b_g1, b_in, w.b_aux_density, na, b_aux, aux, na};                              // :302-307
    out[6] = {crs->b_g2, 0, w.b_input_density, ni, b_in, in, ni};                                 // :312-317
    out[7] = {crs->b_g2, b_in, w.b_aux_density, na, b_aux, aux, na};                              // :318
}

}  // namespace

// B proofs of one shape in flight: one proof between prove_begin and prove_end (B = 1, unbatched jobs with host folds), or
// a sub-batch of bb_groth16_prove_batch (batched jobs, one H pipeline for all items).  Every exit -- error paths included --
// first drains every started job and the two streams that touch the buffers below (the DevBufs go back to the cache when
// this object dies), then destroys the events.
struct bb_prove {
    bb_ctx* ctx;
    const bb_crs* crs;
    std::vector<bb_witness> w;
    uint32_t B;
    bool batched;
    size_t m;
    uint32_t log_m;
    DevBuf d_abc, d_tmp, d_in, d_aux;             // d_abc: rows a_0 .. a_{B-1}, b_0 .., c_0 .. of m Fr; item i's h ends in a_i
    bool in_place = false;                        // B = 1, device witness: the MSMs and the evaluation read the caller's arrays
    const Fr *in_p = nullptr, *aux_p = nullptr;   // the witnesses on the device: d_in / d_aux, or the caller's arrays
    int end_evals = 0;                            // bb_groth16_prove_end: 0 = with the three vectors or without, 1 = with, -1 = without
    std::unique_ptr<StageTimer> tm;               // profile mode: the r1cs.* or r1cs_owner.* stages of a proof from the witness
    uint64_t r1cs_terms = 0;                      // the units of the r1cs.* stages
    cudaStream_t up = nullptr;
    cudaEvent_t ev_up = nullptr, ev_h = nullptr;
    Slot slot[8];
    bb_msm_job* jobs[8] = {};
    int s = BB_OK;                                // a failure to queue, reported at the end
    bool h_queued = false;
    std::vector<int> status;                      // after prove_wait: item i's status in job k at [k * B + i] ...
    std::vector<G1X> sums1;                       // ... and its point at [k * B + i] (k < 6) or [(k - 6) * B + i]
    std::vector<G2X> sums2;
    bb_prove(bb_ctx* c, const bb_crs* k, const bb_witness* items, uint32_t b, bool bat, size_t m_, uint32_t lm)
        : ctx(c), crs(k), w(items, items + b), B(b), batched(bat), m(m_), log_m(lm) {}
    ~bb_prove() {
        std::vector<int> st(B);
        std::vector<G2X> pts(B);
        for (auto& j : jobs) if (j) { msm_wait(j, st.data(), pts.data()); j = nullptr; }
        if (ctx) cudaStreamSynchronize(ctx->main_stream);
        if (up) cudaStreamSynchronize(up);
        if (ev_up) cudaEventDestroy(ev_up);
        if (ev_h) cudaEventDestroy(ev_h);
    }
};

namespace {

// profile mode: the origin of the jobs' device timeline (bb_profile_read "tl.<job>.<mark>")
int profile_epoch(bb_ctx* ctx) {
    if (!ctx->opt_profile) return BB_OK;
    if (!ctx->epoch_ev) BB_CUDA(cudaEventCreate(&ctx->epoch_ev));
    BB_CUDA(cudaEventRecord(ctx->epoch_ev, ctx->main_stream));
    return BB_OK;
}

void prove_start(bb_prove* P, int k) {
    const Slot& j = P->slot[k];
    if (P->s == BB_OK)
        P->s = msm_start(P->ctx, j.bases, j.off, j.dens, j.n, j.src, true, j.n, BB_FORM_MONTGOMERY, k == 0 ? P->ev_h : P->ev_up, &P->jobs[k],
                         job_tag[k], job_critical[k], P->batched ? P->B : 0, j.stride);
}

// The H pipeline (prover.rs:221-240) of the B items on the high-priority main stream: a, b, c from the witnesses or from
// `fill`, zero padded to m.  With `evals` (device buffers of m coset evaluations of a, b, c of one proof -- computed
// elsewhere, bb_h_coset_evals) only the last transform remains: mul_assign, sub_assign, divide_by_z_on_coset, icoset_fft
// (:232-237).
int h_pipeline(bb_prove* P, const void* const* evals, const BatchAbcFill* fill) {
    bb_ctx* ctx = P->ctx;
    cudaStream_t st = ctx->main_stream;
    const bb_witness& w0 = P->w[0];
    const size_t n = w0.n_constraints, m = P->m, B = P->B;
    if (!P->d_tmp.p) BB_TRY(P->d_tmp.alloc(ctx, (P->batched ? 3 * B : 1) * m * 32));     // (an owner stage may have made it)
    if (evals) return h_poly_final_device(ctx, st, (Fr*)evals[0], (const Fr*)evals[1], (const Fr*)evals[2], P->d_tmp.as<Fr>(), P->log_m);
    BB_TRY(P->d_abc.alloc(ctx, 3 * B * m * 32));
    Fr* abc = P->d_abc.as<Fr>();
    if (fill) {                                          // a, b, c evaluated on the device from the uploaded witnesses
        if (!P->batched) {                               // bb_groth16_prove_r1cs's stages (bb_profile_read)
            P->tm.reset(new StageTimer(ctx, st));
            P->tm->mark("r1cs.begin");
        }
        BB_CUDA(cudaStreamWaitEvent(st, P->ev_up, 0));
        if (P->tm) P->tm->mark("r1cs.upload", P->r1cs_terms);
        BB_TRY((*fill)(st, (uint32_t)B, abc, m, P->in_p, P->aux_p));
        if (P->tm) P->tm->mark("r1cs.eval", P->r1cs_terms);
    } else {
        for (size_t i = 0; i < B; i++) {
            const void* srcs[3] = {P->w[i].a, P->w[i].b, P->w[i].c};
            for (size_t k = 0; k < 3 && n; k++)
                BB_CUDA(cudaMemcpyAsync(abc + (k * B + i) * m, srcs[k], n * 32, w0.on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
        }
        if (!w0.on_device) ctx->h2d_bytes += B * 3 * n * 32;
    }
    if (m > n) BB_CUDA(cudaMemset2DAsync(abc + n, m * 32, 0, (m - n) * 32, 3 * B, st));   // coeffs.resize(m, zero), domain.rs:69
    if (P->batched) return h_poly_batch_device(ctx, st, abc, P->d_tmp.as<Fr>(), P->log_m, (uint32_t)B);
    return h_poly_device(ctx, st, abc, abc + m, abc + 2 * m, P->d_tmp.as<Fr>(), P->log_m);
}

// The H pipeline and the h MSM behind it
int prove_queue_h(bb_prove* P, const void* const* evals, const BatchAbcFill* fill) {
    NvtxRange range(evals ? "bb: H pipeline (last transform) + h MSM" : "bb: H pipeline + h MSM");
    int s = h_pipeline(P, evals, fill);
    if (s == BB_OK && cudaEventRecord(P->ev_h, P->ctx->main_stream) != cudaSuccess) { set_error("cudaEventRecord(H pipeline done) failed"); s = BB_ERR_CUDA; }
    if (s != BB_OK) { P->s = s; return s; }
    P->slot[0].src = evals ? evals[0] : P->d_abc.p;
    prove_start(P, 0);
    P->h_queued = true;
    return P->s;
}

// Queues the uploads and the MSMs of the B proofs (prover.rs:221-318).  h_inline: the H pipeline and the h MSM are queued
// here, FIRST -- they are the longest dependency chain of a proof and run on high-priority streams, the seven witness MSMs
// fill the machine around them.  Otherwise prove_end queues them (multi-GPU: the coset evaluations arrive from other ranks
// while the witness MSMs already run); `head`, if any, is queued on the main stream behind the upload and ahead of the
// witness MSMs (the owner stage of bb_groth16_prove_r1cs_begin; a failure to queue it fails the call).  A failure to queue a
// job is kept in P->s.
int prove_queue(bb_prove* P, bool h_inline, const BatchAbcFill* fill, const ProveHead* head = nullptr) {
    bb_ctx* ctx = P->ctx;
    const bb_witness& w0 = P->w[0];
    const size_t ni = w0.n_inputs, na = w0.n_aux, B = P->B;
    P->up = ctx->pick_stream();
    BB_CUDA(cudaEventCreateWithFlags(&P->ev_up, cudaEventDisableTiming));
    BB_CUDA(cudaEventCreateWithFlags(&P->ev_h, cudaEventDisableTiming));
    if (P->in_place) {
        P->in_p = (const Fr*)w0.input_assignment;
        P->aux_p = (const Fr*)(na ? w0.aux_assignment : w0.input_assignment);      // no aux: never read
    } else {
        BB_TRY(P->d_in.alloc(ctx, B * ni * 32)); BB_TRY(P->d_aux.alloc(ctx, B * na * 32));
        const cudaMemcpyKind kind = w0.on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        for (size_t i = 0; i < B; i++) {
            if (ni) BB_CUDA(cudaMemcpyAsync((char*)P->d_in.p + i * ni * 32, P->w[i].input_assignment, ni * 32, kind, P->up));
            if (na) BB_CUDA(cudaMemcpyAsync((char*)P->d_aux.p + i * na * 32, P->w[i].aux_assignment, na * 32, kind, P->up));
        }
        if (!w0.on_device) ctx->h2d_bytes += B * (ni + na) * 32;
        P->in_p = P->d_in.as<Fr>();
        P->aux_p = P->d_aux.as<Fr>();
    }
    BB_CUDA(cudaEventRecord(P->ev_up, P->up));
    slot_table(P->crs, w0, P->m, P->in_p, P->aux_p, P->slot);
    if (head) {
        cudaStream_t st = ctx->main_stream;
        P->tm.reset(new StageTimer(ctx, st));
        P->tm->mark("r1cs_owner.begin");
        BB_CUDA(cudaStreamWaitEvent(st, P->ev_up, 0));
        P->tm->mark("r1cs_owner.upload", 0);
        BB_TRY(P->d_tmp.alloc(ctx, P->m * 32));
        BB_TRY((*head)(st, P->in_p, P->aux_p, P->d_tmp.as<Fr>(), *P->tm));
    }
    if (h_inline) prove_queue_h(P, nullptr, fill);
    // all eight MSMs are in flight before the first wait (prover.rs:244-318); the G2 MSM has the longest chain of the seven
    // (Fp2 arithmetic): it goes first, on the other high-priority stream
    for (int k : {7, 1, 2, 3, 4, 5, 6}) prove_start(P, k);
    return BB_OK;
}

// wait() x8 (prover.rs:339-354); always drains every started job.  The eight waits run on eight short-lived host threads:
// jobs tend to finish together, and an unbatched job's wait ends with a host-side Horner fold of its window sums (255
// doublings: 0.2 ms for G1, 0.5 ms for G2 on one core), so the folds overlap.  job_status[k]: job k's own status.
void prove_wait(bb_prove* P, int job_status[8]) {
    const size_t B = P->B;
    P->status.assign(8 * B, BB_OK);
    P->sums1.assign(6 * B, G1X::identity());
    P->sums2.assign(2 * B, G2X::identity());
    std::thread waiters[8];
    for (int k = 0; k < 8; k++) {
        job_status[k] = BB_OK;
        bb_msm_job* job = P->jobs[k];
        P->jobs[k] = nullptr;
        if (!job) continue;
        void* pts = k < 6 ? (void*)&P->sums1[k * B] : (void*)&P->sums2[(k - 6) * B];
        waiters[k] = std::thread([=] {
            cudaSetDevice(P->ctx->device);
            job_status[k] = msm_wait(job, &P->status[k * B], pts);
        });
    }
    for (auto& t : waiters) if (t.joinable()) t.join();
}

// The 960-byte partial sums of the listed items, to affine with one inversion for all their G1 points and one for all
// their G2 points
void write_partials(const bb_prove* P, const std::vector<uint32_t>& items, uint8_t* out) {
    const size_t nk = items.size(), B = P->B;
    std::vector<G1X> p1(6 * nk);
    std::vector<G2X> p2(2 * nk);
    for (size_t q = 0; q < nk; q++) {
        for (size_t k = 0; k < 6; k++) p1[6 * q + k] = P->sums1[k * B + items[q]];
        for (size_t k = 0; k < 2; k++) p2[2 * q + k] = P->sums2[k * B + items[q]];
    }
    std::vector<G1Affine> a1(6 * nk);
    std::vector<G2Affine> a2(2 * nk);
    batch_to_affine<Fp>(p1.data(), p1.size(), a1.data());
    batch_to_affine<Fp2>(p2.data(), p2.size(), a2.data());
    for (size_t q = 0; q < nk; q++) {
        std::memcpy(out + q * BB_PARTIALS_BYTES, &a1[6 * q], 6 * 96);
        std::memcpy(out + q * BB_PARTIALS_BYTES + 576, &a2[2 * q], 2 * 192);
    }
}

// r1cs: a proof from a resident constraint system (bb_groth16_prove_r1cs_begin), NULL for bb_groth16_prove_begin's
int prove_begin_impl(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, bool h_inline, bb_prove** out, const R1csStart* r1cs = nullptr) {
    NvtxRange range("bb: prove_begin (uploads, queue MSMs)");
    if (!ctx || !crs || !w || !out) { set_error("bb_groth16_prove: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t m;
    uint32_t log_m;
    BB_TRY(domain_size(w->n_constraints, &m, &log_m));
    BB_TRY(profile_epoch(ctx));
    std::unique_ptr<bb_prove> P(new bb_prove(ctx, crs, w, 1, false, m, log_m));
    if (r1cs) {
        P->in_place = w->on_device != 0;
        P->end_evals = r1cs->split ? 1 : -1;
        P->r1cs_terms = r1cs->units;
        BB_TRY(prove_queue(P.get(), !r1cs->split, r1cs->split ? nullptr : &r1cs->fill, r1cs->head ? &r1cs->head : nullptr));
    } else {
        BB_TRY(prove_queue(P.get(), h_inline, nullptr));
    }
    *out = P.release();
    return BB_OK;
}

// Queues the H pipeline if prove_begin did not, waits for the eight MSMs and writes the 960-byte partial sums.  Frees the
// state.
int prove_end_impl(bb_prove* Praw, const void* const* evals, uint8_t* partials) {
    NvtxRange range("bb: prove_end (waits, folds)");
    std::unique_ptr<bb_prove> P(Praw);
    if (!Praw || !partials) { set_error("bb_groth16_prove_end: null argument"); return BB_ERR_ARG; }
    if ((P->end_evals > 0 && !evals) || (P->end_evals < 0 && evals)) {
        set_error("bb_groth16_prove_end: %s", evals ? "this proof ran its whole H pipeline in bb_groth16_prove_r1cs_begin: no evaluation vectors"
                                                    : "this proof's H pipeline was split by polynomial: the three evaluation vectors are needed");
        return BB_ERR_ARG;
    }
    BB_CUDA(cudaSetDevice(P->ctx->device));
    if (!P->h_queued && P->s == BB_OK) prove_queue_h(P.get(), evals, nullptr);
    int job_status[8];
    prove_wait(P.get(), job_status);
    if (P->tm && P->ctx->opt_profile && cudaStreamSynchronize(P->ctx->main_stream) == cudaSuccess) P->tm->report(0);
    if (P->s != BB_OK) return P->s;
    const int s = proof_status(P->status.data(), 1, delta_is_identity(P->crs));
    if (s != BB_OK) return prove_error(P->crs, s);
    write_partials(P.get(), {0}, partials);
    return BB_OK;
}

int prove_partials_impl(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, uint8_t* partials) {
    if (!partials) { set_error("bb_groth16_prove_partials: null argument"); return BB_ERR_ARG; }
    bb_prove* P = nullptr;
    BB_TRY(prove_begin_impl(ctx, crs, w, true, &P));
    return prove_end_impl(P, nullptr, partials);
}

// The terms of A, B, C that depend only on the key and on (r, s) -- prover.rs:326-337:
//   g_a = delta_g1 r + alpha_g1,  g_b = delta_g2 s + beta_g2,  g_c = delta_g1 rs + alpha_g1 s + beta_g1 r
struct ProofStatic { G1X g_a, g_c; G2X g_b; };

void finalize_static(const bb_crs* crs, const Fr& r, const Fr& s, ProofStatic* out) {
    Fr rs = fr_to_canonical(fr_from_canonical(r) * fr_from_canonical(s));        // rs.mul_assign(&s), :332-333
    out->g_a = g1_host_mul(G1X::from_affine(crs->delta_g1), r.l);                 // :326-327
    out->g_a.add_mixed(crs->alpha_g1);
    out->g_b = g2_host_mul(G2X::from_affine(crs->delta_g2), s.l);                 // :328-329
    out->g_b.add_mixed(crs->beta_g2);
    out->g_c = g1_host_mul(G1X::from_affine(crs->delta_g1), rs.l);                // :335-337
    out->g_c.add(g1_host_mul(G1X::from_affine(crs->alpha_g1), s.l));
    out->g_c.add(g1_host_mul(G1X::from_affine(crs->beta_g1), r.l));
}

int finalize_impl(const bb_crs* crs, const uint8_t* partials, size_t count, const Fr& r, const Fr& s, const ProofStatic& stat, uint8_t* proof) {
    G1X sum1[6];
    G2X sum2[2];
    for (auto& p : sum1) p = G1X::identity();
    for (auto& p : sum2) p = G2X::identity();
    for (size_t c = 0; c < count; c++) {
        const uint8_t* base = partials + c * BB_PARTIALS_BYTES;
        for (int k = 0; k < 6; k++) { G1Affine a; std::memcpy(&a, base + 96 * k, 96); sum1[k].add_mixed(a); }
        for (int k = 0; k < 2; k++) { G2Affine a; std::memcpy(&a, base + 576 + 192 * k, 192); sum2[k].add_mixed(a); }
    }
    G1X g_a = stat.g_a, g_c = stat.g_c;
    G2X g_b = stat.g_b;
    G1X a_answer = sum1[2];                                                       // :339-343
    a_answer.add(sum1[3]);
    g_a.add(a_answer);
    G1X b1_answer = sum1[4];                                                      // :345-354
    b1_answer.add(sum1[5]);
    // the two scalar multiplications that need MSM results sit between the last device result and the proof
    // bytes: they run side by side (0.2 ms each on one core)
    G1X a_s;
    std::thread side([&] { a_s = g1_host_mul(a_answer, s.l); });
    const G1X b_r = g1_host_mul(b1_answer, r.l);
    G2X b2_answer = sum2[0];
    b2_answer.add(sum2[1]);
    g_b.add(b2_answer);
    side.join();
    g_c.add(a_s);
    g_c.add(b_r);
    g_c.add(sum1[0]);
    g_c.add(sum1[1]);
    G1X ac[2] = {g_a, g_c};                                                       // :356-360: to_affine, one inversion for A and C
    G1Affine ac_aff[2];
    batch_to_affine<Fp>(ac, 2, ac_aff);
    encode_compressed(ac_aff[0], proof);                                          // lib.rs:39-45
    encode_compressed(g_b.to_affine(), proof + 48);
    encode_compressed(ac_aff[1], proof + 144);
    return BB_OK;
}


// ---- many witnesses of one circuit against one key (bb_groth16_prove_batch) --------------------------------------------
// A sub-batch of B items is one H pipeline for all items on the main stream and EIGHT MSM jobs, each over the B scalar
// vectors of its slot (msm_start with batch = B): the launches per sub-batch are those of one proof plus B - 1 H pipelines,
// and the window folds run on the device.  The host work -- the scalar multiplications by r, s, rs -- is the single-proof
// code, run for the items side by side.

// fn(i) for i < n on a pool of host threads, one per CPU this process may run on
void parallel_for(size_t n, const std::function<void(size_t)>& fn) {
    if (!n) return;
    size_t cpus = 1;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) cpus = (size_t)CPU_COUNT(&set);
    const size_t k = std::max<size_t>(1, std::min(cpus, n));
    std::atomic<size_t> next{0};
    auto body = [&] { for (size_t i; (i = next.fetch_add(1)) < n;) fn(i); };
    std::vector<std::thread> pool;
    for (size_t j = 1; j < k; j++) pool.emplace_back(body);
    body();
    for (auto& th : pool) th.join();
}

bool same_density(const uint64_t* a, const uint64_t* b, size_t bits) {
    if (!a || !b) return a == b;
    return std::memcmp(a, b, (bits + 63) / 64 * 8) == 0;
}

// Proofs per sub-batch: prove_batch_max if set, and at most what one job's 2^32 bucket entries, its result staging block
// and the device memory (free plus the context's cached blocks, against an estimate per proof) hold
size_t batch_limit(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, size_t m, size_t count) {
    Slot js[8];
    slot_table(crs, *w, m, nullptr, nullptr, js);
    size_t k = count;
    if (ctx->opt_prove_batch_max > 0) k = std::min(k, (size_t)ctx->opt_prove_batch_max);
    k = std::min(k, (bb_ctx::PINNED_BLOCK - 32) / (sizeof(G2X) + 4));
    size_t free_b = 0, total_b = 0;
#if defined(__CUDACC__)
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); free_b = 0; }
#else
    free_b = (size_t)1 << 40;                          // the sources compiled for host threads (tests/native): no device to ask
#endif
    {
        std::lock_guard<std::mutex> g(ctx->mu);
        for (auto& kv : ctx->free_blocks) free_b += kv.first;
    }
    const double budget = 0.85 * (double)free_b;
    auto fits = [&](size_t b) {
        double bytes = (double)b * (6 * m + w->n_inputs + w->n_aux) * 32.0;        // a, b, c and their scratch; the witnesses
        for (auto& j : js) {
            if (!j.bases) continue;
            uint64_t slots = 0;
            bytes += (double)msm_batch_bytes(ctx, j.bases, j.n, j.n_dense, (uint32_t)b, &slots);
            if (slots >= (1ull << 32)) return false;
        }
        return bytes <= budget;
    };
    while (k > 1 && !fits(k)) k -= std::max<size_t>(1, k / 8);
    return std::max<size_t>(1, k);
}

// Items 0 .. B - 1 of w: queue, wait, finalise.  Returns a failure of the sub-batch as a whole (it then stands for every
// item); otherwise status[] holds each item's bb_groth16_prove status.
int prove_sub_batch(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, uint32_t B, size_t m, uint32_t log_m, const uint8_t* r_bytes,
                    const uint8_t* s_bytes, uint8_t* proofs, int* status, double* host_tail_ms, const BatchAbcFill* fill) {
    bb_prove P(ctx, crs, w, B, true, m, log_m);
    BB_TRY(prove_queue(&P, true, fill));
    if (P.s != BB_OK) return P.s;
    // while the device works: the MSM-independent terms of every item
    std::vector<ProofStatic> stat(B);
    std::vector<Fr> rr(B), ss(B);
    for (uint32_t i = 0; i < B; i++) { std::memcpy(rr[i].l, r_bytes + 32 * i, 32); std::memcpy(ss[i].l, s_bytes + 32 * i, 32); }
    const bool bad_delta = delta_is_identity(crs);
    if (!bad_delta) parallel_for(B, [&](size_t i) { finalize_static(crs, rr[i], ss[i], &stat[i]); });
    int job_status[8];
    prove_wait(&P, job_status);
    const auto t_waited = std::chrono::steady_clock::now();
    // the density assert is a per-item status; anything else a job failed with is the sub-batch's
    for (int k = 0; k < 8; k++) if (job_status[k] != BB_OK && job_status[k] != BB_ERR_DENSITY_MISMATCH) return job_status[k];
    std::vector<uint32_t> ok;
    for (uint32_t i = 0; i < B; i++) {
        status[i] = proof_status(&P.status[i], B, bad_delta);
        if (status[i] == BB_OK) ok.push_back(i);
    }
    std::vector<uint8_t> partials(ok.size() * BB_PARTIALS_BYTES);
    write_partials(&P, ok, partials.data());
    parallel_for(ok.size(), [&](size_t q) {
        const uint32_t i = ok[q];
        finalize_impl(crs, &partials[q * BB_PARTIALS_BYTES], 1, rr[i], ss[i], stat[i], proofs + (size_t)i * BB_PROOF_BYTES);
    });
    *host_tail_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_waited).count();
    return BB_OK;
}

}  // namespace

namespace bb {

int prove_batch_check(const char* fn, const bb_ctx* ctx, const bb_crs* crs, size_t count, const void* r, const void* s, const void* proofs,
                      const int* status) {
    if (!ctx || !crs || crs->ctx != ctx) { set_error("%s: null argument or a key of another context", fn); return BB_ERR_ARG; }
    if (crs->shard_count != 1) { set_error("%s needs an unsharded CRS", fn); return BB_ERR_ARG; }
    if (count && (!r || !s || !proofs || !status)) { set_error("%s: null argument", fn); return BB_ERR_ARG; }
    return BB_OK;
}

int prove_batch_impl(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, size_t count, const uint8_t* r, const uint8_t* s,
                     uint8_t* proofs, int* status, const BatchAbcFill* fill) {
    BB_TRY(prove_batch_check("bb_groth16_prove_batch", ctx, crs, count, r, s, proofs, status));
    if (!count) return BB_OK;
    if (!w) { set_error("bb_groth16_prove_batch: null argument"); return BB_ERR_ARG; }
    const bb_witness& w0 = w[0];
    for (size_t i = 0; i < count; i++) {
        const bb_witness& wi = w[i];
        if (wi.n_constraints != w0.n_constraints || wi.n_inputs != w0.n_inputs || wi.n_aux != w0.n_aux || (wi.on_device != 0) != (w0.on_device != 0) ||
            !same_density(wi.a_aux_density, w0.a_aux_density, w0.n_aux) || !same_density(wi.b_input_density, w0.b_input_density, w0.n_inputs) ||
            !same_density(wi.b_aux_density, w0.b_aux_density, w0.n_aux)) {
            set_error("bb_groth16_prove_batch: item %zu differs from item 0 in its shape or its densities", i);
            return BB_ERR_ARG;
        }
        if ((wi.n_constraints && !fill && (!wi.a || !wi.b || !wi.c)) || (wi.n_inputs && !wi.input_assignment) || (wi.n_aux && !wi.aux_assignment) ||
            (wi.n_inputs && !wi.b_input_density) || (wi.n_aux && (!wi.a_aux_density || !wi.b_aux_density))) {
            set_error("bb_groth16_prove_batch: item %zu has a null array", i);
            return BB_ERR_ARG;
        }
    }
    std::memset(proofs, 0, count * BB_PROOF_BYTES);
    size_t m;
    uint32_t log_m;
    if (domain_size(w0.n_constraints, &m, &log_m) != BB_OK) {     // every item alike
        for (size_t i = 0; i < count; i++) status[i] = BB_ERR_POLYNOMIAL_DEGREE_TOO_LARGE;
        return BB_OK;
    }
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange range("bb: prove_batch");
    BB_TRY(profile_epoch(ctx));
    const size_t k = batch_limit(ctx, crs, &w0, m, count);
    double tail = 0;
    size_t subs = 0;
    for (size_t lo = 0; lo < count; lo += k, subs++) {
        const uint32_t B = (uint32_t)std::min(k, count - lo);
        const int rc = prove_sub_batch(ctx, crs, w + lo, B, m, log_m, r + 32 * lo, s + 32 * lo, proofs + lo * BB_PROOF_BYTES, status + lo, &tail, fill);
        for (uint32_t i = 0; i < B; i++) {
            if (rc != BB_OK) status[lo + i] = rc;          // a failure of the sub-batch as a whole: none of its items has a proof
            if (status[lo + i] != BB_OK) std::memset(proofs + (lo + i) * BB_PROOF_BYTES, 0, BB_PROOF_BYTES);
        }
    }
    if (ctx->opt_profile) {
        ctx->prof_add("prove_batch.host_tail", tail, subs, count);      // host ms from the last MSM result to the proof bytes
        ctx->prof_add("prove_batch.sub_batches", 0, subs, count);
    }
    return BB_OK;
}
}  // namespace bb

extern "C" {

int bb_groth16_prove_partials(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, uint8_t* partials) {
    return prove_partials_impl(ctx, crs, w, partials);
}

int bb_groth16_prove_begin(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, bb_prove** out) {
    return prove_begin_impl(ctx, crs, w, false, out);
}

int bb_groth16_prove_end(bb_prove* state, const void* d_evals_a, const void* d_evals_b, const void* d_evals_c, uint8_t* partials) {
    const bool any = d_evals_a || d_evals_b || d_evals_c;
    if (any && !(d_evals_a && d_evals_b && d_evals_c)) { delete state; set_error("bb_groth16_prove_end: all three evaluation vectors or none"); return BB_ERR_ARG; }
    const void* ev[3] = {d_evals_a, d_evals_b, d_evals_c};
    return prove_end_impl(state, any ? ev : nullptr, partials);
}

// from_coeffs (zero padding to m), ifft and coset_fft of ONE of the polynomials a, b, c (prover.rs:225-230) into a
// device buffer of m Fr.  _async queues the copy and the two transforms on the high-priority stream and returns;
// _wait blocks until every queued evaluation is there (and hands the scratch buffers back).
int bb_h_coset_evals_async(bb_ctx* ctx, const void* poly, size_t n_constraints, int on_device, void* d_out) {
    if (!ctx || !d_out || (n_constraints && !poly)) { set_error("bb_h_coset_evals: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t m;
    uint32_t log_m;
    BB_TRY(domain_size(n_constraints, &m, &log_m));
    cudaStream_t st = ctx->main_stream;
    void* d_tmp = nullptr;
    BB_TRY(ctx->alloc(m * 32, &d_tmp));
    {
        std::lock_guard<std::mutex> g(ctx->mu);
        ctx->h_evals_scratch.push_back(d_tmp);            // released by bb_h_coset_evals_wait, after the stream has drained
    }
    if (m > n_constraints) BB_CUDA(cudaMemsetAsync((char*)d_out + n_constraints * 32, 0, (m - n_constraints) * 32, st));
    if (n_constraints) BB_CUDA(cudaMemcpyAsync(d_out, poly, n_constraints * 32, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    if (!on_device) ctx->h2d_bytes += n_constraints * 32;
    return h_poly_evals_device(ctx, st, (Fr*)d_out, (Fr*)d_tmp, log_m);
}

int bb_h_coset_evals_wait(bb_ctx* ctx) {
    if (!ctx) { set_error("bb_h_coset_evals_wait: null argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    cudaError_t e = cudaStreamSynchronize(ctx->main_stream);
    std::vector<void*> scratch;
    {
        std::lock_guard<std::mutex> g(ctx->mu);
        scratch.swap(ctx->h_evals_scratch);
    }
    for (void* p : scratch) ctx->release(p);
    if (e != cudaSuccess) { set_error("bb_h_coset_evals: %s", cudaGetErrorString(e)); return BB_ERR_CUDA; }
    return BB_OK;
}

int bb_h_coset_evals(bb_ctx* ctx, const void* poly, size_t n_constraints, int on_device, void* d_out) {
    std::unique_ptr<StageTimer> tm;                       // profile mode: the stage h_coset_evals (copy, padding, transforms)
    if (ctx && ctx->opt_profile && cudaSetDevice(ctx->device) == cudaSuccess) {
        tm.reset(new StageTimer(ctx, ctx->main_stream));
        tm->mark("h_coset_evals.begin");
    }
    int s = bb_h_coset_evals_async(ctx, poly, n_constraints, on_device, d_out);
    if (tm) tm->mark("h_coset_evals");
    int w = ctx ? bb_h_coset_evals_wait(ctx) : BB_OK;
    if (tm && s == BB_OK && w == BB_OK) tm->report(n_constraints);
    return s != BB_OK ? s : w;
}

int bb_groth16_finalize(const bb_crs* crs, const uint8_t* partials, size_t count, const uint8_t* r_bytes, const uint8_t* s_bytes,
                        uint8_t* proof) {
    if (!crs || !partials || !count || !r_bytes || !s_bytes || !proof) { set_error("bb_groth16_finalize: null argument"); return BB_ERR_ARG; }
    if (delta_is_identity(crs)) return prove_error(crs, BB_ERR_UNEXPECTED_IDENTITY);
    Fr r, s;
    std::memcpy(r.l, r_bytes, 32);
    std::memcpy(s.l, s_bytes, 32);
    ProofStatic stat;
    finalize_static(crs, r, s, &stat);
    return finalize_impl(crs, partials, count, r, s, stat, proof);
}

static_assert(sizeof(ProofStatic) == BB_PROOF_STATIC_BYTES, "ProofStatic layout");

int bb_groth16_finalize_static(const bb_crs* crs, const uint8_t* r_bytes, const uint8_t* s_bytes, uint8_t* static_out) {
    if (!crs || !r_bytes || !s_bytes || !static_out) { set_error("bb_groth16_finalize_static: null argument"); return BB_ERR_ARG; }
    Fr r, s;
    std::memcpy(r.l, r_bytes, 32);
    std::memcpy(s.l, s_bytes, 32);
    ProofStatic stat;
    finalize_static(crs, r, s, &stat);
    std::memcpy(static_out, &stat, sizeof stat);
    return BB_OK;
}

int bb_groth16_finalize_with(const bb_crs* crs, const uint8_t* partials, size_t count, const uint8_t* r_bytes, const uint8_t* s_bytes,
                             const uint8_t* static_in, uint8_t* proof) {
    if (!crs || !partials || !count || !r_bytes || !s_bytes || !static_in || !proof) { set_error("bb_groth16_finalize_with: null argument"); return BB_ERR_ARG; }
    if (delta_is_identity(crs)) return prove_error(crs, BB_ERR_UNEXPECTED_IDENTITY);
    Fr r, s;
    std::memcpy(r.l, r_bytes, 32);
    std::memcpy(s.l, s_bytes, 32);
    ProofStatic stat;
    std::memcpy(&stat, static_in, sizeof stat);
    return finalize_impl(crs, partials, count, r, s, stat, proof);
}

// ---- tuning: measure, don't guess ---------------------------------------------------------------------
// The MSM has forms whose ranking depends on the machine, the key size and the number of shards (resident
// window multiples trade 16x the base storage and colder gathers for fewer buckets and deeper halving rounds).
// A key lives for many proofs, so the choice is made once per key by timing real proofs of each form on this
// device (the way FFT and convolution libraries plan), and a form is only eligible if its partial sums are
// byte-identical to the default form's.
namespace {
struct Tuning { const char* name; long precompute; long rows_log; long groups; };   // groups: 1 = G1 vectors, 2 = G2 vectors
const Tuning kTunings[] = {
    {"per-window bucket sets, no tables", 0, 3, 3},
    {"one bucket set over resident window multiples, halving rounds down to ~8 rows per bucket", 2, 3, 3},
    {"one bucket set over resident window multiples, halving rounds down to ~16 rows per bucket", 2, 4, 3},
    {"one bucket set over resident window multiples, halving rounds down to ~4 rows per bucket", 2, 2, 3},
    {"one bucket set over resident window multiples, halving rounds down to ~32 rows per bucket", 2, 5, 3},
    {"one bucket set over resident window multiples for the G2 vector only (~8 rows), per-window bucket sets for G1", 2, 3, 2},
    {"one bucket set over resident window multiples for the G1 vectors only (~8 rows), per-window bucket sets for G2", 2, 3, 1},
};
constexpr int kNumTunings = (int)(sizeof kTunings / sizeof kTunings[0]);
}  // namespace

int bb_tuning_count(void) { return kNumTunings; }
const char* bb_tuning_name(int index) { return index >= 0 && index < kNumTunings ? kTunings[index].name : nullptr; }

namespace {
// tables for the vectors of the groups in `groups` (bit 0 = G1, bit 1 = G2); the other vectors lose theirs
int crs_tables(bb_ctx* ctx, bb_crs* crs, long groups) {
    for (bb_bases* b : {crs->h, crs->l, crs->a, crs->b_g1, crs->b_g2}) {
        if (!b) continue;
        if (groups & (b->group == BB_G1 ? 1 : 2)) BB_TRY(bases_build_table(ctx, b));
        else bb_bases_drop_table(b);
    }
    return BB_OK;
}
}  // namespace

int bb_crs_precompute(bb_ctx* ctx, bb_crs* crs) {
    if (!ctx || !crs || crs->ctx != ctx) { set_error("bb_crs_precompute: bad argument"); return BB_ERR_ARG; }
    return crs_tables(ctx, crs, 3);
}
int bb_crs_drop_tables(bb_crs* crs) {
    if (!crs) { set_error("bb_crs_drop_tables: null argument"); return BB_ERR_ARG; }
    for (bb_bases* b : {crs->h, crs->l, crs->a, crs->b_g1, crs->b_g2})
        if (b) bb_bases_drop_table(b);
    return BB_OK;
}

int bb_crs_apply_tuning(bb_ctx* ctx, bb_crs* crs, int index) {
    if (!ctx || !crs || crs->ctx != ctx || index < 0 || index >= kNumTunings) { set_error("bb_crs_apply_tuning: bad argument"); return BB_ERR_ARG; }
    BB_CUDA(cudaSetDevice(ctx->device));
    BB_CUDA(cudaDeviceSynchronize());                  // nothing may still read a table that is about to go
    const Tuning& t = kTunings[index];
    int s = BB_OK;
    if (t.precompute) s = crs_tables(ctx, crs, t.groups);
    if (s != BB_OK || !t.precompute) bb_crs_drop_tables(crs);
    ctx->opt_msm_precompute = s == BB_OK ? t.precompute : 0;
    ctx->opt_msm_precompute_groups = s == BB_OK ? t.groups : 3;
    ctx->opt_msm_unified_rows_log = s == BB_OK ? t.rows_log : 3;
    return s;
}

int bb_groth16_autotune(bb_ctx* ctx, bb_crs* crs, const bb_witness* w, int reps, int* chosen, double* ms_out) {
    if (!ctx || !crs || crs->ctx != ctx || !w) { set_error("bb_groth16_autotune: bad argument"); return BB_ERR_ARG; }
    if (reps < 1) reps = 3;
    uint8_t ref[BB_PARTIALS_BYTES], got[BB_PARTIALS_BYTES];
    double ms[kNumTunings];
    int best = 0;
    // A shard of a window-sharded key owns the windows w = index mod count of its base range, and the window size differs
    // between the forms (the table forms take it from the vector, the default from the job): the (base, window) pairs a
    // shard sums -- and with them its partial sums -- are comparable only after all shards are added up.  For a sharded
    // key this call therefore only MEASURES (every form must still prove without an error) and leaves the default form
    // configured: all shards must run the same form, which is a collective decision (distributed.autotune_sharded).
    const bool whole_key = crs->shard_count == 1;
    for (int i = 0; i < kNumTunings; i++) {
        ms[i] = -1.0;                                   // -1: not available here (the tables do not fit)
        int s = bb_crs_apply_tuning(ctx, crs, i);
        if (s != BB_OK) { if (i == 0) return s; continue; }
        std::memset(got, 0, sizeof got);
        s = prove_partials_impl(ctx, crs, w, got);             // first proof of this form: builds caches, checked
        if (s != BB_OK) {
            if (i == 0) return s;                       // the witness / key itself fails: nothing to tune
            ms[i] = -2.0;                               // -2: this form failed where the default did not
            continue;
        }
        if (i == 0) std::memcpy(ref, got, sizeof ref);
        else if (whole_key && std::memcmp(ref, got, sizeof ref) != 0) { ms[i] = -3.0; continue; }     // -3: different partial sums -- never eligible
        double fastest = 1e300;
        for (int k = 0; k < reps && s == BB_OK; k++) {
            const auto t0 = std::chrono::steady_clock::now();
            s = prove_partials_impl(ctx, crs, w, got);
            const double dt = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            if (dt < fastest) fastest = dt;
        }
        if (s != BB_OK) { if (i == 0) return s; ms[i] = -2.0; continue; }
        ms[i] = fastest;
        if (ms[i] < ms[best]) best = i;
    }
    if (ms_out) for (int i = 0; i < kNumTunings; i++) ms_out[i] = ms[i];
    if (chosen) *chosen = best;
    return bb_crs_apply_tuning(ctx, crs, whole_key ? best : 0);
}

int bb_groth16_prove(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, const uint8_t* r_bytes, const uint8_t* s_bytes, uint8_t* proof) {
    if (!crs || !r_bytes || !s_bytes || !proof) { set_error("bb_groth16_prove: null argument"); return BB_ERR_ARG; }
    if (crs->shard_count != 1) { set_error("bb_groth16_prove needs an unsharded CRS; use prove_partials + finalize"); return BB_ERR_ARG; }
    return prove_single(ctx, crs, [&](bb_prove** P) { return prove_begin_impl(ctx, crs, w, true, P); }, r_bytes, s_bytes, proof);
}

const char* bb_groth16_prove_message(const bb_crs* crs, int status) { return crs ? prove_status_message(crs, status) : nullptr; }

int bb_groth16_prove_batch(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, size_t count, const uint8_t* r, const uint8_t* s,
                           uint8_t* proofs, int* status) {
    return prove_batch_impl(ctx, crs, w, count, r, s, proofs, status);
}

}  // extern "C"

namespace bb {

int prove_begin_r1cs(bb_ctx* ctx, const bb_crs* crs, const bb_witness* w, const R1csStart& start, bb_prove** out) {
    return prove_begin_impl(ctx, crs, w, false, out, &start);
}

// one proof on an unsharded key: `begin` queues it, the five scalar multiplications that need no MSM result run on the
// host meanwhile, then the waits and the finalisation
int prove_single(bb_ctx* ctx, const bb_crs* crs, const std::function<int(bb_prove**)>& begin, const uint8_t* r_bytes, const uint8_t* s_bytes,
                 uint8_t* proof) {
    uint8_t partials[BB_PARTIALS_BYTES];
    std::memset(partials, 0, sizeof partials);
    Fr r, s;
    std::memcpy(r.l, r_bytes, 32);
    std::memcpy(s.l, s_bytes, 32);
    // profile mode: host-side milestones of one prove, ms since entry (bb_profile_read "host.<mark>")
    const auto t_entry = std::chrono::steady_clock::now();
    auto since = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_entry).count(); };
    bb_prove* P = nullptr;
    BB_TRY(begin(&P));
    const double t_queued = since();
    // the five scalar multiplications that need no MSM result run on the host while the device works
    ProofStatic stat;
    if (!delta_is_identity(crs)) finalize_static(crs, r, s, &stat);
    const double t_static = since();
    BB_TRY(prove_end_impl(P, nullptr, partials));     // reports delta = identity as well (prover.rs:320-324)
    const double t_waited = since();
    int rc = finalize_impl(crs, partials, 1, r, s, stat, proof);
    if (ctx && ctx->opt_profile) {
        ctx->prof_add("host.queued", t_queued, 1, 0);          // everything launched
        ctx->prof_add("host.static_done", t_static, 1, 0);     // MSM-independent scalar multiplications done
        ctx->prof_add("host.msms_done", t_waited, 1, 0);       // all eight results folded on the host
        ctx->prof_add("host.proof_done", since(), 1, 0);
    }
    return rc;
}

}  // namespace bb
