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
// The per-point rules, square roots and subgroup tests are encoding.cuh's.
// Kernels (one thread per point):
//   k_decode_g1      the 2n A and C points (or n packed points for the diagnostic)
//   k_decode_g2      the n B points
//   k_proof_status   folds the three element codes into the status byte, zeroes all points of an invalid proof
//   k_encode_proofs  the inverse: Proof::write of n affine triples
//
// Parameters::read / VerifyingKey::read (groth16/src/lib.rs:158-218, 289-398) of a key file into a resident bb_crs / bb_vk:
// the u32 length prefixes are walked on the host, every point is decoded on the device by
//   k_params_decode_g1 / k_params_decode_g2   one thread per uncompressed point: flags, canonical coordinates,
//                                             Montgomery form, curve equation and subgroup test (checked sections), the
//                                             identity rule; the point goes straight to its index in the resident vector
// and the first failure in file order is kept in one word, atomicMin((ordinal << 3) | why).  Host bytes are streamed in
// chunks through two pinned staging blocks (copy of chunk k + 1 on a copy stream while chunk k decodes on the main
// stream); device bytes are decoded in place.
#include <cstring>

#include "bb_internal.cuh"
#include "encoding.cuh"

using namespace bb;

namespace {

constexpr unsigned DECODE_THREADS = 64;

// point j of rows x parts: bytes base + (j % rows) * stride + (j / rows) * part_offset -> out[j / rows][j % rows]
__global__ void __launch_bounds__(DECODE_THREADS) k_decode_g1(const uint8_t* __restrict__ base, size_t stride, size_t rows, size_t parts,
                                                              size_t part_offset, int check_subgroup, G1Affine* out0, G1Affine* out1,
                                                              uint8_t* why) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= rows * parts) return;
    size_t row = j % rows, part = j / rows;
    Decoded<Fp> d = decode_compressed<Fp>(base + row * stride + part * part_offset, check_subgroup != 0);
    (part ? out1 : out0)[row] = d.p;
    why[j] = (uint8_t)d.why;
}
__global__ void __launch_bounds__(DECODE_THREADS) k_decode_g2(const uint8_t* __restrict__ base, size_t stride, size_t rows,
                                                              int check_subgroup, G2Affine* out, uint8_t* why) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= rows) return;
    Decoded<Fp2> d = decode_compressed<Fp2>(base + j * stride, check_subgroup != 0);
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
__global__ void __launch_bounds__(128) k_encode_proofs(const G1Affine* __restrict__ a, const G2Affine* __restrict__ b,
                                                       const G1Affine* __restrict__ c, size_t n, uint8_t* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t* o = out + i * 192;
    encode_compressed(a[i], o);
    encode_compressed(b[i], o + 48);
    encode_compressed(c[i], o + 144);
}

constexpr size_t MAX_PROOFS = (size_t)1 << 31;

// ---- Parameters::read: uncompressed points (from_uncompressed / _unchecked, then bellman's identity rule) ----------
BB_D void first_failure(unsigned long long* first, unsigned long long code) {
#if defined(__CUDACC__)
    atomicMin(first, code);
#else
    unsigned long long old = __atomic_load_n(first, __ATOMIC_SEQ_CST);
    while (old > code && !__atomic_compare_exchange_n(first, &old, code, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
#endif
}

// n points at src (stride 96 / 192) -> out[0 .. n); point i has ordinal ord0 + i in the file.  A point behind the first
// failure seen so far is skipped: only the first failure in file order is reported.
template <class F>
BB_D void params_decode(const uint8_t* __restrict__ src, size_t n, uint64_t ord0, int checked, int allow_identity, Affine<F>* out,
                        unsigned long long* first) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long ord = ord0 + i;
    if (*(volatile unsigned long long*)first < (ord << 3)) return;
    Affine<F> p;
    int why = read_uncompressed(src + i * 2 * sizeof(F), checked != 0, allow_identity != 0, &p);
    if (why) first_failure(first, (ord << 3) | (unsigned)why);
    else out[i] = p;
}
__global__ void __launch_bounds__(DECODE_THREADS) k_params_decode_g1(const uint8_t* __restrict__ src, size_t n, uint64_t ord0, int checked,
                                                                     int allow_identity, G1Affine* out, unsigned long long* first) {
    params_decode(src, n, ord0, checked, allow_identity, out, first);
}
__global__ void __launch_bounds__(DECODE_THREADS) k_params_decode_g2(const uint8_t* __restrict__ src, size_t n, uint64_t ord0, int checked,
                                                                     int allow_identity, G2Affine* out, unsigned long long* first) {
    params_decode(src, n, ord0, checked, allow_identity, out, first);
}

// ---- Parameters::write (lib.rs:258-287): to_uncompressed, the inverse of the decoders above -----------------------------
// n points -> out[0 .. 96 n) (G2: 192 n), one thread per point; prefix != 0: thread 0 also writes n as the big-endian u32 in
// the four bytes before out (launched with at least one thread)
BB_D void store_prefix(uint8_t* o, size_t n) {
    o[0] = (uint8_t)(n >> 24); o[1] = (uint8_t)(n >> 16); o[2] = (uint8_t)(n >> 8); o[3] = (uint8_t)n;
}
template <class F>
BB_D void params_encode(const Affine<F>* __restrict__ pts, size_t n, int prefix, uint8_t* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (prefix && i == 0) store_prefix(out - 4, n);
    if (i < n) store_uncompressed(pts[i], out + i * 2 * sizeof(F));
}
__global__ void __launch_bounds__(128) k_params_encode_g1(const G1Affine* __restrict__ pts, size_t n, int prefix, uint8_t* out) {
    params_encode(pts, n, prefix, out);
}
__global__ void __launch_bounds__(128) k_params_encode_g2(const G2Affine* __restrict__ pts, size_t n, int prefix, uint8_t* out) {
    params_encode(pts, n, prefix, out);
}

constexpr int PARAMS_SECTIONS = 12, VK_SECTIONS = 7;
const char* const kSection[PARAMS_SECTIONS] = {"alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "delta_g1", "delta_g2",
                                               "ic", "h", "l", "a", "b_g1", "b_g2"};
const char* const kWhy[6] = {"", "flag bits", "coordinate not below p", "not on the curve", "not in the prime-order subgroup", ""};
bool section_g2(int s) { return s == BB_PARAMS_BETA_G2 || s == BB_PARAMS_GAMMA_G2 || s == BB_PARAMS_DELTA_G2 || s == BB_PARAMS_B_G2; }
size_t point_bytes(int s) { return section_g2(s) ? 192 : 96; }

// Where the sections of a key file lie, from its length prefixes: complete points only, so that nothing sized by a
// prefix exceeds the buffer
struct Layout {
    int sections = 0;                      // sections reached (their complete points are decoded)
    size_t off[PARAMS_SECTIONS] = {};      // byte offset of the section's first point
    size_t count[PARAMS_SECTIONS] = {};    // complete points present
    uint64_t ord0[PARAMS_SECTIONS] = {};   // ordinal of its first point in the file
    size_t declared[6] = {};               // the six prefixes as read
    bool eof = false;                      // the buffer ends inside the key: at eof_section, after eof_index of its points,
    bool eof_prefix = false;               // (or inside its length prefix) at byte eof_offset
    int eof_section = -1;
    size_t eof_index = 0, eof_offset = 0;
    size_t end = 0;                        // bytes of the key (complete keys)
};

int walk_layout(bb_ctx* ctx, const uint8_t* bytes, size_t len, bool on_device, int sections, Layout* L) {
    size_t off = 0;
    uint64_t ord = 0;
    for (int s = 0; s < sections; s++) {
        const size_t size = point_bytes(s);
        size_t want = 1;
        L->sections = s + 1;
        if (s >= BB_PARAMS_IC) {
            if (len - off < 4) { L->eof = L->eof_prefix = true; L->eof_section = s; L->eof_index = 0; L->eof_offset = off; L->sections = s; break; }
            uint8_t b[4];
            if (on_device) {
                BB_CUDA(cudaMemcpy(b, bytes + off, 4, cudaMemcpyDeviceToHost));
                ctx->d2h_bytes += 4;
            } else {
                std::memcpy(b, bytes + off, 4);
            }
            want = ((size_t)b[0] << 24) | ((size_t)b[1] << 16) | ((size_t)b[2] << 8) | b[3];
            L->declared[s - BB_PARAMS_IC] = want;
            off += 4;
        }
        const size_t have = (len - off) / size;
        L->off[s] = off;
        L->ord0[s] = ord;
        L->count[s] = want < have ? want : have;
        off += L->count[s] * size;
        ord += L->count[s];
        if (L->count[s] < want) { L->eof = true; L->eof_section = s; L->eof_index = L->count[s]; L->eof_offset = off; break; }
    }
    L->end = off;
    return BB_OK;
}

// caller's host buffer in page-locked memory (then copied to the device without the staging memcpy)
bool host_pinned(const void* p, size_t len) {
#if defined(__CUDACC__)
    for (const void* q : {p, (const void*)((const uint8_t*)p + len - 1)}) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, q) != cudaSuccess) { cudaGetLastError(); return false; }
        if (a.type != cudaMemoryTypeHost) return false;
    }
    return true;
#else
    (void)p; (void)len;
    return false;
#endif
}

struct Events {                           // destroyed with the call
    cudaEvent_t e[4] = {nullptr, nullptr, nullptr, nullptr};
    ~Events() { for (auto x : e) if (x) cudaEventDestroy(x); }
};

int params_read_impl(bb_ctx* ctx, const void* bytes, size_t len, int on_device, int checked, int sections, bb_crs** crs_out,
                     bb_vk** vk_out, bb_params_report* report) {
    const char* fn = sections == PARAMS_SECTIONS ? "bb_params_read" : "bb_vk_read";
    if (crs_out) *crs_out = nullptr;
    if (vk_out) *vk_out = nullptr;
    bb_params_report rep{};
    rep.section = -1;
    if (report) *report = rep;
    if (!ctx || (len && !bytes) || (sections == PARAMS_SECTIONS ? !crs_out : !vk_out)) {
        set_error("%s: null argument", fn);
        return BB_ERR_ARG;
    }
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("params_read");
    const uint8_t* src = (const uint8_t*)bytes;
    Layout L;
    BB_TRY(walk_layout(ctx, src, len, on_device != 0, sections, &L));
    for (int k = 0; k < 6; k++) rep.len[k] = L.declared[k];

    // destinations at their final size (complete points only): alpha; beta_g1, delta_g1; the G2 points in bb_vk's order
    // delta, gamma, beta; ic; the five vectors
    DevBuf d_alpha, d_g1x, d_g2, d_vec[6], d_first;
    BB_TRY(d_alpha.alloc(ctx, sizeof(G1Affine)));
    BB_TRY(d_g1x.alloc(ctx, 2 * sizeof(G1Affine)));
    BB_TRY(d_g2.alloc(ctx, 3 * sizeof(G2Affine)));
    for (int k = 0; k < sections - BB_PARAMS_IC; k++) {
        const int s = BB_PARAMS_IC + k;
        BB_TRY(d_vec[k].alloc(ctx, (L.count[s] ? L.count[s] : 1) * point_bytes(s)));
    }
    BB_TRY(d_first.alloc(ctx, 8));
    void* dest[PARAMS_SECTIONS] = {d_alpha.p, d_g1x.p, d_g2.as<G2Affine>() + 2, d_g2.as<G2Affine>() + 1, d_g1x.as<G1Affine>() + 1, d_g2.p};
    for (int k = 0; k < sections - BB_PARAMS_IC; k++) dest[BB_PARAMS_IC + k] = d_vec[k].p;

    cudaStream_t st = ctx->main_stream;
    // host input: device staging blocks, events and the pinned blocks' lock live until the stream is drained below
    DevBuf d_stage[2];
    Events ev;                                                    // copied[b], decoded[b]
    std::unique_lock<std::mutex> stage_lock(ctx->read_mu, std::defer_lock);
    StageTimer tm(ctx, st);
    tm.mark("params.begin");
    BB_CUDA(cudaMemsetAsync(d_first.p, 0xff, 8, st));
    unsigned long long* first = d_first.as<unsigned long long>();
    uint64_t points = 0;
    auto launch = [&](int s, const uint8_t* p, size_t lo, size_t n) {
        const int chk = s <= BB_PARAMS_IC || checked ? 1 : 0, allow = s < BB_PARAMS_IC ? 1 : 0;
        const uint64_t ord = L.ord0[s] + lo;
        if (section_g2(s))
            k_params_decode_g2<<<cdiv(n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(p, n, ord, chk, allow, (G2Affine*)dest[s] + lo, first);
        else
            k_params_decode_g1<<<cdiv(n, DECODE_THREADS), DECODE_THREADS, 0, st>>>(p, n, ord, chk, allow, (G1Affine*)dest[s] + lo, first);
        ctx->count_launch();
        tm.mark(section_g2(s) ? "params.g2" : "params.g1");
        points += n;
    };

    if (on_device) {                                              // in place: one launch per section
        for (int s = 0; s < L.sections; s++)
            if (L.count[s]) launch(s, src + L.off[s], 0, L.count[s]);
        BB_CUDA(cudaGetLastError());
    } else if (L.end) {
        // chunks of whole points; chunk k is copied into device block k % 2 on the copy stream while chunk k - 1 decodes
        const size_t chunk = (size_t)ctx->opt_params_read_chunk;
        const size_t cap = chunk < 192 ? 192 : chunk;             // one point at least
        const bool direct = host_pinned(bytes, len);
        if (!direct) {
            stage_lock.lock();
            if (ctx->read_stage_bytes < cap) {
                for (auto& p : ctx->read_stage) { if (p) cudaFreeHost(p); p = nullptr; }
                ctx->read_stage_bytes = 0;
                for (auto& p : ctx->read_stage) BB_CUDA(cudaMallocHost(&p, cap));
                ctx->read_stage_bytes = cap;
            }
        }
        BB_TRY(d_stage[0].alloc(ctx, cap));
        BB_TRY(d_stage[1].alloc(ctx, cap));
        for (auto& e : ev.e) BB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        cudaEvent_t* copied = ev.e;
        cudaEvent_t* decoded = ev.e + 2;
        cudaStream_t cp = ctx->pick_stream();
        size_t k = 0;
        for (int s = 0; s < L.sections; s++) {
            const size_t size = point_bytes(s), per = chunk / size ? chunk / size : 1;
            for (size_t lo = 0; lo < L.count[s]; lo += per, k++) {
                const size_t n = L.count[s] - lo < per ? L.count[s] - lo : per, nb = n * size;
                const int b = (int)(k & 1);
                const uint8_t* h = src + L.off[s] + lo * size;
                if (k >= 2) BB_CUDA(cudaStreamWaitEvent(cp, decoded[b], 0));     // chunk k - 2 has left block b
                if (!direct) {
                    if (k >= 2) BB_CUDA(cudaEventSynchronize(copied[b]));        // ... and its pinned block
                    std::memcpy(ctx->read_stage[b], h, nb);
                    h = (const uint8_t*)ctx->read_stage[b];
                }
                BB_CUDA(cudaMemcpyAsync(d_stage[b].p, h, nb, cudaMemcpyHostToDevice, cp));
                ctx->h2d_bytes += nb;
                BB_CUDA(cudaEventRecord(copied[b], cp));
                BB_CUDA(cudaStreamWaitEvent(st, copied[b], 0));
                tm.mark("params.upload");
                launch(s, d_stage[b].as<uint8_t>(), lo, n);
                BB_CUDA(cudaEventRecord(decoded[b], st));
            }
        }
        BB_CUDA(cudaGetLastError());
        // every copy is behind an event the main stream waited for: draining it drains the copy stream's work too
    }
    unsigned long long bad = ~0ull;
    BB_CUDA(cudaMemcpyAsync(&bad, first, 8, cudaMemcpyDeviceToHost, st));
    G1Affine g1[3];
    G2Affine g2[3];                                               // delta, gamma, beta
    BB_CUDA(cudaMemcpyAsync(&g1[0], d_alpha.p, sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(&g1[1], d_g1x.p, 2 * sizeof(G1Affine), cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaMemcpyAsync(g2, d_g2.p, sizeof g2, cudaMemcpyDeviceToHost, st));
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(points);

    if (bad != ~0ull) {                                           // the first invalid point in file order
        const uint64_t ord = bad >> 3;
        const int why = (int)(bad & 7);
        int s = 0;
        while (s + 1 < L.sections && ord >= L.ord0[s + 1]) s++;
        rep.section = s;
        rep.index = (size_t)(ord - L.ord0[s]);
        rep.why = why;
        rep.consumed = L.off[s] + rep.index * point_bytes(s);
        if (s < BB_PARAMS_IC) {
            if (why == WHY_IDENTITY) set_error("%s: point at infinity", kSection[s]);
            else set_error("%s: invalid %s (%s)", kSection[s], section_g2(s) ? "G2" : "G1", kWhy[why]);
        } else {
            if (why == WHY_IDENTITY) set_error("%s[%zu]: point at infinity", kSection[s], rep.index);
            else set_error("%s[%zu]: invalid %s (%s)", kSection[s], rep.index, section_g2(s) ? "G2" : "G1", kWhy[why]);
        }
        if (report) *report = rep;
        return BB_ERR_IO_INVALID_DATA;
    }
    if (L.eof) {
        rep.section = L.eof_section;
        rep.index = L.eof_index;
        rep.consumed = L.eof_offset;
        if (L.eof_section < BB_PARAMS_IC)
            set_error("%s: unexpected end of file (failed to fill whole buffer)", kSection[L.eof_section]);
        else if (L.eof_prefix)
            set_error("%s: unexpected end of file in the length prefix (failed to fill whole buffer)", kSection[L.eof_section]);
        else
            set_error("%s[%zu]: unexpected end of file (failed to fill whole buffer)", kSection[L.eof_section], L.eof_index);
        if (report) *report = rep;
        return BB_ERR_IO_UNEXPECTED_EOF;
    }

    rep.consumed = L.end;
    auto bases = [&](int s) {
        bb_bases* b = new bb_bases();
        b->ctx = ctx; b->group = section_g2(s) ? BB_G2 : BB_G1; b->n = L.count[s]; b->global_offset = 0; b->global_len = L.count[s];
        b->d_points = d_vec[s - BB_PARAMS_IC].take();
        return b;
    };
    bb_bases* ic = vk_out ? bases(BB_PARAMS_IC) : nullptr;
    if (crs_out) {
        bb_bases* vec[5];
        for (int k = 0; k < 5; k++) vec[k] = bases(BB_PARAMS_H + k);
        const G1Affine vg1[3] = {g1[0], g1[1], g1[2]};
        const G2Affine vg2[2] = {g2[2], g2[0]};
        *crs_out = crs_adopt(ctx, vec, vg1, vg2);
    }
    if (vk_out) *vk_out = vk_adopt(ctx, (G1Affine*)d_alpha.take(), (G2Affine*)d_g2.take(), ic);
    if (report) *report = rep;
    return BB_OK;
}

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

int bb_params_read(bb_ctx* ctx, const void* bytes, size_t len, int on_device, int checked, bb_crs** crs_out, bb_vk** vk_out,
                   bb_params_report* report) {
    return params_read_impl(ctx, bytes, len, on_device, checked, PARAMS_SECTIONS, crs_out, vk_out, report);
}

int bb_vk_read(bb_ctx* ctx, const void* bytes, size_t len, int on_device, bb_vk** vk_out, bb_params_report* report) {
    return params_read_impl(ctx, bytes, len, on_device, 1, VK_SECTIONS, nullptr, vk_out, report);
}

int bb_params_write(bb_ctx* ctx, const bb_crs* crs, const bb_vk* vk, int vk_only, void* out, size_t cap, int out_on_device, size_t* len_out) {
    if (!ctx || !crs || !vk || !len_out) { set_error("bb_params_write: null argument"); return BB_ERR_ARG; }
    const CrsView K = crs_view(crs);
    const VkView V = vk_view(vk);
    if (K.ctx != ctx || V.ctx != ctx) { set_error("bb_params_write: the key lives on another context"); return BB_ERR_ARG; }
    if (K.shard_count > 1) { set_error("bb_params_write: shard %u of a sharded key: only a whole key can be written", K.shard_count); return BB_ERR_ARG; }
    const size_t n_ic = V.ic->n;
    size_t len = 868 + 96 * n_ic;
    if (!vk_only) len += 5 * 4 + 96 * (K.vec[0]->n + K.vec[1]->n + K.vec[2]->n + K.vec[3]->n) + 192 * K.vec[4]->n;
    BB_CUDA(cudaSetDevice(ctx->device));
    G1Affine v_alpha;
    G2Affine v_g2[3];                                             // delta, gamma, beta
    BB_CUDA(cudaMemcpy(&v_alpha, V.d_alpha, sizeof v_alpha, cudaMemcpyDeviceToHost));
    BB_CUDA(cudaMemcpy(v_g2, V.d_g2, sizeof v_g2, cudaMemcpyDeviceToHost));
    if (std::memcmp(&v_alpha, &K.g1[0], sizeof v_alpha) || std::memcmp(&v_g2[2], &K.g2[0], sizeof(G2Affine)) ||
        std::memcmp(&v_g2[0], &K.g2[1], sizeof(G2Affine))) {
        set_error("bb_params_write: not this key's verifying key (alpha_g1, beta_g2 or delta_g2 differ)");
        return BB_ERR_ARG;
    }
    *len_out = len;
    if (!out) return BB_OK;
    if (cap < len) { set_error("bb_params_write: %zu bytes of room for a %zu-byte key", cap, len); return BB_ERR_ARG; }
    NvtxRange nvtx("params_write");
    cudaStream_t st = ctx->main_stream;
    StageTimer tm(ctx, st);
    tm.mark("params.begin");
    DevBuf d_out, d_g1x;
    uint8_t* o = (uint8_t*)out;
    if (!out_on_device) {
        BB_TRY(d_out.alloc(ctx, len));
        o = d_out.as<uint8_t>();
    }
    const G1Affine g1x[2] = {K.g1[1], K.g1[2]};                  // beta_g1, delta_g1: only the crs holds them
    BB_TRY(d_g1x.alloc(ctx, sizeof g1x));
    BB_CUDA(cudaMemcpyAsync(d_g1x.p, g1x, sizeof g1x, cudaMemcpyHostToDevice, st));
    size_t off = 0;
    auto g1 = [&](const void* pts, size_t n, bool prefix) {
        if (prefix) off += 4;
        k_params_encode_g1<<<cdiv(n ? n : 1, 128), 128, 0, st>>>((const G1Affine*)pts, n, prefix ? 1 : 0, o + off);
        ctx->count_launch();
        off += 96 * n;
    };
    auto g2 = [&](const void* pts, size_t n, bool prefix) {
        if (prefix) off += 4;
        k_params_encode_g2<<<cdiv(n ? n : 1, 128), 128, 0, st>>>((const G2Affine*)pts, n, prefix ? 1 : 0, o + off);
        ctx->count_launch();
        off += 192 * n;
    };
    g1(V.d_alpha, 1, false);                                      // VerifyingKey::write (lib.rs:143-156)
    g1(d_g1x.as<G1Affine>(), 1, false);
    g2(V.d_g2 + 2, 1, false);
    g2(V.d_g2 + 1, 1, false);
    g1(d_g1x.as<G1Affine>() + 1, 1, false);
    g2(V.d_g2, 1, false);
    g1(V.ic->d_points, n_ic, true);
    if (!vk_only) {                                               // then h, l, a, b_g1, b_g2 (lib.rs:258-287)
        for (int k = 0; k < 4; k++) g1(K.vec[k]->d_points, K.vec[k]->n, true);
        g2(K.vec[4]->d_points, K.vec[4]->n, true);
    }
    BB_CUDA(cudaGetLastError());
    tm.mark("params.encode");
    if (!out_on_device) {
        BB_CUDA(cudaMemcpyAsync(out, o, len, cudaMemcpyDeviceToHost, st));
        ctx->d2h_bytes += len;
    }
    tm.mark("params.download");
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(len);
    return BB_OK;
}

}  // extern "C"
