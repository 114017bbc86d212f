// bellman_b200: synthetic workload for the benchmark -- the MiMC chain of
// bellman/groth16/tests/common/mod.rs:48-129 run through what
// groth16's ProvingAssignment records during synthesis (groth16/src/prover.rs:73-145,
// 193-215).  Upstream this is user circuit code plus bookkeeping on the CPU, unchanged by this
// back-end; it lives here only so that bench.py can produce a valid witness of the
// benchmark's size without going through the test oracle.  Host code, product-side field
// arithmetic (mp.cuh host path).
#include "bb_internal.cuh"

using namespace bb;

namespace {

struct SplitMix {
    uint64_t s;
    uint64_t next() {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
    }
};

// uniform in [0, r): rejection sampling on 255-bit draws
Fr random_fr(SplitMix& g) {
    for (;;) {
        uint64_t c[4] = {g.next(), g.next(), g.next(), g.next() & 0x7fffffffffffffffull};
        Fr v;
        std::memcpy(v.l, c, 32);
        bool lt = false;
        for (int i = 7; i >= 0; i--) {
            if (v.l[i] < bbc::FR_MOD[i]) { lt = true; break; }
            if (v.l[i] > bbc::FR_MOD[i]) break;
        }
        if (lt) return fr_from_canonical(v);
    }
}

inline void put(uint64_t* dst, size_t i, const Fr& v) { std::memcpy(dst + 4 * i, v.l, 32); }
inline void set_bit(uint64_t* bits, size_t i) { bits[i >> 6] |= 1ull << (i & 63); }

// canonical scalars < 2^254 < r from a counter-based generator: element i of stream `seed` is the
// same on every device, so base-range shards of a synthetic CRS agree across ranks
__global__ void __launch_bounds__(256) k_synth_scalars(Fr* out, size_t n, uint64_t seed, uint64_t first) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        uint64_t z = seed + 0x9E3779B97F4A7C15ull * (4 * (first + i) + j + 1);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z ^= z >> 31;
        if (j == 3) z &= 0x3fffffffffffffffull;
        v.l[2 * j] = (uint32_t)z;
        v.l[2 * j + 1] = (uint32_t)(z >> 32);
    }
    out[i] = v;
}

// partial[b] = sum over this CTA's grid-stride share of mont(a_i, b_i) = a_i b_i R^-1 (canonical inputs)
__global__ void __launch_bounds__(256) k_fr_dot(const Fr* __restrict__ a, const Fr* __restrict__ b, size_t n, Fr* partial) {
    __shared__ Fr sh[256];
    Fr acc = Fr::zero();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) acc = acc + a[i] * b[i];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (uint32_t s = blockDim.x / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] = sh[threadIdx.x] + sh[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}

}  // namespace

extern "C" {

int bb_diag_fr_dot(bb_ctx* ctx, const void* d_a, const void* d_b, size_t n, void* out_fr) {
    if (!ctx || !out_fr || (n && (!d_a || !d_b))) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    const unsigned blocks = 1024;
    DevBuf d_p;
    BB_TRY(d_p.alloc(ctx, blocks * sizeof(Fr)));
    k_fr_dot<<<blocks, 256, 0, ctx->main_stream>>>((const Fr*)d_a, (const Fr*)d_b, n, d_p.as<Fr>());
    ctx->count_launch();
    BB_CUDA(cudaGetLastError());
    std::vector<Fr> h(blocks);
    BB_CUDA(cudaMemcpyAsync(h.data(), d_p.p, blocks * sizeof(Fr), cudaMemcpyDeviceToHost, ctx->main_stream));
    BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    Fr acc = Fr::zero();
    for (const Fr& v : h) acc = acc + v;
    acc = acc * fr_r2();                                 // (sum a b R^-1) R^2 R^-1 = sum a b, canonical
    std::memcpy(out_fr, acc.l, 32);
    return BB_OK;
}

// d_out[i] = pseudorandom canonical scalar < 2^254, i < n, resident in HBM (bench inputs)
int bb_synth_scalars_device(bb_ctx* ctx, uint64_t seed, size_t n, void* d_out) {
    if (!ctx || (n && !d_out)) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    if (n) { k_synth_scalars<<<cdiv(n, 256), 256, 0, ctx->main_stream>>>((Fr*)d_out, n, seed, 0); ctx->count_launch(); }
    BB_CUDA(cudaGetLastError());
    BB_CUDA(cudaStreamSynchronize(ctx->main_stream));
    return BB_OK;
}

// Base vector [k_i]G, k_i = stream `seed`, produced on the device straight into a bb_bases
// (no host round trip): global indices [global_offset, global_offset + n) of a vector of global_len.
int bb_synth_bases(bb_ctx* ctx, int group, uint64_t seed, size_t n, size_t global_offset, size_t global_len, bb_bases** out) {
    if (!ctx || !out || (group != BB_G1 && group != BB_G2) || global_offset + n > global_len) return BB_ERR_ARG;
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t stride = group == BB_G1 ? sizeof(G1Affine) : sizeof(G2Affine);
    void* d = nullptr;
    BB_TRY(ctx->alloc((n ? n : 1) * stride, &d));
    DevBuf d_k;
    BB_TRY(d_k.alloc(ctx, n * 32));
    cudaStream_t st = ctx->main_stream;
    if (n) { k_synth_scalars<<<cdiv(n, 256), 256, 0, st>>>(d_k.as<Fr>(), n, seed, global_offset); ctx->count_launch(); }
    int s = fixed_base_mul_device(ctx, group, d_k.as<Fr>(), n, false, d, st);
    if (s == BB_OK && cudaStreamSynchronize(st) != cudaSuccess) s = BB_ERR_CUDA;
    if (s != BB_OK) { ctx->release(d); return s; }
    bb_bases* b = new bb_bases();
    b->ctx = ctx; b->group = group; b->d_points = d; b->n = n; b->global_offset = global_offset; b->global_len = global_len;
    *out = b;
    return BB_OK;
}

// shape[0..6] = num_inputs, num_aux, num_constraints, m, a_aux_density_total,
//               b_input_density_total, b_aux_density_total
int bb_synth_mimc_shape(size_t rounds, uint64_t* shape) {
    if (!rounds || !shape) return BB_ERR_ARG;
    size_t n = 2 * rounds + 2, m = 1;
    while (m < n) m *= 2;
    shape[0] = 2; shape[1] = 2 * rounds + 1; shape[2] = n; shape[3] = m;
    shape[4] = 2 * rounds; shape[5] = 1; shape[6] = rounds;
    return BB_OK;
}

// a,b,c: n Fr; inputs: 2 Fr; aux: 2*rounds+1 Fr (all Montgomery); density bitmaps zeroed and
// filled here (LSB-first words).  Constants and preimage: splitmix64(seed), rejection sampled.
int bb_synth_mimc_witness(size_t rounds, uint64_t seed, uint64_t* a, uint64_t* b, uint64_t* c, uint64_t* inputs, uint64_t* aux,
                          uint64_t* a_aux_density, uint64_t* b_input_density, uint64_t* b_aux_density) {
    if (!rounds || !a || !b || !c || !inputs || !aux || !a_aux_density || !b_input_density || !b_aux_density) return BB_ERR_ARG;
    const size_t num_aux = 2 * rounds + 1;
    std::memset(a_aux_density, 0, ((num_aux + 63) / 64) * 8);
    std::memset(b_aux_density, 0, ((num_aux + 63) / 64) * 8);
    b_input_density[0] = 0;
    SplitMix g{seed};
    std::vector<Fr> constants(rounds);
    for (auto& k : constants) k = random_fr(g);
    Fr xl = random_fr(g), xr = random_fr(g);
    const Fr one = fr_one();
    put(inputs, 0, one);                                  // alloc_input(ONE), prover.rs:204
    size_t n_aux = 0, row = 0;
    put(aux, n_aux, xl); size_t xl_idx = n_aux++;          // "preimage xl"
    put(aux, n_aux, xr); n_aux++;                          // "preimage xr" (only ever appears in C)
    bool xl_is_input = false;
    for (size_t i = 0; i < rounds; i++) {
        const Fr& ci = constants[i];
        Fr t = xl + ci;                                    // <xl + Ci*ONE, w>
        Fr tmp = t.sqr();
        put(aux, n_aux, tmp); size_t tmp_idx = n_aux++;
        // tmp = (xL + Ci)^2 :  A = B = xl + Ci, C = tmp
        put(a, row, t); put(b, row, t); put(c, row, tmp); row++;
        if (!xl_is_input) { set_bit(a_aux_density, xl_idx); set_bit(b_aux_density, xl_idx); }
        if (!ci.is_zero()) set_bit(b_input_density, 0);    // eval skips zero coefficients, prover.rs:31
        Fr nw = t * tmp + xr;
        bool last = i + 1 == rounds;
        size_t nw_idx = 0;
        if (last) put(inputs, 1, nw);                      // "image" public input
        else { put(aux, n_aux, nw); nw_idx = n_aux++; }
        // new_xL = xR + tmp*(xL + Ci) :  A = tmp, B = xl + Ci, C = new_xl - xr
        put(a, row, tmp); put(b, row, t); put(c, row, nw - xr); row++;
        set_bit(a_aux_density, tmp_idx);
        xr = xl;
        xl = nw; xl_idx = nw_idx; xl_is_input = last;
    }
    // x_i * 0 = 0 for every input (prover.rs:208-215)
    Fr image;
    std::memcpy(image.l, inputs + 4, 32);
    put(a, row, one); put(b, row, Fr::zero()); put(c, row, Fr::zero()); row++;
    put(a, row, image); put(b, row, Fr::zero()); put(c, row, Fr::zero()); row++;
    return (n_aux == num_aux && row == 2 * rounds + 2) ? BB_OK : BB_ERR_ARG;
}

// The matrices of the circuit above, in the order its LinearCombinations push their terms
// (groth16/tests/common/mod.rs:48-129); the input rows are left to bb_r1cs_create.
int bb_synth_mimc_r1cs(size_t rounds, uint64_t seed, uint64_t* a_off, uint32_t* a_vars, uint64_t* a_coeffs,
                       uint64_t* b_off, uint32_t* b_vars, uint64_t* b_coeffs, uint64_t* c_off, uint32_t* c_vars, uint64_t* c_coeffs) {
    if (!rounds || !a_off || !a_vars || !a_coeffs || !b_off || !b_vars || !b_coeffs || !c_off || !c_vars || !c_coeffs) return BB_ERR_ARG;
    SplitMix g{seed};
    std::vector<Fr> constants(rounds);
    for (auto& k : constants) k = random_fr(g);
    const Fr one = fr_one(), minus_one = Fr::zero() - fr_one();
    struct Csr {
        uint64_t* off; uint32_t* vars; uint64_t* coeffs; size_t row = 0, t = 0;
        void term(uint32_t v, const Fr& k) { vars[t] = v; put(coeffs, t, k); t++; }
        void end_row() { off[++row] = t; }
    } A{a_off, a_vars, a_coeffs}, B{b_off, b_vars, b_coeffs}, C{c_off, c_vars, c_coeffs};
    a_off[0] = b_off[0] = c_off[0] = 0;
    const uint32_t ONE = 0, IMAGE = 1, AUX = 2;
    uint32_t n_aux = 0;
    uint32_t xl = AUX + n_aux++, xr = AUX + n_aux++;       // preimage xl, xr
    for (size_t i = 0; i < rounds; i++) {
        const Fr& ci = constants[i];
        const uint32_t tmp = AUX + n_aux++;
        // tmp = (xL + Ci)^2
        A.term(xl, one); A.term(ONE, ci); A.end_row();
        B.term(xl, one); B.term(ONE, ci); B.end_row();
        C.term(tmp, one); C.end_row();
        const uint32_t nw = i + 1 == rounds ? IMAGE : AUX + n_aux++;
        // new_xL = xR + tmp*(xL + Ci)
        A.term(tmp, one); A.end_row();
        B.term(xl, one); B.term(ONE, ci); B.end_row();
        C.term(nw, one); C.term(xr, minus_one); C.end_row();
        xr = xl;
        xl = nw;
    }
    return (n_aux == 2 * rounds + 1 && A.t == 3 * rounds && B.t == 4 * rounds && C.t == 3 * rounds) ? BB_OK : BB_ERR_ARG;
}

}  // extern "C"
