// bellman_b200: the constraint system resident on the device.  ProvingAssignment::enforce
// (bellman/groth16/src/prover.rs:105-145) evaluates every linear combination of every constraint
// on the caller's CPU, one field product per term, inside synthesis.  Nothing in that work depends
// on anything but the circuit's shape and the witness, so the handle here keeps the A, B and C
// matrices in HBM beside the key and computes a = A z, b = B z, c = C z as a sparse
// matrix-vector product over Fr, with z = input_assignment || aux_assignment.
//
// Layout (built on the host at create time, DESIGN.md 4.8):
//   the three matrices as ONE CSR of 3 N rows (N = constraints incl. the appended input rows;
//   row g = matrix g / N, constraint g % N), uint32 offsets;
//   per term a uint32 variable index (inputs first, then aux) whose bit 31 marks coefficient one
//   (eval skips that product, prover.rs:47-49), and its Fr coefficient (Montgomery) at the same
//   position; terms with coefficient zero are dropped (they add nothing, and the densities are
//   taken before);
//   the row ids binned by length: <= 32 terms one thread per row, 33..2048 one warp per row,
//   more one CTA of 256 threads per row.  Each bin lists its rows in ascending g, so the rows of
//   one matrix are one contiguous run inside each bin: bin_rows[bin][matrix] counts them, and the
//   owner of one polynomial evaluates its matrix alone over those runs (bb_groth16_prove_r1cs_begin).
#include <algorithm>
#include <memory>
#include <vector>

#include "bb_internal.cuh"

using namespace bb;

namespace {

constexpr uint32_t ONE_FLAG = R1CS_ONE_FLAG;
constexpr uint32_t SHORT_MAX = R1CS_SHORT_MAX;   // terms: one thread per row up to here
constexpr uint32_t WARP_MAX = R1CS_WARP_MAX;     // one warp per row up to here, one CTA above
constexpr int GROUP_THREADS = 256;

struct EvalArgs {
    const uint32_t* off;
    const uint32_t* idx;
    const Fr* coef;
    const Fr* input;
    const Fr* aux;
    Fr *out_a, *out_b, *out_c;
    uint32_t n_inputs;
    uint32_t n;                        // rows per matrix
};

__device__ __forceinline__ Fr r1cs_term(const EvalArgs& A, uint32_t k) {
    const uint32_t v = A.idx[k], var = v & ~ONE_FLAG;
    const Fr z = var < A.n_inputs ? A.input[var] : A.aux[var - A.n_inputs];
    return (v & ONE_FLAG) ? z : A.coef[k] * z;
}

__device__ __forceinline__ void r1cs_put(const EvalArgs& A, uint32_t g, const Fr& v) {
    Fr* o = g < A.n ? A.out_a : g < 2 * A.n ? A.out_b : A.out_c;
    o[g - (g < A.n ? 0 : g < 2 * A.n ? A.n : 2 * A.n)] = v;
}

// rows of at most SHORT_MAX terms (MiMC-like rows of 1-3 terms, empty rows): one thread each
__global__ void __launch_bounds__(128) k_r1cs_rows_thread(EvalArgs A, const uint32_t* __restrict__ rows, uint32_t count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t g = rows[i];
    Fr acc = Fr::zero();
    for (uint32_t k = A.off[g], e = A.off[g + 1]; k < e; k++) acc = acc + r1cs_term(A, k);
    r1cs_put(A, g, acc);
}

// long rows: GROUP threads per row stride over its terms, then a tree of Fr additions in shared memory
template <int GROUP>
__global__ void __launch_bounds__(GROUP_THREADS) k_r1cs_rows_group(EvalArgs A, const uint32_t* __restrict__ rows, uint32_t count) {
    __shared__ Fr sh[GROUP_THREADS];
    const uint32_t lane = threadIdx.x % GROUP, slot = blockIdx.x * (GROUP_THREADS / GROUP) + threadIdx.x / GROUP;
    Fr acc = Fr::zero();
    uint32_t g = 0;
    if (slot < count) {
        g = rows[slot];
        for (uint32_t k = A.off[g] + lane, e = A.off[g + 1]; k < e; k += GROUP) acc = acc + r1cs_term(A, k);
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (uint32_t s = GROUP / 2; s > 0; s >>= 1) {
        if (lane < s) sh[threadIdx.x] = sh[threadIdx.x] + sh[threadIdx.x + s];
        __syncthreads();
    }
    if (lane == 0 && slot < count) r1cs_put(A, g, sh[threadIdx.x]);
}

// The three row kernels on `st`: count[b] rows listed at rows[b] for the short, warp and CTA bin; an empty bin is not launched
int rows_queue(bb_ctx* ctx, cudaStream_t st, const EvalArgs& A, const uint32_t* const rows[3], const uint32_t count[3]) {
    if (count[0]) { k_r1cs_rows_thread<<<cdiv(count[0], 128), 128, 0, st>>>(A, rows[0], count[0]); ctx->count_launch(); }
    if (count[1]) {
        k_r1cs_rows_group<32><<<cdiv(count[1], GROUP_THREADS / 32), GROUP_THREADS, 0, st>>>(A, rows[1], count[1]);
        ctx->count_launch();
    }
    if (count[2]) { k_r1cs_rows_group<GROUP_THREADS><<<count[2], GROUP_THREADS, 0, st>>>(A, rows[2], count[2]); ctx->count_launch(); }
    BB_CUDA(cudaGetLastError());
    return BB_OK;
}

// which_is_unsatisfied over evaluated rows: row k fails when a[k] b[k] != c[k] (Montgomery product, limb equality; every
// value is below r).  A failing row lowers *first, counts itself in *count and, with bits, sets bit k of the LSB-first
// words (the uint64 density words' bytes).  A satisfied witness issues no atomics.
__global__ void __launch_bounds__(256) k_r1cs_check(const Fr* __restrict__ a, const Fr* __restrict__ b, const Fr* __restrict__ c,
                                                    uint32_t n, uint32_t* __restrict__ first, uint32_t* __restrict__ count,
                                                    uint32_t* __restrict__ bits) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || a[k] * b[k] == c[k]) return;
    atomicMin(first, k);
    atomicAdd(count, 1u);
    if (bits) atomicOr(bits + k / 32, 1u << (k % 32));
}

bool fr_geq_modulus(const uint32_t* v) {
    for (int i = 7; i >= 0; i--) {
        if (v[i] > bbc::FR_MOD[i]) return true;
        if (v[i] < bbc::FR_MOD[i]) return false;
    }
    return true;
}

}  // namespace

struct bb_r1cs {
    bb_ctx* ctx = nullptr;
    size_t n_inputs = 0, n_aux = 0, n = 0;              // n: constraints including the appended input rows
    uint64_t nnz[3] = {0, 0, 0}, unit[3] = {0, 0, 0};    // terms the evaluation reads per matrix, and those with coefficient one
    std::vector<uint64_t> a_aux_density, b_input_density, b_aux_density;
    void *d_off = nullptr, *d_idx = nullptr, *d_coef = nullptr, *d_rows = nullptr;
    uint32_t n_short = 0, n_warp = 0, n_cta = 0;
    uint32_t bin_rows[3][3] = {};                        // [bin][matrix]: rows of matrix A, B, C in the short, warp, CTA bin
    ~bb_r1cs() {
        for (void* p : {d_off, d_idx, d_coef, d_rows})
            if (p) ctx->release(p);
    }
};

namespace {

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// The witness checks of eval and prove.  outputs_aligned: the caller's device outputs, if any, are 16-byte aligned.
int check_witness(const char* fn, const bb_ctx* ctx, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux, size_t n_aux,
                  int on_device, bool outputs_aligned) {
    if (R->ctx != ctx) { set_error("%s: the constraint system lives on another context", fn); return BB_ERR_ARG; }
    if (n_inputs != R->n_inputs || n_aux != R->n_aux) {
        set_error("%s: witness has %zu inputs and %zu aux values, the constraint system %zu and %zu", fn, n_inputs, n_aux, R->n_inputs, R->n_aux);
        return BB_ERR_ARG;
    }
    if (!input || (n_aux && !aux)) { set_error("%s: null witness pointer", fn); return BB_ERR_ARG; }
    if ((on_device && !(aligned16(input) && aligned16(aux))) || !outputs_aligned) {
        set_error("%s: device arrays must be 16-byte aligned", fn);
        return BB_ERR_ARG;
    }
    return BB_OK;
}

// z = input || aux on the device: the caller's arrays, or their upload on `st`
int stage_witness(bb_ctx* ctx, cudaStream_t st, const void* input, size_t n_inputs, const void* aux, size_t n_aux, int on_device,
                  DevBuf (&up)[2], const Fr** d_in, const Fr** d_aux) {
    BB_TRY(device_input(ctx, st, input, n_inputs * 32, on_device, up[0], d_in));
    return device_input(ctx, st, aux, n_aux * 32, on_device, up[1], d_aux);
}

// queues the evaluation of all 3 N rows on `st`
int r1cs_eval_queue(bb_ctx* ctx, cudaStream_t st, const bb_r1cs* R, const Fr* d_in, const Fr* d_aux, Fr* oa, Fr* ob, Fr* oc) {
    const CsrMatrix M{(const uint32_t*)R->d_off, (const uint32_t*)R->d_idx, (const Fr*)R->d_coef, (const uint32_t*)R->d_rows,
                      R->n_short, R->n_warp, R->n_cta, (uint32_t)R->n};
    return csr_eval_queue(ctx, st, M, d_in, (uint32_t)R->n_inputs, d_aux, oa, ob, oc);
}

// The owner stage of polynomial i (0 = a, 1 = b, 2 = c) on `st`: <M_i,k, z> for k < n straight into out (m Fr) over matrix
// i's runs of the three bins -- the other two matrices are not read -- zeros up to m (domain.rs:69), then ifft + coset_fft
// in place (prover.rs:225-230) with tmp (m Fr) as scratch
int r1cs_owner_queue(bb_ctx* ctx, cudaStream_t st, const bb_r1cs* R, int i, const Fr* d_in, const Fr* d_aux, Fr* out, size_t m, uint32_t log_m,
                     Fr* tmp, StageTimer& tm) {
    const size_t n = R->n;
    const EvalArgs A{(const uint32_t*)R->d_off, (const uint32_t*)R->d_idx, (const Fr*)R->d_coef, d_in, d_aux, out, out, out,
                     (uint32_t)R->n_inputs, (uint32_t)n};     // matrix i's rows land in out whichever output r1cs_put picks
    const uint32_t* order = (const uint32_t*)R->d_rows;
    const uint32_t bin_start[3] = {0, R->n_short, R->n_short + R->n_warp};
    const uint32_t* rows[3];
    uint32_t count[3];
    for (int b = 0; b < 3; b++) {
        uint32_t lo = bin_start[b];
        for (int q = 0; q < i; q++) lo += R->bin_rows[b][q];
        rows[b] = order + lo;
        count[b] = R->bin_rows[b][i];
    }
    BB_TRY(rows_queue(ctx, st, A, rows, count));
    if (m > n) BB_CUDA(cudaMemsetAsync(out + n, 0, (m - n) * 32, st));
    tm.mark("r1cs_owner.eval", R->nnz[i]);
    BB_TRY(h_poly_evals_device(ctx, st, out, tmp, log_m));
    tm.mark("r1cs_owner.transforms", m);
    return BB_OK;
}

// The bb_witness bb_groth16_prove would take for this witness, without a, b, c
bb_witness r1cs_witness(const bb_r1cs* R, const void* input, const void* aux, int on_device) {
    bb_witness w{};
    w.n_constraints = R->n;
    w.input_assignment = input; w.n_inputs = R->n_inputs;
    w.aux_assignment = aux; w.n_aux = R->n_aux;
    w.a_aux_density = R->a_aux_density.data();
    w.b_input_density = R->b_input_density.data();
    w.b_aux_density = R->b_aux_density.data();
    w.on_device = on_device;
    return w;
}

// The replicated start: a, b, c into the H pipeline's rows (stride m) by the combined bins
R1csStart r1cs_replicated(bb_ctx* ctx, const bb_r1cs* R) {
    R1csStart st{false, {}, {}, R->nnz[0] + R->nnz[1] + R->nnz[2]};
    st.fill = [ctx, R](cudaStream_t s, uint32_t, Fr* abc, size_t m, const Fr* d_in, const Fr* d_aux) -> int {
        return r1cs_eval_queue(ctx, s, R, d_in, d_aux, abc, abc + m, abc + 2 * m);
    };
    return st;
}

// bb_r1cs_check(_batch) after the argument checks: `count` witnesses (row-major, bb_groth16_prove_r1cs_batch's layout)
// checked item by item on the main stream through one a, b, c block and, for host witnesses, one upload block.  The
// per-item first rows and counts stay on the device until one download at the end; bits (count = 1 only) likewise.
int r1cs_check_run(bb_ctx* ctx, const bb_r1cs* R, const void* inputs, const void* aux, size_t count, int on_device, size_t* first,
                   size_t* n_unsat, uint64_t* bits) {
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("r1cs_check");
    cudaStream_t st = ctx->main_stream;
    const size_t n = R->n, ni = R->n_inputs, na = R->n_aux, words = (n + 63) / 64;
    DevBuf d_abc, d_res, d_bits, up[2];
    BB_TRY(d_abc.alloc(ctx, 3 * n * 32));
    BB_TRY(d_res.alloc(ctx, 2 * count * 4));                     // first[count], then n_unsat[count]
    uint32_t *r_first = d_res.as<uint32_t>(), *r_count = r_first + count;
    BB_CUDA(cudaMemsetAsync(r_first, 0xFF, count * 4, st));
    BB_CUDA(cudaMemsetAsync(r_count, 0, count * 4, st));
    if (bits) {
        BB_TRY(d_bits.alloc(ctx, words * 8));
        BB_CUDA(cudaMemsetAsync(d_bits.p, 0, words * 8, st));
    }
    if (!on_device) {
        BB_TRY(up[0].alloc(ctx, ni * 32));
        BB_TRY(up[1].alloc(ctx, na * 32));
    }
    Fr* oa = d_abc.as<Fr>();
    StageTimer tm(ctx, st);
    tm.mark("r1cs_check.begin");
    for (size_t i = 0; i < count; i++) {
        const char* in_i = (const char*)inputs + i * ni * 32;
        const char* aux_i = na ? (const char*)aux + i * na * 32 : nullptr;
        const Fr *d_in = (const Fr*)in_i, *d_aux = (const Fr*)aux_i;
        if (!on_device) {                                          // the stream orders this copy after item i - 1's reads
            BB_CUDA(cudaMemcpyAsync(up[0].p, in_i, ni * 32, cudaMemcpyHostToDevice, st));
            if (na) BB_CUDA(cudaMemcpyAsync(up[1].p, aux_i, na * 32, cudaMemcpyHostToDevice, st));
            ctx->h2d_bytes += (ni + na) * 32;
            d_in = up[0].as<Fr>();
            d_aux = up[1].as<Fr>();
        }
        tm.mark("r1cs_check.upload");
        BB_TRY(r1cs_eval_queue(ctx, st, R, d_in, d_aux, oa, oa + n, oa + 2 * n));
        tm.mark("r1cs_check.eval");
        k_r1cs_check<<<cdiv(n, 256), 256, 0, st>>>(oa, oa + n, oa + 2 * n, (uint32_t)n, r_first + i, r_count + i, d_bits.as<uint32_t>());
        ctx->count_launch();
        BB_CUDA(cudaGetLastError());
        tm.mark("r1cs_check.compare");
    }
    std::vector<uint32_t> res(2 * count);
    BB_CUDA(cudaMemcpyAsync(res.data(), r_first, 2 * count * 4, cudaMemcpyDeviceToHost, st));
    if (bits) BB_CUDA(cudaMemcpyAsync(bits, d_bits.p, words * 8, cudaMemcpyDeviceToHost, st));
    ctx->d2h_bytes += 2 * count * 4 + (bits ? words * 8 : 0);
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(R->nnz[0] + R->nnz[1] + R->nnz[2]);
    for (size_t i = 0; i < count; i++) {
        first[i] = res[i] == 0xFFFFFFFFu ? SIZE_MAX : res[i];
        if (n_unsat) n_unsat[i] = res[count + i];
    }
    return BB_OK;
}

}  // namespace

namespace bb {

int csr_eval_queue(bb_ctx* ctx, cudaStream_t st, const CsrMatrix& M, const Fr* input, uint32_t n_inputs, const Fr* aux, Fr* oa, Fr* ob,
                   Fr* oc) {
    const EvalArgs A{M.off, M.idx, M.coef, input, aux, oa, ob, oc, n_inputs, M.n};
    const uint32_t* const rows[3] = {M.rows, M.rows + M.n_short, M.rows + M.n_short + M.n_warp};
    const uint32_t count[3] = {M.n_short, M.n_warp, M.n_cta};
    return rows_queue(ctx, st, A, rows, count);
}

R1csView r1cs_view(const bb_r1cs* R) {
    return R1csView{R->ctx, R->n, R->n_inputs, R->n_aux, R->nnz[0] + R->nnz[1] + R->nnz[2], (const uint32_t*)R->d_off,
                    (const uint32_t*)R->d_idx, (const Fr*)R->d_coef};
}

}  // namespace bb

extern "C" {

int bb_r1cs_create(bb_ctx* ctx, const bb_r1cs_desc* d, bb_r1cs** out) {
    if (!ctx || !d || !out) { set_error("bb_r1cs_create: null argument"); return BB_ERR_ARG; }
    if (d->n_inputs == 0) { set_error("bb_r1cs_create: no inputs (ONE is input 0)"); return BB_ERR_ARG; }
    const size_t ni = d->n_inputs, nv = d->n_inputs + d->n_aux, rows = d->n_constraints, n = rows + ni;
    if (nv >= ONE_FLAG || nv < ni) { set_error("bb_r1cs_create: %zu inputs + %zu aux variables: at most 2^31 - 1", ni, d->n_aux); return BB_ERR_ARG; }
    if (n >= ((size_t)1 << 31) / 3 + 1 || n < rows) { set_error("bb_r1cs_create: %zu constraints: too many", rows); return BB_ERR_ARG; }
    const bb_r1cs_matrix* mats[3] = {&d->a, &d->b, &d->c};
    static const char* const name[3] = {"A", "B", "C"};
    uint64_t total = ni;
    for (int m = 0; m < 3; m++) {                               // shape first: offsets from 0, non-decreasing
        const bb_r1cs_matrix& M = *mats[m];
        if (!M.row_offsets) { set_error("bb_r1cs_create: %s has no row offsets", name[m]); return BB_ERR_ARG; }
        if (M.row_offsets[0] != 0) { set_error("bb_r1cs_create: %s row_offsets[0] = %llu, not 0", name[m], (unsigned long long)M.row_offsets[0]); return BB_ERR_ARG; }
        for (size_t k = 0; k < rows; k++)
            if (M.row_offsets[k + 1] < M.row_offsets[k]) { set_error("bb_r1cs_create: %s row_offsets decrease at row %zu", name[m], k); return BB_ERR_ARG; }
        const uint64_t terms = M.row_offsets[rows];
        if (terms && (!M.vars || !M.coeffs)) { set_error("bb_r1cs_create: %s has %llu terms and a null array", name[m], (unsigned long long)terms); return BB_ERR_ARG; }
        total += terms;
        if (total >= ((uint64_t)1 << 32)) { set_error("bb_r1cs_create: more than 2^32 - 1 terms"); return BB_ERR_ARG; }
    }
    std::unique_ptr<bb_r1cs> R(new bb_r1cs());
    R->ctx = ctx; R->n_inputs = ni; R->n_aux = d->n_aux; R->n = n;
    const size_t aux_words = (d->n_aux + 63) / 64, in_words = (ni + 63) / 64;
    R->a_aux_density.assign(aux_words ? aux_words : 1, 0);
    R->b_input_density.assign(in_words, 0);
    R->b_aux_density.assign(aux_words ? aux_words : 1, 0);
    const Fr one = fr_one();
    std::vector<uint32_t> off(3 * n + 1), idx, rbins[3];
    std::vector<Fr> coef;
    idx.reserve(total);
    coef.reserve(total);
    auto bin = [&](uint32_t g, uint64_t len) { rbins[len <= SHORT_MAX ? 0 : len <= WARP_MAX ? 1 : 2].push_back(g); };
    for (int m = 0; m < 3; m++) {
        const bb_r1cs_matrix& M = *mats[m];
        const Fr* cf = (const Fr*)M.coeffs;
        for (size_t k = 0; k < rows; k++) {
            const uint32_t g = (uint32_t)(m * n + k);
            off[g] = (uint32_t)idx.size();
            for (uint64_t t = M.row_offsets[k]; t < M.row_offsets[k + 1]; t++) {
                const uint32_t v = M.vars[t];
                Fr c;
                std::memcpy(c.l, cf + t, 32);
                if (v >= nv) { set_error("bb_r1cs_create: %s row %zu term %llu: variable %u of %zu", name[m], k, (unsigned long long)(t - M.row_offsets[k]), v, nv); return BB_ERR_ARG; }
                if (fr_geq_modulus(c.l)) { set_error("bb_r1cs_create: %s row %zu term %llu: coefficient not below r", name[m], k, (unsigned long long)(t - M.row_offsets[k])); return BB_ERR_ARG; }
                if (c.is_zero()) continue;                       // eval: a zero coefficient neither adds nor marks (prover.rs:31-44)
                if (v >= ni) {
                    if (m == 0) R->a_aux_density[(v - ni) >> 6] |= 1ull << ((v - ni) & 63);
                    if (m == 1) R->b_aux_density[(v - ni) >> 6] |= 1ull << ((v - ni) & 63);
                } else if (m == 1) {
                    R->b_input_density[v >> 6] |= 1ull << (v & 63);
                }
                const bool unit = c == one;
                idx.push_back(v | (unit ? ONE_FLAG : 0u));
                coef.push_back(c);
                R->unit[m] += unit;
            }
            bin(g, idx.size() - off[g]);
        }
        for (size_t i = 0; i < ni; i++) {                        // x_i * 0 = 0 for every input (prover.rs:208-215)
            const uint32_t g = (uint32_t)(m * n + rows + i);
            off[g] = (uint32_t)idx.size();
            if (m == 0) { idx.push_back((uint32_t)i | ONE_FLAG); coef.push_back(one); R->unit[0]++; }
            bin(g, idx.size() - off[g]);
        }
        R->nnz[m] = idx.size() - off[(size_t)m * n];
        for (int b = 0; b < 3; b++) {                            // this matrix's run in each bin: what the bin gained since the last matrix
            uint32_t before = 0;
            for (int q = 0; q < m; q++) before += R->bin_rows[b][q];
            R->bin_rows[b][m] = (uint32_t)rbins[b].size() - before;
        }
    }
    off[3 * n] = (uint32_t)idx.size();
    R->n_short = (uint32_t)rbins[0].size(); R->n_warp = (uint32_t)rbins[1].size(); R->n_cta = (uint32_t)rbins[2].size();
    std::vector<uint32_t> order;
    order.reserve(3 * n);
    for (auto& b : rbins) order.insert(order.end(), b.begin(), b.end());
    BB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->main_stream;
    StageTimer tm(ctx, st);
    tm.mark("r1cs.begin");
    BB_TRY(ctx->alloc(off.size() * 4, &R->d_off));
    BB_TRY(ctx->alloc((idx.size() ? idx.size() : 1) * 4, &R->d_idx));
    BB_TRY(ctx->alloc((coef.size() ? coef.size() : 1) * 32, &R->d_coef));
    BB_TRY(ctx->alloc(order.size() * 4, &R->d_rows));
    BB_CUDA(cudaMemcpyAsync(R->d_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice, st));
    if (idx.size()) BB_CUDA(cudaMemcpyAsync(R->d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, st));
    if (coef.size()) BB_CUDA(cudaMemcpyAsync(R->d_coef, coef.data(), coef.size() * 32, cudaMemcpyHostToDevice, st));
    BB_CUDA(cudaMemcpyAsync(R->d_rows, order.data(), order.size() * 4, cudaMemcpyHostToDevice, st));
    tm.mark("r1cs.upload");
    BB_CUDA(cudaStreamSynchronize(st));                           // the host vectors go out of scope
    tm.report(idx.size());
    *out = R.release();
    return BB_OK;
}

void bb_r1cs_destroy(bb_r1cs* r) { delete r; }

int bb_r1cs_info(const bb_r1cs* R, uint64_t* shape, uint64_t* a_aux_density, uint64_t* b_input_density, uint64_t* b_aux_density) {
    if (!R || !shape) { set_error("bb_r1cs_info: null argument"); return BB_ERR_ARG; }
    const uint64_t s[BB_R1CS_SHAPE_WORDS] = {R->n, R->n_inputs, R->n_aux, R->nnz[0], R->nnz[1], R->nnz[2], R->unit[0], R->unit[1], R->unit[2]};
    std::memcpy(shape, s, sizeof s);
    const size_t aux_words = (R->n_aux + 63) / 64, in_words = (R->n_inputs + 63) / 64;
    if (a_aux_density) std::memcpy(a_aux_density, R->a_aux_density.data(), aux_words * 8);
    if (b_input_density) std::memcpy(b_input_density, R->b_input_density.data(), in_words * 8);
    if (b_aux_density) std::memcpy(b_aux_density, R->b_aux_density.data(), aux_words * 8);
    return BB_OK;
}

int bb_r1cs_eval(bb_ctx* ctx, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux, size_t n_aux, int in_on_device,
                 void* a, void* b, void* c, int out_on_device) {
    if (!ctx || !R || !a || !b || !c) { set_error("bb_r1cs_eval: null argument"); return BB_ERR_ARG; }
    BB_TRY(check_witness("bb_r1cs_eval", ctx, R, input, n_inputs, aux, n_aux, in_on_device,
                         !out_on_device || (aligned16(a) && aligned16(b) && aligned16(c))));
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("r1cs_eval");
    cudaStream_t st = ctx->main_stream;
    const size_t n = R->n;
    StageTimer tm(ctx, st);
    tm.mark("r1cs.begin");
    DevBuf up[2], d_out;
    const Fr *d_in, *d_aux;
    BB_TRY(stage_witness(ctx, st, input, n_inputs, aux, n_aux, in_on_device, up, &d_in, &d_aux));
    tm.mark("r1cs.upload");
    Fr *oa = (Fr*)a, *ob = (Fr*)b, *oc = (Fr*)c;
    if (!out_on_device) {
        BB_TRY(d_out.alloc(ctx, 3 * n * 32));
        oa = d_out.as<Fr>(); ob = oa + n; oc = ob + n;
    }
    BB_TRY(r1cs_eval_queue(ctx, st, R, d_in, d_aux, oa, ob, oc));
    tm.mark("r1cs.eval");
    if (!out_on_device) {
        BB_CUDA(cudaMemcpyAsync(a, oa, n * 32, cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(b, ob, n * 32, cudaMemcpyDeviceToHost, st));
        BB_CUDA(cudaMemcpyAsync(c, oc, n * 32, cudaMemcpyDeviceToHost, st));
        ctx->d2h_bytes += 3 * n * 32;
    }
    tm.mark("r1cs.download");
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(R->nnz[0] + R->nnz[1] + R->nnz[2]);
    return BB_OK;
}

int bb_groth16_prove_r1cs(bb_ctx* ctx, const bb_crs* crs, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux,
                          size_t n_aux, int on_device, const uint8_t r[32], const uint8_t s[32], uint8_t proof[192]) {
    if (!ctx || !crs || !R || !r || !s || !proof) { set_error("bb_groth16_prove_r1cs: null argument"); return BB_ERR_ARG; }
    BB_TRY(check_witness("bb_groth16_prove_r1cs", ctx, R, input, n_inputs, aux, n_aux, on_device, true));
    if (crs_view(crs).shard_count != 1) { set_error("bb_groth16_prove needs an unsharded CRS; use prove_partials + finalize"); return BB_ERR_ARG; }
    NvtxRange nvtx("prove_r1cs");
    // create_proof from here on (prover.rs:217-360): the H pipeline evaluates a, b, c on its own stream after the upload,
    // the witness MSMs do not wait for the evaluation
    const bb_witness w = r1cs_witness(R, input, aux, on_device);
    const R1csStart start = r1cs_replicated(ctx, R);
    return prove_single(ctx, crs, [&](bb_prove** P) { return prove_begin_r1cs(ctx, crs, &w, start, P); }, r, s, proof);
}

int bb_groth16_prove_r1cs_begin(bb_ctx* ctx, const bb_crs* crs, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux,
                                size_t n_aux, int on_device, unsigned own, void* const d_evals[3], bb_prove** out) {
    static const char* const fn = "bb_groth16_prove_r1cs_begin";
    if (out) *out = nullptr;
    if (!ctx || !crs || !R || !out) { set_error("%s: null argument", fn); return BB_ERR_ARG; }
    if (crs_view(crs).ctx != ctx) { set_error("%s: the key lives on another context", fn); return BB_ERR_ARG; }
    BB_TRY(check_witness(fn, ctx, R, input, n_inputs, aux, n_aux, on_device, true));
    if (own > 7) { set_error("%s: own = %u: bits 0, 1, 2 are a, b, c", fn, own); return BB_ERR_ARG; }
    if (own && !d_evals) { set_error("%s: own = %u without evaluation vectors", fn, own); return BB_ERR_ARG; }
    for (int i = 0; i < 3; i++)
        if ((own >> i & 1) && (!d_evals[i] || !aligned16(d_evals[i]))) {
            set_error("%s: evaluation vector %c is %s", fn, "abc"[i], d_evals[i] ? "not 16-byte aligned" : "null");
            return BB_ERR_ARG;
        }
    BB_CUDA(cudaSetDevice(ctx->device));
    NvtxRange nvtx("prove_r1cs_begin");
    const bb_witness w = r1cs_witness(R, input, aux, on_device);
    R1csStart start = d_evals ? R1csStart{true, {}, {}, 0} : r1cs_replicated(ctx, R);
    if (own) {
        size_t m;
        uint32_t log_m;
        BB_TRY(domain_size(R->n, &m, &log_m));
        start.head = [=](cudaStream_t st, const Fr* d_in, const Fr* d_aux, Fr* tmp, StageTimer& tm) -> int {
            for (int i = 0; i < 3; i++)
                if (own >> i & 1) BB_TRY(r1cs_owner_queue(ctx, st, R, i, d_in, d_aux, (Fr*)d_evals[i], m, log_m, tmp, tm));
            return BB_OK;
        };
    }
    return prove_begin_r1cs(ctx, crs, &w, start, out);
}

// bb_groth16_prove_batch with the evaluation as its fill: each sub-batch uploads its witnesses once and evaluates every
// item's a, b, c straight into the rows its H pipeline transforms
int bb_groth16_prove_r1cs_batch(bb_ctx* ctx, const bb_crs* crs, const bb_r1cs* R, const void* inputs, size_t n_inputs, const void* aux,
                                size_t n_aux, size_t count, int on_device, const uint8_t* r, const uint8_t* s, uint8_t* proofs, int* status) {
    if (!R) { set_error("bb_groth16_prove_r1cs_batch: null argument"); return BB_ERR_ARG; }
    if (!count) return prove_batch_impl(ctx, crs, nullptr, 0, r, s, proofs, status);
    BB_TRY(check_witness("bb_groth16_prove_r1cs_batch", ctx, R, inputs, n_inputs, aux, n_aux, on_device, true));
    const size_t n = R->n;
    std::vector<bb_witness> ws(count);
    for (size_t i = 0; i < count; i++) {
        bb_witness& w = ws[i];
        w.n_constraints = n; w.n_inputs = n_inputs; w.n_aux = n_aux;
        w.input_assignment = (const char*)inputs + i * n_inputs * 32;
        w.aux_assignment = n_aux ? (const char*)aux + i * n_aux * 32 : nullptr;
        w.a_aux_density = R->a_aux_density.data();
        w.b_input_density = R->b_input_density.data();
        w.b_aux_density = R->b_aux_density.data();
        w.on_device = on_device;
    }
    const BatchAbcFill fill = [&](cudaStream_t st, uint32_t B, Fr* abc, size_t m, const Fr* d_in, const Fr* d_aux) -> int {
        for (uint32_t i = 0; i < B; i++)
            BB_TRY(r1cs_eval_queue(ctx, st, R, d_in + (size_t)i * n_inputs, d_aux + (size_t)i * n_aux, abc + (size_t)i * m,
                                   abc + ((size_t)B + i) * m, abc + (2 * (size_t)B + i) * m));
        return BB_OK;
    };
    return prove_batch_impl(ctx, crs, ws.data(), count, r, s, proofs, status, &fill);
}

int bb_diag_r1cs_owner_stage(bb_ctx* ctx, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux, size_t n_aux,
                             int on_device, int poly, void* d_out) {
    if (!ctx || !R || !d_out || poly < 0 || poly > 2) { set_error("bb_diag_r1cs_owner_stage: bad argument"); return BB_ERR_ARG; }
    BB_TRY(check_witness("bb_diag_r1cs_owner_stage", ctx, R, input, n_inputs, aux, n_aux, on_device, aligned16(d_out)));
    BB_CUDA(cudaSetDevice(ctx->device));
    size_t m;
    uint32_t log_m;
    BB_TRY(domain_size(R->n, &m, &log_m));
    cudaStream_t st = ctx->main_stream;
    StageTimer tm(ctx, st);
    tm.mark("r1cs_owner.begin");
    DevBuf up[2], tmp;
    const Fr *d_in, *d_aux;
    BB_TRY(stage_witness(ctx, st, input, n_inputs, aux, n_aux, on_device, up, &d_in, &d_aux));
    tm.mark("r1cs_owner.upload", 0);
    BB_TRY(tmp.alloc(ctx, m * 32));
    BB_TRY(r1cs_owner_queue(ctx, st, R, poly, d_in, d_aux, (Fr*)d_out, m, log_m, tmp.as<Fr>(), tm));
    BB_CUDA(cudaStreamSynchronize(st));
    tm.report(0);
    return BB_OK;
}

int bb_r1cs_check(bb_ctx* ctx, const bb_r1cs* R, const void* input, size_t n_inputs, const void* aux, size_t n_aux, int on_device,
                  size_t* first, size_t* count, uint64_t* unsat_bits) {
    if (!ctx || !R || !first || !count) { set_error("bb_r1cs_check: null argument"); return BB_ERR_ARG; }
    BB_TRY(check_witness("bb_r1cs_check", ctx, R, input, n_inputs, aux, n_aux, on_device, true));
    return r1cs_check_run(ctx, R, input, aux, 1, on_device, first, count, unsat_bits);
}

int bb_r1cs_check_batch(bb_ctx* ctx, const bb_r1cs* R, const void* inputs, size_t n_inputs, const void* aux, size_t n_aux, size_t count,
                        int on_device, size_t* first, size_t* n_unsat) {
    if (!ctx || !R) { set_error("bb_r1cs_check_batch: null argument"); return BB_ERR_ARG; }
    if (!count) return BB_OK;
    if (!first) { set_error("bb_r1cs_check_batch: null argument"); return BB_ERR_ARG; }
    BB_TRY(check_witness("bb_r1cs_check_batch", ctx, R, inputs, n_inputs, aux, n_aux, on_device, true));
    return r1cs_check_run(ctx, R, inputs, aux, count, on_device, first, n_unsat, nullptr);
}

}  // extern "C"
