// bellman_b200 internal: 32 x 255 tables of byte multiples of a fixed base, for scalar multiplications by at most 32
// mixed additions (bb_fixed_base_mul in capi.cu, the Psi_i of bb_groth16_verify_each in verify.cu).
#pragma once
#include "bb_internal.cuh"

namespace bb {

// table[w*255 + d-1] = d * 2^(8w) * G, affine
template <class F>
struct FixedTable {
    Affine<F>* d_table = nullptr;
};

template <class F>
inline void batch_to_affine_host(const std::vector<XYZZ<F>>& in, std::vector<Affine<F>>& out) {
    size_t n = in.size();
    out.resize(n);
    std::vector<F> pre(n);
    F acc = FieldOps<F>::one();
    for (size_t i = 0; i < n; i++) { pre[i] = acc; acc = acc * in[i].ZZZ; }       // no identities in the table
    F inv = FieldOps<F>::inv(acc);
    for (size_t i = n; i-- > 0;) {
        F zi3 = inv * pre[i];
        inv = inv * in[i].ZZZ;
        F zi2 = (zi3 * in[i].ZZ).sqr();
        out[i] = {in[i].X * zi2, in[i].Y * zi3};
    }
}

// gen must not be the identity.  The table is cudaMalloc'ed: the owner frees t.d_table with cudaFree.
template <class F>
inline int build_fixed_table(FixedTable<F>& t, const Affine<F>& gen) {
    if (t.d_table) return BB_OK;
    std::vector<XYZZ<F>> pts(32 * 255);
    XYZZ<F> base = XYZZ<F>::from_affine(gen);
    for (int w = 0; w < 32; w++) {
        XYZZ<F> cur = base;
        for (int d = 1; d <= 255; d++) { pts[w * 255 + d - 1] = cur; cur.add(base); }
        base = cur;
    }
    std::vector<Affine<F>> aff;
    batch_to_affine_host(pts, aff);
    BB_CUDA(cudaMalloc(&t.d_table, aff.size() * sizeof(Affine<F>)));
    BB_CUDA(cudaMemcpy(t.d_table, aff.data(), aff.size() * sizeof(Affine<F>), cudaMemcpyHostToDevice));
    return BB_OK;
}

}  // namespace bb
