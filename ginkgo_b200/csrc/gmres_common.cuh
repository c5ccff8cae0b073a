// What the GMRES loop kernels (gmres_kernels.cu) and the fused GMRES iteration (fused_gmres.cu) share:
// the Givens update of one Hessenberg column, and the workspace offset of the fused multi-dot (after the
// one-column workspace of fused_common.cuh).
#pragma once
#include "fused_common.cuh"

namespace b200 {
namespace gmres {

// workspace of the fused iteration (b200_gmres_fused_work_size): the one-column workspace of
// fused_common.cuh (the SpMV + dot's and the passes' partials), then those of the multi-dot, one per CTA
// and basis
constexpr int kFusedMdCtasPerSm = 4;
inline int64_t fused_md_offset(const b200_ctx* ctx) { return fused::work_size(ctx); }
inline int64_t fused_work_size(const b200_ctx* ctx, int64_t krylov_dim)
{
    return fused_md_offset(ctx) + (int64_t)ctx->num_sms * kFusedMdCtasPerSm * (krylov_dim + 1);
}

// Right-hand side i of hessenberg_qr (reference/solver/common_gmres_kernels.cpp): the `iter` stored
// Givens rotations applied to the new Hessenberg column, new (cos, sin) from a scaled hypot, and the
// residual-norm update |rnc[iter + 1]|.
template <typename V>
__device__ __forceinline__ void givens_column(int64_t i, V* gsin, int64_t sins, V* gcos, int64_t coss,
                                              V* residual_norm, V* rnc, int64_t rncs, V* hess, int64_t hs,
                                              int64_t iter, uint64_t* final_iter_nums)
{
    final_iter_nums[i]++;
    V hj = hess[i];
    for (int64_t j = 0; j < iter; ++j) {
        const V c = gcos[j * coss + i], s = gsin[j * sins + i];
        const V hj1 = hess[(j + 1) * hs + i];
        const V temp = c * hj + s * hj1;
        const V next = -s * hj + c * hj1;
        hess[j * hs + i] = temp;
        hj = next;
    }
    // hj == hessenberg(iter), as rotated so far
    const V this_hess = hj;
    const V next_hess = hess[(iter + 1) * hs + i];
    V c, s;
    if (this_hess == V(0)) {
        c = V(0);
        s = V(1);
    } else {
        const V scale = fabs(this_hess) + fabs(next_hess);
        const V a = fabs(this_hess / scale), bq = fabs(next_hess / scale);
        const V hyp = scale * sqrt(a * a + bq * bq);
        c = this_hess / hyp;
        s = next_hess / hyp;
    }
    gcos[iter * coss + i] = c;
    gsin[iter * sins + i] = s;
    hess[iter * hs + i] = c * this_hess + s * next_hess;
    hess[(iter + 1) * hs + i] = V(0);
    const V old = rnc[iter * rncs + i];
    const V nxt = -s * old;
    rnc[(iter + 1) * rncs + i] = nxt;
    rnc[iter * rncs + i] = c * old;
    residual_norm[i] = fabs(nxt);
}

}  // namespace gmres
}  // namespace b200
