// What the fused device-resident solvers (fused_cg.cu, fused_bicgstab.cu) share: the shape of their
// step kernels and the stopping check their last CTA runs.
#pragma once
#include "common.cuh"

namespace b200 {
namespace fused {

constexpr int kThreads = 512;

// the reference's criteria, evaluated by ONE thread (core/stop/combined.cpp:33-52)
template <typename V>
__device__ void finish_scalars(V rho_new, V rr, V* sc, int32_t* ctl)
{
    sc[1] = sc[0];
    sc[0] = rho_new;
    sc[3] = rr;
    const int32_t iter = ctl[1] + 1;
    ctl[1] = iter;
    const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];
    const bool has_it = max_iters >= 0, has_res = res_kind != 0;
    uint8_t status = 0;
    uint8_t id = 1;
    for (int k = 0; k < 2 && status == 0; ++k) {
        const bool is_it = (k == 0) == (iter_first != 0);
        if (is_it) {
            if (!has_it) continue;
            if (iter >= max_iters) status = (id & kIdMask) | kFinalizedMask;
            ++id;
        } else {
            if (!has_res) continue;
            const V tau = res_kind == 1 ? sqrt(rr) : sqrt(fabs(rho_new));
            if (tau <= sc[5]) status = kConvergedMask | (id & kIdMask) | kFinalizedMask;
            ++id;
        }
    }
    ctl[0] = status;
}

inline int ew_grid(const b200_ctx* ctx, int64_t n)
{
    int64_t g = ceildiv(n, kThreads * 4);
    const int64_t cap = (int64_t)ctx->num_sms * 4;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace fused
}  // namespace b200
