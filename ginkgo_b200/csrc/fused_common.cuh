// What the fused device-resident solvers (fused_cg.cu, fused_bicgstab.cu, fused_gmres.cu) share: the
// shape of their step kernels, the grid-wide sums and the stopping check their last CTA runs.
#pragma once
#include "common.cuh"

namespace b200 {
namespace fused {

constexpr int kThreads = 512;

// the reference's criteria (core/stop/combined.cpp:33-52), evaluated by ONE thread: Iteration (ctl[2],
// -1 = none) and a residual norm (ctl[3], 0 = none) in the user's order (ctl[4]) with ids 1 and 2.
// Returns the stopping status of iteration `iter`, 0 while running; converged(res_kind) says whether the
// residual criterion holds and is evaluated only where it is checked; `finalized` is OR-ed into a stop.
template <typename Converged>
__device__ __forceinline__ uint8_t criteria_status(int32_t iter, const int32_t* ctl, Converged converged,
                                                   uint8_t finalized)
{
    const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];
    const bool has_it = max_iters >= 0, has_res = res_kind != 0;
    uint8_t status = 0;
    uint8_t id = 1;
    for (int k = 0; k < 2 && status == 0; ++k) {
        const bool is_it = (k == 0) == (iter_first != 0);
        if (is_it) {
            if (!has_it) continue;
            if (iter >= max_iters) status = (id & kIdMask) | finalized;
            ++id;
        } else {
            if (!has_res) continue;
            if (converged(res_kind)) status = kConvergedMask | (id & kIdMask) | finalized;
            ++id;
        }
    }
    return status;
}

// the top-of-iteration check of the fused CG / BiCGStab: rho and ||r||^2 shifted into sc, the iteration
// counted, the status (finalized) into ctl[0]
template <typename V>
__device__ void finish_scalars(V rho_new, V rr, V* sc, int32_t* ctl)
{
    sc[1] = sc[0];
    sc[0] = rho_new;
    sc[3] = rr;
    const int32_t iter = ctl[1] + 1;
    ctl[1] = iter;
    ctl[0] = criteria_status(
        iter, ctl,
        [&](int32_t res_kind) {
            const V tau = res_kind == 1 ? sqrt(rr) : sqrt(fabs(rho_new));
            return tau <= sc[5];
        },
        kFinalizedMask);
}

// K sums of one value per thread over the grid: per-CTA partials, a ticket, and the CTA that arrives last
// adds the partials in a fixed order.  Returns true in that CTA only, whose thread 0 then holds the sums
// in a[]; the ticket is back at 0.
template <typename V, int K>
__device__ __forceinline__ bool grid_sums(V (&a)[K], V* __restrict__ partials, unsigned int* counter, V* red,
                                          bool* is_last)
{
    const int tid = threadIdx.x;
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] = block_sum(a[k], red);
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) partials[K * blockIdx.x + k] = a[k];
        __threadfence();
        const unsigned int ticket = atomicAdd(counter, 1u);
        *is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!*is_last) return false;
    __threadfence();
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] = V(0);
    for (int c = tid; c < (int)gridDim.x; c += kThreads)
#pragma unroll
        for (int k = 0; k < K; ++k) a[k] += __ldcg(partials + K * c + k);
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] = block_sum(a[k], red);
    if (tid == 0) *counter = 0u;
    return true;
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
