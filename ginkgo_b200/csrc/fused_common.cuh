// What the seven fused device-resident paths share (fused_{cg,bicgstab,gmres}.cu, their k-column twins
// fused_{cg,bicgstab,gmres}_mrhs.cu through fused_mrhs.cuh, and fused_minres.cu): the control block and its
// start, the stopping check their last CTA runs, the grid-wide ticket, the grid-wide sums of the one-column
// step kernels and the one-column workspace.
//
// Control  ctl[8] (int32), on the device, polled by the host between batches of iterations:
//   0 the stopping_status byte (one column; 0 = running), or nonzero once EVERY column has stopped (k
//     columns, whose bytes are in status[k]).  Once ctl[0] != 0 every kernel is a no-op (BiCGStab: except
//     the step_xr that pays a pending finalize), so a graph of several iterations can be replayed past
//     the stop.
//   1 iterations done, 2 max_iters (-1 none), 3 res_kind (0 none, 1 ResidualNorm, 2 ImplicitResidualNorm),
//   4 iter_first (Iteration is the first criterion)
//   5..7 the path's own; each file header says what it keeps there
#pragma once
#include "common.cuh"

namespace b200 {
namespace fused {

constexpr int kThreads = 512;

// ctl[0..4] at the start of a solve: running, `first_iter` iterations done (-1 when the first check
// counts itself to 0), and the criteria
__device__ __forceinline__ void start_control(int32_t* ctl, int32_t max_iters, int32_t res_kind,
                                              int32_t iter_first, int32_t first_iter)
{
    ctl[0] = 0;
    ctl[1] = first_iter;
    ctl[2] = max_iters;
    ctl[3] = res_kind;
    ctl[4] = iter_first;
}

// max_iters as ctl[2] holds it: negative for none, larger counts saturate
inline int32_t clamp_iters(int64_t max_iters)
{
    return (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);
}

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

// criteria_status of CG and BiCGStab: the residual norm is ||r|| = sqrt(rr) for ResidualNorm and
// sqrt|rho| for ImplicitResidualNorm, converged at tau <= threshold.  rho and threshold are read only
// where the residual criterion is checked.
template <typename V>
__device__ __forceinline__ uint8_t residual_status(int32_t iter, const int32_t* ctl, V rr, const V& rho,
                                                   const V& threshold, uint8_t finalized)
{
    return criteria_status(
        iter, ctl,
        [&](int32_t res_kind) {
            const V tau = res_kind == 1 ? sqrt(rr) : sqrt(fabs(rho));
            return tau <= threshold;
        },
        finalized);
}

// the top-of-iteration check of CG and BiCGStab on column c of k (sc[s*k + c]; one column: k = 1, c = 0):
// rho shifted into prev_rho (s = 0 -> 1), ||r||^2 into s = 3, iteration `iter` checked against the
// threshold in s = 5 (finalized).  Returns the status; the caller stores it.
template <typename V>
__device__ __forceinline__ uint8_t top_check(int32_t iter, const int32_t* ctl, V rho_new, V rr, V* sc, int64_t k,
                                             int c)
{
    sc[k + c] = sc[c];
    sc[c] = rho_new;
    sc[3 * k + c] = rr;
    return residual_status(iter, ctl, rr, rho_new, sc[5 * k + c], kFinalizedMask);
}

// top_check of the one-column CG / BiCGStab: the iteration counted, the status into ctl[0]
template <typename V>
__device__ void finish_scalars(V rho_new, V rr, V* sc, int32_t* ctl)
{
    const int32_t iter = ctl[1] + 1;
    ctl[1] = iter;
    ctl[0] = top_check(iter, ctl, rho_new, rr, sc, 1, 0);
}

// the baseline norm tau0 of the residual criterion and its threshold = factor * tau0: baseline 0 keeps
// *tau0 (rhs_norm, ||b|| preset by the host), 1 takes the measured initial residual norm
// (initial_resnorm), 2 is absolute
template <typename V>
__device__ __forceinline__ void set_threshold(int baseline, const V& measured, V* tau0, V* threshold, V factor)
{
    if (baseline == 1) *tau0 = measured;
    if (baseline == 2) *tau0 = V(1);
    *threshold = factor * *tau0;
}

// The ticket of a grid-wide reduction, taken by every thread of every CTA.  Before it, whoever wrote the
// CTA's partials has fenced them, and the CTA has read ctl and the scalars that the last CTA may then
// overwrite.  Thread 0 takes a ticket; returns true, after a barrier, in the CTA that took the last one.
// That CTA fences before it reads the partials and resets *counter to 0 after them.
__device__ __forceinline__ bool last_ticket(unsigned int* counter, bool* is_last)
{
    if (threadIdx.x == 0) {
        const unsigned int ticket = atomicAdd(counter, 1u);
        *is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    return *is_last;
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
    }
    if (!last_ticket(counter, is_last)) return false;
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

// ew_grid's cap on the CTAs of a one-column step kernel, and the bound on those of the SpMV + dot
// (csr::max_grid_size)
inline int64_t max_ctas(const b200_ctx* ctx) { return (int64_t)ctx->num_sms * 4; }

inline int ew_grid(const b200_ctx* ctx, int64_t n)
{
    int64_t g = ceildiv(n, kThreads * 4);
    const int64_t cap = max_ctas(ctx);
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// The one-column workspace `work` (b200_{cg,minres}_fused_work_size elements): the SpMV + dot's per-CTA
// partials, then the step kernels' (2 per CTA), then 64 spare.  GMRES appends its multi-dot's partials
// (gmres_common.cuh).
template <typename V>
V* step_partials(const b200_ctx* ctx, V* work)
{
    return work + max_ctas(ctx);
}
inline int64_t work_size(const b200_ctx* ctx) { return max_ctas(ctx) + 2 * max_ctas(ctx) + 64; }

}  // namespace fused
}  // namespace b200
