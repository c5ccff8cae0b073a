// Fused BiCGStab iteration for sm_90a: rho / alpha / beta / gamma / omega are produced AND consumed on
// the device, five launches per iteration, no host round trip.
//
// The reference drives BiCGStab from the host with about 16 launches and two blocking device->host
// reads of the stopping flags per iteration (core/solver/bicgstab.cpp:95-233: dot, criterion check,
// step_1, preconditioner, SpMV, dot, step_2, norm, criterion check, finalize, preconditioner, SpMV,
// two dots, step_3).  The same recurrence, regrouped around its three global reductions (d is the
// inverted diagonal of a scalar Jacobi preconditioner, or absent):
//
//   step_p     p = r + tmp (p - omega v), tmp = rho/prev_rho*alpha/omega; y = d.p     reads 4n, writes 2n
//   spmv_dot2  v = A y  and  beta = rr.v   (SpMV epilogue)                            matrix + 3n
//   step_s     alpha = rho/beta; s = r - alpha v; z = d.s; ||s||^2; mid check         reads 3n, writes 2n
//   spmv_dot2  t = A z,  gamma = s.t  and  beta = t.t   (SpMV epilogue)               matrix + 3n
//   step_xr    omega = gamma/beta; x += alpha y + omega z; r = s - omega t;
//              rho' = rr.r; ||r||^2; swap rho / prev_rho; top-of-iteration check      reads 6n, writes 2n
//
// = 2 matrix + 25 n values per iteration (Identity preconditioner: 23 n, d is not read), against 36 n for
// the reference's kernel sequence.  Element-wise arithmetic is the reference's, operation for operation
// (reference/solver/bicgstab_kernels.cpp:63-170), so given the same scalars p, y, s, z, x, r are the bits
// of bicgstab::step_1/2/3 + the scalar Jacobi apply.
//
// Stopping is the reference's: Iteration and (Implicit)ResidualNorm in the user's order with ids 1 and 2
// (fused_common.cuh), at the top of the iteration on r (step_xr's last CTA) and again in mid-iteration on
// s with the same iteration number (step_s's last CTA).  A stop at the mid check owes x the update of
// bicgstab::finalize, x += alpha y: step_s writes the status into ctl[0], which turns the second SpMV
// into a no-op, and raises ctl[5]; step_xr of the same iteration, seeing ctl[5], does only x += alpha y
// and clears it.  step_xr always follows step_s in an iteration, so x is final before a host that polls
// ctl between iterations can see the stop.  Once stopped and finalized every kernel is a no-op.
//
// Scalars  sc[16]: 0 rho, 1 prev_rho, 2 beta (rr.v, then t.t), 3 ||r||^2, 4 tau0 (baseline norm),
//                  5 threshold = reduction_factor * tau0, 6 alpha, 7 omega, 8 gamma, 9 ||s||^2
// Control  ctl[0..4] of fused_common.cuh; 5 finalize pending (x += alpha y still owed after a stop at the
//                  mid check), 6..7 unused
#include "csr_launch.cuh"
#include "fused_common.cuh"

namespace b200 {
namespace fbicgstab {

using namespace fused;  // kThreads, grid_sums, residual_status, finish_scalars, set_threshold, ew_grid

template <typename V>
__global__ void __launch_bounds__(kThreads)
    step_p_kernel(int64_t n, V* __restrict__ p, const V* __restrict__ r, const V* __restrict__ v,
                  V* __restrict__ y, const V* __restrict__ inv_diag, const V* __restrict__ sc,
                  const int32_t* __restrict__ ctl)
{
    if (ctl[0] != 0) return;
    const V rho = sc[0], prev = sc[1], alpha = sc[6], omega = sc[7];
    const bool plain = !(prev * omega != V(0));
    const V tmp = plain ? V(0) : rho / prev * alpha / omega;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * kThreads) {
        const V ri = r[i];
        const V pi = plain ? ri : ri + tmp * (p[i] - omega * v[i]);
        p[i] = pi;
        y[i] = inv_diag ? pi * inv_diag[i] : pi;
    }
}

// the mid-iteration check on s (core/solver/bicgstab.cpp:170-186), by ONE thread: the criteria of
// finish_scalars with the iteration number and rho of the top check and ||s|| as the residual norm
template <typename V>
__device__ void mid_check(V ss, const V* sc, int32_t* ctl)
{
    const uint8_t status = residual_status(ctl[1], ctl, ss, sc[0], sc[5], kFinalizedMask);
    if (status != 0) {
        ctl[0] = status;
        ctl[5] = 1;  // bicgstab::finalize is owed: step_xr pays it
    }
}

template <typename V>
__global__ void __launch_bounds__(kThreads)
    step_s_kernel(int64_t n, const V* __restrict__ r, const V* __restrict__ v, V* __restrict__ s,
                  V* __restrict__ z, const V* __restrict__ inv_diag, V* __restrict__ sc,
                  int32_t* __restrict__ ctl, V* __restrict__ partials, unsigned int* __restrict__ counter)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    const V beta = sc[2];
    const bool update = beta != V(0);
    const V alpha = update ? sc[0] / beta : V(0);
    V a[1] = {V(0)};
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * kThreads) {
        const V ri = r[i];
        const V si = update ? ri - alpha * v[i] : ri;
        s[i] = si;
        z[i] = inv_diag ? si * inv_diag[i] : si;
        a[0] += si * si;
    }
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (threadIdx.x == 0) {
        sc[6] = alpha;
        sc[9] = a[0];
        mid_check(a[0], sc, ctl);
    }
}

// INIT: r already holds b - A x; sets rr = r and computes rho = rr.r, ||r||^2 and the baseline.
template <typename V, bool INIT>
__global__ void __launch_bounds__(kThreads)
    step_xr_kernel(int64_t n, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ s,
                   const V* __restrict__ t, const V* __restrict__ y, const V* __restrict__ z,
                   V* __restrict__ rr, V* __restrict__ sc, int32_t* __restrict__ ctl,
                   V* __restrict__ partials, unsigned int* __restrict__ counter, int baseline, V factor)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    const int tid = threadIdx.x;
    const bool pending = !INIT && ctl[5] != 0;
    if (!INIT && !pending && ctl[0] != 0) return;
    V a[2] = {V(0), V(0)};
    if (pending) {
        // bicgstab::finalize after a stop at the mid check (reference/solver/bicgstab_kernels.cpp:155-170)
        const V alpha = sc[6];
        for (int64_t i = blockIdx.x * (int64_t)kThreads + tid; i < n; i += (int64_t)gridDim.x * kThreads)
            x[i] += alpha * y[i];
    } else {
        const V beta = sc[2];
        const V omega = INIT ? V(0) : (beta != V(0) ? sc[8] / beta : V(0));
        const V alpha = INIT ? V(0) : sc[6];
        for (int64_t i = blockIdx.x * (int64_t)kThreads + tid; i < n; i += (int64_t)gridDim.x * kThreads) {
            V ri, rri;
            if (INIT) {
                ri = r[i];
                rri = ri;
                rr[i] = ri;
            } else {
                x[i] += alpha * y[i] + omega * z[i];
                ri = s[i] - omega * t[i];
                r[i] = ri;
                rri = rr[i];
            }
            a[0] += rri * ri;
            a[1] += ri * ri;
        }
    }
    // every CTA read ctl[5] and the scalars before it took its ticket: the last one may write them
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (tid == 0) {
        if (pending) {
            ctl[5] = 0;
            return;
        }
        if (INIT) {
            set_threshold(baseline, sqrt(a[1]), sc + 4, sc + 5, factor);
        } else {
            sc[7] = sc[2] != V(0) ? sc[8] / sc[2] : V(0);
        }
        finish_scalars(a[0], a[1], sc, ctl);
    }
}

template <typename V>
__global__ void init_scalars_kernel(V* sc, int32_t* ctl, int32_t max_iters, int32_t res_kind,
                                    int32_t iter_first)
{
    // rho = prev_rho = alpha = beta = gamma = omega = 1 (reference bicgstab::initialize); the INIT
    // finish moves rho to prev_rho
    sc[0] = V(1);
    sc[1] = V(1);
    sc[2] = V(1);
    sc[3] = V(0);
    sc[6] = V(1);
    sc[7] = V(1);
    sc[8] = V(1);
    sc[9] = V(0);
    start_control(ctl, max_iters, res_kind, iter_first, -1);  // the INIT finish counts to 0
    ctl[5] = 0;
}

}  // namespace fbicgstab
}  // namespace b200

extern "C" {

#define B200_DEF_FBICGSTAB(V, VT)                                                                 \
    b200_status b200_bicgstab_fused_init_##V(                                                     \
        b200_ctx* ctx, int64_t n, const VT* r, VT* rr, VT* p, VT* v, VT* y, VT* s, VT* t, VT* z,  \
        VT* sc, int32_t* ctl, VT* work, int64_t max_iters, int32_t res_kind, int32_t iter_first,  \
        int32_t baseline, VT reduction_factor)                                                    \
    {                                                                                             \
        B200_REQUIRE(ctx && sc && ctl && work, "null argument");                                  \
        b200::fbicgstab::init_scalars_kernel<VT><<<1, 1, 0, ctx->stream>>>(                       \
            sc, ctl, b200::fused::clamp_iters(max_iters), res_kind, iter_first);                  \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        VT* zeroed[6] = {p, v, y, s, t, z};                                                       \
        for (VT * a : zeroed) B200_CUDA_CHECK(cudaMemsetAsync(a, 0, sizeof(VT) * n, ctx->stream)); \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fbicgstab::step_xr_kernel<VT, true><<<grid, b200::fused::kThreads, 0, ctx->stream>>>( \
            n, nullptr, const_cast<VT*>(r), nullptr, nullptr, nullptr, nullptr, rr, sc, ctl,      \
            b200::fused::step_partials(ctx, work), ctx->counters + b200::kStepCounter, baseline,  \
            reduction_factor);                                                                    \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_bicgstab_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* r,      \
                                               const VT* v, VT* y, const VT* inv_diag,            \
                                               const VT* sc, const int32_t* ctl)                  \
    {                                                                                             \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fbicgstab::step_p_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(      \
            n, p, r, v, y, inv_diag, sc, ctl);                                                    \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_bicgstab_fused_step_s_##V(b200_ctx* ctx, int64_t n, const VT* r,             \
                                               const VT* v, VT* s, VT* z, const VT* inv_diag,     \
                                               VT* sc, int32_t* ctl, VT* work)                    \
    {                                                                                             \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fbicgstab::step_s_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(      \
            n, r, v, s, z, inv_diag, sc, ctl, b200::fused::step_partials(ctx, work),              \
            ctx->counters + b200::kStepCounter);                                                  \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_bicgstab_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r,           \
                                                const VT* s, const VT* t, const VT* y,            \
                                                const VT* z, const VT* rr, VT* sc, int32_t* ctl,  \
                                                VT* work)                                         \
    {                                                                                             \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fbicgstab::step_xr_kernel<VT, false><<<grid, b200::fused::kThreads, 0,              \
                                                     ctx->stream>>>(                              \
            n, x, r, s, t, y, z, const_cast<VT*>(rr), sc, ctl,                                    \
            b200::fused::step_partials(ctx, work), ctx->counters + b200::kStepCounter, 0, VT(0)); \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }

B200_DEF_FBICGSTAB(f64, double)
B200_DEF_FBICGSTAB(f32, float)

/* c = A b, *dot_out = w . c and (dot2_out != NULL) *dot2_out = c . c in one launch; w has one     */
/* entry per row.  `work` and `ctl` as for b200_csr_spmv_dot_*.  With num_rows == 0 both are 0.    */
#define B200_DEF_SPMV_DOT2(V, VT, I, IT)                                                          \
    b200_status b200_csr_spmv_dot2_##V##_##I(                                                     \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,             \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,       \
        VT* c, const VT* w, VT* dot_out, VT* dot2_out, VT* work, const int32_t* ctl)              \
    {                                                                                             \
        return b200::csr::launch_spmv_dot<VT, IT, false, b200::csr::kDotW2>(                      \
            ctx, plan, num_rows, nnz, row_ptrs, col_idxs, values, nullptr, b, nullptr, c, w,      \
            dot_out, dot2_out, work, ctl);                                                        \
    }

B200_DEF_SPMV_DOT2(f64, double, i32, int32_t)
B200_DEF_SPMV_DOT2(f64, double, i64, int64_t)
B200_DEF_SPMV_DOT2(f32, float, i32, int32_t)
B200_DEF_SPMV_DOT2(f32, float, i64, int64_t)

}  // extern "C"
