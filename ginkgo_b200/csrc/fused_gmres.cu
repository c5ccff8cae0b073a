// Fused GMRES iteration for sm_90a: the Hessenberg column, the Givens rotations, the residual estimate and
// the stopping check stay on the device, no host round trip; modified Gram-Schmidt takes j + 3 launches at
// Krylov index j, classical Gram-Schmidt 4 and CGS2 6.
//
// The reference drives one MGS iteration from the host (core/solver/gmres.cpp:453-530): a blocking
// criterion check, the preconditioner, the SpMV, j + 1 dots and j + 1 sub_scaled, norm2, inv_scale and
// hessenberg_qr -- 2j + 7 launches.  The same recurrence, regrouped around its global reductions (w is
// the new Krylov vector, held in place in basis j + 1; h the Hessenberg column of iteration j; d the
// inverted diagonal of a scalar Jacobi preconditioner):
//
//   scale       v_j = w / h_j (the previous final pass's norm; j = 0 is scaled by init / restart);
//               z = d . v_j                                       reads 2n (d: 3n), writes n (d: 2n)
//   [block Jacobi: z = M v_j, b200_gmres_fused_block_apply]
//   spmv_dot2   w = A z (A v_j), h_0 = v_0 . w in the SpMV epilogue              matrix + 3n
//   pass i      w -= h_{i-1} v_{i-1}; h_i = v_i . w                     i = 1..j, 4n each
//   final       w -= h_j v_j; h_{j+1} = ||w||; the Givens update of hessenberg_qr; the criteria
//               checked on |rnc[j+1]| for the top of iteration j + 1              3n
//
// CGS: scale, spmv_dot2 (h_0), the CTL multi_dot of gmres_kernels.cu (h_1..h_j in one pass), and one final
// pass subtracting h_0 v_0, h_1 v_1, ... element by element in basis order (the loop's sequential
// sub_scaled) -- four launches whatever j is.  CGS2: a plain subtract pass, a second multi_dot over bases
// 0..j into haux, and the final pass subtracting with haux and adding haux into h (the loop's add_scaled).
//
// Element-wise arithmetic is the loop's operation for operation: sub_scaled's `w -= h v` (skipped for
// h == 0), inv_scale's division, the scalar Jacobi apply's product; the Givens update is the function
// the loop's hessenberg_qr kernel runs (gmres_common.cuh).  Dots and norms are per-CTA partials summed
// in CTA order by the CTA that takes the last ticket.
//
// Stopping is the reference's (core/solver/gmres.cpp:453): Iteration and ResidualNorm in the user's
// order with ids 1 and 2, WITHOUT the finalized bit (the final solve_krylov / multi_axpy set it).  The
// status goes into ctl[0] and into the solver's stop_status byte; once ctl[0] != 0 every kernel of the
// iteration is a no-op, so a graph of several iterations may be replayed past the stop.
//
// Scalars  sc[8]:  0 ||w|| of the last final pass (the divisor of the next scale), 1 tau0 (baseline
//                  norm), 2 threshold = reduction_factor * tau0
// Control  ctl[0..4] of fused_common.cuh (res_kind 0 or 1); 5..7 unused, cleared by init
#include "csr_launch.cuh"
#include "fused_common.cuh"
#include "gmres_common.cuh"

namespace b200 {
namespace fgmres {

using namespace fused;  // kThreads, criteria_status, start_control, grid_sums, ew_grid

// the criteria of fused_common.cuh on the GMRES residual estimate tau, by ONE thread, WITHOUT the
// finalized bit (core/solver/gmres.cpp:453 checks with set_finalized = false)
template <typename V>
__device__ void check(V tau, const V* sc, int32_t* ctl, uint8_t* stop)
{
    const int32_t iter = ctl[1] + 1;
    ctl[1] = iter;
    const uint8_t status = criteria_status(iter, ctl, [&](int32_t) { return tau <= sc[2]; }, uint8_t(0));
    if (status != 0) {
        stop[0] = status;
        ctl[0] = status;
    }
}

// rnorm holds ||b - A x|| (the loop's norm2), v_0, rnc[0], fin and the Givens arrays are set by the
// loop's initialize / restart kernels; sc[1] holds ||b|| for the rhs_norm baseline
template <typename V>
__global__ void init_kernel(const V* rnorm, V* sc, int32_t* ctl, uint8_t* stop, int32_t max_iters,
                            int32_t res_kind, int32_t iter_first, int32_t baseline, V factor)
{
    set_threshold(baseline, rnorm[0], sc + 1, sc + 2, factor);
    sc[0] = V(0);
    start_control(ctl, max_iters, res_kind, iter_first, -1);  // the check counts to 0
    ctl[5] = ctl[6] = ctl[7] = 0;
    stop[0] = 0;
    check(rnorm[0], sc, ctl, stop);
}

template <typename V>
__global__ void __launch_bounds__(kThreads)
    scale_kernel(int64_t n, V* __restrict__ v, V* __restrict__ z, const V* __restrict__ inv_diag,
                 const V* __restrict__ sc, const int32_t* __restrict__ ctl, bool divide)
{
    if (ctl[0] != 0) return;
    const V h = sc[0];
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        V vi = v[i];
        if (divide) {
            vi /= h;
            v[i] = vi;
        }
        if (inv_diag) z[i] = vi * inv_diag[i];
    }
}

// MGS pass i: w -= h[i-1] v_{i-1}; h[i] = v_i . w
template <typename V>
__global__ void __launch_bounds__(kThreads)
    mgs_pass_kernel(int64_t n, V* __restrict__ w, const V* __restrict__ v_prev, const V* __restrict__ v_i,
                    V* __restrict__ hcol, int64_t i, const int32_t* __restrict__ ctl, V* __restrict__ partials,
                    unsigned int* __restrict__ counter)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    const V h = hcol[i - 1];
    V a[1] = {V(0)};
    for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
        V wr = w[r];
        if (h != V(0)) wr -= h * v_prev[r];
        w[r] = wr;
        a[0] += v_i[r] * wr;
    }
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (threadIdx.x == 0) hcol[i] = a[0];
}

// subtract pass: w -= coef[i] v_i for i = first..j, element by element in basis order (each the rounding
// of one sub_scaled, skipped for coef[i] == 0).  FINAL: also ||w||; the last CTA adds haux[0..j] into the
// Hessenberg column (CGS2, the loop's add_scaled), sets h[j+1] = ||w||, runs the Givens update and the
// check for the top of iteration j + 1.  MGS: first = j, coef = hcol; CGS: first = 0, coef = hcol; CGS2:
// a plain pass with coef = hcol, then the final one with coef = haux.
template <typename V, bool FINAL>
__global__ void __launch_bounds__(kThreads)
    sub_pass_kernel(int64_t n, V* __restrict__ w, const V* __restrict__ krylov, int64_t first, const V* coef,
                    const V* haux, V* hcol, int64_t j, V* gsin, V* gcos, V* rnorm, V* rnc, uint64_t* fin,
                    uint8_t* stop, V* sc, int32_t* ctl, V* __restrict__ partials, unsigned int* __restrict__ counter)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    V a[1] = {V(0)};
    for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
        V wr = w[r];
        for (int64_t i = first; i <= j; ++i) {
            const V h = coef[i];
            if (h != V(0)) wr -= h * krylov[i * n + r];
        }
        w[r] = wr;
        if (FINAL) a[0] += wr * wr;
    }
    if (!FINAL) return;
    // every CTA read ctl and the coefficients before it took its ticket: the last one may write them
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (threadIdx.x == 0) {
        if (haux)
            for (int64_t i = 0; i <= j; ++i) hcol[i] += haux[i];
        const V nrm = sqrt(a[0]);
        hcol[j + 1] = nrm;
        sc[0] = nrm;
        gmres::givens_column<V>(0, gsin, 1, gcos, 1, rnorm, rnc, 1, hcol, 1, j, fin);
        check(rnorm[0], sc, ctl, stop);
    }
}

}  // namespace fgmres
}  // namespace b200

extern "C" {

#define B200_DEF_FGMRES(V, VT)                                                                    \
    int64_t b200_gmres_fused_work_size_##V(const b200_ctx* ctx, int64_t krylov_dim)               \
    {                                                                                             \
        return b200::gmres::fused_work_size(ctx, krylov_dim);                                     \
    }                                                                                             \
    b200_status b200_gmres_fused_init_##V(b200_ctx* ctx, const VT* rnorm, VT* sc, int32_t* ctl,   \
                                          uint8_t* stop, int64_t max_iters, int32_t res_kind,     \
                                          int32_t iter_first, int32_t baseline,                   \
                                          VT reduction_factor)                                    \
    {                                                                                             \
        B200_REQUIRE(ctx && rnorm && sc && ctl && stop, "null argument");                         \
        b200::fgmres::init_kernel<VT><<<1, 1, 0, ctx->stream>>>(                                  \
            rnorm, sc, ctl, stop, b200::fused::clamp_iters(max_iters), res_kind, iter_first,      \
            baseline, reduction_factor);                                                          \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_gmres_fused_scale_##V(b200_ctx* ctx, int64_t n, VT* v, VT* z,                \
                                           const VT* inv_diag, const VT* sc, const int32_t* ctl,  \
                                           int32_t divide)                                        \
    {                                                                                             \
        B200_REQUIRE(ctx && v && sc && ctl && (z || !inv_diag), "null argument");                 \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fgmres::scale_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(          \
            n, v, z, inv_diag, sc, ctl, divide != 0);                                             \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_gmres_fused_mgs_pass_##V(b200_ctx* ctx, int64_t n, VT* w, const VT* v_prev,  \
                                              const VT* v_i, VT* hcol, int64_t i,                 \
                                              const int32_t* ctl, VT* work)                       \
    {                                                                                             \
        B200_REQUIRE(ctx && w && v_prev && v_i && hcol && ctl && work, "null argument");          \
        B200_REQUIRE(i >= 1, "pass index must be >= 1");                                          \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fgmres::mgs_pass_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(       \
            n, w, v_prev, v_i, hcol, i, ctl, b200::fused::step_partials(ctx, work),               \
            ctx->counters + b200::kStepCounter);                                                  \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_gmres_fused_sub_pass_##V(b200_ctx* ctx, int64_t n, VT* w, const VT* krylov,  \
                                              const VT* coef, int64_t j, const int32_t* ctl)      \
    {                                                                                             \
        B200_REQUIRE(ctx && w && krylov && coef && ctl, "null argument");                         \
        B200_REQUIRE(j >= 0, "negative Krylov index");                                            \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fgmres::sub_pass_kernel<VT, false><<<grid, b200::fused::kThreads, 0, ctx->stream>>>( \
            n, w, krylov, 0, coef, nullptr, nullptr, j, nullptr, nullptr, nullptr, nullptr,       \
            nullptr, nullptr, nullptr, const_cast<int32_t*>(ctl), nullptr, nullptr);              \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_gmres_fused_final_pass_##V(                                                  \
        b200_ctx* ctx, int64_t n, VT* w, const VT* krylov, int64_t first, const VT* coef,         \
        const VT* haux, VT* hcol, int64_t j, VT* gsin, VT* gcos, VT* rnorm, VT* rnc,              \
        uint64_t* fin, uint8_t* stop, VT* sc, int32_t* ctl, VT* work)                             \
    {                                                                                             \
        B200_REQUIRE(ctx && w && krylov && coef && hcol && gsin && gcos && rnorm && rnc && fin && \
                         stop && sc && ctl && work,                                               \
                     "null argument");                                                            \
        B200_REQUIRE(j >= 0 && first >= 0 && first <= j, "need 0 <= first <= j");                 \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fgmres::sub_pass_kernel<VT, true><<<grid, b200::fused::kThreads, 0, ctx->stream>>>( \
            n, w, krylov, first, coef, haux, hcol, j, gsin, gcos, rnorm, rnc, fin, stop, sc, ctl, \
            b200::fused::step_partials(ctx, work), ctx->counters + b200::kStepCounter);           \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }

B200_DEF_FGMRES(f64, double)
B200_DEF_FGMRES(f32, float)

}  // extern "C"
