// Fused BiCGStab iteration for k = 2..32 right-hand sides of one system, sm_90a: the regrouping of
// fused_bicgstab.cu with every vector n x k row-major (stride k) and every scalar per column.  Each
// SpMV is one matrix pass for all k columns.  d is the inverted diagonal of a scalar Jacobi
// preconditioner, or absent (Identity).
//
//   step_p     p_j = r_j + tmp_j (p_j - omega_j v_j), tmp_j = rho_j/prev_rho_j*alpha_j/omega_j
//              (p_j = r_j if prev_rho_j*omega_j == 0); y_j = d.p_j                reads 3nk + n, writes 2nk
//   spmv_mdot2 v = A y for all columns, beta_j = rr_j.v_j in the epilogue         matrix + 3nk
//   step_s     alpha_j = rho_j/beta_j (0 and s_j = r_j if beta_j == 0); s_j = r_j - alpha_j v_j;
//              z_j = d.s_j; ||s_j||^2; the mid-iteration check of every running column
//                                                                                 reads 2nk + n, writes 2nk
//   spmv_mdot2 t = A z, gamma_j = s_j.t_j and beta_j = t_j.t_j in the epilogue    matrix + 3nk
//   step_xr    omega_j = gamma_j/beta_j (0 if beta_j == 0); x_j += alpha_j y_j + omega_j z_j;
//              r_j = s_j - omega_j t_j; rho_j = rr_j.r_j; ||r_j||^2; the top-of-iteration check
//                                                                                 reads 6nk, writes 2nk
//
// = 2 matrix + 23 n k + 2 n values per iteration, against 2 matrix + 36 n k for the reference's
// kernel sequence on an n x k Dense and k (2 matrix + 25 n) for k one-column fused solves.  Element-
// wise arithmetic is the reference's, operation for operation (reference/solver/bicgstab_kernels.cpp:
// 65-178), so given the same scalars p, y, s, z, x, r are the bits of bicgstab::step_1/2/3/finalize +
// the scalar Jacobi apply.  As in the reference, every element-wise step skips a stopped column
// (its x, r and p are not touched again); the SpMVs compute every column.
//
// Stopping is the reference's (core/solver/bicgstab.cpp:95-233), per column: Iteration and
// (Implicit)ResidualNorm in the user's order with ids 1 and 2, at the top of the iteration on r_j
// (step_xr's last CTA, finalized) and again mid-iteration on s_j with the same iteration number and
// rho_j (step_s's last CTA, NOT finalized).  A column stopped at the mid check owes the update of
// bicgstab::finalize, x_j += alpha_j y_j: step_s raises ctl[5], and step_xr of the same iteration pays
// it (a stopped, unfinalized column) and sets the finalized bit, so it is paid once.  ctl[0] is raised
// only once every column has stopped -- at a top check, or at a mid check, which also turns the second
// SpMV into a no-op.  Then every kernel is a no-op except the step_xr that pays what is owed, so a
// graph of several iterations can be replayed past the stop.  Every iteration ends with step_xr, so a
// stop the host reads between iterations has its finalizes paid.
//
// Layout, grids, per-column sums and the SpMV: fused_mrhs.cuh (the SpMV with the DotW2 epilogue).
//
// Scalars  sc[10k]: sc[s*k + j] for column j, s = 0 rho, 1 prev_rho, 2 beta (rr.v, then t.t),
//                   3 ||r||^2, 4 tau0 (baseline norm), 5 threshold = reduction_factor * tau0,
//                   6 alpha, 7 omega, 8 gamma, 9 ||s||^2
// Status   status[k]: the reference's stopping_status byte of every column (0 = running)
// Control  ctl[0..4] of fused_common.cuh; 5 some column owes its finalize (stopped at the mid check),
//                   6..7 unused
#include "fused_mrhs.cuh"

namespace b200 {
namespace fbicgstabm {

using fused::kThreads;  // step kernels
using namespace mrhs;

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    step_p_kernel(int64_t n, int64_t k, V* __restrict__ p, const V* __restrict__ r, const V* __restrict__ v,
                  V* __restrict__ y, const V* __restrict__ inv_diag, const V* __restrict__ sc,
                  const uint8_t* __restrict__ status, const int32_t* __restrict__ ctl)
{
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    if (j >= k || has_stopped(status[j])) return;
    const V rho = sc[j], prev = sc[k + j], alpha = sc[6 * k + j], omega = sc[7 * k + j];
    const bool plain = !(prev * omega != V(0));
    const V tmp = plain ? V(0) : rho / prev * alpha / omega;
    for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n; row += (int64_t)gridDim.x * kRows) {
        const int64_t e = row * k + j;
        const V ri = r[e];
        const V pi = plain ? ri : ri + tmp * (p[e] - omega * v[e]);
        p[e] = pi;
        y[e] = inv_diag ? pi * inv_diag[row] : pi;
    }
}

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    step_s_kernel(int64_t n, int64_t k, const V* __restrict__ r, const V* __restrict__ v, V* __restrict__ s,
                  V* __restrict__ z, const V* __restrict__ inv_diag, V* __restrict__ sc,
                  uint8_t* __restrict__ status, int32_t* __restrict__ ctl, V* __restrict__ partials,
                  unsigned int* __restrict__ counter)
{
    __shared__ V red[1][kThreads / 32][P];
    __shared__ V tot[1][kMaxCols];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    const bool run = j < k && !has_stopped(status[j]);
    const V beta = run ? sc[2 * k + j] : V(0);
    const bool update = beta != V(0);
    const V alpha = update ? sc[j] / beta : V(0);
    V a[1] = {V(0)};
    if (run)
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            const V ri = r[e];
            const V si = update ? ri - alpha * v[e] : ri;
            s[e] = si;
            z[e] = inv_diag ? si * inv_diag[row] : si;
            a[0] += si * si;
        }
    cta_column_sums<V, P, 1, kThreads>(a, red);
    if (!grid_column_sums<V, 1, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    if (threadIdx.x != 0) return;
    // the mid-iteration check of every running column (core/solver/bicgstab.cpp:170-186): the top
    // check's iteration number and rho, ||s|| as the residual norm, the finalized bit not set.  This and
    // step_xr's top check restate fused::residual_status / top_check and mrhs::all_stopped: through the
    // helpers these kernels need more registers and run slower (DESIGN.md section 4).
    const int32_t iter = ctl[1];
    bool all_stopped = true, owed = false;
    for (int c = 0; c < (int)k; ++c) {
        uint8_t st = status[c];
        if (!has_stopped(st)) {
            const V b = sc[2 * k + c];
            sc[6 * k + c] = b != V(0) ? sc[c] / b : V(0);
            const V ss = tot[0][c], rho = sc[c], threshold = sc[5 * k + c];
            sc[9 * k + c] = ss;
            st = fused::criteria_status(
                iter, ctl,
                [&](int32_t res_kind) {
                    const V tau = res_kind == 1 ? sqrt(ss) : sqrt(fabs(rho));
                    return tau <= threshold;
                },
                0);
            if (st != 0) {
                status[c] = st;
                owed = true;
            }
        }
        all_stopped = all_stopped && has_stopped(st);
    }
    if (owed) ctl[5] = 1;
    if (all_stopped) ctl[0] = 1;
}

// INIT: r already holds b - A x and every column runs; sets rr = r and computes rho = rr.r, ||r||^2
// and each column's baseline (no x / r update)
template <typename V, int P, bool INIT>
__global__ void __launch_bounds__(kThreads)
    step_xr_kernel(int64_t n, int64_t k, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ s,
                   const V* __restrict__ t, const V* __restrict__ y, const V* __restrict__ z,
                   V* __restrict__ rr, V* __restrict__ sc, uint8_t* __restrict__ status,
                   int32_t* __restrict__ ctl, V* __restrict__ partials, unsigned int* __restrict__ counter,
                   int baseline, V factor)
{
    __shared__ V red[2][kThreads / 32][P];
    __shared__ V tot[2][kMaxCols];
    __shared__ bool is_last;
    const bool pending = !INIT && ctl[5] != 0;
    const bool iterating = INIT || ctl[0] == 0;
    if (!pending && !iterating) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    const uint8_t st = j < k ? status[j] : uint8_t(0);
    const bool owes = !INIT && j < k && has_stopped(st) && !(st & kFinalizedMask);
    const bool run = iterating && j < k && !has_stopped(st);
    V a[2] = {V(0), V(0)};
    if (owes) {
        // bicgstab::finalize after a stop at this iteration's mid check
        // (reference/solver/bicgstab_kernels.cpp:163-178)
        const V alpha = sc[6 * k + j];
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            x[e] += alpha * y[e];
        }
    } else if (run) {
        const V beta = INIT ? V(0) : sc[2 * k + j];
        const V omega = INIT ? V(0) : (beta != V(0) ? sc[8 * k + j] / beta : V(0));
        const V alpha = INIT ? V(0) : sc[6 * k + j];
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            V ri, rri;
            if (INIT) {
                ri = r[e];
                rri = ri;
                rr[e] = ri;
            } else {
                x[e] += alpha * y[e] + omega * z[e];
                ri = s[e] - omega * t[e];
                r[e] = ri;
                rri = rr[e];
            }
            a[0] += rri * ri;
            a[1] += ri * ri;
        }
    }
    // every CTA read ctl, status and the scalars before it took its ticket: the last one may write them
    cta_column_sums<V, P, 2, kThreads>(a, red);
    if (!grid_column_sums<V, 2, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    if (threadIdx.x != 0) return;
    bool all_stopped = true;
    const int32_t iter = iterating ? ctl[1] + 1 : ctl[1];
    if (iterating) ctl[1] = iter;
    for (int c = 0; c < (int)k; ++c) {
        uint8_t stc = status[c];
        if (has_stopped(stc)) {
            if (!(stc & kFinalizedMask)) status[c] = stc = uint8_t(stc | kFinalizedMask);  // paid
        } else if (iterating) {
            // the top-of-iteration check (fused::finish_scalars per column)
            const V rho_new = tot[0][c], rrn = tot[1][c];
            if (INIT) {
                // baseline: 0 rhs_norm (sc[4k + c] preset to ||b_c||), 1 initial_resnorm, 2 absolute
                if (baseline == 1) sc[4 * k + c] = sqrt(rrn);
                if (baseline == 2) sc[4 * k + c] = V(1);
                sc[5 * k + c] = factor * sc[4 * k + c];
            } else {
                sc[7 * k + c] = sc[2 * k + c] != V(0) ? sc[8 * k + c] / sc[2 * k + c] : V(0);
            }
            sc[k + c] = sc[c];
            sc[c] = rho_new;
            sc[3 * k + c] = rrn;
            const V threshold = sc[5 * k + c];
            stc = fused::criteria_status(
                iter, ctl,
                [&](int32_t res_kind) {
                    const V tau = res_kind == 1 ? sqrt(rrn) : sqrt(fabs(rho_new));
                    return tau <= threshold;
                },
                kFinalizedMask);
            status[c] = stc;
        }
        all_stopped = all_stopped && has_stopped(stc);
    }
    ctl[5] = 0;
    ctl[0] = all_stopped ? 1 : 0;
}

template <typename V>
__global__ void init_scalars_kernel(int64_t k, V* sc, uint8_t* status, int32_t* ctl, int32_t max_iters,
                                    int32_t res_kind, int32_t iter_first)
{
    // rho = prev_rho = alpha = beta = gamma = omega = 1 (reference bicgstab::initialize); the INIT
    // check moves rho to prev_rho
    const int j = threadIdx.x;
    if (j < k) {
        for (int s : {0, 1, 2, 6, 7, 8}) sc[s * k + j] = V(1);
        sc[3 * k + j] = V(0);
        sc[9 * k + j] = V(0);
        status[j] = 0;
    }
    if (j == 0) {
        fused::start_control(ctl, max_iters, res_kind, iter_first, -1);  // the INIT check counts to 0
        ctl[5] = 0;
    }
}

// ---- host side of the entry points ----------------------------------------------------------------
#define B200_FBM_REQUIRE(ctx, n, k)                                                    \
    B200_REQUIRE(ctx, "null argument");                                                \
    B200_REQUIRE((n) >= 0 && (k) >= 2 && (k) <= kMaxCols, "k must be in [2, 32]")

template <typename V, bool INIT>
b200_status step_xr(b200_ctx* ctx, int64_t n, int64_t k, V* x, V* r, const V* s, const V* t, const V* y,
                    const V* z, V* rr, V* sc, uint8_t* status, int32_t* ctl, V* work, int baseline, V factor)
{
    B200_FBM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl && work, "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = work + step_partials_offset<DotW2>(ctx, k);
#define B200_XR(PP)                                                                                      \
    step_xr_kernel<V, PP, INIT><<<grid, kThreads, 0, ctx->stream>>>(n, k, x, r, s, t, y, z, rr, sc, status, \
                                                                    ctl, partials, ctx->counters + kStepCounter, \
                                                                    baseline, factor)
    B200_MRHS_BY_LANES(P, B200_XR)
#undef B200_XR
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status init(b200_ctx* ctx, int64_t n, int64_t k, const V* r, V* rr, V* p, V* v, V* y, V* s, V* t, V* z,
                 V* sc, uint8_t* status, int32_t* ctl, V* work, int64_t max_iters, int32_t res_kind,
                 int32_t iter_first, int32_t baseline, V factor)
{
    B200_FBM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl && work, "null argument");
    init_scalars_kernel<V><<<1, kMaxCols, 0, ctx->stream>>>(
        k, sc, status, ctl, fused::clamp_iters(max_iters), res_kind, iter_first);
    B200_LAUNCH_CHECK(ctx);
    if (n > 0) {
        V* zeroed[6] = {p, v, y, s, t, z};
        for (V* a : zeroed) B200_CUDA_CHECK(cudaMemsetAsync(a, 0, sizeof(V) * n * k, ctx->stream));
    }
    return step_xr<V, true>(ctx, n, k, nullptr, const_cast<V*>(r), nullptr, nullptr, nullptr, nullptr, rr, sc,
                            status, ctl, work, baseline, factor);
}

template <typename V>
b200_status step_p(b200_ctx* ctx, int64_t n, int64_t k, V* p, const V* r, const V* v, V* y, const V* inv_diag,
                   const V* sc, const uint8_t* status, const int32_t* ctl)
{
    B200_FBM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl, "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
#define B200_P(PP) \
    step_p_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, p, r, v, y, inv_diag, sc, status, ctl)
    B200_MRHS_BY_LANES(P, B200_P)
#undef B200_P
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status step_s(b200_ctx* ctx, int64_t n, int64_t k, const V* r, const V* v, V* s, V* z, const V* inv_diag,
                   V* sc, uint8_t* status, int32_t* ctl, V* work)
{
    B200_FBM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl && work, "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = work + step_partials_offset<DotW2>(ctx, k);
#define B200_S(PP)                                                                                      \
    step_s_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, r, v, s, z, inv_diag, sc, status, ctl, \
                                                             partials, ctx->counters + kStepCounter)
    B200_MRHS_BY_LANES(P, B200_S)
#undef B200_S
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

#undef B200_FBM_REQUIRE

}  // namespace fbicgstabm
}  // namespace b200

extern "C" {

#define B200_DEF_FBICGSTABM(V, VT)                                                                     \
    /* elements of `work` (value type): SpMV partials (2k per CTA), then the steps' (2k per CTA) */    \
    int64_t b200_bicgstab_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                           \
    {                                                                                                  \
        return b200::mrhs::step_partials_offset<b200::mrhs::DotW2>(ctx, k) +                           \
               b200::mrhs::step_cap(ctx) * 2 * k + 64;                                                 \
    }                                                                                                  \
    b200_status b200_bicgstab_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* rr,  \
                                            VT* p, VT* v, VT* y, VT* s, VT* t, VT* z, VT* sc,          \
                                            uint8_t* status, int32_t* ctl, VT* work, int64_t max_iters, \
                                            int32_t res_kind, int32_t iter_first, int32_t baseline,    \
                                            VT reduction_factor)                                       \
    {                                                                                                  \
        return b200::fbicgstabm::init<VT>(ctx, n, k, r, rr, p, v, y, s, t, z, sc, status, ctl, work,   \
                                          max_iters, res_kind, iter_first, baseline, reduction_factor); \
    }                                                                                                  \
    b200_status b200_bicgstab_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p, const VT* r, \
                                              const VT* v, VT* y, const VT* inv_diag, const VT* sc,    \
                                              const uint8_t* status, const int32_t* ctl)               \
    {                                                                                                  \
        return b200::fbicgstabm::step_p<VT>(ctx, n, k, p, r, v, y, inv_diag, sc, status, ctl);         \
    }                                                                                                  \
    b200_status b200_bicgstab_mrhs_step_s_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r,        \
                                              const VT* v, VT* s, VT* z, const VT* inv_diag, VT* sc,   \
                                              uint8_t* status, int32_t* ctl, VT* work)                 \
    {                                                                                                  \
        return b200::fbicgstabm::step_s<VT>(ctx, n, k, r, v, s, z, inv_diag, sc, status, ctl, work);   \
    }                                                                                                  \
    b200_status b200_bicgstab_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* r,      \
                                               const VT* s, const VT* t, const VT* y, const VT* z,     \
                                               const VT* rr, VT* sc, uint8_t* status, int32_t* ctl,    \
                                               VT* work)                                               \
    {                                                                                                  \
        return b200::fbicgstabm::step_xr<VT, false>(ctx, n, k, x, r, s, t, y, z, const_cast<VT*>(rr),  \
                                                    sc, status, ctl, work, 0, VT(0));                  \
    }

B200_DEF_FBICGSTABM(f64, double)
B200_DEF_FBICGSTABM(f32, float)

/* c = A b for k = 2..32 columns of the row-major b, c and w (stride k), dots[j] = w_j . c_j and,   */
/* unless dots2 is NULL, dots2[j] = c_j . c_j in one launch.  `work` provides the per-CTA partials  */
/* (b200_bicgstab_mrhs_work_size elements); ctl may be NULL.  With num_rows == 0 the sums are 0.    */
#define B200_DEF_SPMV_MDOT2(V, VT, I, IT)                                                              \
    b200_status b200_csr_spmv_mdot2_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,       \
                                              int64_t nnz, const IT* row_ptrs, const IT* col_idxs,     \
                                              const VT* values, const VT* b, int64_t k, VT* c,         \
                                              const VT* w, VT* dots, VT* dots2, VT* work,              \
                                              const int32_t* ctl)                                      \
    {                                                                                                  \
        B200_REQUIRE(num_rows == 0 || w, "null argument");                                             \
        return b200::mrhs::spmv_mdot<VT, IT, b200::mrhs::DotW2>(ctx, num_rows, num_cols, nnz, row_ptrs, \
                                                                col_idxs, values, b, k, c, w, dots,    \
                                                                dots2, work, ctl);                     \
    }

B200_DEF_SPMV_MDOT2(f64, double, i32, int32_t)
B200_DEF_SPMV_MDOT2(f64, double, i64, int64_t)
B200_DEF_SPMV_MDOT2(f32, float, i32, int32_t)
B200_DEF_SPMV_MDOT2(f32, float, i64, int64_t)

}  // extern "C"
