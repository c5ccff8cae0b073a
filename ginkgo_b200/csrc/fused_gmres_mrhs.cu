// Fused GMRES iteration for k = 2..32 right-hand sides of one system, sm_90a: the regrouping of
// fused_gmres.cu with every vector n x k row-major (stride k) and every Hessenberg entry, Givens
// rotation and residual estimate per column.  The k-wide SpMV is one matrix pass for all columns.
//
// The arrays the host's restart block shares with the loop kernels keep the loop's layout
// (core/solver/gmres.cpp:342-362), so gmres_initialize, gmres_restart, gmres_solve_krylov and
// gmres_multi_axpy run on them unchanged with nrhs = k:
//   krylov  n (kd+1) x k: basis i, column c at krylov[(i n + r) k + c]
//   hcol    row j of the kd x (kd+1) k Hessenberg: H(i, j) of column c at hcol[i k + c]
//   gsin, gcos (kd x k), rnc, haux ((kd+1) x k), rnorm, fin: stride k
//
// At Krylov index j (w is basis j+1, d the inverted diagonal of a scalar Jacobi preconditioner):
//   scale        v_j = w / h_j (j > 0); z = d . v_j                    reads 2nk (d: +n), writes nk (d: 2nk)
//   spmv_mdot2   w = A z (A v_j) for all columns, h_0 = v_0 . w          matrix + 3nk (fused_bicgstab_mrhs.cu)
//   mgs_pass i   w -= h_{i-1} v_{i-1}; h_i = v_i . w, i = 1..j                    4nk each
//   final_pass   w -= h_j v_j; ||w||; last CTA: h_{j+1}, the Givens update of hessenberg_qr, the
//                criteria for the top of iteration j + 1, ctl[0]                   3nk
// CGS: scale, the SpMV, multi_dot (h_1..h_j of every column in one pass over the bases, 16 bases per
// sweep in registers) and a final pass subtracting h_0 v_0, h_1 v_1, ... in basis order.  CGS2: a
// plain sub_pass, a second multi_dot over bases 0..j into haux, and the final pass subtracting haux
// and adding it into h (the loop's add_scaled).
//
// Element-wise arithmetic is the loop's operation for operation: sub_scaled's `w -= h v` (skipped for
// h == 0), inv_scale's division, the scalar Jacobi product, gmres::givens_column per column with
// stride k.  Sums: fused_mrhs.cuh's fixed shuffle tree per column and CTA partials added in a fixed
// order by the CTA with the last ticket; no floating-point atomics.
//
// Stopping is the loop's, per column (core/solver/gmres.cpp:453): Iteration and ResidualNorm in the
// user's order with ids 1 and 2, WITHOUT the finalized bit (multi_axpy sets it), on tau_c =
// |rnc_c[j+1]| against threshold_c.  The iteration counter is shared.  A stopped column is masked as
// hessenberg_qr masks it: its fin, gsin, gcos, rnc and Hessenberg entries are not written, and the
// element-wise and dot work of these kernels skips it (the SpMV computes every column; nothing reads
// a stopped column's new basis or h_0).  ctl[0] is raised only once every column has stopped; then
// every kernel is a no-op, so a graph of several iterations may be replayed past the stop.
//
// Scalars  sc[3k]: sc[s*k + c], s = 0 ||w|| of the last final pass (the divisor of the next scale),
//                  1 tau0 (baseline norm), 2 threshold = reduction_factor * tau0
// Status   status[k]: the loop's stopping_status byte of every column (0 = running)
// Control  ctl[0..4] of fused_common.cuh (res_kind 0 or 1); 5..7 unused, cleared by init
#include "fused_mrhs.cuh"
#include "gmres_common.cuh"

namespace b200 {
namespace fgmresm {

using fused::kThreads;  // scale and the passes
using namespace mrhs;

constexpr int kMdThreads = 256;
constexpr int kMdBases = 16;  // bases per sweep of the multi-dot (register accumulators)

inline int64_t md_cap(const b200_ctx* ctx) { return (int64_t)ctx->num_sms * kStepCtasPerSm; }
// `work`: the SpMV's partials (DotW2), the passes' (k per CTA), the multi-dot's ((kd+1) k per CTA)
inline int64_t md_offset(const b200_ctx* ctx, int64_t k)
{
    return step_partials_offset<DotW2>(ctx, k) + step_cap(ctx) * k;
}
inline int64_t work_size(const b200_ctx* ctx, int64_t k, int64_t krylov_dim)
{
    return md_offset(ctx, k) + md_cap(ctx) * (krylov_dim + 1) * k + 64;
}

template <typename V>
__device__ __forceinline__ uint8_t column_status(int32_t iter, const int32_t* ctl, V tau, V threshold)
{
    return fused::criteria_status(iter, ctl, [&](int32_t) { return tau <= threshold; }, uint8_t(0));
}

// rnorm holds ||b_c - A x_c|| (the loop's norm2); v_0, rnc, fin, gsin and gcos are set by the loop's
// initialize / restart kernels; sc[k + c] holds ||b_c|| for the rhs_norm baseline
template <typename V>
__global__ void init_kernel(int64_t k, const V* rnorm, V* sc, uint8_t* status, int32_t* ctl, int32_t max_iters,
                            int32_t res_kind, int32_t iter_first, int32_t baseline, V factor)
{
    const int c = threadIdx.x;
    if (c == 0) {
        fused::start_control(ctl, max_iters, res_kind, iter_first, 0);
        ctl[5] = ctl[6] = ctl[7] = 0;
    }
    __syncthreads();
    if (c < k) {
        fused::set_threshold(baseline, rnorm[c], sc + k + c, sc + 2 * k + c, factor);
        sc[c] = V(0);
        status[c] = column_status(0, ctl, rnorm[c], sc[2 * k + c]);
    }
    __syncthreads();
    if (c == 0 && all_stopped(k, status)) ctl[0] = 1;
}

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    scale_kernel(int64_t n, int64_t k, V* __restrict__ v, V* __restrict__ z, const V* __restrict__ inv_diag,
                 const V* __restrict__ sc, const uint8_t* __restrict__ status, const int32_t* __restrict__ ctl,
                 bool divide)
{
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    if (j >= k || has_stopped(status[j])) return;
    const V h = sc[j];
    for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n; row += (int64_t)gridDim.x * kRows) {
        const int64_t e = row * k + j;
        V vi = v[e];
        if (divide) {
            vi /= h;
            v[e] = vi;
        }
        if (inv_diag) z[e] = vi * inv_diag[row];
    }
}

// MGS pass i: w -= h_{i-1} v_{i-1}; h_i = v_i . w
template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    mgs_pass_kernel(int64_t n, int64_t k, V* __restrict__ w, const V* __restrict__ v_prev,
                    const V* __restrict__ v_i, V* __restrict__ hcol, int64_t i, const uint8_t* __restrict__ status,
                    const int32_t* __restrict__ ctl, V* __restrict__ partials, unsigned int* __restrict__ counter)
{
    __shared__ V red[1][kThreads / 32][P];
    __shared__ V tot[1][kMaxCols];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    const bool run = j < k && !has_stopped(status[j]);
    V a[1] = {V(0)};
    if (run) {
        const V h = hcol[(i - 1) * k + j];
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            V wr = w[e];
            if (h != V(0)) wr -= h * v_prev[e];
            w[e] = wr;
            a[0] += v_i[e] * wr;
        }
    }
    cta_column_sums<V, P, 1, kThreads>(a, red);
    if (!grid_column_sums<V, 1, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    const int c = threadIdx.x;
    if (c < k && !has_stopped(status[c])) hcol[i * k + c] = tot[0][c];
}

// subtract pass: w -= coef_i v_i for i = first..j, element by element in basis order (each the rounding
// of one sub_scaled, skipped for coef_i == 0).  FINAL: also ||w||; the last CTA adds haux into the
// Hessenberg column (CGS2), sets h_{j+1} = ||w||, runs the Givens update and the check for the top of
// iteration j + 1 of every running column.  MGS: first = j, coef = hcol; CGS: first = 0, coef = hcol;
// CGS2: a plain pass with coef = hcol, then the final one with coef = haux.
template <typename V, int P, bool FINAL>
__global__ void __launch_bounds__(kThreads)
    sub_pass_kernel(int64_t n, int64_t k, V* __restrict__ w, const V* __restrict__ krylov, int64_t first,
                    const V* coef, const V* haux, V* hcol, int64_t j, V* gsin, V* gcos, V* rnorm, V* rnc,
                    uint64_t* fin, uint8_t* status, V* sc, int32_t* ctl, V* __restrict__ partials,
                    unsigned int* __restrict__ counter)
{
    __shared__ V red[1][kThreads / 32][P];
    __shared__ V tot[1][kMaxCols];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int lane = threadIdx.x % P;
    const bool run = lane < k && !has_stopped(status[lane]);
    V a[1] = {V(0)};
    if (run)
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + lane;
            V wr = w[e];
            for (int64_t i = first; i <= j; ++i) {
                const V h = coef[i * k + lane];
                if (h != V(0)) wr -= h * krylov[i * n * k + e];
            }
            w[e] = wr;
            if (FINAL) a[0] += wr * wr;
        }
    if (!FINAL) return;
    // every CTA read ctl, the statuses and the coefficients before it took its ticket: the last one
    // may write them
    cta_column_sums<V, P, 1, kThreads>(a, red);
    if (!grid_column_sums<V, 1, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    const int c = threadIdx.x;
    const int32_t iter = ctl[1] + 1;
    if (c < k && !has_stopped(status[c])) {
        if (haux)
            for (int64_t i = 0; i <= j; ++i) hcol[i * k + c] += haux[i * k + c];
        const V nrm = sqrt(tot[0][c]);
        hcol[(j + 1) * k + c] = nrm;
        sc[c] = nrm;
        gmres::givens_column<V>(c, gsin, k, gcos, k, rnorm, rnc, k, hcol, k, j, fin);
        status[c] = column_status(iter, ctl, rnorm[c], sc[2 * k + c]);
    }
    __syncthreads();
    if (c == 0) {
        ctl[1] = iter;
        if (all_stopped(k, status)) ctl[0] = 1;
    }
}

// hcol[i k + c] = v_i . w for i < num_bases and every running column c, in one pass over the bases:
// kMdBases bases per sweep in registers, w read once per sweep.  The partials of every (basis, column)
// go to the workspace; the CTA with the last ticket adds them in CTA order, one warp each.
template <typename V, int P>
__global__ void __launch_bounds__(kMdThreads, 2)
    multi_dot_kernel(int64_t n, int64_t k, int64_t num_bases, const V* __restrict__ krylov, const V* __restrict__ w,
                     V* __restrict__ hcol, const uint8_t* __restrict__ status, const int32_t* __restrict__ ctl,
                     V* __restrict__ partials, unsigned int* __restrict__ counter)
{
    __shared__ V red[kMdBases][kMdThreads / 32][P];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    constexpr int kRows = kMdThreads / P;
    const int tid = threadIdx.x, j = tid % P;
    const bool run = j < k && !has_stopped(status[j]);
    const int64_t per_cta = num_bases * k;
    for (int64_t i0 = 0; i0 < num_bases; i0 += kMdBases) {
        const int nb = (int)((num_bases - i0) < kMdBases ? (num_bases - i0) : kMdBases);
        V acc[kMdBases];
#pragma unroll
        for (int q = 0; q < kMdBases; ++q) acc[q] = V(0);
        if (run)
            for (int64_t row = blockIdx.x * (int64_t)kRows + tid / P; row < n; row += (int64_t)gridDim.x * kRows) {
                const int64_t e = row * k + j;
                const V wv = w[e];
                V kv[kMdBases];
#pragma unroll
                for (int q = 0; q < kMdBases; ++q) kv[q] = q < nb ? krylov[(i0 + q) * n * k + e] : V(0);
#pragma unroll
                for (int q = 0; q < kMdBases; ++q)
                    if (q < nb) acc[q] += kv[q] * wv;
            }
        if (i0 > 0) __syncthreads();  // the previous sweep's reads of red are done
        cta_column_sums<V, P, kMdBases, kMdThreads>(acc, red);
        if (tid < k)
#pragma unroll
            for (int q = 0; q < kMdBases; ++q)
                if (q < nb) partials[blockIdx.x * per_cta + (i0 + q) * k + tid] = acc[q];
    }
    if (tid < k) __threadfence();
    last_cta_sums<kMdThreads>(per_cta, partials, counter, &is_last, [&](int64_t idx, V s) {
        if (!has_stopped(status[idx % k])) hcol[idx] = s;  // a stopped column keeps its Hessenberg entries
    });
}

// ---- host side of the entry points ----------------------------------------------------------------
#define B200_FGM_REQUIRE(ctx, n, k)                                                    \
    B200_REQUIRE(ctx, "null argument");                                                \
    B200_REQUIRE((n) >= 0 && (k) >= 2 && (k) <= kMaxCols, "k must be in [2, 32]")

template <typename V>
b200_status init(b200_ctx* ctx, int64_t k, const V* rnorm, V* sc, uint8_t* status, int32_t* ctl, int64_t max_iters,
                 int32_t res_kind, int32_t iter_first, int32_t baseline, V factor)
{
    B200_FGM_REQUIRE(ctx, 0, k);
    B200_REQUIRE(rnorm && sc && status && ctl, "null argument");
    init_kernel<V><<<1, kMaxCols, 0, ctx->stream>>>(k, rnorm, sc, status, ctl,
                                                   fused::clamp_iters(max_iters), res_kind, iter_first, baseline,
                                                   factor);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status scale(b200_ctx* ctx, int64_t n, int64_t k, V* v, V* z, const V* inv_diag, const V* sc,
                  const uint8_t* status, const int32_t* ctl, int32_t divide)
{
    B200_FGM_REQUIRE(ctx, n, k);
    B200_REQUIRE(v && sc && status && ctl && (z || !inv_diag), "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
#define B200_SC(PP) \
    scale_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, v, z, inv_diag, sc, status, ctl, divide != 0)
    B200_MRHS_BY_LANES(P, B200_SC)
#undef B200_SC
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status mgs_pass(b200_ctx* ctx, int64_t n, int64_t k, V* w, const V* v_prev, const V* v_i, V* hcol, int64_t i,
                     const uint8_t* status, const int32_t* ctl, V* work)
{
    B200_FGM_REQUIRE(ctx, n, k);
    B200_REQUIRE(w && v_prev && v_i && hcol && status && ctl && work, "null argument");
    B200_REQUIRE(i >= 1, "pass index must be >= 1");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = work + step_partials_offset<DotW2>(ctx, k);
#define B200_MG(PP)                                                                                      \
    mgs_pass_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, w, v_prev, v_i, hcol, i, status, ctl, \
                                                               partials, ctx->counters + kStepCounter)
    B200_MRHS_BY_LANES(P, B200_MG)
#undef B200_MG
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V, bool FINAL>
b200_status sub_pass(b200_ctx* ctx, int64_t n, int64_t k, V* w, const V* krylov, int64_t first, const V* coef,
                     const V* haux, V* hcol, int64_t j, V* gsin, V* gcos, V* rnorm, V* rnc, uint64_t* fin,
                     uint8_t* status, V* sc, int32_t* ctl, V* work)
{
    B200_FGM_REQUIRE(ctx, n, k);
    B200_REQUIRE(w && krylov && coef && status && ctl, "null argument");
    B200_REQUIRE(j >= 0 && first >= 0 && first <= j, "need 0 <= first <= j");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = FINAL ? work + step_partials_offset<DotW2>(ctx, k) : nullptr;
#define B200_SP(PP)                                                                                       \
    sub_pass_kernel<V, PP, FINAL><<<grid, kThreads, 0, ctx->stream>>>(n, k, w, krylov, first, coef, haux, \
                                                                      hcol, j, gsin, gcos, rnorm, rnc, fin, \
                                                                      status, sc, ctl, partials,          \
                                                                      ctx->counters + kStepCounter)
    B200_MRHS_BY_LANES(P, B200_SP)
#undef B200_SP
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status multi_dot(b200_ctx* ctx, int64_t n, int64_t k, int64_t num_bases, int64_t krylov_dim, const V* krylov,
                      const V* w, V* hcol, const uint8_t* status, const int32_t* ctl, V* work)
{
    B200_FGM_REQUIRE(ctx, n, k);
    B200_REQUIRE(krylov && w && hcol && status && ctl && work, "null argument");
    B200_REQUIRE(num_bases <= krylov_dim + 1, "more bases than the workspace holds");
    if (num_bases <= 0) return B200_OK;
    const int P = lanes_for(k);
    const int grid = rows_grid<kMdThreads>(n, P, md_cap(ctx));
    V* partials = work + md_offset(ctx, k);
#define B200_MD(PP)                                                                                        \
    multi_dot_kernel<V, PP><<<grid, kMdThreads, 0, ctx->stream>>>(n, k, num_bases, krylov, w, hcol, status, \
                                                                  ctl, partials, ctx->counters + kMultiDotCounter)
    B200_MRHS_BY_LANES(P, B200_MD)
#undef B200_MD
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

#undef B200_FGM_REQUIRE

}  // namespace fgmresm
}  // namespace b200

extern "C" {

#define B200_DEF_FGMRESM(V, VT)                                                                               \
    int64_t b200_gmres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k, int64_t krylov_dim)                  \
    {                                                                                                         \
        return b200::fgmresm::work_size(ctx, k, krylov_dim);                                                  \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_init_##V(b200_ctx* ctx, int64_t k, const VT* rnorm, VT* sc, uint8_t* status,   \
                                         int32_t* ctl, int64_t max_iters, int32_t res_kind, int32_t iter_first, \
                                         int32_t baseline, VT reduction_factor)                               \
    {                                                                                                         \
        return b200::fgmresm::init<VT>(ctx, k, rnorm, sc, status, ctl, max_iters, res_kind, iter_first,       \
                                       baseline, reduction_factor);                                           \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_scale_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v, VT* z,                   \
                                          const VT* inv_diag, const VT* sc, const uint8_t* status,            \
                                          const int32_t* ctl, int32_t divide)                                 \
    {                                                                                                         \
        return b200::fgmresm::scale<VT>(ctx, n, k, v, z, inv_diag, sc, status, ctl, divide);                  \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_mgs_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* v_prev,     \
                                             const VT* v_i, VT* hcol, int64_t i, const uint8_t* status,       \
                                             const int32_t* ctl, VT* work)                                    \
    {                                                                                                         \
        return b200::fgmresm::mgs_pass<VT>(ctx, n, k, w, v_prev, v_i, hcol, i, status, ctl, work);            \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t k, int64_t num_bases,          \
                                              int64_t krylov_dim, const VT* krylov, const VT* w, VT* hcol,    \
                                              const uint8_t* status, const int32_t* ctl, VT* work)            \
    {                                                                                                         \
        return b200::fgmresm::multi_dot<VT>(ctx, n, k, num_bases, krylov_dim, krylov, w, hcol, status, ctl,   \
                                            work);                                                            \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_sub_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov,     \
                                             const VT* coef, int64_t j, const uint8_t* status,                \
                                             const int32_t* ctl)                                              \
    {                                                                                                         \
        return b200::fgmresm::sub_pass<VT, false>(ctx, n, k, w, krylov, 0, coef, nullptr, nullptr, j,         \
                                                  nullptr, nullptr, nullptr, nullptr, nullptr,                \
                                                  const_cast<uint8_t*>(status), nullptr,                      \
                                                  const_cast<int32_t*>(ctl), nullptr);                        \
    }                                                                                                         \
    b200_status b200_gmres_mrhs_final_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov,   \
                                               int64_t first, const VT* coef, const VT* haux, VT* hcol,       \
                                               int64_t j, VT* gsin, VT* gcos, VT* rnorm, VT* rnc,             \
                                               uint64_t* fin, uint8_t* status, VT* sc, int32_t* ctl,          \
                                               VT* work)                                                      \
    {                                                                                                         \
        B200_REQUIRE(hcol && gsin && gcos && rnorm && rnc && fin && sc && work, "null argument");              \
        return b200::fgmresm::sub_pass<VT, true>(ctx, n, k, w, krylov, first, coef, haux, hcol, j, gsin, gcos, \
                                                 rnorm, rnc, fin, status, sc, ctl, work);                     \
    }

B200_DEF_FGMRESM(f64, double)
B200_DEF_FGMRESM(f32, float)

}  // extern "C"
