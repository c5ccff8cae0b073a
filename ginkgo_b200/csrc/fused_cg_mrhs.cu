// Fused CG iteration for k = 2..32 right-hand sides of one system, sm_90a: the regrouping of
// fused_cg.cu with every vector n x k row-major (stride k) and every scalar per column.  One
// matrix pass per iteration serves all k columns.
//
//   step_p    p_j = z_j + (rho_j/prev_rho_j) p_j                     reads 2nk, writes nk
//   spmv_mdot q = A p for all k columns, pq_j = p_j.q_j in the epilogue  matrix + 2nk (p gathered)
//   step_xr   alpha_j = rho_j/pq_j; x_j += alpha_j p_j; r_j -= alpha_j q_j; z_j = M^-1 r_j;
//             rho'_j = r_j.z_j; rr_j = r_j.r_j; per-column check (last CTA)  reads 4nk + n, writes 3nk
//
// = matrix + 12 n k + n values per iteration (13 n k in the count of fused_cg.cu, which reads the
// diagonal once per column), against k (matrix + 13 n) for k one-column solves.  The
// reference runs the same loop on an n x k Dense and masks every element-wise step by the column's
// stopping_status (common/unified/solver/cg_kernels.cpp:74,99); so do step_p and step_xr here: a
// stopped column's x, r and p are not touched again.  The SpMV computes every column (as the
// reference's Csr::apply does); its q of a stopped column is never read.
//
// Row / lane layout, bounded grids, per-column sums and the SpMV (its DotB epilogue) are those of
// fused_mrhs.cuh: q is bit-identical to b200_csr_spmv_* with num_rhs = k, and the per-CTA partials
// (k per CTA, 2k for step_xr) fit a fixed workspace.
//
// Scalars  sc[6k]:  sc[s*k + j] for column j, s = 0 rho, 1 prev_rho, 2 pq, 3 rr, 4 tau0 (baseline
//                   norm), 5 threshold = reduction_factor * tau0
// Status   status[k]: the reference's stopping_status byte of every column (0 = running)
// Control  ctl[0..4] of fused_common.cuh; 5..7 unused
#include "fused_mrhs.cuh"

namespace b200 {
namespace fcgm {

using fused::kThreads;  // step kernels
using namespace mrhs;   // layout, grids, column sums, the SpMV (fused_mrhs.cuh)

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    step_p_kernel(int64_t n, int64_t k, V* __restrict__ p, const V* __restrict__ z, const V* __restrict__ sc,
                  const uint8_t* __restrict__ status, const int32_t* __restrict__ ctl)
{
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    if (j >= k || has_stopped(status[j])) return;
    const V rho = sc[j], prev = sc[k + j];
    const bool plain = (prev == V(0));
    const V beta = plain ? V(0) : rho / prev;
    for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n; row += (int64_t)gridDim.x * kRows) {
        const int64_t e = row * k + j;
        const V zi = z[e];
        p[e] = plain ? zi : zi + beta * p[e];
    }
}

// INIT: r already holds b - A x and every column runs; computes z, rho, rr (no x / r update) and
// each column's baseline
template <typename V, int P, bool INIT>
__global__ void __launch_bounds__(kThreads)
    step_xr_kernel(int64_t n, int64_t k, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ p,
                   const V* __restrict__ q, V* __restrict__ z, const V* __restrict__ inv_diag, V* __restrict__ sc,
                   uint8_t* __restrict__ status, int32_t* __restrict__ ctl, V* __restrict__ partials,
                   unsigned int* __restrict__ counter, int baseline, V factor)
{
    __shared__ V red[2][kThreads / 32][P];
    __shared__ V tot[2][kMaxCols];
    __shared__ bool is_last;
    if (!INIT && ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int j = threadIdx.x % P;
    const bool run = j < k && !has_stopped(status[j]);
    const V pq = run ? sc[2 * k + j] : V(0);
    const bool update = !INIT && run && pq != V(0);
    const V alpha = update ? sc[j] / pq : V(0);
    V a[2] = {V(0), V(0)};
    if (run)
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            V ri = r[e];
            if (update) {
                x[e] += alpha * p[e];
                ri -= alpha * q[e];
                r[e] = ri;
            }
            const V zi = inv_diag ? ri * inv_diag[row] : ri;
            z[e] = zi;
            a[0] += ri * zi;
            a[1] += ri * ri;
        }
    cta_column_sums<V, P, 2, kThreads>(a, red);
    if (!grid_column_sums<V, 2, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    if (threadIdx.x != 0) return;
    // the top-of-iteration check of every running column
    const int32_t iter = ctl[1] + 1;
    ctl[1] = iter;
    for (int c = 0; c < (int)k; ++c) {
        if (has_stopped(status[c])) continue;
        const V rr = tot[1][c];
        if (INIT) fused::set_threshold(baseline, sqrt(rr), sc + 4 * k + c, sc + 5 * k + c, factor);
        status[c] = fused::top_check(iter, ctl, tot[0][c], rr, sc, k, c);
    }
    if (all_stopped(k, status)) ctl[0] = 1;
}

template <typename V>
__global__ void init_scalars_kernel(int64_t k, V* sc, uint8_t* status, int32_t* ctl, int32_t max_iters,
                                    int32_t res_kind, int32_t iter_first)
{
    const int j = threadIdx.x;
    if (j < k) {
        sc[j] = V(1);  // becomes prev_rho = 1 after the INIT check (reference cg::initialize)
        sc[k + j] = V(1);
        sc[2 * k + j] = V(0);
        sc[3 * k + j] = V(0);
        status[j] = 0;
    }
    if (j == 0) fused::start_control(ctl, max_iters, res_kind, iter_first, -1);  // the INIT check counts to 0
}

// ---- host side of the entry points ----------------------------------------------------------------
template <typename V, bool INIT>
b200_status step_xr(b200_ctx* ctx, int64_t n, int64_t k, V* x, V* r, const V* p, const V* q, V* z,
                    const V* inv_diag, V* sc, uint8_t* status, int32_t* ctl, V* work, int baseline, V factor)
{
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = work + step_partials_offset<DotB>(ctx, k);
#define B200_XR(PP)                                                                                   \
    step_xr_kernel<V, PP, INIT><<<grid, kThreads, 0, ctx->stream>>>(n, k, x, r, p, q, z, inv_diag, sc, \
                                                                    status, ctl, partials,            \
                                                                    ctx->counters + kStepCounter,     \
                                                                    baseline, factor)
    B200_MRHS_BY_LANES(P, B200_XR)
#undef B200_XR
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status init(b200_ctx* ctx, int64_t n, int64_t k, const V* r, V* z, V* p, V* q, const V* inv_diag, V* sc,
                 uint8_t* status, int32_t* ctl, V* work, int64_t max_iters, int32_t res_kind, int32_t iter_first,
                 int32_t baseline, V factor)
{
    B200_REQUIRE(ctx && sc && status && ctl && work, "null argument");
    B200_REQUIRE(n >= 0 && k >= 2 && k <= kMaxCols, "k must be in [2, 32]");
    init_scalars_kernel<V><<<1, kMaxCols, 0, ctx->stream>>>(k, sc, status, ctl, fused::clamp_iters(max_iters),
                                                           res_kind, iter_first);
    B200_LAUNCH_CHECK(ctx);
    if (n > 0) {
        B200_CUDA_CHECK(cudaMemsetAsync(p, 0, sizeof(V) * n * k, ctx->stream));
        B200_CUDA_CHECK(cudaMemsetAsync(q, 0, sizeof(V) * n * k, ctx->stream));
    }
    return step_xr<V, true>(ctx, n, k, nullptr, const_cast<V*>(r), p, q, z, inv_diag, sc, status, ctl, work,
                            baseline, factor);
}

template <typename V>
b200_status step_p(b200_ctx* ctx, int64_t n, int64_t k, V* p, const V* z, const V* sc, const uint8_t* status,
                   const int32_t* ctl)
{
    B200_REQUIRE(ctx && sc && status && ctl, "null argument");
    B200_REQUIRE(n >= 0 && k >= 2 && k <= kMaxCols, "k must be in [2, 32]");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
#define B200_P(PP) step_p_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, p, z, sc, status, ctl)
    B200_MRHS_BY_LANES(P, B200_P)
#undef B200_P
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

}  // namespace fcgm
}  // namespace b200

extern "C" {

#define B200_DEF_FCGM(V, VT)                                                                         \
    /* elements of `work` (value type): SpMV partials (k per CTA), then step_xr's (2k per CTA) */     \
    int64_t b200_cg_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                               \
    {                                                                                                \
        return b200::mrhs::step_partials_offset<b200::mrhs::DotB>(ctx, k) +                         \
               b200::mrhs::step_cap(ctx) * 2 * k + 64;                                               \
    }                                                                                                \
    b200_status b200_cg_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* z, VT* p, \
                                      VT* q, const VT* inv_diag, VT* sc, uint8_t* status, int32_t* ctl, \
                                      VT* work, int64_t max_iters, int32_t res_kind,                \
                                      int32_t iter_first, int32_t baseline, VT reduction_factor)    \
    {                                                                                                \
        return b200::fcgm::init<VT>(ctx, n, k, r, z, p, q, inv_diag, sc, status, ctl, work, max_iters, \
                                    res_kind, iter_first, baseline, reduction_factor);               \
    }                                                                                                \
    b200_status b200_cg_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p, const VT* z,     \
                                        const VT* sc, const uint8_t* status, const int32_t* ctl)     \
    {                                                                                                \
        return b200::fcgm::step_p<VT>(ctx, n, k, p, z, sc, status, ctl);                             \
    }                                                                                                \
    b200_status b200_cg_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* r,          \
                                         const VT* p, const VT* q, VT* z, const VT* inv_diag, VT* sc, \
                                         uint8_t* status, int32_t* ctl, VT* work)                    \
    {                                                                                                \
        B200_REQUIRE(ctx && sc && status && ctl && work, "null argument");                           \
        B200_REQUIRE(n >= 0 && k >= 2 && k <= b200::fcgm::kMaxCols, "k must be in [2, 32]");        \
        return b200::fcgm::step_xr<VT, false>(ctx, n, k, x, r, p, q, z, inv_diag, sc, status, ctl,   \
                                              work, 0, VT(0));                                       \
    }

B200_DEF_FCGM(f64, double)
B200_DEF_FCGM(f32, float)

/* q = A p for k = 2..32 columns of the row-major p and q (stride k) and dots[j] = p_j . q_j in one */
/* launch (square A; p is also the dot operand).  `work` provides the per-CTA partials               */
/* (b200_cg_mrhs_work_size elements); ctl may be NULL.  With num_rows == 0 the dots are 0.          */
#define B200_DEF_SPMV_MDOT(V, VT, I, IT)                                                             \
    b200_status b200_csr_spmv_mdot_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,      \
                                             int64_t nnz, const IT* row_ptrs, const IT* col_idxs,    \
                                             const VT* values, const VT* b, int64_t k, VT* c,        \
                                             VT* dots, VT* work, const int32_t* ctl)                 \
    {                                                                                                \
        return b200::mrhs::spmv_mdot<VT, IT, b200::mrhs::DotB>(ctx, num_rows, num_cols, nnz, row_ptrs, \
                                                               col_idxs, values, b, k, c, nullptr, dots, \
                                                               nullptr, work, ctl);                     \
    }

B200_DEF_SPMV_MDOT(f64, double, i32, int32_t)
B200_DEF_SPMV_MDOT(f64, double, i64, int64_t)
B200_DEF_SPMV_MDOT(f32, float, i32, int32_t)
B200_DEF_SPMV_MDOT(f32, float, i64, int64_t)

}  // extern "C"
