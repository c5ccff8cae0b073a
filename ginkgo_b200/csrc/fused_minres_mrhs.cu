// Fused MINRES iteration for k = 2..32 right-hand sides of one system, sm_90a: the regrouping of
// fused_minres.cu with every vector n x k row-major (stride k) and every scalar per column.  One
// matrix pass per iteration serves all k columns (d is the inverted diagonal of a scalar Jacobi
// preconditioner, or absent):
//
//   spmv_sub_mdot  v = A z - v for all columns, alpha_c = z_c.v_c in the epilogue         matrix + 3nk
//   lanczos        v_c -= alpha_c q_c; beta_c = v_c.(d v_c); minres::step_1 per running
//                  column in the last CTA                                                  3nk + n
//   update         minres::step_2 with z~ = d v recomputed and without q_prev; the last CTA
//                  swaps gamma / beta per column, counts the iteration and checks every
//                  running column                                                         11nk + n
//
// = matrix + 17 n k + 2 n values per iteration, against k (matrix + 19 n) for k one-column solves.
// The loop runs the same body on an n x k Dense (core/solver/minres.cpp:199-285) and masks
// minres::step_1 / step_2 by the column's stopping_status; so do lanczos and update here: no scalar,
// x, p, q, v or z of a stopped column is written.  The SpMV computes every column (as Csr::apply
// does); a stopped column's v and alpha are never read.  Unlike the one-column lanczos, v -= alpha q
// runs for alpha == 0 too: with a 1 x k alpha, Dense::sub_scaled does not skip a zero scalar
// (dense_blas1.cu: add_scaled).
//
// Row / lane layout, bounded grids, per-column sums and the SpMV (its SubDotB epilogue) are those of
// fused_mrhs.cuh: v is bit-identical to b200_csr_advanced_spmv_* with (1, -1) and num_rhs = k.
// Element-wise arithmetic and the scalar recurrence are krylov_steps.cu's (fused_minres.cuh).
//
// p and p_prev trade places every iteration for all columns at once (a pointer swap in the loop), so
// update picks their roles from the parity of the shared counter ctl[1], as fused_minres.cu does; the
// last CTA increments it only after every other CTA took its ticket.
//
// Stopping is the loop's, per column: Iteration and ImplicitResidualNorm (sqrt|tau_c| <= threshold_c)
// in the user's order with ids 1 and 2, checked by init for iteration 0 and by update's last CTA for
// the next iteration.  ctl[0] is raised only once every column has stopped; then every kernel is a
// no-op, so a graph of several iterations can be replayed past the stop.
//
// Scalars  sc[16k]: sc[s*k + c] for column c, with the slots s of fused_minres.cu's sc[16]
// Status   status[k]: the loop's stopping_status byte of every column (0 = running)
// Control  ctl[0..4] of fused_common.cuh (res_kind 0 or 2); 5..7 unused, cleared by init
#include "fused_minres.cuh"
#include "fused_mrhs.cuh"

namespace b200 {
namespace fminresm {

using fused::kThreads;  // lanczos and update
using namespace mrhs;   // layout, grids, column sums, the SpMV (fused_mrhs.cuh)
using fminres::safe_divide;

inline int64_t work_size(const b200_ctx* ctx, int64_t k)
{
    return step_partials_offset<SubDotB>(ctx, k) + step_cap(ctx) * k + 64;
}

// the check of one column, as fused_minres.cu's: sqrt|tau| <= threshold for ImplicitResidualNorm
template <typename V>
__device__ __forceinline__ uint8_t tau_status(int32_t iter, const int32_t* ctl, V tau, V threshold)
{
    return fused::criteria_status(
        iter, ctl, [&](int32_t) { return sqrt(fabs(tau)) <= threshold; }, kFinalizedMask);
}

// sc[4k + c] holds the baseline norm (||b_c|| or ||r0_c||, from the host) unless it is absolute
template <typename V>
__global__ void init_kernel(int64_t k, V* sc, uint8_t* status, int32_t* ctl, int32_t max_iters, int32_t res_kind,
                            int32_t iter_first, int32_t baseline, V factor)
{
    const int c = threadIdx.x;
    if (c == 0) {
        fused::start_control(ctl, max_iters, res_kind, iter_first, 0);
        ctl[5] = ctl[6] = ctl[7] = 0;
    }
    __syncthreads();
    if (c < k) {
        fused::set_threshold(baseline, sc[4 * k + c], sc + 4 * k + c, sc + 5 * k + c, factor);
        status[c] = tau_status(0, ctl, sc[6 * k + c], sc[5 * k + c]);
    }
    __syncthreads();
    if (c == 0 && all_stopped(k, status)) ctl[0] = 1;
}

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    lanczos_kernel(int64_t n, int64_t k, V* __restrict__ v, const V* __restrict__ q, const V* __restrict__ inv_diag,
                   V* __restrict__ sc, const uint8_t* __restrict__ status, const int32_t* __restrict__ ctl,
                   V* __restrict__ partials, unsigned int* __restrict__ counter)
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
        const V alpha = sc[j];
        for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < n;
             row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            V vi = v[e];
            vi -= alpha * q[e];
            v[e] = vi;
            const V zt = inv_diag ? vi * inv_diag[row] : vi;
            a[0] += vi * zt;
        }
    }
    // every CTA read alpha and the statuses before it took its ticket: the last one may overwrite them
    cta_column_sums<V, P, 1, kThreads>(a, red);
    if (!grid_column_sums<V, 1, kThreads>(a, k, partials, counter, tot, &is_last)) return;
    const int c = threadIdx.x;
    if (c < k && !has_stopped(status[c])) fminres::step_1(tot[0][c], sc + c, k);
}

template <typename V, int P>
__global__ void __launch_bounds__(kThreads)
    update_kernel(int64_t n, int64_t k, V* __restrict__ x, V* __restrict__ p0, V* __restrict__ p1,
                  V* __restrict__ z, V* __restrict__ q, V* __restrict__ v, const V* __restrict__ inv_diag,
                  V* __restrict__ sc, uint8_t* __restrict__ status, int32_t* __restrict__ ctl,
                  unsigned int* __restrict__ counter)
{
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    constexpr int kRows = kThreads / P;
    const int tid = threadIdx.x;
    const int32_t iter = ctl[1];
    // the loop swaps p and p_prev before step_2: iteration i writes p1 when i is even, p0 when odd
    V* __restrict__ p = (iter & 1) ? p0 : p1;
    const V* __restrict__ pp = (iter & 1) ? p1 : p0;
    const int j = tid % P;
    if (j < k && !has_stopped(status[j])) {
        const V alpha = sc[j], beta = sc[k + j], gamma = sc[2 * k + j], delta = sc[3 * k + j];
        const V ce = sc[10 * k + j] * sc[7 * k + j];
        for (int64_t row = blockIdx.x * (int64_t)kRows + tid / P; row < n; row += (int64_t)gridDim.x * kRows) {
            const int64_t e = row * k + j;
            const V gp = gamma * pp[e];
            const V dp = delta * p[e];
            const V num = (z[e] - gp) - dp;
            const V pn = safe_divide(num, alpha);
            p[e] = pn;
            const V cep = ce * pn;
            x[e] = x[e] + cep;
            const V vv = v[e];
            const V tmp = q[e];
            q[e] = safe_divide(vv, beta);
            v[e] = tmp * beta;
            const V zt = inv_diag ? vv * inv_diag[row] : vv;
            z[e] = safe_divide(zt, beta);
        }
    }
    // the ticket of grid_column_sums without the sums: every CTA has read ctl[1], the statuses and the
    // scalars
    __syncthreads();
    if (tid == 0) __threadfence();
    if (!fused::last_ticket(counter, &is_last)) return;
    const int32_t next = iter + 1;
    if (tid < k && !has_stopped(status[tid])) {
        // std::swap(gamma, beta) of the loop, by value
        const V beta = sc[k + tid];
        sc[k + tid] = sc[2 * k + tid];
        sc[2 * k + tid] = beta;
        status[tid] = tau_status(next, ctl, sc[6 * k + tid], sc[5 * k + tid]);
    }
    __syncthreads();
    if (tid == 0) {
        *counter = 0u;
        ctl[1] = next;
        if (all_stopped(k, status)) ctl[0] = 1;
    }
}

// ---- host side of the entry points ----------------------------------------------------------------
#define B200_FMM_REQUIRE(ctx, n, k)                                                    \
    B200_REQUIRE(ctx, "null argument");                                                \
    B200_REQUIRE((n) >= 0 && (k) >= 2 && (k) <= kMaxCols, "k must be in [2, 32]")

template <typename V>
b200_status init(b200_ctx* ctx, int64_t k, V* sc, uint8_t* status, int32_t* ctl, int64_t max_iters,
                 int32_t res_kind, int32_t iter_first, int32_t baseline, V factor)
{
    B200_FMM_REQUIRE(ctx, 0, k);
    B200_REQUIRE(sc && status && ctl, "null argument");
    init_kernel<V><<<1, kMaxCols, 0, ctx->stream>>>(k, sc, status, ctl, fused::clamp_iters(max_iters), res_kind,
                                                   iter_first, baseline, factor);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status lanczos(b200_ctx* ctx, int64_t n, int64_t k, V* v, const V* q, const V* inv_diag, V* sc,
                    const uint8_t* status, const int32_t* ctl, V* work)
{
    B200_FMM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl && work, "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
    V* partials = work + step_partials_offset<SubDotB>(ctx, k);
#define B200_LZ(PP)                                                                                     \
    lanczos_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, v, q, inv_diag, sc, status, ctl, partials, \
                                                              ctx->counters + kStepCounter)
    B200_MRHS_BY_LANES(P, B200_LZ)
#undef B200_LZ
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
b200_status update(b200_ctx* ctx, int64_t n, int64_t k, V* x, V* p0, V* p1, V* z, V* q, V* v, const V* inv_diag,
                   V* sc, uint8_t* status, int32_t* ctl)
{
    B200_FMM_REQUIRE(ctx, n, k);
    B200_REQUIRE(sc && status && ctl, "null argument");
    const int P = lanes_for(k);
    const int grid = rows_grid<kThreads>(n, P, step_cap(ctx));
#define B200_UP(PP)                                                                                    \
    update_kernel<V, PP><<<grid, kThreads, 0, ctx->stream>>>(n, k, x, p0, p1, z, q, v, inv_diag, sc, status, \
                                                             ctl, ctx->counters + kStepCounter)
    B200_MRHS_BY_LANES(P, B200_UP)
#undef B200_UP
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

#undef B200_FMM_REQUIRE

}  // namespace fminresm
}  // namespace b200

extern "C" {

#define B200_DEF_FMINRESM(V, VT)                                                                               \
    /* elements of `work` (value type): SpMV partials (k per CTA), then lanczos' (k per CTA) */                \
    int64_t b200_minres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                                     \
    {                                                                                                          \
        return b200::fminresm::work_size(ctx, k);                                                              \
    }                                                                                                          \
    b200_status b200_minres_mrhs_init_##V(b200_ctx* ctx, int64_t k, VT* sc, uint8_t* status, int32_t* ctl,      \
                                          int64_t max_iters, int32_t res_kind, int32_t iter_first,             \
                                          int32_t baseline, VT reduction_factor)                               \
    {                                                                                                          \
        return b200::fminresm::init<VT>(ctx, k, sc, status, ctl, max_iters, res_kind, iter_first, baseline,    \
                                        reduction_factor);                                                     \
    }                                                                                                          \
    b200_status b200_minres_mrhs_lanczos_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v, const VT* q,           \
                                             const VT* inv_diag, VT* sc, const uint8_t* status,                \
                                             const int32_t* ctl, VT* work)                                     \
    {                                                                                                          \
        return b200::fminresm::lanczos<VT>(ctx, n, k, v, q, inv_diag, sc, status, ctl, work);                  \
    }                                                                                                          \
    b200_status b200_minres_mrhs_update_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* p0, VT* p1, VT* z, \
                                            VT* q, VT* v, const VT* inv_diag, VT* sc, uint8_t* status,         \
                                            int32_t* ctl)                                                      \
    {                                                                                                          \
        return b200::fminresm::update<VT>(ctx, n, k, x, p0, p1, z, q, v, inv_diag, sc, status, ctl);           \
    }

B200_DEF_FMINRESM(f64, double)
B200_DEF_FMINRESM(f32, float)

/* c = A b - c for k = 2..32 columns of the row-major b and c (stride k) and dots[j] = b_j . c_j in one */
/* launch: the advanced SpMV with (alpha, beta) = (1, -1).  `work` provides the per-CTA partials        */
/* (b200_minres_mrhs_work_size elements); ctl may be NULL.  With num_rows == 0 the dots are 0.          */
#define B200_DEF_SPMV_SUB_MDOT(V, VT, I, IT)                                                                 \
    b200_status b200_csr_spmv_sub_mdot_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,          \
                                                 int64_t nnz, const IT* row_ptrs, const IT* col_idxs,        \
                                                 const VT* values, const VT* b, int64_t k, VT* c, VT* dots,  \
                                                 VT* work, const int32_t* ctl)                               \
    {                                                                                                        \
        return b200::mrhs::spmv_mdot<VT, IT, b200::mrhs::SubDotB>(ctx, num_rows, num_cols, nnz, row_ptrs,   \
                                                                  col_idxs, values, b, k, c, nullptr, dots, \
                                                                  nullptr, work, ctl);                      \
    }

B200_DEF_SPMV_SUB_MDOT(f64, double, i32, int32_t)
B200_DEF_SPMV_SUB_MDOT(f64, double, i64, int64_t)
B200_DEF_SPMV_SUB_MDOT(f32, float, i32, int32_t)
B200_DEF_SPMV_SUB_MDOT(f32, float, i64, int64_t)

}  // extern "C"
