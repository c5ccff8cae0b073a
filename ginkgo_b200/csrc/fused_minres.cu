// Fused MINRES iteration for sm_90a: the Lanczos scalars, the Givens rotations and the stopping check
// are produced AND consumed on the device, three launches per iteration, no host round trip.
//
// The reference drives MINRES from the host with about ten launches and a blocking device->host read
// of the stopping flags per iteration (core/solver/minres.cpp:199-285: criterion check, advanced SpMV,
// dot, sub_scaled, preconditioner, dot, minres::step_1, minres::step_2).  The same recurrence,
// regrouped around its two global reductions (d is the inverted diagonal of a scalar Jacobi
// preconditioner, or absent):
//
//   spmv_sub_dot  v = A z - v  and  alpha = z.v   (advanced SpMV, dot in its epilogue)  matrix + 3n
//   lanczos       v -= alpha q;  beta = v.(d v);  minres::step_1 in the last CTA        reads 3n, writes n
//   update        minres::step_2 with z~ = d v recomputed and without q_prev; the last
//                 CTA swaps gamma / beta, counts the iteration and checks the next one   reads 7n, writes 5n
//
// = matrix + 19 n values per iteration, against 26 n for the reference's kernel sequence: q_prev is
// written there and never read, and z~ = d v is stored only to be read back by step_2.  Element-wise
// arithmetic and the scalar recurrence are those of krylov_steps.cu (minres_step_1 / minres_step_2),
// operation for operation, so given the same sums every vector and scalar has the loop's bits.
//
// p and p_prev trade places every iteration (a pointer swap in the loop).  A graph bakes pointers in,
// so update takes both buffers and picks their roles from the parity of the iteration counter ctl[1]
// it reads at entry; the last CTA increments the counter only after every other CTA took its ticket.
// One graph serves every batch whatever the parity of check_every.
//
// Stopping is the reference's with the implicit residual norm: Iteration and ImplicitResidualNorm
// (sqrt|tau| <= factor * tau0) in the user's order with ids 1 and 2 (fused_common.cuh), checked by
// init for iteration 0 and at the end of every update for the next iteration -- the loop's order
// (check, step_1, step_2, check).  Once ctl[0] != 0 every kernel is a no-op at entry, so a graph of k
// iterations can be replayed past the stop.
//
// Scalars  sc[16]: 0 alpha, 1 beta, 2 gamma, 3 delta, 4 tau0 (baseline norm), 5 threshold =
//                  reduction_factor * tau0, 6 tau, 7 eta, 8 eta_next, 9 cos_prev, 10 cos, 11 sin_prev,
//                  12 sin
// Control  ctl[0..4] of fused_common.cuh (res_kind 0 or 2); 5..7 unused, cleared by init
#include "csr_launch.cuh"
#include "fused_minres.cuh"

namespace b200 {
namespace fminres {

using namespace fused;  // kThreads, grid_sums, last_ticket, criteria_status, set_threshold, ew_grid

template <typename V>
__global__ void __launch_bounds__(kThreads)
    lanczos_kernel(int64_t n, V* __restrict__ v, const V* __restrict__ q, const V* __restrict__ inv_diag,
                   V* __restrict__ sc, const int32_t* __restrict__ ctl, V* __restrict__ partials,
                   unsigned int* __restrict__ counter)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    const V alpha = sc[0];
    const bool sub = alpha != V(0);  // Dense::sub_scaled skips a zero scalar
    V a[1] = {V(0)};
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        V vi = v[i];
        if (sub) {
            vi -= alpha * q[i];
            v[i] = vi;
        }
        const V zt = inv_diag ? vi * inv_diag[i] : vi;
        a[0] += vi * zt;
    }
    // every CTA read alpha before it took its ticket: the last one may overwrite the scalars
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (threadIdx.x == 0) step_1(a[0], sc, 1);
}

template <typename V>
__global__ void __launch_bounds__(kThreads)
    update_kernel(int64_t n, V* __restrict__ x, V* __restrict__ p0, V* __restrict__ p1, V* __restrict__ z,
                  V* __restrict__ q, V* __restrict__ v, const V* __restrict__ inv_diag, V* __restrict__ sc,
                  int32_t* __restrict__ ctl, unsigned int* __restrict__ counter)
{
    __shared__ bool is_last;
    if (ctl[0] != 0) return;
    const int tid = threadIdx.x;
    const int32_t iter = ctl[1];
    // the loop swaps p and p_prev before step_2: iteration k writes p1 when k is even, p0 when odd
    V* __restrict__ p = (iter & 1) ? p0 : p1;
    const V* __restrict__ pp = (iter & 1) ? p1 : p0;
    const V alpha = sc[0], beta = sc[1], gamma = sc[2], delta = sc[3];
    const V ce = sc[10] * sc[7];
    for (int64_t i = blockIdx.x * (int64_t)kThreads + tid; i < n; i += (int64_t)gridDim.x * kThreads) {
        const V gp = gamma * pp[i];
        const V dp = delta * p[i];
        const V num = (z[i] - gp) - dp;
        const V pn = safe_divide(num, alpha);
        p[i] = pn;
        const V cep = ce * pn;
        x[i] = x[i] + cep;
        const V vv = v[i];
        const V tmp = q[i];
        q[i] = safe_divide(vv, beta);
        v[i] = tmp * beta;
        const V zt = inv_diag ? vv * inv_diag[i] : vv;
        z[i] = safe_divide(zt, beta);
    }
    // the ticket of fused::grid_sums without the sums: every CTA has read ctl[1] and the scalars
    __syncthreads();
    if (tid == 0) __threadfence();
    if (!last_ticket(counter, &is_last) || tid != 0) return;
    *counter = 0u;
    // std::swap(gamma, beta) of the loop, by value
    sc[1] = gamma;
    sc[2] = beta;
    const int32_t next = iter + 1;
    ctl[1] = next;
    const V tau = sc[6];
    ctl[0] = criteria_status(
        next, ctl, [&](int32_t) { return sqrt(fabs(tau)) <= sc[5]; }, kFinalizedMask);
}

// sc[4] holds the baseline norm (||b|| or ||r0||, from the host) unless it is absolute
template <typename V>
__global__ void init_kernel(V* sc, int32_t* ctl, int32_t max_iters, int32_t res_kind, int32_t iter_first,
                            int32_t baseline, V factor)
{
    set_threshold(baseline, sc[4], sc + 4, sc + 5, factor);  // baseline 1: the host put ||r0|| in sc[4]
    start_control(ctl, max_iters, res_kind, iter_first, 0);
    ctl[5] = ctl[6] = ctl[7] = 0;
    const V tau = sc[6];
    ctl[0] = criteria_status(
        0, ctl, [&](int32_t) { return sqrt(fabs(tau)) <= sc[5]; }, kFinalizedMask);
}

// the (alpha, beta) = (1, -1) of the advanced SpMV, as device scalars
__device__ double one_neg_one_f64[2] = {1.0, -1.0};
__device__ float one_neg_one_f32[2] = {1.0f, -1.0f};

}  // namespace fminres
}  // namespace b200

extern "C" {

#define B200_DEF_FMINRES(V, VT)                                                                   \
    /* elements of `work` (value type) the fused kernels need */                                  \
    int64_t b200_minres_fused_work_size_##V(const b200_ctx* ctx)                                  \
    {                                                                                             \
        return b200::fused::work_size(ctx);                                                       \
    }                                                                                             \
    b200_status b200_minres_fused_init_##V(b200_ctx* ctx, VT* sc, int32_t* ctl, int64_t max_iters, \
                                           int32_t res_kind, int32_t iter_first, int32_t baseline, \
                                           VT reduction_factor)                                   \
    {                                                                                             \
        B200_REQUIRE(ctx && sc && ctl, "null argument");                                          \
        b200::fminres::init_kernel<VT><<<1, 1, 0, ctx->stream>>>(                                 \
            sc, ctl, b200::fused::clamp_iters(max_iters), res_kind, iter_first, baseline,         \
            reduction_factor);                                                                    \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_minres_fused_lanczos_##V(b200_ctx* ctx, int64_t n, VT* v, const VT* q,       \
                                              const VT* inv_diag, VT* sc, const int32_t* ctl,     \
                                              VT* work)                                           \
    {                                                                                             \
        B200_REQUIRE(ctx && sc && ctl && work, "null argument");                                  \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fminres::lanczos_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(       \
            n, v, q, inv_diag, sc, ctl, b200::fused::step_partials(ctx, work),                    \
            ctx->counters + b200::kStepCounter);                                                  \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }                                                                                             \
    b200_status b200_minres_fused_update_##V(b200_ctx* ctx, int64_t n, VT* x, VT* p0, VT* p1,     \
                                             VT* z, VT* q, VT* v, const VT* inv_diag, VT* sc,     \
                                             int32_t* ctl)                                        \
    {                                                                                             \
        B200_REQUIRE(ctx && sc && ctl, "null argument");                                          \
        const int grid = b200::fused::ew_grid(ctx, n);                                            \
        b200::fminres::update_kernel<VT><<<grid, b200::fused::kThreads, 0, ctx->stream>>>(        \
            n, x, p0, p1, z, q, v, inv_diag, sc, ctl, ctx->counters + b200::kStepCounter);        \
        B200_LAUNCH_CHECK(ctx);                                                                   \
        return B200_OK;                                                                           \
    }

B200_DEF_FMINRES(f64, double)
B200_DEF_FMINRES(f32, float)

/* c = A b - c and *dot_out = b . c in one launch: the advanced SpMV with (alpha, beta) = (1, -1),  */
/* the dot in its epilogue.  Arguments, plan, work and ctl as for b200_csr_spmv_dot_*.               */
#define B200_DEF_SPMV_SUB_DOT(V, VT, I, IT)                                                       \
    b200_status b200_csr_spmv_sub_dot_##V##_##I(                                                  \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,             \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,       \
        VT* c, VT* dot_out, VT* work, const int32_t* ctl)                                         \
    {                                                                                             \
        VT* ab = nullptr;                                                                         \
        B200_CUDA_CHECK(cudaGetSymbolAddress((void**)&ab, b200::fminres::one_neg_one_##V));       \
        return b200::csr::launch_spmv_dot<VT, IT, true, b200::csr::kDotB>(                        \
            ctx, plan, num_rows, nnz, row_ptrs, col_idxs, values, ab, b, ab + 1, c, nullptr,      \
            dot_out, nullptr, work, ctl);                                                         \
    }

B200_DEF_SPMV_SUB_DOT(f64, double, i32, int32_t)
B200_DEF_SPMV_SUB_DOT(f64, double, i64, int64_t)
B200_DEF_SPMV_SUB_DOT(f32, float, i32, int32_t)
B200_DEF_SPMV_SUB_DOT(f32, float, i64, int64_t)

}  // extern "C"
