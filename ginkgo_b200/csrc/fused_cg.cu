// Fused CG iteration for sm_90a: alpha / beta / rho are produced AND consumed on
// the device, three launches per iteration, no host round trip.
//
// The reference drives CG from the host with 8 launches and a blocking
// device->host copy per iteration (core/solver/cg.cpp:142-180: preconditioner
// apply, dot, norm2 + stopping check, step_1, SpMV, dot, step_2).  The same
// recurrence, regrouped around its two unavoidable global reductions:
//
//   step_p   p = z + (rho/prev_rho) p                                  reads 2n, writes n
//   spmv_dot q = A p  and  pq = p.q   (fused in the SpMV epilogue)     matrix + 2n
//   step_xr  alpha = rho/pq; x += alpha p; r -= alpha q; z = M^-1 r;
//            rho' = r.z; rr = r.r; stopping check (in the last CTA)    reads 5n, writes 3n
//
// = matrix + 13 n values per iteration (SURVEY.md section 8d), against 19 n for
// the reference's kernel sequence.  The stopping check is the reference's
// (core/stop/{combined,iteration,residual_norm}.cpp): Iteration and
// (Implicit)ResidualNorm in the user's order, ids 1 and 2, written into a
// device control block; once ctl[0] != 0 every kernel of later iterations is a
// no-op, so a CUDA graph of k iterations can be replayed blindly and the host
// only reads the control block every k iterations.
//
// Scalars  sc[8]: 0 rho, 1 prev_rho, 2 pq, 3 rr, 4 tau0 (baseline norm),
//                 5 threshold = reduction_factor * tau0, 6/7 local partial sums
//                 (multi-GPU: all-reduced between step_xr and finish)
// Control  ctl[0..4] of fused_common.cuh; 5..7 unused
#include "csr_launch.cuh"
#include "fused_common.cuh"

namespace b200 {
namespace fcg {

using namespace fused;  // kThreads, grid_sums, finish_scalars, set_threshold, ew_grid

template <typename V>
__global__ void __launch_bounds__(kThreads)
    step_p_kernel(int64_t n, V* __restrict__ p, const V* __restrict__ z, const V* __restrict__ sc,
                  const int32_t* __restrict__ ctl)
{
    if (ctl[0] != 0) return;
    const V rho = sc[0], prev = sc[1];
    const bool plain = (prev == V(0));
    const V beta = plain ? V(0) : rho / prev;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n;
         i += (int64_t)gridDim.x * kThreads) {
        const V zi = z[i];
        p[i] = plain ? zi : zi + beta * p[i];
    }
}

// INIT: r already holds b - A x; computes z, rho, rr (no x/r update) and the baseline.
template <typename V, bool INIT>
__global__ void __launch_bounds__(kThreads)
    step_xr_kernel(int64_t n, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ p,
                   const V* __restrict__ q, V* __restrict__ z, const V* __restrict__ inv_diag,
                   V* __restrict__ sc, int32_t* __restrict__ ctl, V* __restrict__ partials,
                   unsigned int* __restrict__ counter, int finalize, int baseline, V factor)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (!INIT && ctl[0] != 0) return;
    const int tid = threadIdx.x;
    const V pq = sc[2];
    const bool update = !INIT && pq != V(0);
    const V alpha = update ? sc[0] / pq : V(0);
    V a[2] = {V(0), V(0)};  // rho = r.z, rr = r.r
    for (int64_t i = blockIdx.x * (int64_t)kThreads + tid; i < n;
         i += (int64_t)gridDim.x * kThreads) {
        V ri = r[i];
        if (update) {
            x[i] += alpha * p[i];
            ri -= alpha * q[i];
            r[i] = ri;
        }
        const V zi = inv_diag ? ri * inv_diag[i] : ri;
        z[i] = zi;
        a[0] += ri * zi;
        a[1] += ri * ri;
    }
    if (!grid_sums(a, partials, counter, red, &is_last)) return;
    if (tid == 0) {
        if (!finalize) {
            sc[6] = a[0];
            sc[7] = a[1];
        } else {
            if (INIT) set_threshold(baseline, sqrt(a[1]), sc + 4, sc + 5, factor);
            finish_scalars(a[0], a[1], sc, ctl);
        }
    }
}

// multi-GPU: after the all-reduce of sc[6..7] (and of sc[2] for pq)
template <typename V, bool INIT>
__global__ void finish_kernel(V* sc, int32_t* ctl, int baseline, V factor)
{
    if (!INIT && ctl[0] != 0) return;
    if (INIT) {
        // baseline: 1 initial_resnorm, 2 absolute, 3 rhs_norm with sc[4] = global ||b||^2,
        // 0 rhs_norm with sc[4] = ||b|| already
        if (baseline == 3) sc[4] = sqrt(sc[4]);
        set_threshold(baseline, sqrt(sc[7]), sc + 4, sc + 5, factor);
    }
    finish_scalars(sc[6], sc[7], sc, ctl);
}

template <typename V>
__global__ void init_scalars_kernel(V* sc, int32_t* ctl, int32_t max_iters, int32_t res_kind,
                                    int32_t iter_first)
{
    sc[0] = V(1);  // becomes prev_rho = 1 after the INIT finish (reference cg::initialize)
    sc[1] = V(1);
    sc[2] = V(0);
    sc[3] = V(0);
    sc[6] = V(0);
    sc[7] = V(0);
    start_control(ctl, max_iters, res_kind, iter_first, -1);  // the INIT finish counts to 0
}

}  // namespace fcg
}  // namespace b200

struct b200_graph {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
};

extern "C" {

// ---- CUDA-graph helpers: capture a sequence of C-ABI calls on the context's stream -------
b200_status b200_graph_begin_capture(b200_ctx* ctx)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    B200_CUDA_CHECK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    return B200_OK;
}

b200_status b200_graph_end_capture(b200_ctx* ctx, b200_graph** out)
{
    B200_REQUIRE(ctx && out, "null argument");
    b200_graph* g = new b200_graph();
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &g->graph);
    if (e == cudaSuccess) e = cudaGraphInstantiate(&g->exec, g->graph, 0);
    if (e != cudaSuccess) {
        b200::set_error("graph capture failed: %s", cudaGetErrorString(e));
        if (g->graph) cudaGraphDestroy(g->graph);
        delete g;
        cudaGetLastError();
        return B200_ERR_CUDA;
    }
    *out = g;
    return B200_OK;
}

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    B200_REQUIRE(ctx && graph, "null argument");
    B200_CUDA_CHECK(cudaGraphLaunch(graph->exec, ctx->stream));
    return B200_OK;
}

void b200_graph_destroy(b200_graph* graph)
{
    if (!graph) return;
    if (graph->exec) cudaGraphExecDestroy(graph->exec);
    if (graph->graph) cudaGraphDestroy(graph->graph);
    delete graph;
}

#define B200_DEF_FCG(V, VT)                                                                      \
    /* elements of `work` (value type) the fused kernels need for a matrix of this size */       \
    int64_t b200_cg_fused_work_size_##V(const b200_ctx* ctx)                                     \
    {                                                                                            \
        return b200::fused::work_size(ctx);                                                      \
    }                                                                                            \
    b200_status b200_cg_fused_init_##V(                                                          \
        b200_ctx* ctx, int64_t n, const VT* r, VT* z, VT* p, VT* q, const VT* inv_diag, VT* sc,  \
        int32_t* ctl, VT* work, int64_t max_iters, int32_t res_kind, int32_t iter_first,         \
        int32_t baseline, VT reduction_factor, int32_t finalize)                                 \
    {                                                                                            \
        B200_REQUIRE(ctx && sc && ctl && work, "null argument");                                 \
        b200::fcg::init_scalars_kernel<VT><<<1, 1, 0, ctx->stream>>>(                            \
            sc, ctl, b200::fused::clamp_iters(max_iters), res_kind, iter_first);                 \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        B200_CUDA_CHECK(cudaMemsetAsync(p, 0, sizeof(VT) * n, ctx->stream));                     \
        B200_CUDA_CHECK(cudaMemsetAsync(q, 0, sizeof(VT) * n, ctx->stream));                     \
        const int grid = b200::fcg::ew_grid(ctx, n);                                             \
        b200::fcg::step_xr_kernel<VT, true><<<grid, b200::fcg::kThreads, 0, ctx->stream>>>(      \
            n, nullptr, const_cast<VT*>(r), p, q, z, inv_diag, sc, ctl,                          \
            b200::fused::step_partials(ctx, work), ctx->counters + b200::kStepCounter, finalize, \
            baseline, reduction_factor);                                                         \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        return B200_OK;                                                                          \
    }                                                                                            \
    b200_status b200_cg_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* z,           \
                                         const VT* sc, const int32_t* ctl)                       \
    {                                                                                            \
        const int grid = b200::fcg::ew_grid(ctx, n);                                             \
        b200::fcg::step_p_kernel<VT><<<grid, b200::fcg::kThreads, 0, ctx->stream>>>(n, p, z, sc, \
                                                                                    ctl);        \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        return B200_OK;                                                                          \
    }                                                                                            \
    b200_status b200_cg_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r, const VT* p,   \
                                          const VT* q, VT* z, const VT* inv_diag, VT* sc,        \
                                          int32_t* ctl, VT* work, int32_t finalize)              \
    {                                                                                            \
        const int grid = b200::fcg::ew_grid(ctx, n);                                             \
        b200::fcg::step_xr_kernel<VT, false><<<grid, b200::fcg::kThreads, 0, ctx->stream>>>(     \
            n, x, r, p, q, z, inv_diag, sc, ctl, b200::fused::step_partials(ctx, work),          \
            ctx->counters + b200::kStepCounter, finalize, 0, VT(0));                             \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        return B200_OK;                                                                          \
    }                                                                                            \
    b200_status b200_cg_fused_finish_##V(b200_ctx* ctx, VT* sc, int32_t* ctl, int32_t init,      \
                                         int32_t baseline, VT reduction_factor)                  \
    {                                                                                            \
        if (init)                                                                                \
            b200::fcg::finish_kernel<VT, true><<<1, 1, 0, ctx->stream>>>(sc, ctl, baseline,      \
                                                                         reduction_factor);      \
        else                                                                                     \
            b200::fcg::finish_kernel<VT, false><<<1, 1, 0, ctx->stream>>>(sc, ctl, baseline,     \
                                                                          reduction_factor);     \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        return B200_OK;                                                                          \
    }

B200_DEF_FCG(f64, double)
B200_DEF_FCG(f32, float)

/* c = A b and *dot_out = b . c in one launch (square A; b is also the dot operand).  `work`  */
/* provides the per-CTA partials (b200_cg_fused_work_size elements); ctl may be NULL.  With   */
/* num_rows == 0 the dot is 0.                                                                */
#define B200_DEF_SPMV_DOT(V, VT, I, IT)                                                          \
    b200_status b200_csr_spmv_dot_##V##_##I(                                                     \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,            \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,      \
        VT* c, VT* dot_out, VT* work, const int32_t* ctl)                                        \
    {                                                                                            \
        return b200::csr::launch_spmv_dot<VT, IT, false, b200::csr::kDotB>(                      \
            ctx, plan, num_rows, nnz, row_ptrs, col_idxs, values, nullptr, b, nullptr, c,        \
            nullptr, dot_out, nullptr, work, ctl);                                               \
    }

B200_DEF_SPMV_DOT(f64, double, i32, int32_t)
B200_DEF_SPMV_DOT(f64, double, i64, int64_t)
B200_DEF_SPMV_DOT(f32, float, i32, int32_t)
B200_DEF_SPMV_DOT(f32, float, i64, int64_t)

}  // extern "C"
