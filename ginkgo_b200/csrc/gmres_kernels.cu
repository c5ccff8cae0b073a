// GMRES kernels -- replaces gko::kernels::cuda::{common_gmres,gmres}::*
// (reference common/unified/solver/common_gmres_kernels.cpp:25-160 and
// common/unified/solver/gmres_kernels.cpp:25-120); arithmetic contract
// reference/solver/common_gmres_kernels.cpp:27-195 and
// reference/solver/gmres_kernels.cpp:27-99.
//
// Layouts (core/solver/gmres.cpp:342-362): krylov_bases is a tall
// ((krylov_dim+1)*rows) x cols Dense, basis i = rows [i*rows, (i+1)*rows);
// hessenberg_iter is the (iter+2) x cols column of the current iteration.
#include "elementwise.cuh"
#include "gmres_common.cuh"

namespace b200 {
namespace gmres {

template <typename V>
b200_status initialize(b200_ctx* ctx, int64_t rows, int64_t cols, int64_t krylov_dim, const V* b,
                       int64_t bs, V* residual, int64_t rs, V* gsin, int64_t sins, V* gcos,
                       int64_t coss, uint8_t* stop)
{
    // rows of work: `rows` residual rows, then krylov_dim givens rows, then 1 status row
    return launch_ew(ctx, rows + krylov_dim + 1, cols, [=] __device__(int64_t i, int64_t j) {
        if (i < rows) {
            residual[i * rs + j] = b[i * bs + j];
        } else if (i < rows + krylov_dim) {
            const int64_t k = i - rows;
            gsin[k * sins + j] = V(0);
            gcos[k * coss + j] = V(0);
        } else {
            stop[j] = 0;
        }
    });
}

template <typename V>
b200_status restart(b200_ctx* ctx, int64_t rows, int64_t cols, const V* residual, int64_t rs,
                    const V* residual_norm, V* rnc, V* krylov, int64_t ks,
                    uint64_t* final_iter_nums)
{
    return launch_ew(ctx, rows + 1, cols, [=] __device__(int64_t i, int64_t j) {
        if (i == rows) {
            rnc[j] = residual_norm[j];
            final_iter_nums[j] = 0;
        } else {
            krylov[i * ks + j] = residual[i * rs + j] / residual_norm[j];
        }
    });
}

// One thread per right-hand side: k stored Givens rotations applied to the new
// Hessenberg column, new (cos, sin) from a scaled hypot, residual-norm update.
template <typename V>
__global__ void hessenberg_qr_kernel(int64_t cols, V* gsin, int64_t sins, V* gcos, int64_t coss,
                                     V* residual_norm, V* rnc, int64_t rncs, V* hess, int64_t hs,
                                     int64_t iter, uint64_t* final_iter_nums, const uint8_t* stop)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= cols || has_stopped(stop[i])) return;
    givens_column(i, gsin, sins, gcos, coss, residual_norm, rnc, rncs, hess, hs, iter, final_iter_nums);
}

// Back substitution on the transposed-stored Hessenberg:
// H(i,j) lives at hessenberg[j * hs + i * cols + k]  (core/solver/gmres.cpp:351-362)
template <typename V>
__global__ void solve_krylov_kernel(int64_t cols, const V* rnc, int64_t rncs, const V* hess,
                                    int64_t hs, V* y, int64_t ys, const uint64_t* final_iter_nums,
                                    const uint8_t* stop)
{
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= cols || is_finalized(stop[k])) return;
    const int64_t n = (int64_t)final_iter_nums[k];
    for (int64_t i = n - 1; i >= 0; --i) {
        V temp = rnc[i * rncs + k];
        for (int64_t j = i + 1; j < n; ++j) temp -= hess[j * hs + i * cols + k] * y[j * ys + k];
        y[i * ys + k] = temp / hess[i * hs + i * cols + k];
    }
}

template <typename V>
__global__ void multi_axpy_status_kernel(int64_t cols, uint8_t* stop)
{
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < cols && has_stopped(stop[j])) stop[j] |= kFinalizedMask;
}

template <typename V>
b200_status multi_axpy(b200_ctx* ctx, int64_t rows, int64_t cols, const V* krylov, int64_t ks,
                       const V* y, int64_t ys, V* out, int64_t os, const uint64_t* final_iter_nums,
                       uint8_t* stop)
{
    b200_status st = launch_ew(ctx, rows, cols, [=] __device__(int64_t i, int64_t k) {
        if (is_finalized(stop[k])) return;
        const int64_t n = (int64_t)final_iter_nums[k];
        V acc = V(0);
        for (int64_t j = 0; j < n; ++j) acc += krylov[(i + j * rows) * ks + k] * y[j * ys + k];
        out[i * os + k] = acc;
    });
    if (st != B200_OK || cols == 0) return st;
    multi_axpy_status_kernel<V><<<(unsigned)ceildiv(cols, 256), 256, 0, ctx->stream>>>(cols, stop);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

// multi_dot: h(i,k) = sum_r basis_i(r,k) * w(r,k) for all i < num_bases in ONE pass.
// grid.x CTAs each own a strided set of row chunks; a thread keeps w(r) in a
// register and walks the bases, so w is read once and every basis once.
constexpr int kMdThreads = 256;
constexpr int kMdMaxBases = 16;  // bases handled per sweep (register accumulators)

// VW consecutive rows per thread (one 16-byte load per basis when VW * sizeof(V) == 16):
// 17 x 16 B in flight per thread, enough memory-level parallelism to stream HBM -- with one
// 4-byte element per load the kernel stayed far below the HBM roofline.
template <typename V, int VW>
struct alignas(sizeof(V) * VW) md_vec {
    V v[VW];
};

// CTL: the fused GMRES iteration's instance, a no-op once its control word ctl[0] says it stopped.
template <typename V, int VW, bool CTL = false>
__global__ void __launch_bounds__(kMdThreads)
    multi_dot_kernel(int64_t rows, int64_t cols, int64_t num_bases, const V* __restrict__ krylov,
                     int64_t ks, const V* __restrict__ w, int64_t wstride, V* __restrict__ partials,
                     unsigned int* __restrict__ counter, V* __restrict__ hcol, int64_t hs,
                     const int32_t* __restrict__ ctl = nullptr)
{
    __shared__ V red[32];
    __shared__ bool is_last;
    if (CTL && ctl[0] != 0) return;
    const int tid = threadIdx.x;
    using vec = md_vec<V, VW>;
    for (int64_t i0 = 0; i0 < num_bases; i0 += kMdMaxBases) {
        const int nb = (int)((num_bases - i0) < kMdMaxBases ? (num_bases - i0) : kMdMaxBases);
        for (int64_t k = 0; k < cols; ++k) {
            V acc[kMdMaxBases];
#pragma unroll
            for (int q = 0; q < kMdMaxBases; ++q) acc[q] = V(0);
            for (int64_t r = (blockIdx.x * (int64_t)kMdThreads + tid) * VW; r < rows;
                 r += (int64_t)gridDim.x * kMdThreads * VW) {
                vec wv, kv[kMdMaxBases];
                if (VW == 1) {
                    wv.v[0] = w[r * wstride + k];
#pragma unroll
                    for (int q = 0; q < kMdMaxBases; ++q)
                        kv[q].v[0] = q < nb ? krylov[((i0 + q) * rows + r) * ks + k] : V(0);
                } else {  // ks == wstride == 1, cols == 1, rows % VW == 0, aligned (host checks)
                    wv = *reinterpret_cast<const vec*>(w + r);
#pragma unroll
                    for (int q = 0; q < kMdMaxBases; ++q) {
                        if (q < nb)
                            kv[q] = *reinterpret_cast<const vec*>(krylov + (i0 + q) * rows + r);
                    }
                }
#pragma unroll
                for (int q = 0; q < kMdMaxBases; ++q) {
                    if (q < nb) {
#pragma unroll
                        for (int e = 0; e < VW; ++e) acc[q] += kv[q].v[e] * wv.v[e];
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < kMdMaxBases; ++q) {
                if (q < nb) {
                    const V s = block_sum(acc[q], red);
                    if (tid == 0) partials[((i0 + q) * cols + k) * gridDim.x + blockIdx.x] = s;
                }
            }
        }
    }
    if (tid == 0) {
        __threadfence();
        const unsigned int ticket = atomicAdd(counter, 1u);
        is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) {
        __threadfence();
        // one warp per (basis, column): lanes stride over the per-CTA partials, fixed shuffle
        // tree -- deterministic, and not a serial chain of gridDim.x dependent L2 reads
        const int lane = tid & 31, wrp = tid >> 5;
        for (int64_t e = wrp; e < num_bases * cols; e += kMdThreads / 32) {
            V s = V(0);
            for (int g = lane; g < (int)gridDim.x; g += 32) s += __ldcg(partials + e * gridDim.x + g);
            s = warp_sum(s);
            if (lane == 0) {
                const int64_t i = e / cols, k = e - i * cols;
                hcol[i * hs + k] = s;
            }
        }
        if (tid == 0) *counter = 0u;
    }
}

template <typename V>
b200_status multi_dot(b200_ctx* ctx, int64_t rows, int64_t cols, int64_t num_bases, const V* krylov,
                      int64_t ks, const V* w, int64_t ws, V* hcol, int64_t hs)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    if (num_bases <= 0 || cols <= 0) return B200_OK;
    constexpr int kVW = 16 / (int)sizeof(V);
    const bool vec_ok = cols == 1 && ks == 1 && ws == 1 && rows % kVW == 0 &&
                        ((uintptr_t)krylov % 16) == 0 && ((uintptr_t)w % 16) == 0;
    // exactly one resident wave: the kernel keeps 16 accumulators + 17 vector loads per thread (128
    // registers -> 2 CTAs per SM); the old cap of 3 CTAs per SM left a half-empty second wave behind
    // the first
    static thread_local int per_sm[2] = {0, 0};
    int& occ = per_sm[vec_ok ? 1 : 0];
    if (occ == 0) {
        if (vec_ok)
            B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, multi_dot_kernel<V, kVW>,
                                                                          kMdThreads, 0));
        else
            B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, multi_dot_kernel<V, 1>,
                                                                          kMdThreads, 0));
        if (occ < 1) occ = 1;
    }
    int grid = (int)ceildiv(rows, (int64_t)kMdThreads * (vec_ok ? kVW : 1) * 2);
    if (grid > ctx->num_sms * occ) grid = ctx->num_sms * occ;
    if (grid < 1) grid = 1;
    V* partials = (V*)ctx->scratch(sizeof(V) * grid * num_bases * cols);
    if (!partials) return B200_ERR_ALLOC;
    if (vec_ok)
        multi_dot_kernel<V, kVW><<<grid, kMdThreads, 0, ctx->stream>>>(
            rows, cols, num_bases, krylov, ks, w, ws, partials, ctx->counters, hcol, hs);
    else
        multi_dot_kernel<V, 1><<<grid, kMdThreads, 0, ctx->stream>>>(
            rows, cols, num_bases, krylov, ks, w, ws, partials, ctx->counters, hcol, hs);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

// h[i] = v_i . w for i < num_bases, one right-hand side, skipped once ctl[0] != 0: the multi-dot of the
// fused GMRES iteration (CGS / CGS2).  The per-CTA partials live in the caller's workspace at
// fused_md_offset (the pointer is baked into a graph, ctx->scratch may move), at most
// kFusedMdCtasPerSm CTAs per SM.
template <typename V>
b200_status fused_multi_dot(b200_ctx* ctx, int64_t rows, int64_t num_bases, const V* krylov, const V* w,
                            V* hcol, const int32_t* ctl, V* work)
{
    B200_REQUIRE(ctx && krylov && w && hcol && ctl && work, "null argument");
    if (num_bases <= 0) return B200_OK;
    constexpr int kVW = 16 / (int)sizeof(V);
    const bool vec_ok = rows % kVW == 0 && ((uintptr_t)krylov % 16) == 0 && ((uintptr_t)w % 16) == 0;
    static thread_local int per_sm[2] = {0, 0};
    int& occ = per_sm[vec_ok ? 1 : 0];
    if (occ == 0) {
        if (vec_ok)
            B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, multi_dot_kernel<V, kVW, true>,
                                                                          kMdThreads, 0));
        else
            B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, multi_dot_kernel<V, 1, true>,
                                                                          kMdThreads, 0));
        occ = occ < 1 ? 1 : (occ > kFusedMdCtasPerSm ? kFusedMdCtasPerSm : occ);
    }
    int grid = (int)ceildiv(rows, (int64_t)kMdThreads * (vec_ok ? kVW : 1) * 2);
    if (grid > ctx->num_sms * occ) grid = ctx->num_sms * occ;
    if (grid < 1) grid = 1;
    V* partials = work + fused_md_offset(ctx);
    if (vec_ok)
        multi_dot_kernel<V, kVW, true><<<grid, kMdThreads, 0, ctx->stream>>>(
            rows, 1, num_bases, krylov, 1, w, 1, partials, ctx->counters + kMultiDotCounter, hcol, 1, ctl);
    else
        multi_dot_kernel<V, 1, true><<<grid, kMdThreads, 0, ctx->stream>>>(
            rows, 1, num_bases, krylov, 1, w, 1, partials, ctx->counters + kMultiDotCounter, hcol, 1, ctl);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

}  // namespace gmres
}  // namespace b200

extern "C" {

#define B200_DEF_GMRES(V, VT)                                                                  \
    b200_status b200_common_gmres_initialize_##V(                                              \
        b200_ctx* ctx, int64_t rows, int64_t cols, int64_t krylov_dim, const VT* b,            \
        int64_t bs, VT* residual, int64_t rs, VT* gsin, int64_t sins, VT* gcos, int64_t coss,  \
        uint8_t* stop)                                                                         \
    {                                                                                          \
        return b200::gmres::initialize<VT>(ctx, rows, cols, krylov_dim, b, bs, residual, rs,   \
                                           gsin, sins, gcos, coss, stop);                      \
    }                                                                                          \
    b200_status b200_common_gmres_hessenberg_qr_##V(                                           \
        b200_ctx* ctx, int64_t cols, VT* gsin, int64_t sins, VT* gcos, int64_t coss,           \
        VT* residual_norm, VT* rnc, int64_t rncs, VT* hess, int64_t hs, int64_t iter,          \
        uint64_t* final_iter_nums, const uint8_t* stop)                                        \
    {                                                                                          \
        if (cols <= 0) return B200_OK;                                                         \
        b200::gmres::hessenberg_qr_kernel<VT>                                                  \
            <<<(unsigned)b200::ceildiv(cols, 128), 128, 0, ctx->stream>>>(                     \
                cols, gsin, sins, gcos, coss, residual_norm, rnc, rncs, hess, hs, iter,        \
                final_iter_nums, stop);                                                        \
        B200_LAUNCH_CHECK(ctx);                                                                \
        return B200_OK;                                                                        \
    }                                                                                          \
    b200_status b200_common_gmres_solve_krylov_##V(                                            \
        b200_ctx* ctx, int64_t cols, const VT* rnc, int64_t rncs, const VT* hess, int64_t hs,  \
        VT* y, int64_t ys, const uint64_t* final_iter_nums, const uint8_t* stop)               \
    {                                                                                          \
        if (cols <= 0) return B200_OK;                                                         \
        b200::gmres::solve_krylov_kernel<VT>                                                   \
            <<<(unsigned)b200::ceildiv(cols, 128), 128, 0, ctx->stream>>>(                     \
                cols, rnc, rncs, hess, hs, y, ys, final_iter_nums, stop);                      \
        B200_LAUNCH_CHECK(ctx);                                                                \
        return B200_OK;                                                                        \
    }                                                                                          \
    b200_status b200_gmres_restart_##V(b200_ctx* ctx, int64_t rows, int64_t cols,              \
                                       const VT* residual, int64_t rs,                         \
                                       const VT* residual_norm, VT* rnc, VT* krylov,           \
                                       int64_t ks, uint64_t* final_iter_nums)                  \
    {                                                                                          \
        return b200::gmres::restart<VT>(ctx, rows, cols, residual, rs, residual_norm, rnc,     \
                                        krylov, ks, final_iter_nums);                          \
    }                                                                                          \
    b200_status b200_gmres_multi_axpy_##V(b200_ctx* ctx, int64_t rows, int64_t cols,           \
                                          const VT* krylov, int64_t ks, const VT* y,           \
                                          int64_t ys, VT* out, int64_t os,                     \
                                          const uint64_t* final_iter_nums, uint8_t* stop)      \
    {                                                                                          \
        return b200::gmres::multi_axpy<VT>(ctx, rows, cols, krylov, ks, y, ys, out, os,        \
                                           final_iter_nums, stop);                             \
    }                                                                                          \
    b200_status b200_gmres_multi_dot_##V(b200_ctx* ctx, int64_t rows, int64_t cols,            \
                                         int64_t num_bases, const VT* krylov, int64_t ks,      \
                                         const VT* next_krylov, int64_t ns, VT* hcol,          \
                                         int64_t hs)                                           \
    {                                                                                          \
        return b200::gmres::multi_dot<VT>(ctx, rows, cols, num_bases, krylov, ks, next_krylov, \
                                          ns, hcol, hs);                                       \
    }                                                                                          \
    b200_status b200_gmres_fused_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t num_bases,    \
                                               const VT* krylov, const VT* w, VT* hcol,        \
                                               const int32_t* ctl, VT* work)                   \
    {                                                                                          \
        return b200::gmres::fused_multi_dot<VT>(ctx, n, num_bases, krylov, w, hcol, ctl,       \
                                                work);                                         \
    }

B200_DEF_GMRES(f64, double)
B200_DEF_GMRES(f32, float)

}  // extern "C"
