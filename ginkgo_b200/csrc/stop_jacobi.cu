// Stopping-criterion checks and Jacobi preconditioner application.
//
// residual_norm / implicit_residual_norm / set_all_statuses replace
// gko::kernels::cuda::{residual_norm,implicit_residual_norm,set_all_statuses}
// (reference common/cuda_hip/stop/residual_norm_kernels.cpp:33-170,
//  contract reference/stop/residual_norm_kernels.cpp:27-92).  The reference
// launches an init kernel + the check kernel and then does TWO blocking 1-byte
// device->host copies; here one kernel writes both flags into a pinned host
// mailbox and a single stream synchronise hands them back.
//
// Jacobi: scalar apply / invert_diagonal replace
// common/unified/preconditioner/jacobi_kernels.cpp:39-105; block apply replaces
// common/cuda_hip/preconditioner/jacobi_{simple,advanced}_apply_kernels
// (contract reference/preconditioner/jacobi_kernels.cpp:419-592).
#include <stdlib.h>

#include "elementwise.cuh"
#include "jacobi_precision.cuh"

namespace b200 {
namespace stop {

template <typename V, bool IMPLICIT>
__global__ void residual_norm_kernel(int64_t cols, const V* tau, const V* orig_tau, V goal,
                                     uint8_t id, bool set_finalized, uint8_t* stop,
                                     uint8_t* device_storage, uint8_t* mailbox)
{
    // single CTA; cols is the number of right-hand sides (small)
    __shared__ int not_conv, changed;
    if (threadIdx.x == 0) {
        not_conv = 0;
        changed = 0;
    }
    __syncthreads();
    for (int64_t i = threadIdx.x; i < cols; i += blockDim.x) {
        const V t = IMPLICIT ? sqrt(fabs(tau[i])) : tau[i];
        uint8_t s = stop[i];
        if (t <= goal * orig_tau[i]) {
            if (!has_stopped(s)) {
                s |= kConvergedMask | (id & kIdMask);
                if (set_finalized) s |= kFinalizedMask;
                stop[i] = s;
            }
            changed = 1;  // reference sets one_changed even if already stopped
        }
        if (!has_stopped(s)) not_conv = 1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint8_t all_conv = not_conv ? 0 : 1;
        const uint8_t one_ch = changed ? 1 : 0;
        if (device_storage) {
            device_storage[0] = all_conv;
            device_storage[1] = one_ch;
        }
        mailbox[0] = all_conv;
        mailbox[1] = one_ch;
    }
}

template <typename V, bool IMPLICIT>
b200_status check(b200_ctx* ctx, int64_t cols, const V* tau, const V* orig_tau, V goal, uint8_t id,
                  int32_t set_finalized, uint8_t* stop, uint8_t* device_storage,
                  int32_t* all_converged, int32_t* one_changed)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    B200_REQUIRE(cols >= 0, "negative size");
    B200_REQUIRE(all_converged && one_changed, "null output");
    uint8_t* dev_view = nullptr;
    B200_CUDA_CHECK(cudaHostGetDevicePointer((void**)&dev_view, ctx->pinned, 0));
    residual_norm_kernel<V, IMPLICIT><<<1, 256, 0, ctx->stream>>>(
        cols, tau, orig_tau, goal, id, set_finalized != 0, stop, device_storage, dev_view);
    B200_LAUNCH_CHECK(ctx);
    B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    *all_converged = ctx->pinned[0];
    *one_changed = ctx->pinned[1];
    return B200_OK;
}

__global__ void set_all_statuses_kernel(int64_t cols, uint8_t id, bool set_finalized, uint8_t* stop)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= cols) return;
    uint8_t s = stop[i];
    if (!has_stopped(s)) {
        s |= (id & kIdMask);
        if (set_finalized) s |= kFinalizedMask;
        stop[i] = s;
    }
}

}  // namespace stop

namespace jacobi {

// One warp per diagonal block (block sizes <= 32): lane r owns row r of the
// inverted block, b_blk is broadcast by shuffles; columns of the block are
// contiguous across lanes in the interleaved storage (coalesced).  With a
// single right-hand side this is a batch of tiny GEMVs at ~0.5 flop/byte:
// HBM-bound, so no tensor cores (SURVEY.md section 7 "Block-Jacobi layout").
// Summation order per row: inner = 0..bs-1, as the reference's apply_block.
// One warp per storage GROUP (32 / pow2(max_block_size) blocks interleaved so that column c
// of all of them is one contiguous run): lane l holds row l % block_offset of sub-block
// l / block_offset, so every load of a block column is a single coalesced run for the whole
// warp.  All MBS columns are fetched before the first multiply (no chain of dependent
// latencies) and stay in registers for every right-hand side.
// CTL: the fused GMRES iteration's instance, a no-op once its control word ctl[0] says it stopped.
template <typename V, typename I, int MBS, bool ADVANCED, bool ADAPTIVE, bool CTL = false>
__global__ void __launch_bounds__(256)
    block_apply_kernel(int64_t num_blocks, int64_t block_offset, int64_t group_offset,
                       int32_t group_power, const uint8_t* __restrict__ block_precisions,
                       const I* __restrict__ block_ptrs, const V* __restrict__ blocks,
                       const V* __restrict__ alpha_p,
                       const V* __restrict__ b, int64_t bs_, int64_t num_rhs,
                       const V* __restrict__ beta_p, V* __restrict__ x, int64_t xs,
                       const int32_t* __restrict__ ctl = nullptr)
{
    if (CTL && ctl[0] != 0) return;
    const int lane = threadIdx.x & 31;
    const int64_t group = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int group_size = 1 << group_power;
    if (group * group_size >= num_blocks) return;
    const int bo = (int)block_offset;
    const int sub = lane / bo;
    const int r = lane - sub * bo;
    const int64_t k = group * group_size + sub;
    int64_t first = 0;
    int bsz = 0;
    if (sub < group_size && k < num_blocks) {
        first = block_ptrs[k];
        bsz = (int)((int64_t)block_ptrs[k + 1] - first);
    }
    const bool valid = r < bsz;
    const int64_t stride = block_offset << group_power;
    // adaptive precision (jacobi_precision.cuh): the block is stored as the type its precision_reduction
    // byte names, addressed in elements of THAT type from the group's base, and widened on load.
    // ADAPTIVE == false (no precision array) is the round-1 kernel unchanged: cfg4's GMRES applies it
    // every iteration.
    const int kind =
        ADAPTIVE ? storage_kind<V>((sub < group_size && k < num_blocks) ? block_precisions[k] : uint8_t(0))
                 : (sizeof(V) == 8 ? (int)kF64 : (int)kF32);
    const void* gbase = blocks + group_offset * group;
    V a[MBS];
    // Two phases: ALL raw loads of the column set first (by storage width), then the conversions.  With
    // the conversion next to each load the branches of gko::half's inf / nan / denormal handling kept
    // the compiler from hoisting the loads: 16 dependent round trips per warp, several times slower
    // on cfg4's blocks.
    const int64_t e0 = lane;
    if (!ADAPTIVE) {
        const V* col0 = blocks + group_offset * group + lane;
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner)
            a[inner] = (valid && inner < bsz) ? col0[inner * stride] : V(0);
    } else
    switch (storage_bytes(kind)) {
    case 8: {
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner)
            a[inner] = (valid && inner < bsz) ? (V) reinterpret_cast<const double*>(gbase)[e0 + inner * stride] : V(0);
        break;
    }
    case 4: {
        uint32_t raw[MBS];
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner)
            raw[inner] = (valid && inner < bsz) ? reinterpret_cast<const uint32_t*>(gbase)[e0 + inner * stride] : 0u;
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner)
            a[inner] = kind == kF32 ? (V)__uint_as_float(raw[inner]) : (V)__hiloint2double((int)raw[inner], 0);
        break;
    }
    default: {
        uint16_t raw[MBS];
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner)
            raw[inner] = (valid && inner < bsz) ? reinterpret_cast<const uint16_t*>(gbase)[e0 + inner * stride]
                                                : uint16_t(0);
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner) {
            const uint32_t w = (uint32_t)raw[inner] << 16;
            a[inner] = kind == kF16     ? (V)gko_half_to_float(raw[inner])
                       : kind == kT32_16 ? (V)__uint_as_float(w)
                                         : (V)__hiloint2double((int)w, 0);
        }
        break;
    }
    }
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const int src0 = sub * bo;
    for (int64_t j = 0; j < num_rhs; ++j) {
        const V bv = valid ? b[(first + r) * bs_ + j] : V(0);
        V acc = V(0);
        if (ADVANCED && valid && beta != V(0)) acc = x[(first + r) * xs + j] * beta;
#pragma unroll
        for (int inner = 0; inner < MBS; ++inner) {
            const V bi = __shfl_sync(0xffffffffu, bv, (src0 + inner) & 31);
            if (valid && inner < bsz) acc += ADVANCED ? (alpha * a[inner]) * bi : a[inner] * bi;
        }
        if (valid) x[(first + r) * xs + j] = acc;
    }
}

// --------------------------------------------------------------------------------------------
// Many right-hand sides: the block apply is a batch of small dense GEMMs  X_k = Binv_k B_k
// (bs x bs times bs x nrhs) -- the one place of the path where tensor cores apply (SURVEY.md 8d,
// north_star).  The reference loops the right-hand sides inside apply_block
// (reference/preconditioner/jacobi_kernels.cpp:415-447; its CUDA backend launches one GEMV kernel
// per block row, common/cuda_hip/preconditioner/jacobi_simple_apply_kernels.cpp:41-55).
// Here: one warp per block, the block's inverse is loaded ONCE into DMMA A-fragments (in its
// stored precision, widened to fp64), then for every tile of 8 right-hand sides
// MT x KS  mma.sync.m8n8k4.f64  (SASS DMMA) accumulate in fp64; fp32 operands are widened, so
// products are exact and only the final store rounds.  Summation order differs from the
// reference's sequential inner loop (k in chunks of 4 inside the tensor core): results agree to
// r<T>, not bit for bit -- the SIMT kernel above stays the path for fewer than 8 (fp32: 16) right-hand sides.
// Roofline: per block bs^2 + 2 bs nrhs values of traffic against 2 bs^2 nrhs flops -- 16 x 16 fp64
// with 32 right-hand sides is 1.6 flop/B, i.e. about 5 TFLOP/s at an H100's 3.35 TB/s: far beyond
// issuing one DFMA per product from shuffled operands (the SIMT kernel: 3 instructions per product
// and lane), well inside the 67 TFLOP/s the H100 SXM data sheet gives its fp64 tensor cores.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}

constexpr int kMmaWarps = 8;

template <typename V, typename I, int MT, bool ADVANCED>
__global__ void __launch_bounds__(kMmaWarps * 32)
    block_apply_mma_kernel(int64_t num_blocks, int64_t block_offset, int64_t group_offset, int32_t group_power,
                           const uint8_t* __restrict__ block_precisions, const I* __restrict__ block_ptrs,
                           const V* __restrict__ blocks, const V* __restrict__ alpha_p,
                           const V* __restrict__ b, int64_t bs_, int64_t num_rhs,
                           const V* __restrict__ beta_p, V* __restrict__ x, int64_t xs)
{
    constexpr int KS = 2 * MT;  // k-steps of 4 covering 8 * MT columns
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kMmaWarps + (threadIdx.x >> 5);
    if (k >= num_blocks) return;
    const int64_t first = block_ptrs[k];
    const int bsz = (int)((int64_t)block_ptrs[k + 1] - first);
    const int gid = lane >> 2, tig = lane & 3;
    const int64_t stride = block_offset << group_power;
    const void* gbase = blocks + group_offset * (k >> group_power);
    const int64_t bo = block_offset * (k & (((int64_t)1 << group_power) - 1));
    const int kind = storage_kind<V>(block_precisions ? block_precisions[k] : uint8_t(0));
    // A fragments: element (row, col) of the inverse, row = 8 mt + gid, col = 4 ks + tig
    double a[MT][KS];
    auto load_frags = [&](auto get) {
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                const int row = 8 * mt + gid, col = 4 * ks + tig;
                a[mt][ks] = (row < bsz && col < bsz) ? get(bo + row + col * stride) : 0.0;
            }
    };
    switch (kind) {  // outside the loops: one branch, then MT * KS independent loads
    case kF64: load_frags([&](int64_t i) { return reinterpret_cast<const double*>(gbase)[i]; }); break;
    case kF32: load_frags([&](int64_t i) { return (double)reinterpret_cast<const float*>(gbase)[i]; }); break;
    default: load_frags([&](int64_t i) { return (double)load_elem(gbase, i, kind, V(0)); }); break;
    }
    double alpha = 1.0, beta = 0.0;
    if (ADVANCED) {
        alpha = (double)*alpha_p;
        beta = (double)*beta_p;
    }
    for (int64_t j0 = 0; j0 < num_rhs; j0 += 8) {
        // B fragments: element (kk, n) of the right-hand-side block, kk = 4 ks + tig, n = gid
        double bf[KS];
        const bool ncol = j0 + gid < num_rhs;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int kk = 4 * ks + tig;
            bf[ks] = (ncol && kk < bsz) ? (double)b[(first + kk) * bs_ + j0 + gid] : 0.0;
        }
        double c[MT][2];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            c[mt][0] = c[mt][1] = 0.0;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) dmma_m8n8k4(c[mt][0], c[mt][1], a[mt][ks], bf[ks]);
        }
        // D fragments: row = 8 mt + gid, columns 2 tig, 2 tig + 1 of the tile
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            const int row = 8 * mt + gid;
            if (row >= bsz) continue;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int64_t col = j0 + 2 * tig + q;
                if (col >= num_rhs) continue;
                V* dst = x + (first + row) * xs + col;
                double v = c[mt][q];
                if (ADVANCED) v = beta != 0.0 ? alpha * v + beta * (double)*dst : alpha * v;
                *dst = (V)v;
            }
        }
    }
}

// which kernel applies the blocks: -1 (default) tensor cores from 8 right-hand sides on, 0 always the SIMT
// kernel (bit-identical to the reference for any number of right-hand sides), 1 always the tensor cores.
// B200_JACOBI_MMA in the environment sets the initial value, b200_jacobi_apply_mode changes it.
inline int& mma_mode()
{
    static int mode = [] {
        const char* env = getenv("B200_JACOBI_MMA");
        return env ? (env[0] == '0' ? 0 : (env[0] == '1' ? 1 : -1)) : -1;
    }();
    return mode;
}
// fp64: 8 right-hand sides fill one DMMA tile, from there on the tensor-core path is the faster one;
// fp32 operands are widened to fp64, the DMMA pipe (not HBM) bounds that path and it overtakes the
// SIMT kernel between 8 and 16 right-hand sides
inline bool use_mma(int64_t num_rhs, size_t value_bytes)
{
    const int m = mma_mode();
    return m == 1 || (m < 0 && num_rhs >= (value_bytes == 8 ? 8 : 16));
}

template <typename V, typename I, bool ADVANCED>
b200_status block_apply(b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size,
                        int64_t block_offset, int64_t group_offset, int32_t group_power,
                        const uint8_t* block_precisions, const I* block_ptrs, const V* blocks,
                        const V* alpha, const V* b, int64_t bs, int64_t num_rhs, const V* beta, V* x,
                        int64_t xs)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    B200_REQUIRE(max_block_size >= 1 && max_block_size <= 32, "max_block_size must be in [1,32]");
    B200_REQUIRE(block_offset >= 1 && (block_offset << group_power) <= 32 && group_power >= 0,
                 "storage scheme does not fit a warp");
    if (num_blocks <= 0 || num_rhs <= 0) return B200_OK;
    if (use_mma(num_rhs, sizeof(V))) {
        const unsigned mgrid = (unsigned)ceildiv(num_blocks, (int64_t)kMmaWarps);
#define B200_BJM(M)                                                                               \
    block_apply_mma_kernel<V, I, M, ADVANCED><<<mgrid, kMmaWarps * 32, 0, ctx->stream>>>(         \
        num_blocks, block_offset, group_offset, group_power, block_precisions, block_ptrs, blocks, \
        alpha, b, bs, num_rhs, beta, x, xs)
        if (max_block_size <= 8)
            B200_BJM(1);
        else if (max_block_size <= 16)
            B200_BJM(2);
        else
            B200_BJM(4);
#undef B200_BJM
        B200_LAUNCH_CHECK(ctx);
        return B200_OK;
    }
    const int64_t groups = ceildiv(num_blocks, int64_t(1) << group_power);
    const unsigned grid = (unsigned)ceildiv(groups * 32, (int64_t)256);
#define B200_BJ(M)                                                                              \
    do {                                                                                        \
        if (block_precisions)                                                                   \
            block_apply_kernel<V, I, M, ADVANCED, true><<<grid, 256, 0, ctx->stream>>>(         \
                num_blocks, block_offset, group_offset, group_power, block_precisions,          \
                block_ptrs, blocks, alpha, b, bs, num_rhs, beta, x, xs);                        \
        else                                                                                    \
            block_apply_kernel<V, I, M, ADVANCED, false><<<grid, 256, 0, ctx->stream>>>(        \
                num_blocks, block_offset, group_offset, group_power, nullptr, block_ptrs,       \
                blocks, alpha, b, bs, num_rhs, beta, x, xs);                                    \
    } while (0)
    if (block_offset <= 4)
        B200_BJ(4);
    else if (block_offset <= 8)
        B200_BJ(8);
    else if (block_offset <= 16)
        B200_BJ(16);
    else
        B200_BJ(32);
#undef B200_BJ
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

// x = M b for one right-hand side with unit strides, as block_apply's SIMT kernel, skipped once ctl[0] != 0
// (the preconditioner step of the fused GMRES iteration, replayed in a graph past the stop)
template <typename V, typename I>
b200_status fused_block_apply(b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,
                              int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,
                              const I* block_ptrs, const V* blocks, const V* b, V* x, const int32_t* ctl)
{
    B200_REQUIRE(ctx != nullptr && ctl != nullptr, "null argument");
    B200_REQUIRE(max_block_size >= 1 && max_block_size <= 32, "max_block_size must be in [1,32]");
    B200_REQUIRE(block_offset >= 1 && (block_offset << group_power) <= 32 && group_power >= 0,
                 "storage scheme does not fit a warp");
    if (num_blocks <= 0) return B200_OK;
    const int64_t groups = ceildiv(num_blocks, int64_t(1) << group_power);
    const unsigned grid = (unsigned)ceildiv(groups * 32, (int64_t)256);
#define B200_BJC(M)                                                                                 \
    do {                                                                                            \
        if (block_precisions)                                                                       \
            block_apply_kernel<V, I, M, false, true, true><<<grid, 256, 0, ctx->stream>>>(          \
                num_blocks, block_offset, group_offset, group_power, block_precisions, block_ptrs,  \
                blocks, nullptr, b, 1, 1, nullptr, x, 1, ctl);                                      \
        else                                                                                        \
            block_apply_kernel<V, I, M, false, false, true><<<grid, 256, 0, ctx->stream>>>(         \
                num_blocks, block_offset, group_offset, group_power, nullptr, block_ptrs, blocks,   \
                nullptr, b, 1, 1, nullptr, x, 1, ctl);                                              \
    } while (0)
    if (block_offset <= 4)
        B200_BJC(4);
    else if (block_offset <= 8)
        B200_BJC(8);
    else if (block_offset <= 16)
        B200_BJC(16);
    else
        B200_BJC(32);
#undef B200_BJC
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

}  // namespace jacobi
}  // namespace b200

extern "C" {

void b200_jacobi_apply_mode(int mode) { b200::jacobi::mma_mode() = mode < 0 ? -1 : (mode ? 1 : 0); }

b200_status b200_set_all_statuses(b200_ctx* ctx, int64_t cols, uint8_t stopping_id,
                                  int32_t set_finalized, uint8_t* stop_status)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    if (cols <= 0) return B200_OK;
    b200::stop::set_all_statuses_kernel<<<(unsigned)b200::ceildiv(cols, 256), 256, 0, ctx->stream>>>(
        cols, stopping_id, set_finalized != 0, stop_status);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

#define B200_DEF_STOP_JACOBI(V, VT)                                                            \
    b200_status b200_residual_norm_##V(b200_ctx* ctx, int64_t cols, const VT* tau,             \
                                       const VT* orig_tau, VT goal, uint8_t id,                \
                                       int32_t set_finalized, uint8_t* stop,                   \
                                       uint8_t* device_storage, int32_t* all_converged,        \
                                       int32_t* one_changed)                                   \
    {                                                                                          \
        return b200::stop::check<VT, false>(ctx, cols, tau, orig_tau, goal, id, set_finalized, \
                                            stop, device_storage, all_converged,               \
                                            one_changed);                                      \
    }                                                                                          \
    b200_status b200_implicit_residual_norm_##V(                                               \
        b200_ctx* ctx, int64_t cols, const VT* tau, const VT* orig_tau, VT goal, uint8_t id,   \
        int32_t set_finalized, uint8_t* stop, uint8_t* device_storage,                         \
        int32_t* all_converged, int32_t* one_changed)                                          \
    {                                                                                          \
        return b200::stop::check<VT, true>(ctx, cols, tau, orig_tau, goal, id, set_finalized,  \
                                           stop, device_storage, all_converged, one_changed);  \
    }                                                                                          \
    b200_status b200_jacobi_invert_diagonal_##V(b200_ctx* ctx, int64_t n, const VT* diag,      \
                                                VT* inv_diag)                                  \
    {                                                                                          \
        return b200::launch_ew(ctx, n, 1, [=] __device__(int64_t i, int64_t) {                 \
            const VT d = diag[i] == VT(0) ? VT(1) : diag[i];                                   \
            inv_diag[i] = VT(1) / d;                                                           \
        });                                                                                    \
    }                                                                                          \
    b200_status b200_jacobi_simple_scalar_apply_##V(b200_ctx* ctx, int64_t rows, int64_t cols, \
                                                    const VT* inv_diag, const VT* b,           \
                                                    int64_t bs, VT* x, int64_t xs)             \
    {                                                                                          \
        return b200::launch_ew(ctx, rows, cols, [=] __device__(int64_t i, int64_t j) {         \
            x[i * xs + j] = b[i * bs + j] * inv_diag[i];                                       \
        });                                                                                    \
    }                                                                                          \
    b200_status b200_jacobi_scalar_apply_##V(b200_ctx* ctx, int64_t rows, int64_t cols,        \
                                             const VT* inv_diag, const VT* alpha,              \
                                             const VT* b, int64_t bs, const VT* beta, VT* x,   \
                                             int64_t xs)                                       \
    {                                                                                          \
        return b200::launch_ew(ctx, rows, cols, [=] __device__(int64_t i, int64_t j) {         \
            x[i * xs + j] = beta[0] * x[i * xs + j] + alpha[0] * b[i * bs + j] * inv_diag[i];  \
        });                                                                                    \
    }

B200_DEF_STOP_JACOBI(f64, double)
B200_DEF_STOP_JACOBI(f32, float)

#define B200_DEF_JACOBI_BLOCK(V, VT, I, IT)                                                    \
    b200_status b200_jacobi_simple_apply_##V##_##I(                                            \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const IT* block_pointers,                   \
        const VT* blocks, const VT* b, int64_t bs, int64_t num_rhs, VT* x, int64_t xs)         \
    {                                                                                          \
        return b200::jacobi::block_apply<VT, IT, false>(                                       \
            ctx, num_blocks, max_block_size, block_offset, group_offset, group_power, nullptr, \
            block_pointers, blocks, nullptr, b, bs, num_rhs, nullptr, x, xs);                  \
    }                                                                                          \
    b200_status b200_jacobi_simple_apply_adaptive_##V##_##I(                                   \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,            \
        const IT* block_pointers, const VT* blocks, const VT* b, int64_t bs, int64_t num_rhs,  \
        VT* x, int64_t xs)                                                                     \
    {                                                                                          \
        return b200::jacobi::block_apply<VT, IT, false>(                                       \
            ctx, num_blocks, max_block_size, block_offset, group_offset, group_power,          \
            block_precisions, block_pointers, blocks, nullptr, b, bs, num_rhs, nullptr, x,     \
            xs);                                                                               \
    }                                                                                          \
    b200_status b200_jacobi_apply_adaptive_##V##_##I(                                          \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,            \
        const IT* block_pointers, const VT* blocks, const VT* alpha, const VT* b, int64_t bs,  \
        int64_t num_rhs, const VT* beta, VT* x, int64_t xs)                                    \
    {                                                                                          \
        return b200::jacobi::block_apply<VT, IT, true>(                                        \
            ctx, num_blocks, max_block_size, block_offset, group_offset, group_power,          \
            block_precisions, block_pointers, blocks, alpha, b, bs, num_rhs, beta, x, xs);     \
    }                                                                                          \
    b200_status b200_jacobi_apply_##V##_##I(                                                   \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const IT* block_pointers,                   \
        const VT* blocks, const VT* alpha, const VT* b, int64_t bs, int64_t num_rhs,           \
        const VT* beta, VT* x, int64_t xs)                                                     \
    {                                                                                          \
        return b200::jacobi::block_apply<VT, IT, true>(                                        \
            ctx, num_blocks, max_block_size, block_offset, group_offset, group_power, nullptr, \
            block_pointers, blocks, alpha, b, bs, num_rhs, beta, x, xs);                       \
    }                                                                                          \
    b200_status b200_gmres_fused_block_apply_##V##_##I(                                        \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,            \
        const IT* block_pointers, const VT* blocks, const VT* b, VT* x, const int32_t* ctl)    \
    {                                                                                          \
        return b200::jacobi::fused_block_apply<VT, IT>(                                        \
            ctx, num_blocks, max_block_size, block_offset, group_offset, group_power,          \
            block_precisions, block_pointers, blocks, b, x, ctl);                              \
    }

B200_DEF_JACOBI_BLOCK(f64, double, i32, int32_t)
B200_DEF_JACOBI_BLOCK(f64, double, i64, int64_t)
B200_DEF_JACOBI_BLOCK(f32, float, i32, int32_t)
B200_DEF_JACOBI_BLOCK(f32, float, i64, int64_t)

}  // extern "C"
