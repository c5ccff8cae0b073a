// Shared device/host helpers for the sm_90a kernels behind include/ginkgo_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/ginkgo_b200.h"

namespace b200 {

void set_error(const char* fmt, ...);

// The CudaExecutor analogue: device, stream, SM count and a stream-ordered
// scratch area shared by all reductions of this context (the reference hands
// every reduction an `array<char>& tmp`; common/cuda_hip/base/
// kernel_launch_reduction.hpp:121-125).
struct Workspace {
    void* ptr = nullptr;
    size_t bytes = 0;
};

}  // namespace b200

struct b200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    int num_sms = 0;
    int max_smem_optin = 0;
    size_t l2_bytes = 0;
    int64_t launches = 0;
    b200::Workspace ws;           // general scratch
    unsigned int* counters = nullptr;  // zero-initialised, self-resetting block counters
    uint8_t* pinned = nullptr;    // small pinned host mailbox (stop flags)
    void* dev_mailbox = nullptr;  // small device mailbox
    // fork / join of independent kernels of ONE operation (csr: the rows split over CTAs next to the
    // main kernel): aux waits for `fork` recorded on stream, stream waits for `join` recorded on aux.
    // Plain event dependencies, so they are captured into CUDA graphs like any other launch.
    cudaStream_t aux = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    // b200_snapshot_*: two slots of a stream-ordered "what did this look like at THIS point of the
    // stream" read-back that does not wait for work enqueued afterwards
    void* snap_dev = nullptr;      // 2 x kSnapBytes device
    uint8_t* snap_host = nullptr;  // 2 x kSnapBytes pinned host
    cudaEvent_t snap_ev[2] = {nullptr, nullptr};
    static constexpr size_t kSnapBytes = 256;

    // returns a scratch pointer of at least `bytes` (stream ordered re-use)
    void* scratch(size_t bytes);
};

#define B200_STR2(x) #x
#define B200_STR(x) B200_STR2(x)

#define B200_CUDA_CHECK(expr)                                                         \
    do {                                                                              \
        cudaError_t e__ = (expr);                                                     \
        if (e__ != cudaSuccess) {                                                     \
            b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,             \
                            cudaGetErrorString(e__));                                 \
            return B200_ERR_CUDA;                                                     \
        }                                                                             \
    } while (0)

#define B200_REQUIRE(cond, msg)                                          \
    do {                                                                 \
        if (!(cond)) {                                                   \
            b200::set_error("%s:%d: %s", __FILE__, __LINE__, msg);       \
            return B200_ERR_INVALID;                                     \
        }                                                                \
    } while (0)

#define B200_LAUNCH_CHECK(ctx)                                                       \
    do {                                                                             \
        (ctx)->launches++;                                                           \
        cudaError_t e__ = cudaGetLastError();                                        \
        if (e__ != cudaSuccess) {                                                    \
            b200::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__,        \
                            cudaGetErrorString(e__));                                \
            return B200_ERR_CUDA;                                                    \
        }                                                                            \
    } while (0)

namespace b200 {

constexpr int kWarp = 32;

__host__ __device__ inline int64_t ceildiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Slots of b200_ctx::counters that the fused solvers' grid-wide sums take their tickets from.  The same
// 256 counters serve the BLAS-1 reductions (dense_blas1.cu: slot t for column tile t of a batch, so any
// of 0..255) and the unfused GMRES multi-dot (slot 0).  Sharing is safe because every kernel that takes
// a ticket resets its slot to 0 in the CTA that takes the last one, and every user launches on
// ctx->stream (directly or in a graph captured on it), so no two kernels hold a slot at the same time.
constexpr int kSpmvDotCounter = 1;   // the SpMV's dot epilogue (csr::DotArgs, mrhs::spmv_mdot)
constexpr int kStepCounter = 2;      // the fused step kernels
constexpr int kMultiDotCounter = 3;  // the multi-dot that honours ctl (GMRES's fused CGS / CGS2)

// stopping_status bit layout (include/ginkgo/core/stop/stopping_status.hpp)
constexpr uint8_t kConvergedMask = 1u << 7;
constexpr uint8_t kFinalizedMask = 1u << 6;
constexpr uint8_t kIdMask = (1u << 6) - 1u;
__device__ __forceinline__ bool has_stopped(uint8_t s) { return (s & kIdMask) != 0; }
__device__ __forceinline__ bool is_finalized(uint8_t s) { return (s & kFinalizedMask) != 0; }

// ---- cache-hinted loads ----------------------------------------------------
// Streaming loads: matrix values / column indices are read exactly once, so
// keep them out of L1 (no_allocate) and mark them evict-first in L2 so they do
// not push the gathered x vector out.  sm_90 global loads are at most 128 bits
// wide; the L2 eviction priority travels as a cache-policy operand
// (createpolicy, below).
__device__ __forceinline__ void ld_stream_128(const double* p, double (&v)[2], uint64_t pol)
{
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
                 : "=d"(v[0]), "=d"(v[1])
                 : "l"(p), "l"(pol));
}
__device__ __forceinline__ void ld_stream_128(const float* p, float (&v)[4], uint64_t pol)
{
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3])
                 : "l"(p), "l"(pol));
}
__device__ __forceinline__ void ld_stream_128(const int32_t* p, int32_t (&v)[4], uint64_t pol)
{
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3])
                 : "l"(p), "l"(pol));
}
__device__ __forceinline__ void ld_stream_128(const int64_t* p, int64_t (&v)[2], uint64_t pol)
{
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;"
                 : "=l"(v[0]), "=l"(v[1])
                 : "l"(p), "l"(pol));
}

// Load 8 consecutive elements (16B-aligned start) with streaming hints, `pol`
// from policy_evict_first().
template <typename T>
__device__ __forceinline__ void ld_stream_x8(const T* p, T (&v)[8], uint64_t pol)
{
    constexpr int W = 16 / (int)sizeof(T);
#pragma unroll
    for (int q = 0; q < 8 / W; ++q) {
        T a[W];
        ld_stream_128(p + q * W, a, pol);
#pragma unroll
        for (int i = 0; i < W; ++i) v[q * W + i] = a[i];
    }
}

// L2 cache policies for narrower accesses (descriptor form)
__device__ __forceinline__ uint64_t policy_evict_first()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_last()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// scalar streaming load (no L1 allocation, L2 evict-first via policy)
__device__ __forceinline__ double ld_stream(const double* p, uint64_t pol)
{
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;"
                 : "=d"(v)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float ld_stream(const float* p, uint64_t pol)
{
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;"
                 : "=f"(v)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ int32_t ld_stream(const int32_t* p, uint64_t pol)
{
    int32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;"
                 : "=r"(v)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ int64_t ld_stream(const int64_t* p, uint64_t pol)
{
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;"
                 : "=l"(v)
                 : "l"(p), "l"(pol));
    return v;
}

// Gather loads of the dense operand: read-only path, L1 allocate (banded
// matrices re-use neighbours), prefer to keep in L2 (evict_last policy).
__device__ __forceinline__ double ld_gather(const double* p, uint64_t pol)
{
    double v;
    asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float ld_gather(const float* p, uint64_t pol)
{
    float v;
    asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
    return v;
}


// ---- mbarrier / bulk async copy (TMA 1-D) / cp.async helpers ---------------
__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy accesses to shared memory must be ordered before the async proxy
// (bulk copy engine) overwrites the same bytes
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra LAB_DONE_%=;\n"
        "bra LAB_WAIT_%=;\n"
        "LAB_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared bulk copy (SASS UBLKCP), completion signalled on `bar`;
// bytes must be a multiple of 16, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                            uint64_t policy)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async(void* dst, const void* src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(dst)), "l"(src),
                 "n"(BYTES)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// streaming store (written once, not re-read by this kernel)
template <typename T>
__device__ __forceinline__ void st_stream(T* p, T v)
{
    __stcs(p, v);
}

// ---- reductions --------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum with a fixed tree (deterministic). `smem` holds >= 32 T.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem)
{
    const int lane = threadIdx.x & 31;
    const int wid = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nw) ? smem[threadIdx.x] : T(0);
    if (wid == 0) v = warp_sum(v);
    return v;  // valid in warp 0 (all lanes)
}

inline int grid_for(int64_t work_items, int block, int num_sms, int max_ctas_per_sm)
{
    int64_t g = ceildiv(work_items, block);
    int64_t cap = (int64_t)num_sms * max_ctas_per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace b200
