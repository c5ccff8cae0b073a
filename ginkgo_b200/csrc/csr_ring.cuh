// csr_ring.cuh -- "CTA ring" CSR SpMV kernel for sm_90a:  c = A b  /  c = alpha A b + beta c  (+ fused b.c)
//
// Replaces gko::kernels::cuda::csr::{spmv, advanced_spmv}
// (reference common/cuda_hip/matrix/csr_kernels.template.cpp:2353-2468); arithmetic contract =
// the reference executor's (reference/matrix/csr_kernels.cpp:47-118): per row, products added
// left to right (LANES == 1), advanced_spmv starting from beta*c and adding (alpha*val)*b.
//
// Design:
//   * one persistent CTA per SM = NW consumer warps + 1 producer warp, NO block barrier in the
//     main loop.  The producer's elected lane walks the CTA's tiles (same row-aligned merge-path
//     tiles as the other kernels: whole rows, < tile_items nonzeros + the last row) and brings
//     each tile's values / col_idxs / row_ptrs slabs into a ring of STAGES shared-memory
//     stages with three cp.async.bulk copies (SASS UBLKCP, L2 evict-first) onto the stage's
//     `full` mbarrier; it only waits for the stage's `empty` mbarrier (count NW).  3-4 stages
//     x ~48 KB are in flight per SM whatever the consumers do -- the HBM stream never waits
//     for a register.
//   * consumers: lane <-> ROW (LANES lanes per row).  A pass = 32/LANES consecutive rows; the
//     passes of the CTA's tiles are dealt round-robin to the warps, every warp runs through the
//     stages at its own pace.  Per pass a lane reads its row's column indices from the stage,
//     issues KB independent gathers of b, then multiplies and adds in storage order from a
//     register accumulator: no product staging in shared memory (staging stores and loads
//     were a large share of the L1TEX data-pipe wavefronts), half the shared-memory wavefronts per
//     nonzero, and on stencils / bands the 32 gathers of one instruction are 32 neighbouring
//     rows at the same offset = 2-3 cache lines instead of one line per diagonal.
//   * a last row that does not fit the stage is streamed from global memory by all consumer
//     warps (named barrier among the consumers only, fixed reduction tree).  Rows longer than
//     kLongRow are taken out of this kernel altogether by the plan (long_rows_kernel: split
//     over CTAs, partial sums combined in chunk order).
// Deterministic: no floating-point atomics; LANES == 1 sums are bit-identical to the reference
// executor (library built with -fmad=false).
#pragma once
#include "csr_kernels.cuh"

namespace b200 {
namespace csr {

// Stage geometry: CAP staged nonzeros; tiles of at most CAP - 512 merge items (so rows up to
// 512 entries ride along with their tile), hence at most (CAP - 512) / kRowW rows.
// Two shapes are shipped (launch_ring_auto): a deep ring (CAP 3584 x 4 stages = 197 KB in
// flight per SM) for matrices whose gathers are local, and a shallow one (CAP 1792 x 2 stages =
// 49 KB) for scattered gathers: the number of outstanding L1 misses is bounded by the L1 data
// capacity (one 128-byte line per pending gather), and L1 is what shared memory leaves of the
// SM's 228 KB -- with the deep ring every kernel of this family ran several times slower on
// uniformly random columns.
template <typename V, typename I, int CAP>
struct RingStage {
    static constexpr int items_max = CAP - 512;
    static constexpr int rp_cap = items_max / kRowW + 8;
    static constexpr size_t hdr_off = 0;  // int64 r0, p0, r1, p1 of the staged tile (r1 < 0: end)
    static constexpr size_t vals_off = 128;
    static constexpr size_t cols_off = vals_off + sizeof(V) * CAP;
    static constexpr size_t rp_off = cols_off + sizeof(I) * CAP;
    static constexpr size_t bytes = (rp_off + sizeof(I) * rp_cap + 127) & ~size_t(127);
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
template <int THREADS>
__device__ __forceinline__ void named_bar_sync()
{
    asm volatile("bar.sync 1, %0;" ::"n"(THREADS) : "memory");
}
// gather of the dense operand without L1 allocation (uniformly random columns: no reuse in an SM)
__device__ __forceinline__ double ld_gather_na(const double* p, uint64_t pol)
{
    double v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;"
                 : "=d"(v)
                 : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float ld_gather_na(const float* p, uint64_t pol)
{
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;"
                 : "=f"(v)
                 : "l"(p), "l"(pol));
    return v;
}

// fused-dot epilogue for any block size (dot_epilogue of csr_kernels.cuh assumes kThreads)
template <typename V, int DOT>
__device__ __forceinline__ void dot_epilogue_any(const DotAcc<V, DOT>& acc, const DotArgs<V>& dot, V* red,
                                                 bool* is_last)
{
    dot_epilogue_impl<0>(acc, dot, red, is_last);
}

template <typename V, typename I, int LANES, bool ADVANCED, int DOT, int NW, int KB, bool GNA, int CAP, int STAGES,
          int NP>
__global__ void __launch_bounds__((NW + NP) * 32, 1)
    ring_kernel(const int64_t* __restrict__ tiles, int64_t num_tiles, int64_t nnz, int64_t num_rows,
                const I* __restrict__ row_ptrs, const I* __restrict__ col_idxs,
                const V* __restrict__ values, const V* __restrict__ alpha_p,
                const V* __restrict__ b, int64_t b_stride, const V* __restrict__ beta_p,
                V* __restrict__ c, int64_t c_stride, DotArgs<V> dot)
{
    using S = RingStage<V, I, CAP>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t full_bar[STAGES];
    __shared__ uint64_t empty_bar[STAGES];
    __shared__ V red[32];
    __shared__ bool is_last;
    if (DOT && dot.ctl && dot.ctl[0] != 0) return;
    wait_for_block(dot);

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], NW);
        }
        fence_mbar_init();
    }
    __syncthreads();

    const int64_t G = gridDim.x;
    const uint64_t pol_first = policy_evict_first();
    DotAcc<V, DOT> dot_acc;

    static_assert(STAGES % NP == 0, "every producer warp owns STAGES / NP stages");
    // tiles of this CTA, in order: t = blockIdx.x + j * G; tile j lives in stage j % STAGES
    const int64_t nmine = num_tiles > (int64_t)blockIdx.x ? (num_tiles - 1 - blockIdx.x) / G + 1 : 0;

    if (warp >= NW) {
        // ------------------------------------------------------------------ producer warps
        // Producer w fills the stages of tiles j = w, w + NP, ... (one elected lane; the extents
        // of its next two tiles are already in registers, so no dependent global load sits between
        // two bulk copies).  With ONE lane walking all tiles, a dependent extent load and some 300
        // instructions per tile made the producer the bottleneck whatever the tile size, and the
        // consumers starved on the full barrier.
        if (lane == 0) {
            const int w = warp - NW;
            const int64_t floor4 = nnz & ~int64_t(3);
            const int64_t rfloor4 = (num_rows + 1) & ~int64_t(3);
            auto load_ext = [&](int64_t j, longlong2& ea, longlong2& eb) {
                if (j < nmine) {
                    const int64_t t = blockIdx.x + j * G;
                    ea = *reinterpret_cast<const longlong2*>(tiles + 2 * t);
                    eb = *reinterpret_cast<const longlong2*>(tiles + 2 * t + 2);
                }
            };
            longlong2 a0e = {0, 0}, b0e = {0, 0}, a1e = {0, 0}, b1e = {0, 0}, a2e = {0, 0}, b2e = {0, 0};
            load_ext(w, a0e, b0e);
            load_ext(w + NP, a1e, b1e);
            int stage = w % STAGES;
            uint32_t ph = 0;
            for (int64_t j = w; j < nmine; j += NP) {
                load_ext(j + 2 * NP, a2e, b2e);
                const int64_t r0 = a0e.x, p0 = a0e.y, r1 = b0e.x, p1 = b0e.y;
                const int64_t a0 = p0 & ~int64_t(3);
                const int64_t ra0 = r0 & ~int64_t(3);
                int64_t pend = p1, rows_end = r1;
                if (r1 > r0 && p1 - a0 > CAP) {  // the last row does not fit: staged without it
                    rows_end = r1 - 1;
                    pend = (int64_t)row_ptrs[rows_end];
                }
                mbar_wait(&empty_bar[stage], ph ^ 1u);
                unsigned char* sp = smem_raw + (size_t)stage * S::bytes;
                longlong2* hdr = reinterpret_cast<longlong2*>(sp + S::hdr_off);
                hdr[0] = a0e;
                hdr[1] = b0e;
                uint32_t cnt = 0, rcnt = 0;
                if (rows_end > r0) {
                    int64_t be = (pend + 3) & ~int64_t(3);
                    int64_t rbe = (rows_end + 4) & ~int64_t(3);
                    if (be > floor4 || rbe > rfloor4) {
                        // the <= 3 trailing entries of the arrays cannot be bulk-copied (16-byte
                        // units): copied by hand (last tile of the matrix only)
                        V* vals_s = reinterpret_cast<V*>(sp + S::vals_off);
                        I* cols_s = reinterpret_cast<I*>(sp + S::cols_off);
                        I* rp_s = reinterpret_cast<I*>(sp + S::rp_off);
                        if (be > floor4) be = floor4;
                        if (rbe > rfloor4) rbe = rfloor4;
                        for (int64_t q = (be > a0 ? be : a0); q < pend; ++q) {
                            vals_s[q - a0] = values[q];
                            cols_s[q - a0] = col_idxs[q];
                        }
                        for (int64_t q = (rbe > ra0 ? rbe : ra0); q <= rows_end; ++q) rp_s[q - ra0] = row_ptrs[q];
                    }
                    cnt = be > a0 ? (uint32_t)(be - a0) : 0u;
                    rcnt = rbe > ra0 ? (uint32_t)(rbe - ra0) : 0u;
                }
                fence_proxy_async();
                mbar_arrive_expect_tx(&full_bar[stage],
                                      cnt * (uint32_t)(sizeof(V) + sizeof(I)) + rcnt * (uint32_t)sizeof(I));
                if (cnt > 0) {
                    tma_load_1d(sp + S::vals_off, values + a0, cnt * (uint32_t)sizeof(V), &full_bar[stage], pol_first);
                    tma_load_1d(sp + S::cols_off, col_idxs + a0, cnt * (uint32_t)sizeof(I), &full_bar[stage],
                                pol_first);
                }
                if (rcnt > 0)
                    tma_load_1d(sp + S::rp_off, row_ptrs + ra0, rcnt * (uint32_t)sizeof(I), &full_bar[stage],
                                pol_first);
                stage += NP;
                if (stage >= STAGES) {
                    stage -= STAGES;
                    ph ^= 1u;
                }
                a0e = a1e;
                b0e = b1e;
                a1e = a2e;
                b1e = b2e;
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers
        V alpha = V(1), beta = V(0);
        if (ADVANCED) {
            alpha = *alpha_p;
            beta = *beta_p;
        }
        const uint64_t pol_last = policy_evict_last();
        constexpr int kRpp = 32 / LANES;
        const int sub = lane % LANES;
        int stage = 0;
        uint32_t ph = 0;
        int base = 0;  // passes dealt so far, modulo NW (identical in all consumer warps)
        for (int64_t j = 0; j < nmine; ++j) {
            mbar_wait(&full_bar[stage], ph);
            const unsigned char* sp = smem_raw + (size_t)stage * S::bytes;
            const int64_t* hdr = reinterpret_cast<const int64_t*>(sp + S::hdr_off);
            const int64_t r0 = hdr[0], p0 = hdr[1], r1 = hdr[2], p1 = hdr[3];
            const int64_t a0 = p0 & ~int64_t(3);
            const bool long_last = r1 > r0 && (p1 - a0) > CAP;
            const int64_t rows_end = long_last ? r1 - 1 : r1;
            if (rows_end > r0) {
                const V* vals_s = reinterpret_cast<const V*>(sp + S::vals_off);
                const I* cols_s = reinterpret_cast<const I*>(sp + S::cols_off);
                const I* rp_l = reinterpret_cast<const I*>(sp + S::rp_off) + (r0 & int64_t(3));
                const int nrows = (int)(rows_end - r0);
                const int npass = (nrows + kRpp - 1) / kRpp;
                int first = warp - base;
                if (first < 0) first += NW;
                for (int pass = first; pass < npass; pass += NW) {
                    const int rloc = pass * kRpp + lane / LANES;
                    const bool rv = rloc < nrows;
                    int s = 0, len = 0;
                    if (rv) {
                        s = (int)((int64_t)rp_l[rloc] - a0);
                        len = (int)((int64_t)rp_l[rloc + 1] - a0) - s;
                    }
                    // rows the plan splits over CTAs are long_rows_kernel's, wherever they sit in the
                    // stage (the split threshold is below the ring's tile size)
                    const bool mine = rv && !(dot.skip_from > 0 && len >= dot.skip_from);
                    if (!mine) len = 0;
                    const int mylen = (len - sub + LANES - 1) / LANES;
                    const int maxlen = __reduce_max_sync(0xffffffffu, mylen);
                    V acc = V(0);
                    if (LANES == 1 && ADVANCED && mine && beta != V(0)) acc = c[(r0 + rloc) * c_stride] * beta;
                    const int i0 = s + sub;
                    for (int j = 0; j < maxlen; j += KB) {
                        I cc[KB];
                        V xx[KB];
#pragma unroll
                        for (int k = 0; k < KB; ++k) {
                            cc[k] = I(0);
                            if (j + k < mylen) cc[k] = cols_s[i0 + (j + k) * LANES];
                        }
#pragma unroll
                        for (int k = 0; k < KB; ++k) {
                            xx[k] = V(0);
                            if (j + k < mylen)
                                xx[k] = GNA ? ld_gather_na(b + (int64_t)cc[k] * b_stride, pol_last)
                                            : ld_gather(b + (int64_t)cc[k] * b_stride, pol_last);
                        }
#pragma unroll
                        for (int k = 0; k < KB; ++k) {
                            if (j + k < mylen) {
                                const V v = vals_s[i0 + (j + k) * LANES];
                                acc += ADVANCED ? (alpha * v) * xx[k] : v * xx[k];
                            }
                        }
                    }
                    if (LANES > 1) {
#pragma unroll
                        for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                        if (ADVANCED && mine && sub == 0 && beta != V(0))
                            acc = c[(r0 + rloc) * c_stride] * beta + acc;
                    }
                    if (mine && sub == 0) {
                        c[(r0 + rloc) * c_stride] = acc;
                        dot_acc.add(dot, b, b_stride, r0 + rloc, acc);
                    }
                }
                base = (base + npass) % NW;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == STAGES) {
                stage = 0;
                ph ^= 1u;
            }
            if (long_last && !(dot.skip_from > 0 && p1 - (int64_t)row_ptrs[r1 - 1] >= dot.skip_from)) {
                // the tile's last row does not fit a stage: all consumer warps stream it from
                // global memory, fixed reduction tree (deterministic); rows the plan splits over
                // CTAs (dot.skip_from) are left to long_rows_kernel
                const int64_t rl = r1 - 1;
                const int64_t sl = (int64_t)row_ptrs[rl];
                V acc = strided_row_sum<V, I, ADVANCED>(sl + tid, p1, NW * 32, col_idxs, values, alpha, b,
                                                        b_stride, pol_first, pol_last);
                acc = warp_sum(acc);
                named_bar_sync<NW * 32>();
                if (lane == 0) red[warp] = acc;
                named_bar_sync<NW * 32>();
                if (warp == 0) {
                    V v = lane < NW ? red[lane] : V(0);
                    v = warp_sum(v);
                    if (lane == 0) {
                        if (ADVANCED && beta != V(0)) v = c[rl * c_stride] * beta + v;
                        c[rl * c_stride] = v;
                        dot_acc.add(dot, b, b_stride, rl, v);
                    }
                }
            }
        }
    }
    if (DOT) dot_epilogue_any(dot_acc, dot, red, &is_last);
}

// shared-memory size + a carve-out that leaves the rest of the SM's 228 KB to L1
template <typename K>
b200_status set_smem_exact(K kernel, size_t bytes)
{
    static thread_local const void* done = nullptr;
    if (done != (const void*)kernel) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        int pct = (int)((bytes + 4096) * 100 / (228 * 1024)) + 1;
        if (pct > 100) pct = 100;
        B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
        done = (const void*)kernel;
    }
    return B200_OK;
}

template <typename V, typename I, int LANES, bool ADVANCED, int DOT, int NW, int KB, bool GNA, int CAP, int STAGES,
          int NP>
b200_status launch_ring(b200_ctx* ctx, int64_t num_tiles, const int64_t* tiles, int64_t nnz,
                        int64_t num_rows, const I* row_ptrs, const I* col_idxs, const V* values,
                        const V* alpha, const V* b, int64_t b_stride, const V* beta, V* c,
                        int64_t c_stride, DotArgs<V> dot, int grid)
{
    using S = RingStage<V, I, CAP>;
    constexpr size_t smem = S::bytes * STAGES;
    static_assert(smem <= 227 * 1024, "ring does not fit the SM's shared memory");
    auto k = ring_kernel<V, I, LANES, ADVANCED, DOT, NW, KB, GNA, CAP, STAGES, NP>;
    b200_status st = set_smem_exact(k, smem);
    if (st != B200_OK) return st;
    k<<<grid, (NW + NP) * 32, smem, ctx->stream>>>(tiles, num_tiles, nnz, num_rows, row_ptrs, col_idxs,
                                                  values, alpha, b, b_stride, beta, c, c_stride, dot);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

}  // namespace csr
}  // namespace b200
