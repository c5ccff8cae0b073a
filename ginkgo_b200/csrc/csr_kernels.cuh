// csr_kernels.cuh -- CSR SpMV kernels for sm_90a (shared by csr_spmv.cu and fused_cg.cu):  c = A b   and   c = alpha A b + beta c   (+ optional fused b.c)
//
// Replaces gko::kernels::cuda::csr::{spmv, advanced_spmv}
// (reference common/cuda_hip/matrix/csr_kernels.template.cpp:2353-2468); the
// arithmetic contract is the reference executor's
// (reference/matrix/csr_kernels.cpp:47-118): per row, products accumulated left
// to right, for advanced_spmv starting from beta*c (never reading c if beta==0)
// and adding (alpha*val)*b.
//
// Kernel design ("row-segmented slab" kernel, single right-hand side):
//   * Partition (b200_csr_plan, the analogue of the reference's `srow`): the
//     merge-path coordinate 2*row + row_ptrs[row] is cut into tiles of kTile
//     items, so every tile owns whole rows, at most kTile/2 of them, and fewer
//     than kTile nonzeros plus its last row.  The plan stores (first row, first
//     nonzero) per tile, so a CTA needs no dependent loads to find its slab.
//   * Persistent CTAs (3 per SM) walk the tiles round-robin with a 2-stage
//     pipeline: while tile i is processed, the col_idxs / values slabs of tile
//     i+1 are brought into shared memory by the bulk-copy engine
//     (cp.async.bulk, SASS UBLKCP, L2 evict-first, mbarrier completion) and its
//     row_ptrs slab by cp.async (LDGSTS) -- the HBM stream never waits for a
//     thread and is perfectly load balanced whatever the row lengths are.
//   * Gather phase: one nonzero per thread-slot, b[col] gathered with an L2
//     evict-last policy, val*b written back in place in shared memory.
//   * Row phase: LANES threads per row add the row's products from shared
//     memory.  LANES == 1 (average row <= 32) is strictly left to right, i.e.
//     bit-identical to the reference executor; LANES > 1 uses a fixed shuffle
//     tree; a last row that does not fit the staging buffer is summed by the
//     whole CTA.  No floating-point atomics anywhere: results are deterministic.
// Base pointers that are not 16-byte aligned take `slab_kernel`, the same
// algorithm with ordinary coalesced loads.  Multiple right-hand sides use a
// thread-per-(row,rhs) kernel with the reference's summation order.
#pragma once
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace b200 {
namespace csr {

constexpr int kThreads = 256;
constexpr int kTile = 2048;           // merge items (2*rows + nnz) per tile
constexpr int kRowW = 2;              // weight of a row in the merge coordinate
constexpr int kMaxRows = kTile / kRowW;
constexpr int kCap = kTile + 512 + 8;  // staged nonzeros per tile (incl. alignment slack)
constexpr int kStages = 3;
constexpr int kCtasPerSm = 2;
constexpr int kGatherUnroll = (kCap + kThreads - 1) / kThreads;  // 11

template <typename I>
__global__ void plan_kernel(const I* __restrict__ row_ptrs, int64_t num_rows, int64_t num_tiles,
                            int64_t tile_items, int64_t* __restrict__ tiles)
{
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t > num_tiles) return;
    const int64_t d = t * tile_items;
    int64_t lo = 0, hi = num_rows;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (kRowW * mid + (int64_t)row_ptrs[mid] >= d)
            hi = mid;
        else
            lo = mid + 1;
    }
    tiles[2 * t] = lo;
    tiles[2 * t + 1] = (int64_t)row_ptrs[lo];
}

// Optional fused dot product (Krylov: q = A p and p.q in one launch): every CTA
// adds its rows' share, publishes its partial(s), and the CTA that arrives last
// sums the partials in CTA order (deterministic).  The kernels' DOT template value:
//   kDotNone   no dot
//   kDotB      result = sum b[row]*c[row]  (CG: the SpMV's own input, square A)
//   kDotW2     result = sum w[row]*c[row] for a caller-given w with one entry per row, and
//              result2 (optional) = sum c[row]*c[row]; two partials per CTA (BiCGStab: rr.v, s.t and t.t)
// `ctl` (optional) is the fused solvers' control block: ctl[0] != 0 (stopped) turns
// the launch into a no-op.
enum : int { kDotNone = 0, kDotB = 1, kDotW2 = 2 };

template <typename V>
struct DotArgs {
    V* partials;            // one per CTA (kDotW2: two)
    unsigned int* counter;  // self-resetting ticket
    V* result;
    const int32_t* ctl;
    // rows with at least this many entries are NOT computed by these kernels (0: none): the plan
    // splits them over CTAs (long_rows_kernel); such a row is always the last row of its tile
    int64_t skip_from;
    // multi-GPU pipelining: before touching b, wait until *wait_flag >= wait_epoch (system scope): the
    // owner block this launch gathers from has landed (dist.cu, b200_halo_*_staged); nullptr: no wait
    const unsigned long long* wait_flag;
    unsigned long long wait_epoch;
    // kDotW2 only
    const V* w;
    V* result2;  // nullptr: the second sum is not written
};

// a thread's share of the fused dot(s); add() is called once per finished row with its c
template <typename V, int DOT>
struct DotAcc {
    V s = V(0);
    __device__ __forceinline__ void add(const DotArgs<V>&, const V* __restrict__ b, int64_t b_stride, int64_t r, V cr)
    {
        if (DOT) s += b[r * b_stride] * cr;
    }
};
template <typename V>
struct DotAcc<V, kDotW2> {
    V s = V(0), s2 = V(0);
    __device__ __forceinline__ void add(const DotArgs<V>& dot, const V* __restrict__, int64_t, int64_t r, V cr)
    {
        s += dot.w[r] * cr;
        s2 += cr * cr;
    }
};

// every CTA's thread 0 polls the flag; the barrier publishes the acquire to the block
template <typename V>
__device__ __forceinline__ void wait_for_block(const DotArgs<V>& dot)
{
    if (dot.wait_flag == nullptr) return;
    if (threadIdx.x == 0) {
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(dot.wait_flag) : "memory");
        } while (v < dot.wait_epoch);
    }
    __syncthreads();
}

// THREADS: the block size when it is a compile-time constant, 0 for blockDim.x
template <int THREADS, typename V, int DOT>
__device__ __forceinline__ void dot_epilogue_impl(const DotAcc<V, DOT>& acc, const DotArgs<V>& dot, V* red,
                                                  bool* is_last)
{
    const int tid = threadIdx.x;
    const int64_t stride = THREADS > 0 ? THREADS : (int)blockDim.x;
    const V s = block_sum(acc.s, red);
    V s2 = V(0);
    if constexpr (DOT == kDotW2) s2 = block_sum(acc.s2, red);
    if (tid == 0) {
        if constexpr (DOT == kDotW2) {
            dot.partials[2 * blockIdx.x] = s;
            dot.partials[2 * blockIdx.x + 1] = s2;
        } else {
            dot.partials[blockIdx.x] = s;
        }
        __threadfence();
        const unsigned int ticket = atomicAdd(dot.counter, 1u);
        *is_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (*is_last) {
        __threadfence();
        V t = V(0), t2 = V(0);
        for (int64_t k = tid; k < (int64_t)gridDim.x; k += stride) {
            if constexpr (DOT == kDotW2) {
                t += __ldcg(dot.partials + 2 * k);
                t2 += __ldcg(dot.partials + 2 * k + 1);
            } else {
                t += __ldcg(dot.partials + k);
            }
        }
        t = block_sum(t, red);
        if constexpr (DOT == kDotW2) t2 = block_sum(t2, red);
        if (tid == 0) {
            *dot.result = t;
            if constexpr (DOT == kDotW2)
                if (dot.result2) *dot.result2 = t2;
            *dot.counter = 0u;
        }
    }
}

template <typename V, int DOT>
__device__ __forceinline__ void dot_epilogue(const DotAcc<V, DOT>& acc, const DotArgs<V>& dot, V* red, bool* is_last)
{
    dot_epilogue_impl<kThreads>(acc, dot, red, is_last);
}

// Row phase shared by both kernels: rows [r0, rows_end) of the tile, products in
// prod[] indexed by (nonzero - a0), row pointers from rp(r).
template <typename V, int LANES, bool ADVANCED, int DOT, typename RowPtr>
__device__ __forceinline__ void row_phase(int64_t r0, int64_t rows_end, int64_t a0, const V* prod,
                                          RowPtr rp, V beta, const V* __restrict__ b,
                                          int64_t b_stride, V* __restrict__ c, int64_t c_stride,
                                          DotAcc<V, DOT>& dot_acc, const DotArgs<V>& dot)
{
    const int64_t skip_from = dot.skip_from;
    constexpr int kRowsPerPass = kThreads / LANES;
    const int tid = threadIdx.x;
    const int sub = tid % LANES;
    const int64_t nrows = rows_end - r0;
    const int64_t passes = (nrows + kRowsPerPass - 1) / kRowsPerPass;
    for (int64_t ps = 0; ps < passes; ++ps) {
        const int64_t r = r0 + ps * kRowsPerPass + tid / LANES;
        bool rv = r < rows_end;
        int64_t s = 0, e = 0;
        if (rv) {
            s = rp(r);
            e = rp(r + 1);
        }
        // rows the plan splits over CTAs (long_rows_kernel) are not this kernel's: with a tile larger
        // than the split threshold such a row can sit anywhere in the tile, not only at its end
        if (skip_from > 0 && e - s >= skip_from) {
            rv = false;
            s = e = 0;
        }
        V acc = V(0);
        if (LANES == 1) {
            if (ADVANCED && rv && beta != V(0)) acc = c[r * c_stride] * beta;
            for (int64_t i = s; i < e; ++i) acc += prod[i - a0];
        } else {
            for (int64_t i = s + sub; i < e; i += LANES) acc += prod[i - a0];
#pragma unroll
            for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (ADVANCED && rv && sub == 0 && beta != V(0)) acc = c[r * c_stride] * beta + acc;
        }
        if (rv && sub == 0) {
            c[r * c_stride] = acc;
            dot_acc.add(dot, b, b_stride, r, acc);
        }
    }
}

// Products of the entries start, start + step, ... (< end) of one row, added to ONE accumulator in
// that order.  Four entries per round: the four (col, val) loads and the four gathers of a round
// are issued before the first add, so a thread keeps 4 gathers in flight instead of 1 -- the sum is
// the same sequence of additions as the plain loop.  (In the Zipf twin of cfg2 about a quarter of
// the nonzeros sit in rows that a single warp sums with this loop.)
template <typename V, typename I, bool ADVANCED>
__device__ __forceinline__ V strided_row_sum(int64_t start, int64_t end, int64_t step,
                                             const I* __restrict__ col_idxs,
                                             const V* __restrict__ values, V alpha,
                                             const V* __restrict__ b, int64_t b_stride,
                                             uint64_t pol_first, uint64_t pol_last, V acc = V(0))
{
    int64_t i = start;
    for (; i + 3 * step < end; i += 4 * step) {
        I col[4];
        V val[4], x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            col[k] = ld_stream(col_idxs + i + k * step, pol_first);
            val[k] = ld_stream(values + i + k * step, pol_first);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = ld_gather(b + (int64_t)col[k] * b_stride, pol_last);
#pragma unroll
        for (int k = 0; k < 4; ++k) acc += ADVANCED ? (alpha * val[k]) * x[k] : val[k] * x[k];
    }
    for (; i < end; i += step) {
        const I col = ld_stream(col_idxs + i, pol_first);
        const V val = ld_stream(values + i, pol_first);
        const V x = ld_gather(b + (int64_t)col * b_stride, pol_last);
        acc += ADVANCED ? (alpha * val) * x : val * x;
    }
    return acc;
}

// last row of a tile that does not fit the staging buffer: whole-CTA sum
template <typename V, typename I, bool ADVANCED, int DOT>
__device__ __forceinline__ void long_row(int64_t rl, int64_t sl, int64_t p1,
                                         const I* __restrict__ col_idxs,
                                         const V* __restrict__ values, V alpha, V beta,
                                         const V* __restrict__ b, int64_t b_stride,
                                         V* __restrict__ c, int64_t c_stride, V* red,
                                         DotAcc<V, DOT>& dot_acc, const DotArgs<V>& dot,
                                         uint64_t pol_first, uint64_t pol_last)
{
    const int tid = threadIdx.x;
    V acc = strided_row_sum<V, I, ADVANCED>(sl + tid, p1, kThreads, col_idxs, values, alpha, b, b_stride,
                                            pol_first, pol_last);
    acc = block_sum(acc, red);
    if (tid == 0) {
        if (ADVANCED && beta != V(0)) acc = c[rl * c_stride] * beta + acc;
        c[rl * c_stride] = acc;
        dot_acc.add(dot, b, b_stride, rl, acc);
    }
}

// --------------------------------------------------------------------------
// gather-pipe kernel: scattered gathers, no block barriers, a gather round always in flight
// --------------------------------------------------------------------------
// Every WARP walks its own sequence of small tiles (the plan's `witems` merge items of the same
// 2*row + row_ptrs[row] coordinate, so every row of a tile but the last fits the strip).  Lane l owns
// the nonzeros p0 + l + 32 k, k < 8: coalesced evict-first slab loads, and the gathers of structured
// matrices fall into few cache lines.  Per iteration a warp
//   1. issues the gathers of tile B (column indices loaded one iteration earlier), together with
//      B's values, the row pointers of B's first kGRows + 1 rows and, when beta != 0, c of those rows;
//   2. loads the column indices of the next tile C and the extents of the tile after it;
//   3. sums the rows of the previous tile A from its shared-memory strip -- row pointers and c come
//      from registers, so the row phase waits for no memory while B's gathers are in flight;
//   4. waits for B, parks its products in the strip (the only one: A is done with it).
// Row sums: LANES lanes per row; LANES == 1 adds left to right starting from beta*c (the reference's
// order), a row of kWideRow or more entries is summed by the whole warp (fixed tree), a last row that
// does not fit the strip by an order-preserving strided sum.  Nothing but __syncwarp is needed.
constexpr int kWTile = 256;             // merge items per warp tile without a plan
constexpr int kWCap = kWTile + 64 + 8;  // staged nonzeros per warp tile
constexpr int kWMaxItems = kWCap - 8;   // largest `witems` a plan may choose
constexpr int kWarpsPerCta = 8;
constexpr int kWCtasPerSm = 2;   // warp_pipe_kernel: two strips per warp
constexpr int kGCtasPerSm = 2;   // gather_pipe_kernel: 16 warps per SM; at 3 (80 registers) it spills and is slower
constexpr int kGRows = 64;       // rows per tile whose row pointers and c come with the prefetch
constexpr int kWideRow = 64;     // LANES == 1: rows of this many entries or more are summed by the whole warp

// Merge items per warp tile, from the matrix's average row length d: about min(56, 240 / d) rows, so
// the nonzeros of a tile fill the 8 gather slots of every lane (256) and its rows stay below kGRows.
// cfg2's column parts (d ~ 3): 280 items, ~56 rows, ~168 nonzeros; d = 15: 272 items, ~240 nonzeros.
inline int64_t witems_for(int64_t num_rows, int64_t nnz)
{
    if (num_rows <= 0 || nnz <= 0) return kWTile;
    const double d = (double)nnz / (double)num_rows;
    const double rows = 240.0 / d < 56.0 ? 240.0 / d : 56.0;
    const int64_t items = (int64_t)(rows * (kRowW + d));
    return items < 2 * kRowW ? 2 * kRowW : (items > kWMaxItems ? kWMaxItems : items);
}

template <typename V, typename I, int LANES, bool ADVANCED, int DOT>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kGCtasPerSm)
    gather_pipe_kernel(const int64_t* __restrict__ tiles, int64_t num_tiles, int64_t nnz,
                       const I* __restrict__ row_ptrs, const I* __restrict__ col_idxs,
                       const V* __restrict__ values, const V* __restrict__ alpha_p,
                       const V* __restrict__ b, int64_t b_stride, const V* __restrict__ beta_p,
                       V* __restrict__ c, int64_t c_stride, DotArgs<V> dot)
{
    __shared__ __align__(16) V prod_all[kWarpsPerCta][kWCap];
    __shared__ V red[32];
    __shared__ bool is_last;
    if (DOT && dot.ctl && dot.ctl[0] != 0) return;
    wait_for_block(dot);

    const int lane = threadIdx.x & 31;
    V* prod = prod_all[threadIdx.x >> 5];
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const bool read_c = ADVANCED && beta != V(0);
    const uint64_t pol_last = policy_evict_last();
    const uint64_t pol_first = policy_evict_first();
    const int64_t W = (int64_t)gridDim.x * kWarpsPerCta;
    int64_t t = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);

    // extents of a tile: rows [r0, r1), nonzeros [p0, p1); empty past the end.  Index type I: a matrix
    // with I = int32 has fewer than 2^31 rows and nonzeros.
    struct Ext {
        I r0, p0, r1, p1;
    };
    auto load_ext = [&](int64_t tt) {
        Ext e{0, 0, 0, 0};
        if (tt < num_tiles) {
            const longlong2 a = *reinterpret_cast<const longlong2*>(tiles + 2 * tt);
            const longlong2 bb = *reinterpret_cast<const longlong2*>(tiles + 2 * tt + 2);
            e = Ext{(I)a.x, (I)a.y, (I)bb.x, (I)bb.y};
        }
        return e;
    };
    auto load_cols = [&](const Ext& e, I (&cols)[8]) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int64_t idx = (int64_t)e.p0 + lane + 32 * k;
            cols[k] = idx < e.p1 ? ld_stream(col_idxs + idx, pol_first) : I(0);
        }
    };
    // row_ptrs[r0 + j] / c[r0 + j] of a tile: j < kGRows from the lanes' prefetch registers (all lanes
    // call these together), beyond that a load
    auto rp_at = [&](const I (&rv)[2], const Ext& e, int j, bool ok) -> I {
        const I v0 = __shfl_sync(0xffffffffu, rv[0], j & 31);
        const I v1 = __shfl_sync(0xffffffffu, rv[1], j & 31);
        if (j < 32) return v0;
        if (j < kGRows) return v1;
        if ((int64_t)e.r0 + j == (int64_t)e.r1) return e.p1;
        return ok ? row_ptrs[(int64_t)e.r0 + j] : I(0);
    };
    auto c_at = [&](const V (&cv)[2], const Ext& e, int j, bool ok) -> V {
        const V v0 = __shfl_sync(0xffffffffu, cv[0], j & 31);
        const V v1 = __shfl_sync(0xffffffffu, cv[1], j & 31);
        if (j < 32) return v0;
        if (j < kGRows) return v1;
        return ok ? c[((int64_t)e.r0 + j) * c_stride] : V(0);
    };
    // row sums of tile A: rows [r0, r0 + nrows), products in the strip at (nonzero - p0)
    auto row_phase = [&](const Ext& e, int nrows, const I (&rv)[2], const V (&cv)[2], DotAcc<V, DOT>& dot_acc) {
        constexpr int kRpp = 32 / LANES;
        const int sub = lane % LANES;
        for (int ps = 0; ps * kRpp < nrows; ++ps) {
            const int rloc = ps * kRpp + lane / LANES;
            const bool rv_ok = rloc < nrows;
            const int64_t r = (int64_t)e.r0 + rloc;
            int64_t s = rp_at(rv, e, rloc, rv_ok);
            int64_t en = rp_at(rv, e, rloc + 1, rv_ok);
            V cr = V(0);
            if (read_c) cr = c_at(cv, e, rloc, rv_ok);
            if (!rv_ok) s = en = 0;
            V acc = V(0);
            const bool wide = LANES == 1 && (en - s) >= kWideRow;
            if (LANES == 1) {
                if (!wide) {
                    if (read_c && rv_ok) acc = cr * beta;
                    for (int64_t i = s; i < en; ++i) acc += prod[i - e.p0];
                }
            } else {
                for (int64_t i = s + sub; i < en; i += LANES) acc += prod[i - e.p0];
#pragma unroll
                for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (read_c && rv_ok && sub == 0) acc = cr * beta + acc;
            }
            if (rv_ok && sub == 0 && !wide) {
                c[r * c_stride] = acc;
                dot_acc.add(dot, b, b_stride, r, acc);
            }
            if (LANES == 1) {
                unsigned wm = __ballot_sync(0xffffffffu, wide);
                while (wm) {
                    const int src = __ffs(wm) - 1;
                    wm &= wm - 1;
                    const int64_t ws = __shfl_sync(0xffffffffu, s, src);
                    const int64_t we = __shfl_sync(0xffffffffu, en, src);
                    V part = V(0);
                    for (int64_t i = ws + lane; i < we; i += 32) part += prod[i - e.p0];
                    part = warp_sum(part);  // fixed tree: deterministic
                    if (lane == src) {
                        if (read_c) part = cr * beta + part;
                        c[r * c_stride] = part;
                        dot_acc.add(dot, b, b_stride, r, part);
                    }
                }
            }
        }
    };

    Ext eB = load_ext(t), eC = load_ext(t + W);
    I cB[8];
    load_cols(eB, cB);
    // tile A: the one whose products sit in the strip
    Ext eA{0, 0, 0, 0};
    int nA = 0;
    I rA[2] = {0, 0};
    V cA[2] = {V(0), V(0)};
    DotAcc<V, DOT> dot_acc;
    for (; t < num_tiles; t += W) {
        // 1. gathers, values, row pointers and c of tile B
        const bool have = eB.r1 > eB.r0;
        V xs[8], vB[8];
        I rB[2] = {0, 0};
        V cvB[2] = {V(0), V(0)};
        if (have) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int64_t idx = (int64_t)eB.p0 + lane + 32 * k;
                const bool ok = idx < eB.p1;
                xs[k] = ok ? ld_gather(b + (int64_t)cB[k] * b_stride, pol_last) : V(0);
                vB[k] = ok ? ld_stream(values + idx, pol_first) : V(0);
            }
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int64_t r = (int64_t)eB.r0 + 32 * q + lane;
                if (r <= eB.r1) rB[q] = row_ptrs[r];
                if (read_c && r < eB.r1) cvB[q] = c[r * c_stride];
            }
        }
        // 2. column indices of tile C, extents of the tile after it
        const Ext eD = load_ext(t + 2 * W);
        I cC[8];
        load_cols(eC, cC);
        // 3. row sums of tile A while all of that is in flight
        if (nA > 0) row_phase(eA, nA, rA, cA, dot_acc);
        __syncwarp();
        // 4. products of tile B into the strip
        nA = 0;
        if (have) {
            const int64_t p0 = eB.p0, p1 = eB.p1;
            const bool long_last = (p1 - p0) > kWCap;
            const int nrows = (int)(eB.r1 - eB.r0);
            const int64_t sl = long_last ? (int64_t)rp_at(rB, eB, nrows - 1, true) : p1;
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (p0 + lane + 32 * k < p1)
                    prod[lane + 32 * k] = ADVANCED ? (alpha * vB[k]) * xs[k] : vB[k] * xs[k];
            // (rare) nonzeros beyond the 256 of the registers that still belong to the strip
            for (int64_t i = p0 + 256 + lane; i < sl; i += 32) {
                const I col = ld_stream(col_idxs + i, pol_first);
                const V val = ld_stream(values + i, pol_first);
                const V x = ld_gather(b + (int64_t)col * b_stride, pol_last);
                prod[i - p0] = ADVANCED ? (alpha * val) * x : val * x;
            }
            // a last row that does not fit the strip: the whole warp sums it
            if (long_last && !(dot.skip_from > 0 && p1 - sl >= dot.skip_from)) {
                const int64_t rl = (int64_t)eB.r1 - 1;
                V acc = strided_row_sum<V, I, ADVANCED>(sl + lane, p1, 32, col_idxs, values, alpha, b,
                                                        b_stride, pol_first, pol_last);
                acc = warp_sum(acc);
                if (lane == 0) {
                    if (read_c) acc = c[rl * c_stride] * beta + acc;
                    c[rl * c_stride] = acc;
                    dot_acc.add(dot, b, b_stride, rl, acc);
                }
            }
            eA = eB;
            nA = long_last ? nrows - 1 : nrows;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                rA[q] = rB[q];
                cA[q] = cvB[q];
            }
        }
        __syncwarp();
        eB = eC;
        eC = eD;
#pragma unroll
        for (int k = 0; k < 8; ++k) cB[k] = cC[k];
    }
    if (nA > 0) row_phase(eA, nA, rA, cA, dot_acc);
    if (DOT) dot_epilogue(dot_acc, dot, red, &is_last);
}

// --------------------------------------------------------------------------
// warp-pipe kernel, software pipelined: the row sums of tile k-1 (shared memory only)
// run while the gathers of tile k and the slab loads of tile k+1 are in flight
// --------------------------------------------------------------------------
template <typename V, typename I, int LANES, bool ADVANCED, int DOT>
__global__ void __launch_bounds__(kWarpsPerCta * 32, kWCtasPerSm)
    warp_pipe_kernel(const int64_t* __restrict__ tiles, int64_t num_tiles, int64_t nnz,
                     const I* __restrict__ row_ptrs, const I* __restrict__ col_idxs,
                     const V* __restrict__ values, const V* __restrict__ alpha_p,
                     const V* __restrict__ b, int64_t b_stride, const V* __restrict__ beta_p,
                     V* __restrict__ c, int64_t c_stride, DotArgs<V> dot)
{
    __shared__ __align__(16) V prod_all[kWarpsPerCta][2][kWCap];
    __shared__ V red[32];
    __shared__ bool is_last;
    if (DOT && dot.ctl && dot.ctl[0] != 0) return;
    wait_for_block(dot);

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const uint64_t pol_last = policy_evict_last();
    const uint64_t pol_first = policy_evict_first();
    const int64_t W = (int64_t)gridDim.x * kWarpsPerCta;
    int64_t t = (int64_t)blockIdx.x * kWarpsPerCta + warp;

    auto load_ext = [&](int64_t tt, int64_t (&e)[4]) {
        if (tt < num_tiles) {
            const longlong2 a = *reinterpret_cast<const longlong2*>(tiles + 2 * tt);
            const longlong2 bb = *reinterpret_cast<const longlong2*>(tiles + 2 * tt + 2);
            e[0] = a.x;
            e[1] = a.y;
            e[2] = bb.x;
            e[3] = bb.y;
        } else {
            e[0] = e[1] = e[2] = e[3] = 0;
        }
    };
    auto load_slab = [&](const int64_t (&e)[4], I (&cols)[8], V (&vals)[8]) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int64_t idx = e[1] + lane + 32 * k;
            const bool ok = idx < e[3];
            cols[k] = ok ? ld_stream(col_idxs + idx, pol_first) : I(0);
            vals[k] = ok ? ld_stream(values + idx, pol_first) : V(0);
        }
    };
    // row sums of a finished tile from its strip (reads shared memory + a few row pointers)
    auto row_phase = [&](const V* prod, int64_t r0, int64_t p0, int nrows, I rp_first, DotAcc<V, DOT>& dot_acc) {
        constexpr int kRpp = 32 / LANES;
        const int sub = lane % LANES;
        for (int ps = 0; ps * kRpp < nrows; ++ps) {
            const int rloc = ps * kRpp + lane / LANES;
            const bool rv = rloc < nrows;
            int64_t s = 0, e = 0;
            if (LANES == 1 && ps == 0) {
                const I nxt_rp = __shfl_down_sync(0xffffffffu, rp_first, 1);
                s = rp_first;
                e = (lane == 31) ? (rv ? (int64_t)row_ptrs[r0 + 32] : 0) : (int64_t)nxt_rp;
            } else if (rv) {
                s = row_ptrs[r0 + rloc];
                e = row_ptrs[r0 + rloc + 1];
            }
            if (!rv) s = e = 0;
            V acc = V(0);
            if (LANES == 1) {
                if (ADVANCED && rv && beta != V(0)) acc = c[(r0 + rloc) * c_stride] * beta;
                for (int64_t i = s; i < e; ++i) acc += prod[i - p0];
            } else {
                for (int64_t i = s + sub; i < e; i += LANES) acc += prod[i - p0];
#pragma unroll
                for (int o = LANES / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (ADVANCED && rv && sub == 0 && beta != V(0))
                    acc = c[(r0 + rloc) * c_stride] * beta + acc;
            }
            if (rv && sub == 0) {
                c[(r0 + rloc) * c_stride] = acc;
                dot_acc.add(dot, b, b_stride, r0 + rloc, acc);
            }
        }
    };

    int64_t cur[4], nxt[4];
    I cols[8];
    V vals[8];
    I rp_cur = 0;
    load_ext(t, cur);
    load_ext(t + W, nxt);
    if (cur[2] > cur[0]) {
        load_slab(cur, cols, vals);
        if (lane <= cur[2] - cur[0]) rp_cur = row_ptrs[cur[0] + lane];
    }
    // the tile whose products are parked and still have to be summed
    int64_t prev_r0 = 0, prev_p0 = 0;
    int prev_nrows = 0;
    I prev_rp = 0;
    int par = 0;
    DotAcc<V, DOT> dot_acc;
    for (; t < num_tiles; t += W) {
        const int64_t r0 = cur[0], p0 = cur[1], r1 = cur[2], p1 = cur[3];
        const bool have = r1 > r0;
        bool long_last = false;
        int64_t rl = 0, sl = p1, pend = p1, rows_end = r1;
        V xs[8];
        if (have) {
            long_last = (p1 - p0) > kWCap;
            rl = r1 - 1;
            sl = long_last ? (int64_t)row_ptrs[rl] : p1;
            pend = long_last ? sl : p1;
            rows_end = long_last ? rl : r1;
            // 1. gathers of this tile go out first
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                xs[k] = V(0);
                if (p0 + lane + 32 * k < pend)
                    xs[k] = ld_gather(b + (int64_t)cols[k] * b_stride, pol_last);
            }
        }
        // 2. slab + row pointers of the next tile, extents of the one after it
        I ncols[8];
        V nvals[8];
        I nrp = 0;
        int64_t nn[4];
        load_ext(t + 2 * W, nn);
        if (nxt[2] > nxt[0]) {
            load_slab(nxt, ncols, nvals);
            if (lane <= nxt[2] - nxt[0]) nrp = row_ptrs[nxt[0] + lane];
        }
        // 3. row sums of the PREVIOUS tile while all of that is in flight
        if (prev_nrows > 0) row_phase(prod_all[warp][par ^ 1], prev_r0, prev_p0, prev_nrows, prev_rp, dot_acc);
        prev_nrows = 0;
        // 4. products of this tile into the other strip
        if (have) {
            V* prod = prod_all[warp][par];
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (p0 + lane + 32 * k < pend)
                    prod[lane + 32 * k] = ADVANCED ? (alpha * vals[k]) * xs[k] : vals[k] * xs[k];
            for (int64_t i = p0 + 256 + lane; i < pend; i += 32) {
                const I col = ld_stream(col_idxs + i, pol_first);
                const V val = ld_stream(values + i, pol_first);
                const V x = ld_gather(b + (int64_t)col * b_stride, pol_last);
                prod[i - p0] = ADVANCED ? (alpha * val) * x : val * x;
            }
            if (long_last && !(dot.skip_from > 0 && p1 - sl >= dot.skip_from)) {
                V acc = strided_row_sum<V, I, ADVANCED>(sl + lane, p1, 32, col_idxs, values, alpha, b,
                                                        b_stride, pol_first, pol_last);
                acc = warp_sum(acc);
                if (lane == 0) {
                    if (ADVANCED && beta != V(0)) acc = c[rl * c_stride] * beta + acc;
                    c[rl * c_stride] = acc;
                    dot_acc.add(dot, b, b_stride, rl, acc);
                }
            }
            prev_r0 = r0;
            prev_p0 = p0;
            prev_nrows = (int)(rows_end - r0);
            prev_rp = rp_cur;
            par ^= 1;
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            cols[k] = ncols[k];
            vals[k] = nvals[k];
        }
        rp_cur = nrp;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            cur[q] = nxt[q];
            nxt[q] = nn[q];
        }
    }
    if (prev_nrows > 0) row_phase(prod_all[warp][par ^ 1], prev_r0, prev_p0, prev_nrows, prev_rp, dot_acc);
    if (DOT) dot_epilogue(dot_acc, dot, red, &is_last);
}

// --------------------------------------------------------------------------
// fallback for unaligned base pointers: one tile per CTA, ordinary loads
// --------------------------------------------------------------------------
template <typename V, typename I, int LANES, bool ADVANCED, int DOT>
__global__ void __launch_bounds__(kThreads, 3)
    slab_kernel(const int64_t* __restrict__ tiles, int64_t nnz, const I* __restrict__ row_ptrs,
                const I* __restrict__ col_idxs, const V* __restrict__ values,
                const V* __restrict__ alpha_p, const V* __restrict__ b, int64_t b_stride,
                const V* __restrict__ beta_p, V* __restrict__ c, int64_t c_stride, DotArgs<V> dot)
{
    __shared__ __align__(16) V prod[kCap];
    __shared__ V red[32];
    __shared__ bool is_last;

    const int tid = threadIdx.x;
    if (DOT && dot.ctl && dot.ctl[0] != 0) return;
    const int64_t r0 = tiles[2 * blockIdx.x], p0 = tiles[2 * blockIdx.x + 1];
    const int64_t r1 = tiles[2 * blockIdx.x + 2], p1 = tiles[2 * blockIdx.x + 3];
    DotAcc<V, DOT> dot_acc;
    if (r1 > r0) {
        const int64_t a0 = p0 & ~int64_t(7);
        V alpha = V(1), beta = V(0);
        if (ADVANCED) {
            alpha = *alpha_p;
            beta = *beta_p;
        }
        const uint64_t pol_last = policy_evict_last();
        const uint64_t pol_first = policy_evict_first();
        const bool long_last = (p1 - a0) > kCap;
        const int64_t rl = r1 - 1;
        const int64_t sl = long_last ? (int64_t)row_ptrs[rl] : p1;
        const int64_t pend = long_last ? sl : p1;
        const int64_t rows_end = long_last ? rl : r1;
        if ((((uintptr_t)col_idxs | (uintptr_t)values) & 31u) == 0) {
            // 8 consecutive nonzeros per thread, 128-bit streaming loads
#pragma unroll 2
            for (int64_t base = a0 + (int64_t)tid * 8; base < pend; base += (int64_t)kThreads * 8) {
                I cols[8];
                V vals[8];
                if (base + 8 <= nnz) {
                    ld_stream_x8(col_idxs + base, cols, pol_first);
                    ld_stream_x8(values + base, vals, pol_first);
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const bool ok = base + k < nnz;
                        cols[k] = ok ? ld_stream(col_idxs + base + k, pol_first) : I(0);
                        vals[k] = ok ? ld_stream(values + base + k, pol_first) : V(0);
                    }
                }
                V xs[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int64_t idx = base + k;
                    xs[k] = (idx >= p0 && idx < pend)
                                ? ld_gather(b + (int64_t)cols[k] * b_stride, pol_last)
                                : V(0);
                }
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    prod[base - a0 + k] = ADVANCED ? (alpha * vals[k]) * xs[k] : vals[k] * xs[k];
            }
        } else {
            for (int64_t i = p0 + tid; i < pend; i += kThreads) {
                const I col = ld_stream(col_idxs + i, pol_first);
                const V val = ld_stream(values + i, pol_first);
                const V x = ld_gather(b + (int64_t)col * b_stride, pol_last);
                prod[i - a0] = ADVANCED ? (alpha * val) * x : val * x;
            }
        }
        __syncthreads();
        row_phase<V, LANES, ADVANCED, DOT>(
            r0, rows_end, a0, prod, [&](int64_t r) { return (int64_t)row_ptrs[r]; }, beta, b, b_stride,
            c, c_stride, dot_acc, dot);
        if (long_last && !(dot.skip_from > 0 && p1 - sl >= dot.skip_from))
            long_row<V, I, ADVANCED, DOT>(rl, sl, p1, col_idxs, values, alpha, beta, b, b_stride, c,
                                          c_stride, red, dot_acc, dot, pol_first, pol_last);
    }
    if (DOT) dot_epilogue(dot_acc, dot, red, &is_last);
}

// thread per (row, rhs): reference summation order, any strides
template <typename V, typename I, bool ADVANCED>
__global__ void __launch_bounds__(256)
    multi_rhs_kernel(int64_t num_rows, int64_t num_rhs, const I* __restrict__ row_ptrs,
                     const I* __restrict__ col_idxs, const V* __restrict__ values,
                     const V* __restrict__ alpha_p, const V* __restrict__ b, int64_t b_stride,
                     const V* __restrict__ beta_p, V* __restrict__ c, int64_t c_stride)
{
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const int64_t total = num_rows * num_rhs;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = t / num_rhs;
        const int64_t j = t - row * num_rhs;
        const int64_t s = row_ptrs[row], e = row_ptrs[row + 1];
        V acc = V(0);
        if (ADVANCED && beta != V(0)) acc = c[row * c_stride + j] * beta;
        for (int64_t k = s; k < e; ++k) {
            const V val = values[k];
            const V x = b[(int64_t)col_idxs[k] * b_stride + j];
            acc += ADVANCED ? (alpha * val) * x : val * x;
        }
        c[row * c_stride + j] = acc;
    }
}

// --------------------------------------------------------------------------
// several right-hand sides: P = 2..32 lanes per row, lane j owns right-hand side j0 + j
// (grid.y walks j0 in steps of P), 32 / P rows per warp.  Per nonzero the P lanes read the same
// (col, value) -- a broadcast -- and gather P CONSECUTIVE entries of the row-major b: one
// coalesced access serves all right-hand sides.  Every (row, rhs) sum is left to right = the
// reference's order.  The reference runs its vector kernel once per right-hand side (grid.y = #rhs,
// common/cuda_hip/matrix/csr_kernels.template.cpp:2103-2109), i.e. streams the matrix nrhs times.
// --------------------------------------------------------------------------
template <typename V, typename I, bool ADVANCED, int P>
__global__ void __launch_bounds__(256)
    multi_rhs_rows_kernel(int64_t num_rows, int64_t num_rhs, const I* __restrict__ row_ptrs,
                          const I* __restrict__ col_idxs, const V* __restrict__ values,
                          const V* __restrict__ alpha_p, const V* __restrict__ b, int64_t b_stride,
                          const V* __restrict__ beta_p, V* __restrict__ c, int64_t c_stride)
{
    constexpr int kRowsPerWarp = 32 / P;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t row = warp * kRowsPerWarp + lane / P;
    const int64_t j = (int64_t)blockIdx.y * P + lane % P;
    if (row >= num_rows) return;
    const bool jv = j < num_rhs;
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const int64_t s = row_ptrs[row], e = row_ptrs[row + 1];
    V acc = V(0);
    if (ADVANCED && jv && beta != V(0)) acc = c[row * c_stride + j] * beta;
    constexpr int kB = 4;
    for (int64_t k = s; k < e; k += kB) {
        I cc[kB];
        V vv[kB], xx[kB];
#pragma unroll
        for (int q = 0; q < kB; ++q) {
            cc[q] = k + q < e ? col_idxs[k + q] : I(0);
            vv[q] = k + q < e ? values[k + q] : V(0);
        }
#pragma unroll
        for (int q = 0; q < kB; ++q) xx[q] = (k + q < e && jv) ? b[(int64_t)cc[q] * b_stride + j] : V(0);
#pragma unroll
        for (int q = 0; q < kB; ++q)
            if (k + q < e) acc += ADVANCED ? (alpha * vv[q]) * xx[q] : vv[q] * xx[q];
    }
    if (jv) c[row * c_stride + j] = acc;
}

// --------------------------------------------------------------------------
// rows split over CTAs (skewed matrices): the plan lists every row with >= kLongRow entries and
// cuts it into chunks of kLongChunk; one CTA per chunk adds its products (thread t takes entries
// t, t + 256, ... in order, then a fixed tree), the CTA that finishes a row last adds the row's
// chunk sums IN CHUNK ORDER and writes c.  Deterministic, no floating-point atomics.  Replaces the
// carry fix-up of the reference's merge-path / load-balance kernels
// (common/cuda_hip/matrix/csr_kernels.template.cpp:208-505), which use atomic_add.
// --------------------------------------------------------------------------
// 1024: a row below the threshold is at most 32 rounds of 32 entries for the one warp that owns it, so
// the static deal of tiles to warps stays balanced; everything longer goes to long_rows_kernel, which
// runs at the gather rate of the memory system (with higher thresholds, single warps summing
// multi-thousand-entry rows of the Zipf twin of cfg2 became the tail of the main kernel)
constexpr int64_t kLongRow = 1024;
constexpr int64_t kLongChunk = 4096;

struct LongRows {
    int64_t num_rows;             // long rows
    int64_t num_chunks;
    const int64_t* row;           // [num_rows] row index, ascending
    const int64_t* chunk_first;   // [num_rows + 1] first chunk of a row
    const int32_t* chunk_row;     // [num_chunks] position of the chunk's row in `row`
    unsigned int* tickets;        // [num_rows] self-resetting
    void* partials;               // [num_chunks] value type
};

template <typename V, typename I, bool ADVANCED>
__global__ void __launch_bounds__(256) long_rows_kernel(LongRows lr, const I* __restrict__ row_ptrs,
                                                       const I* __restrict__ col_idxs,
                                                       const V* __restrict__ values,
                                                       const V* __restrict__ alpha_p,
                                                       const V* __restrict__ b, int64_t b_stride,
                                                       const V* __restrict__ beta_p, V* __restrict__ c,
                                                       int64_t c_stride, const int32_t* ctl,
                                                       const unsigned long long* wait_flag,
                                                       unsigned long long wait_epoch)
{
    __shared__ V red[32];
    __shared__ bool last;
    if (ctl && ctl[0] != 0) return;
    {  // multi-GPU pipelining: the owner block this launch gathers from must have landed (see DotArgs)
        DotArgs<V> w{};
        w.wait_flag = wait_flag;
        w.wait_epoch = wait_epoch;
        wait_for_block(w);
    }
    const int tid = threadIdx.x;
    const int64_t chunk = blockIdx.x;
    const int k = lr.chunk_row[chunk];
    const int64_t row = lr.row[k];
    const int64_t s = (int64_t)row_ptrs[row] + (chunk - lr.chunk_first[k]) * kLongChunk;
    int64_t e = s + kLongChunk;
    const int64_t row_end = row_ptrs[row + 1];
    if (e > row_end) e = row_end;
    V alpha = V(1), beta = V(0);
    if (ADVANCED) {
        alpha = *alpha_p;
        beta = *beta_p;
    }
    const uint64_t pol_last = policy_evict_last();
    const uint64_t pol_first = policy_evict_first();
    V acc = strided_row_sum<V, I, ADVANCED>(s + tid, e, 256, col_idxs, values, alpha, b, b_stride, pol_first,
                                            pol_last);
    acc = block_sum(acc, red);
    V* partials = (V*)lr.partials;
    if (tid == 0) {
        partials[chunk] = acc;
        __threadfence();
        const unsigned nchunks = (unsigned)(lr.chunk_first[k + 1] - lr.chunk_first[k]);
        last = atomicAdd(lr.tickets + k, 1u) == nchunks - 1;
    }
    __syncthreads();
    if (last && tid == 0) {
        __threadfence();
        lr.tickets[k] = 0u;
        V sum = V(0);
        for (int64_t q = lr.chunk_first[k]; q < lr.chunk_first[k + 1]; ++q) sum += __ldcg(partials + q);
        if (ADVANCED && beta != V(0)) sum = c[row * c_stride] * beta + sum;
        c[row * c_stride] = sum;
    }
}

// fused dot: the long rows' share of the dot (b.c, or w.c and c.c with w != nullptr), added in row
// order after the main kernel has written the dot(s) of all other rows
template <typename V>
__global__ void long_rows_dot_fix_kernel(LongRows lr, const V* __restrict__ b, int64_t b_stride,
                                         const V* __restrict__ c, int64_t c_stride, V* result,
                                         const int32_t* ctl, const V* __restrict__ w, V* result2)
{
    if (ctl && ctl[0] != 0) return;
    V t = *result;
    if (w == nullptr) {
        for (int64_t k = 0; k < lr.num_rows; ++k) t += b[lr.row[k] * b_stride] * c[lr.row[k] * c_stride];
    } else {
        V t2 = result2 ? *result2 : V(0);
        for (int64_t k = 0; k < lr.num_rows; ++k) {
            const V cr = c[lr.row[k] * c_stride];
            t += w[lr.row[k]] * cr;
            t2 += cr * cr;
        }
        if (result2) *result2 = t2;
    }
    *result = t;
}

}  // namespace csr
}  // namespace b200
