// csr_launch.cuh -- the CSR plan (the analogue of the reference's `srow`, include/ginkgo/core/matrix/
// csr.hpp:470-507) and the choice / launch of the SpMV kernel variant.
//
// Variants (every one sums a row's products in the same order, so the choice never changes a bit):
//   kCtaRing  csr_ring.cuh   persistent CTA, bulk-copy (cp.async.bulk / UBLKCP) ring of 4 x 48 KB stages,
//                            lane <-> row.  Matrices whose gathers are LOCAL (stencils, bands, FEM).
//   kWarp     gather_pipe    register-prefetched slabs, row pointers and c; the gathers of the next tile are in
//                            flight while a warp sums the rows of the previous one, products parked in a 2.6 KB
//                            strip per warp.  Matrices with SCATTERED gathers (uniformly random columns), small ones.
//   kPipe     warp_pipe      the same tiles, two strips per warp: local gathers on matrices too small for the ring.
//   kSlab     slab_kernel    base pointers without 16-byte alignment.
// The choice is a function of the matrix (b200_csr_plan_tune_*): the locality of its gathers, measured as the
// number of distinct 128-byte lines of b per gather instruction of the lane <-> row schedule on a sample of
// row groups, its size, and the size of b against L2 -- not of a timing (timing is opt-in, B200_CSR_TUNE_TIMING=1).
#pragma once
#include "csr_kernels.cuh"
#include "csr_ring.cuh"

namespace b200 {
namespace csr {

inline int pick_lanes(int64_t num_rows, int64_t nnz)
{
    const double avg = num_rows > 0 ? (double)nnz / (double)num_rows : 0.0;
    if (avg <= 32.0) return 1;
    if (avg <= 64.0) return 2;
    if (avg <= 128.0) return 4;
    if (avg <= 256.0) return 8;
    if (avg <= 512.0) return 16;
    return 32;
}

// ring kernel shape shipped: CAP 3584 nonzeros per stage, tiles of 3072 merge items
constexpr int kRingCap = 3584;
constexpr int kRingItems = kRingCap - 512;

inline int64_t num_tiles_for(int64_t num_rows, int64_t nnz) { return ceildiv(kRowW * num_rows + nnz, kTile); }
inline int64_t num_wtiles_for(int64_t num_rows, int64_t nnz, int64_t items = kWTile)
{
    return ceildiv(kRowW * num_rows + nnz, items);
}
inline int64_t num_rtiles_for(int64_t num_rows, int64_t nnz)
{
    return ceildiv(kRowW * num_rows + nnz, kRingItems);
}

}  // namespace csr
}  // namespace b200

struct b200_csr_plan {
    int64_t num_rows = 0;
    int64_t nnz = 0;
    int64_t num_tiles = 0;
    int64_t* tiles = nullptr;  // device, 2 * (num_tiles + 1): (first row, first nonzero)
    int64_t num_wtiles = 0;
    int64_t* wtiles = nullptr;  // same for the warp kernels' tiles of `witems` items
    int64_t witems = 0;         // witems_for(num_rows, nnz): chosen from the average row length
    int64_t num_rtiles = 0;
    int64_t* rtiles = nullptr;  // same for the ring kernel's kRingItems-item tiles
    int lanes = 1;
    int device = 0;
    int variant = -1;  // kernel variant chosen by b200_csr_plan_tune_*, -1 = not tuned
    float gather_lines = -1.f;  // distinct 128-byte lines of b per gathered element (tune), -1 = unknown
    // rows with >= kLongRow entries (skewed matrices): computed by long_rows_kernel, one CTA per chunk
    // of kLongChunk entries, chunk sums combined in chunk order (csr_kernels.cuh)
    int64_t num_long = 0, num_long_chunks = 0;
    int64_t* long_row = nullptr;          // device [num_long]
    int64_t* long_chunk_first = nullptr;  // device [num_long + 1]
    int32_t* long_chunk_row = nullptr;    // device [num_long_chunks]
    unsigned int* long_tickets = nullptr; // device [num_long], zero, self-resetting
    void* long_partials = nullptr;        // device [num_long_chunks] values (8 bytes each)
    // Column-blocked copy of the matrix (b200_csr_plan_tune_* builds it for scattered gathers into a b
    // larger than L2 keeps): part p holds, row by row, the entries with column in
    // [p * col_block, (p+1) * col_block).  Rows are column-sorted (checked), so applying the parts in
    // order -- part 0 as c = A0 b, part p as c = 1*Ap b + 1*c -- adds every row's products in exactly
    // the original order: same bits, but the gathers of one launch stay inside a slice of b that fits
    // in L2.  The copy holds VALUES: after changing the matrix values in place the caller refreshes it
    // (b200_csr_plan_refresh_values_*); `pos` keeps the split positions for that.
    static constexpr int kMaxParts = 16;
    bool allow_copy = false;  // b200_csr_plan_allow_value_copy: the owner promises to refresh after value changes
    int parts = 0;
    const void* src_cols = nullptr;  // the arrays the copy was made from (identity check)
    const void* src_vals = nullptr;
    void* pos = nullptr;             // I[(parts-1) * num_rows]: first entry of a row in part p+1
    void* part_row_ptrs[kMaxParts] = {};
    void* part_cols[kMaxParts] = {};
    void* part_vals[kMaxParts] = {};
    int64_t part_nnz[kMaxParts] = {};
    int64_t part_bound[kMaxParts + 1] = {};  // part p holds the columns [part_bound[p], part_bound[p+1])
    b200_csr_plan* part_plan[kMaxParts] = {};
    void* ones = nullptr;  // device {1, 1} in the value type
};

namespace b200 {
namespace csr {

template <typename I>
b200_status fill_plan(b200_ctx* ctx, int64_t num_rows, int64_t nnz, const I* row_ptrs,
                      int64_t num_tiles, int64_t* tiles, int64_t tile_items = kTile)
{
    const int block = 256;
    const int grid = (int)ceildiv(num_tiles + 1, block);
    plan_kernel<I><<<grid, block, 0, ctx->stream>>>(row_ptrs, num_rows, num_tiles, tile_items,
                                                    tiles);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

// kernel variants (1 and 3 were the round-1 bulk-copy kernels, superseded by kCtaRing)
enum Variant { kSlab = 0, kWarp = 2, kPipe = 4, kCtaRing = 5 };

inline Variant pick_variant(const void* col_idxs, const void* values,
                            const b200_csr_plan* plan = nullptr)
{
    const uintptr_t a = (uintptr_t)col_idxs | (uintptr_t)values;
    const char* env = getenv("B200_CSR_KERNEL");
    Variant want = (plan && plan->variant >= 0) ? (Variant)plan->variant : kWarp;
    if (env && !strcmp(env, "slab")) want = kSlab;
    if (env && !strcmp(env, "warp")) want = kWarp;
    if (env && !strcmp(env, "pipe")) want = kPipe;
    if (env && !strcmp(env, "ring") && plan && plan->rtiles) want = kCtaRing;
    if (want == kCtaRing && ((a & 15u) || !plan || !plan->rtiles)) want = kWarp;  // bulk copies: 16-byte alignment
    return want;
}

// tile array / tile count a variant works on without a plan (the ring always has one)
inline int64_t variant_tiles(Variant v, int64_t num_rows, int64_t nnz)
{
    return v == kSlab ? num_tiles_for(num_rows, nnz) : num_wtiles_for(num_rows, nnz);
}
inline const int64_t* plan_tiles(const b200_csr_plan* plan, Variant v, int64_t* count)
{
    if (v == kCtaRing) {
        *count = plan->num_rtiles;
        return plan->rtiles;
    }
    if (v == kSlab) {
        *count = plan->num_tiles;
        return plan->tiles;
    }
    *count = plan->num_wtiles;
    return plan->wtiles;
}

// number of CTAs a launch uses (the size of the fused-dot partials array)
inline int grid_size(const b200_ctx* ctx, Variant v, int64_t num_tiles)
{
    if (v == kSlab) return (int)num_tiles;
    if (v == kCtaRing) return (int)(num_tiles < ctx->num_sms ? num_tiles : ctx->num_sms);
    const int64_t need = ceildiv(num_tiles, kWarpsPerCta);
    const int64_t cap = (int64_t)ctx->num_sms * (v == kWarp ? kGCtasPerSm : kWCtasPerSm);
    return (int)(need < cap ? need : cap);
}
inline int max_grid_size(const b200_ctx* ctx) { return ctx->num_sms * 4; }

// ring configuration: short rows need more consumer warps (a pass = 32 rows is one gather round
// trip; cfg3, 7 nnz/row, is faster with 28 warps than with 16), long rows fewer (the banded twin,
// 15 nnz/row, is faster with 16)
template <typename V, typename I, int LANES, bool ADVANCED, int DOT>
b200_status launch_ring_auto(b200_ctx* ctx, int64_t num_tiles, const int64_t* tiles, int64_t nnz,
                             int64_t num_rows, const I* row_ptrs, const I* col_idxs, const V* values,
                             const V* alpha, const V* b, int64_t b_stride, const V* beta, V* c,
                             int64_t c_stride, DotArgs<V> dot, int grid)
{
    constexpr size_t stage = RingStage<V, I, kRingCap>::bytes;
    constexpr int STAGES = stage * 4 <= 225 * 1024 ? 4 : (stage * 3 <= 225 * 1024 ? 3 : 2);
    constexpr int NP = STAGES % 2 == 0 ? 2 : 1;
    const bool short_rows = nnz < 10 * num_rows * LANES;
    if (short_rows)
        return launch_ring<V, I, LANES, ADVANCED, DOT, 28, 8, false, kRingCap, STAGES, NP>(
            ctx, num_tiles, tiles, nnz, num_rows, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c,
            c_stride, dot, grid);
    return launch_ring<V, I, LANES, ADVANCED, DOT, 16, 8, false, kRingCap, STAGES, NP>(
        ctx, num_tiles, tiles, nnz, num_rows, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c,
        c_stride, dot, grid);
}

template <typename V, typename I, int LANES, bool ADVANCED, int DOT>
b200_status launch_one(b200_ctx* ctx, Variant v, int64_t num_tiles, const int64_t* tiles,
                       int64_t nnz, const I* row_ptrs, const I* col_idxs, const V* values,
                       const V* alpha, const V* b, int64_t b_stride, const V* beta, V* c,
                       int64_t c_stride, DotArgs<V> dot, int grid)
{
    if (v == kPipe) {
        warp_pipe_kernel<V, I, LANES, ADVANCED, DOT><<<grid, kWarpsPerCta * 32, 0, ctx->stream>>>(
            tiles, num_tiles, nnz, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c, c_stride,
            dot);
    } else if (v == kWarp) {
        auto k = gather_pipe_kernel<V, I, LANES, ADVANCED, DOT>;
        static bool dbg = getenv("B200_DEBUG") != nullptr;
        if (dbg) {
            int nb = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, kWarpsPerCta * 32, 0);
            fprintf(stderr, "[b200] gather_pipe_kernel: %d CTAs/SM, grid %d, tiles %lld\n", nb, grid,
                    (long long)num_tiles);
            dbg = false;
        }
        k<<<grid, kWarpsPerCta * 32, 0, ctx->stream>>>(tiles, num_tiles, nnz, row_ptrs, col_idxs,
                                                       values, alpha, b, b_stride, beta, c, c_stride,
                                                       dot);
    } else {
        slab_kernel<V, I, LANES, ADVANCED, DOT><<<(unsigned)num_tiles, kThreads, 0, ctx->stream>>>(
            tiles, nnz, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c, c_stride, dot);
    }
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

// num_rows is only needed by the ring variant (row_ptrs tail of the last tile)
template <typename V, typename I, bool ADVANCED, int DOT>
b200_status launch_slab(b200_ctx* ctx, int lanes, Variant v, int64_t num_tiles,
                        const int64_t* tiles, int64_t nnz, const I* row_ptrs, const I* col_idxs,
                        const V* values, const V* alpha, const V* b, int64_t b_stride,
                        const V* beta, V* c, int64_t c_stride, DotArgs<V> dot = DotArgs<V>{},
                        int64_t num_rows = -1)
{
    if (num_tiles <= 0) return B200_OK;
    const int grid = grid_size(ctx, v, num_tiles);
    if (v == kCtaRing) {
        B200_REQUIRE(num_rows >= 0, "ring variant needs num_rows");
        // the ring instantiates three row shapes: 1 lane per row, 4 and 32
#define B200_RING(L)                                                                                \
    return launch_ring_auto<V, I, L, ADVANCED, DOT>(ctx, num_tiles, tiles, nnz, num_rows, row_ptrs, \
                                                    col_idxs, values, alpha, b, b_stride, beta, c, \
                                                    c_stride, dot, grid)
        if (lanes <= 1) B200_RING(1);
        if (lanes <= 8) B200_RING(4);
        B200_RING(32);
#undef B200_RING
    }
#define B200_SLAB(L)                                                                           \
    return launch_one<V, I, L, ADVANCED, DOT>(ctx, v, num_tiles, tiles, nnz, row_ptrs,         \
                                              col_idxs, values, alpha, b, b_stride, beta, c,   \
                                              c_stride, dot, grid)
    switch (lanes) {
    case 1: B200_SLAB(1);
    case 2: B200_SLAB(2);
    case 4: B200_SLAB(4);
    case 8: B200_SLAB(8);
    case 16: B200_SLAB(16);
    default: B200_SLAB(32);
    }
#undef B200_SLAB
}

// one SpMV through a plan: the chosen variant on its tiles and -- for plans with rows split over CTAs --
// the long-row kernel NEXT TO it on the context's auxiliary stream (fork / join events): the two write
// disjoint rows of c, the main kernel of a skewed matrix is latency-bound on its many short rows while the
// long-row kernel runs at the gather rate, so together they take little more than the longer of the two.  The long rows'
// share of the fused dot is added after the join.
template <typename V, typename I, bool ADVANCED, int DOT>
b200_status launch_planned(b200_ctx* ctx, const b200_csr_plan* plan, Variant v, int64_t nnz, const I* row_ptrs,
                           const I* col_idxs, const V* values, const V* alpha, const V* b, int64_t b_stride,
                           const V* beta, V* c, int64_t c_stride, DotArgs<V> dot = DotArgs<V>{})
{
    int64_t nt = 0;
    const int64_t* tiles = plan_tiles(plan, v, &nt);
    const bool has_long = plan->num_long > 0;
    if (has_long) {
        dot.skip_from = kLongRow;
        B200_CUDA_CHECK(cudaEventRecord(ctx->fork, ctx->stream));
        B200_CUDA_CHECK(cudaStreamWaitEvent(ctx->aux, ctx->fork, 0));
    }
    // the main kernel goes FIRST: it is persistent with 2 CTAs (512 threads) per SM and leaves three
    // quarters of the thread slots to the CTAs of the long-row kernel; launched the other way round the
    // long-row grid fills every slot and the two run one after the other
    b200_status st = launch_slab<V, I, ADVANCED, DOT>(ctx, plan->lanes, v, nt, tiles, nnz, row_ptrs, col_idxs, values,
                                                     alpha, b, b_stride, beta, c, c_stride, dot, plan->num_rows);
    if (has_long) {
        LongRows lr{plan->num_long,      plan->num_long_chunks, plan->long_row,     plan->long_chunk_first,
                    plan->long_chunk_row, plan->long_tickets,    plan->long_partials};
        long_rows_kernel<V, I, ADVANCED><<<(unsigned)plan->num_long_chunks, 256, 0, ctx->aux>>>(
            lr, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c, c_stride, DOT ? dot.ctl : nullptr,
            dot.wait_flag, dot.wait_epoch);
        ctx->launches++;
        cudaError_t le = cudaGetLastError();
        if (le == cudaSuccess) le = cudaEventRecord(ctx->join, ctx->aux);
        if (le != cudaSuccess && st == B200_OK) {
            b200::set_error("%s:%d: long_rows_kernel -> %s", __FILE__, __LINE__, cudaGetErrorString(le));
            st = B200_ERR_CUDA;
        }
    }
    if (has_long) {
        // always rejoin (also after a failed launch: a capture must not end with a dangling fork)
        cudaError_t e = cudaStreamWaitEvent(ctx->stream, ctx->join, 0);
        if (st == B200_OK && e != cudaSuccess) {
            b200::set_error("%s:%d: cudaStreamWaitEvent -> %s", __FILE__, __LINE__, cudaGetErrorString(e));
            st = B200_ERR_CUDA;
        }
    }
    if (st != B200_OK || !has_long) return st;
    if (DOT) {
        LongRows lr{plan->num_long,      plan->num_long_chunks, plan->long_row,     plan->long_chunk_first,
                    plan->long_chunk_row, plan->long_tickets,    plan->long_partials};
        long_rows_dot_fix_kernel<V><<<1, 1, 0, ctx->stream>>>(lr, b, b_stride, c, c_stride, dot.result, dot.ctl,
                                                              DOT == kDotW2 ? dot.w : nullptr, dot.result2);
        B200_LAUNCH_CHECK(ctx);
    }
    return B200_OK;
}

// the SpMV + dot on a matrix without rows: there are no tiles, so no SpMV kernel runs and writes the sums
template <typename V>
__global__ void empty_dot_kernel(V* dot_out, V* dot2_out, const int32_t* ctl)
{
    if (ctl && ctl[0] != 0) return;
    *dot_out = V(0);
    if (dot2_out) *dot2_out = V(0);
}

// The SpMV + dot entry points of the fused solvers (b200_csr_spmv_{dot,dot2,sub_dot}_*): c = A b, or
// c = alpha A b + beta c (ADVANCED), and the sums of DOT into dot_out (and dot2_out unless it is null, w
// the second operand of kDotW2) through the plan's variant, which must not be kSlab.  `work` holds the
// per-CTA partials; ctl may be null.  A matrix without rows gets zero sums.
template <typename V, typename I, bool ADVANCED, int DOT>
b200_status launch_spmv_dot(b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t nnz,
                            const I* row_ptrs, const I* col_idxs, const V* values, const V* alpha, const V* b,
                            const V* beta, V* c, const V* w, V* dot_out, V* dot2_out, V* work, const int32_t* ctl)
{
    B200_REQUIRE(ctx && plan && (DOT != kDotW2 || w) && dot_out && work, "null argument (a plan is required)");
    B200_REQUIRE(plan->num_rows == num_rows && plan->nnz == nnz, "plan does not match");
    const Variant v = pick_variant(col_idxs, values, plan);
    B200_REQUIRE(v != kSlab, "col_idxs/values must be 32-byte aligned");
    if (num_rows == 0) {
        empty_dot_kernel<V><<<1, 1, 0, ctx->stream>>>(dot_out, dot2_out, ctl);
        B200_LAUNCH_CHECK(ctx);
        return B200_OK;
    }
    DotArgs<V> dot{work, ctx->counters + kSpmvDotCounter, dot_out, ctl};
    dot.w = w;
    dot.result2 = dot2_out;
    return launch_planned<V, I, ADVANCED, DOT>(ctx, plan, v, nnz, row_ptrs, col_idxs, values, alpha, b, 1, beta, c,
                                               1, dot);
}

}  // namespace csr
}  // namespace b200
