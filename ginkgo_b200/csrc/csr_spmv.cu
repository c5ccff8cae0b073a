// C-ABI entry points of the CSR (and COO-on-CSR) SpMV; kernels in csr_kernels.cuh.
#include <algorithm>
#include <vector>

#include "csr_launch.cuh"
#include "scan.cuh"

namespace b200 {
namespace csr {

template <typename V, typename I, bool ADVANCED>
b200_status spmv_impl(b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows,
                      int64_t num_cols, int64_t nnz, const I* row_ptrs, const I* col_idxs,
                      const V* values, const V* alpha, const V* b, int64_t b_stride,
                      int64_t num_rhs, const V* beta, V* c, int64_t c_stride)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    B200_REQUIRE(num_rows >= 0 && num_cols >= 0 && nnz >= 0 && num_rhs >= 0, "negative size");
    B200_REQUIRE(b_stride >= num_rhs && c_stride >= num_rhs, "stride smaller than num_rhs");
    if (num_rows == 0 || num_rhs == 0) return B200_OK;
    B200_REQUIRE(row_ptrs && c, "null pointer");
    B200_REQUIRE(nnz == 0 || (col_idxs && values && b), "null pointer");
    if (ADVANCED) B200_REQUIRE(alpha && beta, "alpha/beta must be device pointers");

    if (num_rhs > 1) {
        // P lanes per row (next power of two >= num_rhs, at most 32), grid.y chunks of P right-hand sides
        int P = 2;
        while (P < num_rhs && P < 32) P *= 2;
        const int64_t rows_per_block = 256 / P;
        dim3 grid((unsigned)ceildiv(num_rows, rows_per_block), (unsigned)ceildiv(num_rhs, (int64_t)P));
#define B200_MRHS(PP)                                                                             \
    multi_rhs_rows_kernel<V, I, ADVANCED, PP><<<grid, 256, 0, ctx->stream>>>(                     \
        num_rows, num_rhs, row_ptrs, col_idxs, values, alpha, b, b_stride, beta, c, c_stride)
        switch (P) {
        case 2: B200_MRHS(2); break;
        case 4: B200_MRHS(4); break;
        case 8: B200_MRHS(8); break;
        case 16: B200_MRHS(16); break;
        default: B200_MRHS(32); break;
        }
#undef B200_MRHS
        B200_LAUNCH_CHECK(ctx);
        return B200_OK;
    }

    if (plan && plan->parts > 1 && plan->src_cols == (const void*)col_idxs &&
        plan->src_vals == (const void*)values) {
        // column-blocked copy: part 0 starts the row sums, the others continue them
        const V* ones = (const V*)plan->ones;
        for (int p = 0; p < plan->parts; ++p) {
            const b200_csr_plan* sub = plan->part_plan[p];
            const Variant v = pick_variant(plan->part_cols[p], plan->part_vals[p], sub);
            b200_status st;
            if (p == 0 && !ADVANCED)
                st = launch_planned<V, I, false, false>(
                    ctx, sub, v, plan->part_nnz[p], (const I*)plan->part_row_ptrs[p],
                    (const I*)plan->part_cols[p], (const V*)plan->part_vals[p], nullptr, b, b_stride,
                    nullptr, c, c_stride);
            else
                st = launch_planned<V, I, true, false>(
                    ctx, sub, v, plan->part_nnz[p], (const I*)plan->part_row_ptrs[p],
                    (const I*)plan->part_cols[p], (const V*)plan->part_vals[p],
                    ADVANCED ? alpha : ones, b, b_stride, (ADVANCED && p == 0) ? beta : ones + 1, c,
                    c_stride);
            if (st != B200_OK) return st;
        }
        return B200_OK;
    }
    const Variant variant = pick_variant(col_idxs, values, plan);
    int64_t num_tiles = variant_tiles(variant, num_rows, nnz);
    const int64_t* tiles = nullptr;
    int lanes;
    if (plan) {
        B200_REQUIRE(plan->num_rows == num_rows && plan->nnz == nnz,
                     "plan does not match the matrix");
        return launch_planned<V, I, ADVANCED, false>(ctx, plan, variant, nnz, row_ptrs, col_idxs, values, alpha, b,
                                                     b_stride, beta, c, c_stride);
    } else {
        int64_t* tr = (int64_t*)ctx->scratch(2 * (num_tiles + 1) * sizeof(int64_t));
        if (!tr) {
            set_error("scratch allocation failed");
            return B200_ERR_ALLOC;
        }
        b200_status st = fill_plan<I>(ctx, num_rows, nnz, row_ptrs, num_tiles, tr,
                                      variant != kSlab ? kWTile : kTile);
        if (st != B200_OK) return st;
        tiles = tr;
        lanes = pick_lanes(num_rows, nnz);
    }
    return launch_slab<V, I, ADVANCED, false>(ctx, lanes, variant, num_tiles, tiles, nnz, row_ptrs,
                                              col_idxs, values, alpha, b, b_stride, beta, c,
                                              c_stride, DotArgs<V>{}, num_rows);
}

// rows with >= kLongRow entries -> plan->long_*  (synchronises; set-up time)
template <typename I>
__global__ void find_long_rows_kernel(int64_t num_rows, const I* __restrict__ rp, int64_t min_len,
                                      unsigned long long* __restrict__ count, int64_t cap,
                                      int64_t* __restrict__ list)
{
    const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (row >= num_rows) return;
    if ((int64_t)rp[row + 1] - (int64_t)rp[row] >= min_len) {
        const unsigned long long k = atomicAdd(count, 1ull);
        if ((int64_t)k < cap) list[k] = row;
    }
}

inline void plan_free_long(b200_csr_plan* p)
{
    cudaFree(p->long_row);
    cudaFree(p->long_chunk_first);
    cudaFree(p->long_chunk_row);
    cudaFree(p->long_tickets);
    cudaFree(p->long_partials);
    p->long_row = p->long_chunk_first = nullptr;
    p->long_chunk_row = nullptr;
    p->long_tickets = nullptr;
    p->long_partials = nullptr;
    p->num_long = p->num_long_chunks = 0;
}

template <typename I>
b200_status plan_long_rows(b200_ctx* ctx, b200_csr_plan* p, const I* row_ptrs)
{
    if (p->nnz < kLongRow) return B200_OK;
    const int64_t cap = p->nnz / kLongRow;  // there cannot be more
    char* scratch = (char*)ctx->scratch(16 + (size_t)cap * sizeof(int64_t));
    if (!scratch) return B200_ERR_ALLOC;
    unsigned long long* count = (unsigned long long*)scratch;
    int64_t* list = (int64_t*)(scratch + 16);
    B200_CUDA_CHECK(cudaMemsetAsync(count, 0, sizeof(unsigned long long), ctx->stream));
    find_long_rows_kernel<I><<<(unsigned)ceildiv(p->num_rows, 256), 256, 0, ctx->stream>>>(p->num_rows, row_ptrs,
                                                                                           kLongRow, count, cap, list);
    B200_LAUNCH_CHECK(ctx);
    unsigned long long n = 0;
    B200_CUDA_CHECK(cudaMemcpyAsync(&n, count, sizeof n, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (n == 0) return B200_OK;
    std::vector<int64_t> rows((size_t)n);
    B200_CUDA_CHECK(cudaMemcpy(rows.data(), list, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToHost));
    std::sort(rows.begin(), rows.end());
    std::vector<I> ends(2);
    std::vector<int64_t> first((size_t)n + 1, 0);
    std::vector<int32_t> crow;
    for (size_t k = 0; k < (size_t)n; ++k) {
        B200_CUDA_CHECK(cudaMemcpy(ends.data(), row_ptrs + rows[k], 2 * sizeof(I), cudaMemcpyDeviceToHost));
        const int64_t len = (int64_t)ends[1] - (int64_t)ends[0];
        const int64_t chunks = ceildiv(len, kLongChunk);
        first[k + 1] = first[k] + chunks;
        crow.insert(crow.end(), (size_t)chunks, (int32_t)k);
    }
    p->num_long = (int64_t)n;
    p->num_long_chunks = first[(size_t)n];
    bool ok = cudaMalloc((void**)&p->long_row, sizeof(int64_t) * (size_t)n) == cudaSuccess &&
              cudaMalloc((void**)&p->long_chunk_first, sizeof(int64_t) * ((size_t)n + 1)) == cudaSuccess &&
              cudaMalloc((void**)&p->long_chunk_row, sizeof(int32_t) * crow.size()) == cudaSuccess &&
              cudaMalloc((void**)&p->long_tickets, sizeof(unsigned) * (size_t)n) == cudaSuccess &&
              cudaMalloc(&p->long_partials, 8 * crow.size()) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        plan_free_long(p);  // no room: the kernels' own long-row paths take over (correct, slower)
        return B200_OK;
    }
    B200_CUDA_CHECK(cudaMemcpy(p->long_row, rows.data(), sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice));
    B200_CUDA_CHECK(cudaMemcpy(p->long_chunk_first, first.data(), sizeof(int64_t) * ((size_t)n + 1),
                               cudaMemcpyHostToDevice));
    B200_CUDA_CHECK(cudaMemcpy(p->long_chunk_row, crow.data(), sizeof(int32_t) * crow.size(), cudaMemcpyHostToDevice));
    B200_CUDA_CHECK(cudaMemset(p->long_tickets, 0, sizeof(unsigned) * (size_t)n));
    return B200_OK;
}

template <typename I>
b200_status plan_create(b200_ctx* ctx, int64_t num_rows, int64_t nnz, const I* row_ptrs,
                        b200_csr_plan** out)
{
    B200_REQUIRE(ctx && out, "null argument");
    B200_REQUIRE(num_rows >= 0 && nnz >= 0, "negative size");
    b200_csr_plan* p = new b200_csr_plan();
    p->num_rows = num_rows;
    p->nnz = nnz;
    p->num_tiles = num_tiles_for(num_rows, nnz);
    p->witems = witems_for(num_rows, nnz);
    p->num_wtiles = num_wtiles_for(num_rows, nnz, p->witems);
    p->num_rtiles = num_rtiles_for(num_rows, nnz);
    p->lanes = pick_lanes(num_rows, nnz);
    p->device = ctx->device;
    cudaError_t e = cudaMalloc((void**)&p->tiles,
                               2 * (p->num_tiles + p->num_wtiles + p->num_rtiles + 3) * sizeof(int64_t));
    if (e != cudaSuccess) {
        delete p;
        set_error("cudaMalloc failed for csr plan: %s", cudaGetErrorString(e));
        return B200_ERR_ALLOC;
    }
    p->wtiles = p->tiles + 2 * (p->num_tiles + 1);
    p->rtiles = p->wtiles + 2 * (p->num_wtiles + 1);
    if (num_rows > 0) {
        b200_status st = fill_plan<I>(ctx, num_rows, nnz, row_ptrs, p->num_tiles, p->tiles, kTile);
        if (st == B200_OK)
            st = fill_plan<I>(ctx, num_rows, nnz, row_ptrs, p->num_wtiles, p->wtiles, p->witems);
        if (st == B200_OK)
            st = fill_plan<I>(ctx, num_rows, nnz, row_ptrs, p->num_rtiles, p->rtiles, kRingItems);
        if (st == B200_OK) st = plan_long_rows<I>(ctx, p, row_ptrs);
        if (st != B200_OK) {
            plan_free_long(p);
            cudaFree(p->tiles);
            delete p;
            return st;
        }
    }
    *out = p;
    return B200_OK;
}

// ---- column-blocked copy (see b200_csr_plan) ------------------------------------------
template <typename I>
__global__ void unsorted_rows_kernel(int64_t num_rows, const I* __restrict__ rp,
                                     const I* __restrict__ ci, int* __restrict__ flag)
{
    const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (row >= num_rows) return;
    for (int64_t k = rp[row]; k + 1 < (int64_t)rp[row + 1]; ++k)
        if (ci[k] > ci[k + 1]) {
            *flag = 1;
            return;
        }
}

// pos[(p - 1) * num_rows + row] = first entry of `row` with column >= bounds[p], p = 1..parts-1
struct PartBounds {
    int64_t b[b200_csr_plan::kMaxParts + 1];
};
template <typename I>
__global__ void split_positions_kernel(int64_t num_rows, const I* __restrict__ rp,
                                       const I* __restrict__ ci, int parts, PartBounds bounds,
                                       I* __restrict__ pos)
{
    const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (row >= num_rows) return;
    const int64_t s = rp[row], e = rp[row + 1];
    int64_t k = s;
    for (int p = 1; p < parts; ++p) {
        const int64_t bound = bounds.b[p];
        while (k < e && (int64_t)ci[k] < bound) ++k;
        pos[(int64_t)(p - 1) * num_rows + row] = (I)k;
    }
}

template <typename V, typename I>
__global__ void split_copy_kernel(int64_t num_rows, const I* __restrict__ rp,
                                  const I* __restrict__ ci, const V* __restrict__ va, int parts,
                                  const I* __restrict__ pos, int part,
                                  const I* __restrict__ prp, I* __restrict__ pci,
                                  V* __restrict__ pva)
{
    const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (row >= num_rows) return;
    const int64_t s = part == 0 ? (int64_t)rp[row] : (int64_t)pos[(int64_t)(part - 1) * num_rows + row];
    const int64_t e = part == parts - 1 ? (int64_t)rp[row + 1] : (int64_t)pos[(int64_t)part * num_rows + row];
    int64_t out = prp[row];
    for (int64_t k = s; k < e; ++k, ++out) {
        pci[out] = ci[k];
        pva[out] = va[k];
    }
}

template <typename V>
__global__ void plan_ones_kernel(V* p)
{
    p[0] = V(1);
    p[1] = V(1);
}

inline void plan_drop_parts(b200_csr_plan* plan)
{
    for (int p = 0; p < b200_csr_plan::kMaxParts; ++p) {
        cudaFree(plan->part_row_ptrs[p]);
        cudaFree(plan->part_cols[p]);
        cudaFree(plan->part_vals[p]);
        plan->part_row_ptrs[p] = plan->part_cols[p] = plan->part_vals[p] = nullptr;
        if (plan->part_plan[p]) {
            plan_free_long(plan->part_plan[p]);
            cudaFree(plan->part_plan[p]->tiles);
            delete plan->part_plan[p];
            plan->part_plan[p] = nullptr;
        }
    }
    cudaFree(plan->ones);
    plan->ones = nullptr;
    cudaFree(plan->pos);
    plan->pos = nullptr;
    plan->parts = 0;
}

template <typename I>
b200_status plan_create(b200_ctx* ctx, int64_t num_rows, int64_t nnz, const I* row_ptrs,
                        b200_csr_plan** out);

// Builds the copy; returns B200_OK with plan->parts == 0 when the matrix does not qualify
// (unsorted rows, no memory): the caller then simply keeps the original arrays.
// bounds_host (optional): parts + 1 ascending column boundaries, bounds[0] = 0, bounds[parts] = num_cols;
// nullptr: parts equal column blocks
template <typename V, typename I>
b200_status plan_reblock(b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,
                         int64_t nnz, const I* rp, const I* ci, const V* va, int parts,
                         const int64_t* bounds_host = nullptr)
{
    plan_drop_parts(plan);
    if (parts < 2 || num_rows == 0 || nnz == 0) return B200_OK;
    if (parts > b200_csr_plan::kMaxParts) {
        if (bounds_host) return B200_OK;  // cannot honour the requested boundaries
        parts = b200_csr_plan::kMaxParts;
    }
    const unsigned grid = (unsigned)ceildiv(num_rows, 256);
    int* flag = (int*)ctx->scratch(sizeof(int));
    if (!flag) return B200_OK;
    cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream);
    unsorted_rows_kernel<I><<<grid, 256, 0, ctx->stream>>>(num_rows, rp, ci, flag);
    B200_LAUNCH_CHECK(ctx);
    int unsorted = 0;
    B200_CUDA_CHECK(cudaMemcpyAsync(&unsorted, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (unsorted) return B200_OK;
    I* pos = nullptr;
    I* sums = nullptr;
    bool ok = cudaMalloc((void**)&pos, sizeof(I) * (size_t)(parts - 1) * num_rows) == cudaSuccess &&
              cudaMalloc((void**)&sums, sizeof(I) * (size_t)scan::num_tiles(num_rows + 1)) == cudaSuccess &&
              cudaMalloc(&plan->ones, 2 * sizeof(V)) == cudaSuccess;
    const int64_t col_block = ceildiv(num_cols, (int64_t)parts);
    PartBounds pb;
    for (int p = 0; p <= parts; ++p) {
        pb.b[p] = bounds_host ? bounds_host[p] : (p == parts ? num_cols : p * col_block);
        plan->part_bound[p] = pb.b[p];
    }
    b200_status st = B200_OK;
    if (ok) {
        plan_ones_kernel<V><<<1, 1, 0, ctx->stream>>>((V*)plan->ones);
        ctx->launches++;
        split_positions_kernel<I><<<grid, 256, 0, ctx->stream>>>(num_rows, rp, ci, parts, pb, pos);
        ctx->launches++;
    }
    for (int p = 0; p < parts && ok && st == B200_OK; ++p) {
        ok = cudaMalloc(&plan->part_row_ptrs[p], sizeof(I) * (size_t)(num_rows + 1)) == cudaSuccess;
        if (!ok) break;
        I* prp = (I*)plan->part_row_ptrs[p];
        const I* cpos = pos;
        const int np = parts;
        st = scan::exclusive<I>(
            ctx, num_rows + 1,
            [=] __device__(int64_t r) -> I {
                if (r >= num_rows) return I(0);
                const I s = p == 0 ? rp[r] : cpos[(int64_t)(p - 1) * num_rows + r];
                const I e = p == np - 1 ? rp[r + 1] : cpos[(int64_t)p * num_rows + r];
                return e - s;
            },
            prp, sums);
        if (st != B200_OK) break;
        I last = 0;
        B200_CUDA_CHECK(cudaMemcpyAsync(&last, prp + num_rows, sizeof(I), cudaMemcpyDeviceToHost, ctx->stream));
        B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        plan->part_nnz[p] = (int64_t)last;
        const size_t cnt = (size_t)(last > 0 ? last : 1);
        ok = cudaMalloc(&plan->part_cols[p], sizeof(I) * cnt) == cudaSuccess &&
             cudaMalloc(&plan->part_vals[p], sizeof(V) * cnt) == cudaSuccess;
        if (!ok) break;
        split_copy_kernel<V, I><<<grid, 256, 0, ctx->stream>>>(num_rows, rp, ci, va, parts, pos, p, prp,
                                                               (I*)plan->part_cols[p],
                                                               (V*)plan->part_vals[p]);
        ctx->launches++;
        st = plan_create<I>(ctx, num_rows, plan->part_nnz[p], prp, &plan->part_plan[p]);
    }
    cudaStreamSynchronize(ctx->stream);
    cudaFree(sums);
    if (!ok || st != B200_OK) {
        cudaGetLastError();
        cudaFree(pos);
        plan_drop_parts(plan);
        return st;
    }
    plan->pos = pos;
    plan->parts = parts;
    plan->src_cols = ci;
    plan->src_vals = va;
    return B200_OK;
}

// ---- locality of the gathers --------------------------------------------------------------
// For a sample of groups of 32 consecutive rows (= one pass of the ring kernel's lane <-> row
// schedule): how many distinct 128-byte lines of b does the j-th gather instruction touch, per
// gathered element?  Stencils / bands: 32 neighbouring rows at the same offset = 2-3 lines per 32
// elements (~0.08); uniformly random columns: one line per element (1.0).
template <typename V, typename I>
__global__ void gather_lines_kernel(int64_t num_rows, const I* __restrict__ rp, const I* __restrict__ ci,
                                    int64_t groups, int64_t group_stride, unsigned long long* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int64_t g = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (g >= groups) return;
    const int64_t row = g * group_stride + lane;
    int64_t s = 0, len = 0;
    if (row < num_rows) {
        s = rp[row];
        len = (int64_t)rp[row + 1] - s;
    }
    if (len > 64) len = 64;  // the head of long rows is representative
    const int64_t maxlen = __reduce_max_sync(0xffffffffu, (int)len);
    unsigned long long lines = 0, elems = 0;
    constexpr int kPerLine = 128 / (int)sizeof(V);
    for (int64_t j = 0; j < maxlen; ++j) {
        const bool act = j < len;
        const unsigned mask = __ballot_sync(0xffffffffu, act);
        if (act) {
            const long long line = (long long)ci[s + j] / kPerLine;
            const unsigned same = __match_any_sync(mask, line);
            if ((__ffs(same) - 1) == lane) ++lines;  // one leader per distinct line
            ++elems;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lines += __shfl_xor_sync(0xffffffffu, lines, o);
        elems += __shfl_xor_sync(0xffffffffu, elems, o);
    }
    if (lane == 0) {
        atomicAdd(out, lines);
        atomicAdd(out + 1, elems);
    }
}

template <typename V, typename I>
b200_status plan_gather_lines(b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, const I* rp, const I* ci)
{
    plan->gather_lines = 0.f;
    if (num_rows == 0 || plan->nnz == 0) return B200_OK;
    const int64_t all = ceildiv(num_rows, 32);
    const int64_t groups = all < 4096 ? all : 4096;
    const int64_t stride = (all / groups) * 32;  // evenly spread over the matrix
    unsigned long long* cnt = (unsigned long long*)ctx->scratch(2 * sizeof(unsigned long long));
    if (!cnt) return B200_ERR_ALLOC;
    B200_CUDA_CHECK(cudaMemsetAsync(cnt, 0, 2 * sizeof(unsigned long long), ctx->stream));
    gather_lines_kernel<V, I><<<(unsigned)ceildiv(groups * 32, 256), 256, 0, ctx->stream>>>(num_rows, rp, ci, groups,
                                                                                          stride, cnt);
    B200_LAUNCH_CHECK(ctx);
    unsigned long long h[2] = {0, 0};
    B200_CUDA_CHECK(cudaMemcpyAsync(h, cnt, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    plan->gather_lines = h[1] ? (float)((double)h[0] / (double)h[1]) : 0.f;
    return B200_OK;
}

// Set-up time choice of the kernel variant and of the column-blocked copy -- the analogue of the
// reference's `automatical` strategy, which picks from nnz statistics (include/ginkgo/core/matrix/
// csr.hpp).  A function of the matrix, reproducible run to run and under a profiler:
//   gathers local (<= 0.5 line per element) and >= 2 ring tiles per SM, 16-byte aligned arrays  -> kCtaRing
//   gathers local, smaller matrix                                                               -> kPipe
//   gathers scattered                                                                           -> kWarp,
//       plus the column-blocked copy when b exceeds 3/8 of L2 (parts of <= 5/16 of L2 each) and the
//       rows are column-sorted
// Every variant sums a row in the same order, so the choice never changes a result bit.
// B200_CSR_TUNE_TIMING=1 (opt-in) times the candidates on the matrix instead, as round 1 did.
template <typename V, typename I>
b200_status plan_tune(b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,
                      int64_t nnz, const I* row_ptrs, const I* col_idxs, const V* values)
{
    B200_REQUIRE(ctx && plan, "null argument");
    B200_REQUIRE(plan->num_rows == num_rows && plan->nnz == nnz, "plan does not match the matrix");
    plan->variant = kWarp;
    if (num_rows == 0 || nnz == 0) return B200_OK;
    B200_REQUIRE(row_ptrs && col_idxs && values, "null pointer");
    b200_status st = plan_gather_lines<V, I>(ctx, plan, num_rows, row_ptrs, col_idxs);
    if (st != B200_OK) return st;
    const bool local = plan->gather_lines <= 0.5f;
    const bool aligned = (((uintptr_t)col_idxs | (uintptr_t)values | (uintptr_t)row_ptrs) & 15u) == 0;
    const bool big = plan->num_rtiles >= 2 * (int64_t)ctx->num_sms;
    const int64_t warps = (int64_t)ctx->num_sms * kWCtasPerSm * kWarpsPerCta;
    if (local)
        plan->variant = (big && aligned) ? kCtaRing : (plan->num_wtiles >= 4 * warps ? kPipe : kWarp);
    // column-blocked copy: scattered gathers into a b that does not stay in L2 next to the stream
    // (a slice of 5/16 of L2 stays resident: ~16 MB of an H100's 50 MB)
    const size_t b_bytes = (size_t)num_cols * sizeof(V);
    const size_t part_bytes = ctx->l2_bytes * 5 / 16;
    const char* rb = getenv("B200_CSR_REBLOCK");  // "0" never, "N" force N parts
    int parts = 0;
    if (rb)
        parts = atoi(rb);
    else if (plan->allow_copy && !local && b_bytes > ctx->l2_bytes * 3 / 8 && nnz >= 4 * num_rows)
        parts = (int)((b_bytes + part_bytes - 1) / part_bytes);
    if (parts > b200_csr_plan::kMaxParts) parts = b200_csr_plan::kMaxParts;
    if (parts >= 2) {
        st = plan_reblock<V, I>(ctx, plan, num_rows, num_cols, nnz, row_ptrs, col_idxs, values, parts);
        if (st != B200_OK) return st;
        for (int p = 0; p < plan->parts; ++p) {
            plan->part_plan[p]->variant = plan->variant;
            plan->part_plan[p]->gather_lines = plan->gather_lines;
        }
    }
    static const bool timing = getenv("B200_CSR_TUNE_TIMING") && atoi(getenv("B200_CSR_TUNE_TIMING")) != 0;
    if (timing) {
        // opt-in: time every applicable variant on the matrix itself and keep the fastest
        V *b = nullptr, *c = nullptr;
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        if (cudaMalloc((void**)&b, (size_t)num_cols * sizeof(V)) == cudaSuccess &&
            cudaMalloc((void**)&c, (size_t)num_rows * sizeof(V)) == cudaSuccess &&
            cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess) {
            cudaMemsetAsync(b, 0, (size_t)num_cols * sizeof(V), ctx->stream);
            const Variant cand[3] = {kWarp, kPipe, kCtaRing};
            float best = 0.f;
            int best_v = plan->variant;
            for (int k = 0; k < 3 && st == B200_OK; ++k) {
                if (cand[k] == kCtaRing && !aligned) continue;
                plan->variant = cand[k];
                for (int p = 0; p < plan->parts; ++p) plan->part_plan[p]->variant = cand[k];
                float ms = 0.f;
                for (int r = 0; r <= 3 && st == B200_OK; ++r) {  // r == 0 warms up
                    if (r == 1) cudaEventRecord(e0, ctx->stream);
                    st = spmv_impl<V, I, false>(ctx, plan, num_rows, num_cols, nnz, row_ptrs, col_idxs, values,
                                                nullptr, b, 1, 1, nullptr, c, 1);
                }
                cudaEventRecord(e1, ctx->stream);
                if (cudaEventSynchronize(e1) != cudaSuccess) st = B200_ERR_CUDA;
                if (st == B200_OK) cudaEventElapsedTime(&ms, e0, e1);
                if (st == B200_OK && (best == 0.f || ms < 0.97f * best)) {
                    best = ms;
                    best_v = cand[k];
                }
            }
            plan->variant = best_v;
            for (int p = 0; p < plan->parts; ++p) plan->part_plan[p]->variant = best_v;
        }
        cudaGetLastError();
        cudaFree(b);
        cudaFree(c);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
    if (getenv("B200_DEBUG"))
        fprintf(stderr,
                "[b200] csr plan tuned: rows %lld nnz %lld, %.3f lines of b per gathered element -> %s, "
                "column-blocked parts=%d\n",
                (long long)num_rows, (long long)nnz, plan->gather_lines,
                plan->variant == kCtaRing ? "cta_ring" : (plan->variant == kPipe ? "warp_pipe" : "gather_pipe"),
                plan->parts);
    if (st != B200_OK) set_error("csr plan tuning failed: %s", cudaGetErrorString(cudaGetLastError()));
    return st;
}

// one part of the column-blocked copy: c = A_p b (accumulate == 0) or c += A_p b.  Parts applied in
// ascending order reproduce the row sums of the whole matrix bit for bit; any other order (the
// multi-GPU pipeline applies owner blocks in arrival order) changes the association of the sums.
template <typename V, typename I>
b200_status spmv_part(b200_ctx* ctx, const b200_csr_plan* plan, int part, int accumulate, const V* b,
                      int64_t b_stride, V* c, int64_t c_stride, const unsigned long long* wait_flag,
                      unsigned long long wait_epoch)
{
    B200_REQUIRE(ctx && plan && b && c, "null argument");
    B200_REQUIRE(part >= 0 && part < plan->parts, "no such part");
    const b200_csr_plan* sub = plan->part_plan[part];
    if (plan->part_nnz[part] == 0) {  // empty block: only the first one has something to do (c = 0)
        if (!accumulate) {
            B200_REQUIRE(c_stride == 1, "empty first block needs a contiguous c");
            B200_CUDA_CHECK(cudaMemsetAsync(c, 0, sizeof(V) * (size_t)plan->num_rows, ctx->stream));
        }
        return B200_OK;
    }
    const Variant v = pick_variant(plan->part_cols[part], plan->part_vals[part], sub);
    DotArgs<V> dot{};
    dot.wait_flag = wait_flag;
    dot.wait_epoch = wait_epoch;
    const V* ones = (const V*)plan->ones;
    if (!accumulate)
        return launch_planned<V, I, false, false>(ctx, sub, v, plan->part_nnz[part],
                                                  (const I*)plan->part_row_ptrs[part], (const I*)plan->part_cols[part],
                                                  (const V*)plan->part_vals[part], nullptr, b, b_stride, nullptr, c,
                                                  c_stride, dot);
    return launch_planned<V, I, true, false>(ctx, sub, v, plan->part_nnz[part], (const I*)plan->part_row_ptrs[part],
                                             (const I*)plan->part_cols[part], (const V*)plan->part_vals[part], ones, b,
                                             b_stride, ones + 1, c, c_stride, dot);
}

// values of the column-blocked copy again from the caller's (changed) values array
template <typename V, typename I>
__global__ void split_values_kernel(int64_t num_rows, const I* __restrict__ rp, const V* __restrict__ va, int parts,
                                    const I* __restrict__ pos, int part, const I* __restrict__ prp,
                                    V* __restrict__ pva)
{
    const int64_t row = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (row >= num_rows) return;
    const int64_t s = part == 0 ? (int64_t)rp[row] : (int64_t)pos[(int64_t)(part - 1) * num_rows + row];
    const int64_t e = part == parts - 1 ? (int64_t)rp[row + 1] : (int64_t)pos[(int64_t)part * num_rows + row];
    int64_t out = prp[row];
    for (int64_t k = s; k < e; ++k, ++out) pva[out] = va[k];
}

template <typename V, typename I>
b200_status plan_refresh_values(b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, const I* row_ptrs,
                                const V* values)
{
    B200_REQUIRE(ctx && plan, "null argument");
    B200_REQUIRE(plan->num_rows == num_rows, "plan does not match the matrix");
    if (plan->parts < 2) return B200_OK;  // no copy: nothing can be stale
    B200_REQUIRE(row_ptrs && values && plan->pos, "null pointer");
    const unsigned grid = (unsigned)ceildiv(num_rows, 256);
    for (int p = 0; p < plan->parts; ++p) {
        split_values_kernel<V, I><<<grid, 256, 0, ctx->stream>>>(num_rows, row_ptrs, values, plan->parts,
                                                                 (const I*)plan->pos, p,
                                                                 (const I*)plan->part_row_ptrs[p],
                                                                 (V*)plan->part_vals[p]);
        B200_LAUNCH_CHECK(ctx);
    }
    plan->src_vals = values;
    return B200_OK;
}

}  // namespace csr
}  // namespace b200

extern "C" {

/* csr::is_sorted_by_column_index (core/matrix/csr_kernels.hpp; reference/matrix/csr_kernels.cpp
 * `is_sorted_by_column_index`): 1 iff every row's column indices are non-decreasing.  Blocking
 * (the reference returns the flag through a host bool as well). */
#define B200_DEF_IS_SORTED(I, IT)                                                                \
    b200_status b200_csr_is_sorted_by_column_index_##I(b200_ctx* ctx, int64_t num_rows,          \
                                                       const IT* row_ptrs, const IT* col_idxs,   \
                                                       int32_t* is_sorted_host)                  \
    {                                                                                            \
        B200_REQUIRE(ctx && is_sorted_host, "null argument");                                    \
        *is_sorted_host = 1;                                                                     \
        if (num_rows <= 0) return B200_OK;                                                       \
        B200_REQUIRE(row_ptrs != nullptr, "null pointer");                                       \
        int* flag = (int*)ctx->scratch(sizeof(int));                                             \
        if (!flag) {                                                                             \
            b200::set_error("scratch allocation failed");                                        \
            return B200_ERR_ALLOC;                                                               \
        }                                                                                        \
        B200_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));                     \
        b200::csr::unsorted_rows_kernel<IT><<<(unsigned)b200::ceildiv(num_rows, 256), 256, 0,    \
                                              ctx->stream>>>(num_rows, row_ptrs, col_idxs, flag); \
        B200_LAUNCH_CHECK(ctx);                                                                  \
        int unsorted = 0;                                                                        \
        B200_CUDA_CHECK(cudaMemcpyAsync(&unsorted, flag, sizeof(int), cudaMemcpyDeviceToHost,    \
                                        ctx->stream));                                           \
        B200_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));                                     \
        *is_sorted_host = unsorted ? 0 : 1;                                                      \
        return B200_OK;                                                                          \
    }
B200_DEF_IS_SORTED(i32, int32_t)
B200_DEF_IS_SORTED(i64, int64_t)
#undef B200_DEF_IS_SORTED

int b200_csr_plan_variant(const b200_csr_plan* plan) { return plan ? plan->variant : -1; }
/* overrides the tuned choice (0 slab, 2 gather_pipe, 4 warp_pipe, 5 cta_ring): parity tests and
 * experiments run every variant on the same matrix; results are the same bits whatever is set */
void b200_csr_plan_set_variant(b200_csr_plan* plan, int variant)
{
    if (plan && (variant == 0 || variant == 2 || variant == 4 || variant == 5)) plan->variant = variant;
}
void b200_csr_plan_allow_value_copy(b200_csr_plan* plan, int allow)
{
    if (plan) plan->allow_copy = allow != 0;
}
double b200_csr_plan_gather_lines(const b200_csr_plan* plan) { return plan ? (double)plan->gather_lines : -1.0; }
int b200_csr_plan_parts(const b200_csr_plan* plan) { return plan ? plan->parts : 0; }
int64_t b200_csr_plan_num_long_rows(const b200_csr_plan* plan) { return plan ? plan->num_long : 0; }

void b200_csr_plan_destroy(b200_csr_plan* plan)
{
    if (!plan) return;
    cudaSetDevice(plan->device);
    cudaDeviceSynchronize();
    b200::csr::plan_drop_parts(plan);
    b200::csr::plan_free_long(plan);
    cudaFree(plan->tiles);
    delete plan;
}

#define B200_DEF_CSR(V, VT, I, IT)                                                             \
    b200_status b200_csr_plan_create_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t nnz,   \
                                               const IT* row_ptrs, b200_csr_plan** out)        \
    {                                                                                          \
        return b200::csr::plan_create<IT>(ctx, num_rows, nnz, row_ptrs, out);                  \
    }                                                                                          \
    b200_status b200_csr_plan_tune_##V##_##I(b200_ctx* ctx, b200_csr_plan* plan,               \
                                             int64_t num_rows, int64_t num_cols, int64_t nnz,  \
                                             const IT* row_ptrs, const IT* col_idxs,           \
                                             const VT* values)                                 \
    {                                                                                          \
        return b200::csr::plan_tune<VT, IT>(ctx, plan, num_rows, num_cols, nnz, row_ptrs,      \
                                            col_idxs, values);                                 \
    }                                                                                          \
    b200_status b200_csr_plan_refresh_values_##V##_##I(b200_ctx* ctx, b200_csr_plan* plan,     \
                                                       int64_t num_rows, const IT* row_ptrs,   \
                                                       const VT* values)                       \
    {                                                                                          \
        return b200::csr::plan_refresh_values<VT, IT>(ctx, plan, num_rows, row_ptrs, values);  \
    }                                                                                          \
    b200_status b200_csr_plan_split_columns_##V##_##I(                                         \
        b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, int64_t num_cols, int64_t nnz,   \
        const IT* row_ptrs, const IT* col_idxs, const VT* values, int32_t parts,               \
        const int64_t* bounds_host)                                                            \
    {                                                                                          \
        B200_REQUIRE(ctx && plan && bounds_host, "null argument");                             \
        B200_REQUIRE(plan->num_rows == num_rows && plan->nnz == nnz, "plan does not match");   \
        for (int p = 0; p < parts; ++p)                                                        \
            B200_REQUIRE(bounds_host[p] <= bounds_host[p + 1], "bounds must ascend");          \
        B200_REQUIRE(bounds_host[0] == 0 && bounds_host[parts] == num_cols, "bounds must cover the columns"); \
        b200_status st = b200::csr::plan_reblock<VT, IT>(ctx, plan, num_rows, num_cols, nnz, row_ptrs, col_idxs,    \
                                                        values, parts, bounds_host);           \
        if (st == B200_OK)                                                                     \
            for (int p = 0; p < plan->parts; ++p) plan->part_plan[p]->variant = plan->variant; \
        return st;                                                                             \
    }                                                                                          \
    b200_status b200_csr_spmv_part_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan, int32_t part,      \
                                             int32_t accumulate, const VT* b, int64_t b_stride, VT* c,    \
                                             int64_t c_stride, const uint64_t* wait_flag,      \
                                             uint64_t wait_epoch)                              \
    {                                                                                          \
        return b200::csr::spmv_part<VT, IT>(ctx, plan, part, accumulate, b, b_stride, c, c_stride,        \
                                            (const unsigned long long*)wait_flag,              \
                                            (unsigned long long)wait_epoch);                   \
    }                                                                                          \
    b200_status b200_csr_spmv_##V##_##I(                                                       \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,    \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride)                            \
    {                                                                                          \
        return b200::csr::spmv_impl<VT, IT, false>(ctx, plan, num_rows, num_cols, nnz,         \
                                                   row_ptrs, col_idxs, values, nullptr, b,     \
                                                   b_stride, num_rhs, nullptr, c, c_stride);   \
    }                                                                                          \
    b200_status b200_csr_advanced_spmv_##V##_##I(                                              \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values,                 \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, const VT* beta,       \
        VT* c, int64_t c_stride)                                                               \
    {                                                                                          \
        return b200::csr::spmv_impl<VT, IT, true>(ctx, plan, num_rows, num_cols, nnz,          \
                                                  row_ptrs, col_idxs, values, alpha, b,        \
                                                  b_stride, num_rhs, beta, c, c_stride);       \
    }

B200_DEF_CSR(f64, double, i32, int32_t)
B200_DEF_CSR(f64, double, i64, int64_t)
B200_DEF_CSR(f32, float, i32, int32_t)
B200_DEF_CSR(f32, float, i64, int64_t)

}  // extern "C"

// ===========================================================================
// COO on top of the CSR kernels.  A row-sorted COO is a CSR whose row pointers
// are implicit; convert_idxs_to_ptrs (reference/components/
// format_conversion_kernels.cpp, `convert_idxs_to_ptrs`) writes them down once
// (cached in b200_coo_plan) and every apply then runs the slab kernel:
//   spmv2:           c += A b        == advanced(alpha=1, beta=1)
//   advanced_spmv2:  c += alpha A b  == advanced(alpha,   beta=1)
// The slab kernel starts each row from c*beta and adds the products left to
// right, which is exactly the order of the reference's `c(row) += val*b(col)`
// loop (reference/matrix/coo_kernels.cpp:59-97), so no atomics are needed and
// the result is deterministic -- the reference CUDA path uses atomic_add
// (common/cuda_hip/matrix/coo_kernels.cpp:62-231).
// ===========================================================================
struct b200_coo_plan {
    int64_t num_rows = 0;
    int64_t nnz = 0;
    void* row_ptrs = nullptr;  // device, (num_rows + 1) index_type
    b200_csr_plan* csr = nullptr;
    void* ones = nullptr;  // device: {1.0, 1.0} in the plan's value type
    int device = 0;
};

namespace b200 {
namespace coo {

template <typename I>
__global__ void idxs_to_ptrs_kernel(const I* __restrict__ idxs, int64_t nnz, int64_t num_rows,
                                    I* __restrict__ ptrs)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (nnz == 0) {
        if (i <= num_rows) ptrs[i] = 0;
        return;
    }
    if (i >= nnz) return;
    const int64_t cur = idxs[i];
    const int64_t prev = i == 0 ? -1 : (int64_t)idxs[i - 1];
    for (int64_t r = prev + 1; r <= cur; ++r) ptrs[r] = (I)i;
    if (i == nnz - 1) {
        for (int64_t r = cur + 1; r <= num_rows; ++r) ptrs[r] = (I)nnz;
    }
}

template <typename I>
b200_status idxs_to_ptrs(b200_ctx* ctx, const I* idxs, int64_t nnz, int64_t num_rows, I* ptrs)
{
    const int64_t work = nnz == 0 ? num_rows + 1 : nnz;
    idxs_to_ptrs_kernel<I><<<(unsigned)ceildiv(work, 256), 256, 0, ctx->stream>>>(idxs, nnz, num_rows,
                                                                                  ptrs);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

template <typename V>
__global__ void set_ones_kernel(V* p)
{
    p[0] = V(1);
    p[1] = V(1);
}

template <typename V, typename I>
b200_status plan_create(b200_ctx* ctx, int64_t num_rows, int64_t nnz, const I* row_idxs,
                        b200_coo_plan** out)
{
    B200_REQUIRE(ctx && out, "null argument");
    B200_REQUIRE(num_rows >= 0 && nnz >= 0, "negative size");
    b200_coo_plan* p = new b200_coo_plan();
    p->num_rows = num_rows;
    p->nnz = nnz;
    p->device = ctx->device;
    if (cudaMalloc(&p->row_ptrs, (num_rows + 1) * sizeof(I)) != cudaSuccess ||
        cudaMalloc(&p->ones, 2 * sizeof(V)) != cudaSuccess) {
        set_error("cudaMalloc failed for coo plan");
        cudaFree(p->row_ptrs);
        delete p;
        return B200_ERR_ALLOC;
    }
    b200_status st = idxs_to_ptrs<I>(ctx, row_idxs, nnz, num_rows, (I*)p->row_ptrs);
    if (st == B200_OK) {
        set_ones_kernel<V><<<1, 1, 0, ctx->stream>>>((V*)p->ones);
        ctx->launches++;
        st = csr::plan_create<I>(ctx, num_rows, nnz, (const I*)p->row_ptrs, &p->csr);
    }
    if (st != B200_OK) {
        cudaFree(p->row_ptrs);
        cudaFree(p->ones);
        delete p;
        return st;
    }
    *out = p;
    return B200_OK;
}

// mode: 0 spmv, 1 advanced_spmv, 2 spmv2, 3 advanced_spmv2
template <typename V, typename I>
b200_status apply(b200_ctx* ctx, const b200_coo_plan* plan, int mode, int64_t num_rows,
                  int64_t num_cols, int64_t nnz, const I* row_idxs, const I* col_idxs,
                  const V* values, const V* alpha, const V* b, int64_t b_stride, int64_t num_rhs,
                  const V* beta, V* c, int64_t c_stride)
{
    B200_REQUIRE(ctx != nullptr, "ctx is null");
    B200_REQUIRE(num_rows >= 0 && nnz >= 0, "negative size");
    if (num_rows == 0 || num_rhs == 0) return B200_OK;
    if (nnz == 0 && mode >= 2) return B200_OK;  // c += (nothing): the reference loop is empty
    const I* row_ptrs;
    const b200_csr_plan* cplan = nullptr;
    const V* ones;
    if (plan) {
        B200_REQUIRE(plan->num_rows == num_rows && plan->nnz == nnz, "plan does not match");
        row_ptrs = (const I*)plan->row_ptrs;
        cplan = plan->csr;
        ones = (const V*)plan->ones;
    } else {
        // one scratch block: [ones (16 B) | row_ptrs | csr tiles]; the CSR call below
        // must not re-use ctx->scratch, so the tile array is carved out here too
        const csr::Variant variant = csr::pick_variant(col_idxs, values);
        const int64_t num_tiles = csr::variant_tiles(variant, num_rows, nnz);
        const size_t off_ptrs = 16;
        const size_t off_tiles = (off_ptrs + (num_rows + 1) * sizeof(I) + 15) & ~size_t(15);
        const size_t total = off_tiles + 2 * (num_tiles + 1) * sizeof(int64_t);
        char* base = (char*)ctx->scratch(total);
        if (!base) return B200_ERR_ALLOC;
        V* o = (V*)base;
        I* rp = (I*)(base + off_ptrs);
        int64_t* tiles = (int64_t*)(base + off_tiles);
        set_ones_kernel<V><<<1, 1, 0, ctx->stream>>>(o);
        ctx->launches++;
        b200_status st = idxs_to_ptrs<I>(ctx, row_idxs, nnz, num_rows, rp);
        if (st != B200_OK) return st;
        if (num_rhs == 1) {
            st = csr::fill_plan<I>(ctx, num_rows, nnz, rp, num_tiles, tiles,
                                   variant != csr::kSlab ? csr::kWTile : csr::kTile);
            if (st != B200_OK) return st;
            const csr::Variant tma = variant;
            const int lanes = csr::pick_lanes(num_rows, nnz);
            if (mode == 0)
                return csr::launch_slab<V, I, false, false>(ctx, lanes, tma, num_tiles, tiles, nnz,
                                                            rp, col_idxs, values, nullptr, b,
                                                            b_stride, nullptr, c, c_stride);
            return csr::launch_slab<V, I, true, false>(ctx, lanes, tma, num_tiles, tiles, nnz, rp,
                                                       col_idxs, values, (mode == 2) ? o : alpha, b,
                                                       b_stride, (mode == 1) ? beta : o + 1, c,
                                                       c_stride);
        }
        row_ptrs = rp;
        ones = o;
        // multi-rhs CSR path does not touch ctx->scratch
    }
    switch (mode) {
    case 0:
        return csr::spmv_impl<V, I, false>(ctx, cplan, num_rows, num_cols, nnz, row_ptrs, col_idxs,
                                           values, nullptr, b, b_stride, num_rhs, nullptr, c,
                                           c_stride);
    case 1:
        return csr::spmv_impl<V, I, true>(ctx, cplan, num_rows, num_cols, nnz, row_ptrs, col_idxs,
                                          values, alpha, b, b_stride, num_rhs, beta, c, c_stride);
    case 2:
        return csr::spmv_impl<V, I, true>(ctx, cplan, num_rows, num_cols, nnz, row_ptrs, col_idxs,
                                          values, ones, b, b_stride, num_rhs, ones + 1, c,
                                          c_stride);
    default:
        return csr::spmv_impl<V, I, true>(ctx, cplan, num_rows, num_cols, nnz, row_ptrs, col_idxs,
                                          values, alpha, b, b_stride, num_rhs, ones + 1, c,
                                          c_stride);
    }
}

}  // namespace coo
}  // namespace b200

extern "C" {

void b200_coo_plan_destroy(b200_coo_plan* plan)
{
    if (!plan) return;
    b200_csr_plan_destroy(plan->csr);
    cudaSetDevice(plan->device);
    cudaFree(plan->row_ptrs);
    cudaFree(plan->ones);
    delete plan;
}

#define B200_DEF_COO(V, VT, I, IT)                                                             \
    b200_status b200_coo_plan_create_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t nnz,   \
                                               const IT* row_idxs, b200_coo_plan** out)        \
    {                                                                                          \
        return b200::coo::plan_create<VT, IT>(ctx, num_rows, nnz, row_idxs, out);              \
    }                                                                                          \
    b200_status b200_coo_spmv_##V##_##I(                                                       \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values, const VT* b,    \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride)                            \
    {                                                                                          \
        return b200::coo::apply<VT, IT>(ctx, plan, 0, num_rows, num_cols, nnz, row_idxs,       \
                                        col_idxs, values, nullptr, b, b_stride, num_rhs,       \
                                        nullptr, c, c_stride);                                 \
    }                                                                                          \
    b200_status b200_coo_advanced_spmv_##V##_##I(                                              \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values,                 \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, const VT* beta,       \
        VT* c, int64_t c_stride)                                                               \
    {                                                                                          \
        return b200::coo::apply<VT, IT>(ctx, plan, 1, num_rows, num_cols, nnz, row_idxs,       \
                                        col_idxs, values, alpha, b, b_stride, num_rhs, beta,   \
                                        c, c_stride);                                          \
    }                                                                                          \
    b200_status b200_coo_spmv2_##V##_##I(                                                      \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values, const VT* b,    \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride)                            \
    {                                                                                          \
        return b200::coo::apply<VT, IT>(ctx, plan, 2, num_rows, num_cols, nnz, row_idxs,       \
                                        col_idxs, values, nullptr, b, b_stride, num_rhs,       \
                                        nullptr, c, c_stride);                                 \
    }                                                                                          \
    b200_status b200_coo_advanced_spmv2_##V##_##I(                                             \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values,                 \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, VT* c,                \
        int64_t c_stride)                                                                      \
    {                                                                                          \
        return b200::coo::apply<VT, IT>(ctx, plan, 3, num_rows, num_cols, nnz, row_idxs,       \
                                        col_idxs, values, alpha, b, b_stride, num_rhs,         \
                                        nullptr, c, c_stride);                                 \
    }

B200_DEF_COO(f64, double, i32, int32_t)
B200_DEF_COO(f64, double, i64, int64_t)
B200_DEF_COO(f32, float, i32, int32_t)
B200_DEF_COO(f32, float, i64, int64_t)

}  // extern "C"
