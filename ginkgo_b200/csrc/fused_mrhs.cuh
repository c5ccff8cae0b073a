// What the fused iterations for k = 2..32 right-hand sides (fused_cg_mrhs.cu, fused_bicgstab_mrhs.cu,
// fused_gmres_mrhs.cu, fused_minres_mrhs.cu) share: the row / lane layout of their n x k row-major vectors (stride k), the
// bounded grids and the workspace, the per-column sums, the all-stopped test and the SpMV whose epilogue
// sums per-column products.
//
// Layout: P = next power of two >= k lanes per row; lane j works on column j of the k-wide row.
// Grids are bounded and walk the rows grid-stride, so the per-CTA partials fit a fixed workspace.
//
// Sums: per CTA a fixed shuffle tree over the lanes of one column, then the warps in order; the CTA
// that takes the last ticket adds the CTA partials of each column in a fixed order (one warp per
// column).  No floating-point atomics: two runs on the same inputs give the same bits.
#pragma once
#include "fused_common.cuh"

namespace b200 {
namespace mrhs {

constexpr int kMaxCols = 32;
constexpr int kSpmvThreads = 256;
constexpr int kSpmvCtasPerSm = 8;
constexpr int kStepCtasPerSm = 4;

inline int lanes_for(int64_t k)
{
    int P = 2;
    while (P < k && P < kMaxCols) P *= 2;
    return P;
}
inline int64_t spmv_cap(const b200_ctx* ctx) { return (int64_t)ctx->num_sms * kSpmvCtasPerSm; }
inline int64_t step_cap(const b200_ctx* ctx) { return (int64_t)ctx->num_sms * kStepCtasPerSm; }

// rows in flight per CTA sweep = THREADS / P; about 4 sweeps per CTA before the cap is reached
template <int THREADS>
inline int rows_grid(int64_t rows, int P, int64_t cap)
{
    int64_t g = ceildiv(rows, (int64_t)(THREADS / P) * 4);
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// NV sums per column over the CTA: in each warp a fixed shuffle tree over the lanes of one column
// (lane j, j + P, ...), then the warps in order.  Thread j < P returns column j's sums in a[].
template <typename V, int P, int NV, int THREADS>
__device__ __forceinline__ void cta_column_sums(V (&a)[NV], V (&red)[NV][THREADS / 32][P])
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int off = 16; off >= P; off >>= 1)
#pragma unroll
        for (int v = 0; v < NV; ++v) a[v] += __shfl_xor_sync(0xffffffffu, a[v], off);
    if (lane < P)
#pragma unroll
        for (int v = 0; v < NV; ++v) red[v][warp][lane] = a[v];
    __syncthreads();
    if (tid < P)
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            V s = V(0);
            for (int w = 0; w < THREADS / 32; ++w) s += red[v][w][tid];
            a[v] = s;
        }
}

// The last-CTA part of a grid-wide sum of per_cta values per CTA (partials[c * per_cta + idx] from CTA
// c), by every thread once the CTA's partials are written and fenced: the ticket, then in the CTA with
// the last one the partials of every index in CTA order -- one warp per index, lanes over the CTAs, then
// a fixed shuffle tree -- handed to store(idx, sum) by lane 0.  Returns true in that CTA only, after a
// barrier; the ticket is back at 0.
template <int THREADS, typename V, typename Store>
__device__ __forceinline__ bool last_cta_sums(int64_t per_cta, const V* __restrict__ partials,
                                              unsigned int* counter, bool* is_last, Store store)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __syncthreads();
    if (!fused::last_ticket(counter, is_last)) return false;
    __threadfence();
    for (int idx = warp; idx < per_cta; idx += THREADS / 32) {
        V s = V(0);
        for (int c = lane; c < (int)gridDim.x; c += 32) s += __ldcg(partials + c * per_cta + idx);
        s = warp_sum(s);
        if (lane == 0) store(idx, s);
    }
    __syncthreads();
    if (tid == 0) *counter = 0u;
    return true;
}

// the grid-wide part of NV sums per column: thread j < k publishes its column's NV CTA sums, and the CTA
// with the last ticket adds the partials of every (sum, column) into tot[v][j] (last_cta_sums).  Returns
// true in that CTA only, after a barrier; the ticket is back at 0.
template <typename V, int NV, int THREADS>
__device__ __forceinline__ bool grid_column_sums(const V (&a)[NV], int64_t k, V* __restrict__ partials,
                                                 unsigned int* counter, V (&tot)[NV][kMaxCols], bool* is_last)
{
    const int tid = threadIdx.x;
    const int64_t per_cta = NV * k;
    if (tid < k) {
#pragma unroll
        for (int v = 0; v < NV; ++v) partials[blockIdx.x * per_cta + v * k + tid] = a[v];
        __threadfence();
    }
    return last_cta_sums<THREADS>(per_cta, partials, counter, is_last,
                                  [&](int idx, V s) { tot[idx / k][idx % k] = s; });
}

// By thread 0, after every column's status is written: have all k columns stopped?  The callers raise
// ctl[0] = 1 then and otherwise leave ctl[0] as it is, which is the same as writing 0: a kernel that gets
// here started with ctl[0] == 0 (it returns at entry otherwise, and init has just cleared it).
__device__ __forceinline__ bool all_stopped(int64_t k, const uint8_t* status)
{
    bool all = true;
    for (int c = 0; c < (int)k; ++c) all = all && has_stopped(status[c]);
    return all;
}

// `work` of the k-column paths: the SpMV's partials (Epi::NV k per CTA), then the step kernels' from this
// offset on
template <typename Epi>
inline int64_t step_partials_offset(const b200_ctx* ctx, int64_t k)
{
    return spmv_cap(ctx) * Epi::NV * k;
}

// SpMV epilogues: what each (row, column) of c adds to its column's sums, and where the sums go, and
// SUB: whether the SpMV is c = A b - c (the advanced SpMV with (1, -1)) instead of c = A b.
// DotB: dots[j] = sum b_j . c_j (b is the SpMV input: CG's p . A p).
struct DotB {
    static constexpr int NV = 1;
    static constexpr bool SUB = false;
    template <typename V>
    __device__ __forceinline__ static void add(V (&a)[NV], const V* __restrict__ b, const V* __restrict__ w,
                                               int64_t e, V c)
    {
        a[0] += b[e] * c;
    }
    template <typename V>
    __device__ __forceinline__ static void store(const V (&tot)[NV][kMaxCols], V* dots, V* dots2, int j)
    {
        dots[j] = tot[0][j];
    }
};
// DotW2: dots[j] = sum w_j . c_j with a caller-given n x k w, and dots2[j] = sum c_j . c_j unless
// dots2 is null (BiCGStab's rr . v, and s . t with t . t)
struct DotW2 {
    static constexpr int NV = 2;
    static constexpr bool SUB = false;
    template <typename V>
    __device__ __forceinline__ static void add(V (&a)[NV], const V* __restrict__ b, const V* __restrict__ w,
                                               int64_t e, V c)
    {
        a[0] += w[e] * c;
        a[1] += c * c;
    }
    template <typename V>
    __device__ __forceinline__ static void store(const V (&tot)[NV][kMaxCols], V* dots, V* dots2, int j)
    {
        dots[j] = tot[0][j];
        if (dots2) dots2[j] = tot[1][j];
    }
};
// SubDotB: c = A b - c and DotB's sums (MINRES's v = A z - v, alpha = z . v)
struct SubDotB : DotB {
    static constexpr bool SUB = true;
};

// c = A b (Epi::SUB: A b - c) for k columns (b, c, w: stride k), the epilogue's per-column sums into
// dots / dots2.  Lane j gathers column j of the k-wide row of b and every (row, column) sum runs left to
// right: the layout of multi_rhs_rows_kernel (csr_kernels.cuh), so c is bit-identical to b200_csr_spmv_*
// with num_rhs = k.  SUB seeds each sum with c * (-1) before the products, as that kernel's ADVANCED
// mode does with (alpha, beta) = (1, -1) (acc = c beta; acc += (alpha v) x, and 1 * v is exact): c is
// bit-identical to b200_csr_advanced_spmv_* with (1, -1) and num_rhs = k.
template <typename V, typename I, int P, typename Epi>
__global__ void __launch_bounds__(kSpmvThreads)
    spmv_mdot_kernel(int64_t num_rows, int64_t k, const I* __restrict__ row_ptrs, const I* __restrict__ col_idxs,
                     const V* __restrict__ values, const V* __restrict__ b, V* __restrict__ c,
                     const V* __restrict__ w, V* __restrict__ dots, V* __restrict__ dots2,
                     V* __restrict__ partials, unsigned int* __restrict__ counter, const int32_t* __restrict__ ctl)
{
    constexpr int NV = Epi::NV;
    __shared__ V red[NV][kSpmvThreads / 32][P];
    __shared__ V tot[NV][kMaxCols];
    __shared__ bool is_last;
    if (ctl && ctl[0] != 0) return;
    constexpr int kRows = kSpmvThreads / P;
    const int j = threadIdx.x % P;
    const bool jv = j < k;
    V a[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) a[v] = V(0);
    for (int64_t row = blockIdx.x * (int64_t)kRows + threadIdx.x / P; row < num_rows;
         row += (int64_t)gridDim.x * kRows) {
        const int64_t s = row_ptrs[row], e = row_ptrs[row + 1];
        V acc = V(0);
        if (Epi::SUB && jv) acc = c[row * k + j] * V(-1);
        constexpr int kB = 4;
        for (int64_t t = s; t < e; t += kB) {
            I cc[kB];
            V vv[kB], xx[kB];
#pragma unroll
            for (int u = 0; u < kB; ++u) {
                cc[u] = t + u < e ? col_idxs[t + u] : I(0);
                vv[u] = t + u < e ? values[t + u] : V(0);
            }
#pragma unroll
            for (int u = 0; u < kB; ++u) xx[u] = (t + u < e && jv) ? b[(int64_t)cc[u] * k + j] : V(0);
#pragma unroll
            for (int u = 0; u < kB; ++u)
                if (t + u < e) acc += vv[u] * xx[u];
        }
        if (jv) {
            c[row * k + j] = acc;
            Epi::add(a, b, w, row * k + j, acc);
        }
    }
    cta_column_sums<V, P, NV, kSpmvThreads>(a, red);
    if (!grid_column_sums<V, NV, kSpmvThreads>(a, k, partials, counter, tot, &is_last)) return;
    if (threadIdx.x < k) Epi::store(tot, dots, dots2, threadIdx.x);
}

#define B200_MRHS_BY_LANES(P, CALL) \
    switch (P) {                    \
    case 2: CALL(2); break;         \
    case 4: CALL(4); break;         \
    case 8: CALL(8); break;         \
    case 16: CALL(16); break;       \
    default: CALL(32); break;       \
    }

// the host side: checks, the bounded grid (one CTA without rows: it writes zero sums), the launch
template <typename V, typename I, typename Epi>
b200_status spmv_mdot(b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t nnz, const I* row_ptrs,
                      const I* col_idxs, const V* values, const V* b, int64_t k, V* c, const V* w, V* dots,
                      V* dots2, V* partials, const int32_t* ctl)
{
    B200_REQUIRE(ctx && dots && partials, "null argument");
    B200_REQUIRE(num_rows >= 0 && num_cols >= 0 && nnz >= 0, "negative size");
    B200_REQUIRE(k >= 2 && k <= kMaxCols, "k must be in [2, 32]");
    B200_REQUIRE(num_rows == 0 || (row_ptrs && c && b), "null pointer");
    B200_REQUIRE(nnz == 0 || (col_idxs && values), "null pointer");
    const int P = lanes_for(k);
    const int grid = rows_grid<kSpmvThreads>(num_rows, P, spmv_cap(ctx));
#define B200_MD(PP)                                                                                      \
    spmv_mdot_kernel<V, I, PP, Epi><<<grid, kSpmvThreads, 0, ctx->stream>>>(                              \
        num_rows, k, row_ptrs, col_idxs, values, b, c, w, dots, dots2, partials, ctx->counters + kSpmvDotCounter, ctl)
    B200_MRHS_BY_LANES(P, B200_MD)
#undef B200_MD
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
}

}  // namespace mrhs
}  // namespace b200
