// spmv_lab.cu -- experiment harness (NOT product, NOT test): candidate CSR SpMV kernels of
// ginkgo_b200/csrc side by side + memory-system microbenchmarks (stream read, 8-byte gather
// through LSU, through the TMA gather4 path).  Built by scripts/lab/build.sh, run on the GPU box by
// scripts/lab/run.sh; prints one line per measurement.
//   spmv_lab <group> [matrix]     group: micro | base | ring | tma4       matrix: cfg2 | cfg2h | banded | cfg3 | cfg4
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../ginkgo_b200/csrc/csr_launch.cuh"

using namespace b200;
using namespace b200::csr;

#define CK(x)                                                                              \
    do {                                                                                   \
        cudaError_t e_ = (x);                                                              \
        if (e_ != cudaSuccess) {                                                           \
            printf("CUDA error %s at %s:%d (%s)\n", cudaGetErrorString(e_), __FILE__, __LINE__, #x); \
            exit(2);                                                                       \
        }                                                                                  \
    } while (0)

// the device's shape, filled in by main(): SM count and SM clock from cudaDeviceProp; the HBM peak
// (GB/s) from MEASURED_PEAKS.json ("hbm_gbs") when that file is in the working directory, else the
// H100 SXM data sheet's 3.35 TB/s
static int g_sms = 132;
static double g_ghz = 1.98;
static double kPeak = 3350.0;
static const char* g_peak_src = "data sheet";

static void init_device()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    g_sms = prop.multiProcessorCount;
    int khz = 0;
    CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
    if (khz > 0) g_ghz = khz / 1e6;
    if (FILE* f = fopen("MEASURED_PEAKS.json", "r")) {
        char buf[4096];
        const size_t n = fread(buf, 1, sizeof buf - 1, f);
        fclose(f);
        buf[n] = 0;
        if (const char* k = strstr(buf, "\"hbm_gbs\"")) {
            const char* v = strchr(k, ':');
            const double gbs = v ? atof(v + 1) : 0.0;
            if (gbs > 0) {
                kPeak = gbs;
                g_peak_src = "MEASURED_PEAKS.json";
            }
        }
    }
    printf("device %s: %d SMs, max SM clock %.3f GHz, HBM peak %.0f GB/s (%s)\n", prop.name, g_sms, g_ghz, kPeak,
           g_peak_src);
}

// ------------------------------------------------------------------------------ generators
__host__ __device__ inline uint64_t mix64(uint64_t z)
{
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ inline uint64_t hash3(uint64_t s, uint64_t a, uint64_t b)
{
    return mix64(mix64(s * 0x9E3779B97F4A7C15ull + a) + b * 0xBF58476D1CE4E5B9ull);
}
__host__ __device__ inline double unit(uint64_t h) { return (double)(h >> 11) * (2.0 / 9007199254740992.0) - 1.0; }

template <typename V, int PR>
__global__ void gen_random(int64_t n, int64_t ncols, int64_t col0, int* rp, int* ci, V* va, bool diag)
{
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r > n) return;
    rp[r] = (int)(r * PR);
    if (r == n) return;
    int64_t c[PR];
    const int64_t span = ncols - PR + 1;
    for (int k = 0; k < PR; ++k) c[k] = (int64_t)(hash3(1, r, k) % (uint64_t)span);
    for (int i = 1; i < PR; ++i) {  // insertion sort
        int64_t v = c[i];
        int j = i - 1;
        while (j >= 0 && c[j] > v) {
            c[j + 1] = c[j];
            --j;
        }
        c[j + 1] = v;
    }
    for (int k = 0; k < PR; ++k) {
        ci[r * PR + k] = (int)(col0 + c[k] + k);
        va[r * PR + k] = (V)unit(hash3(101, r, k));
    }
}
// cfg2a: the rows of cfg2 restricted to the columns [0, ncols/2): what the first launch of the
// 2-block column-blocked copy streams (variable row lengths, 40 MB of x)
template <typename V, int PR>
__global__ void gen_random_half(int64_t n, int64_t ncols, const int* rp, int* cnt, int* ci, V* va)
{
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    int64_t c[PR];
    const int64_t span = ncols - PR + 1;
    for (int k = 0; k < PR; ++k) c[k] = (int64_t)(hash3(1, r, k) % (uint64_t)span);
    for (int i = 1; i < PR; ++i) {
        int64_t v = c[i];
        int j = i - 1;
        while (j >= 0 && c[j] > v) {
            c[j + 1] = c[j];
            --j;
        }
        c[j + 1] = v;
    }
    int m = 0;
    for (int k = 0; k < PR; ++k)
        if (c[k] + k < ncols / 2) {
            if (rp) {
                ci[rp[r] + m] = (int)(c[k] + k);
                va[rp[r] + m] = (V)unit(hash3(101, r, k));
            }
            ++m;
        }
    if (cnt) cnt[r] = m;
}
template <typename V>
__global__ void gen_band_fill(int64_t n, int hb, const int* rp, int* ci, V* va)
{
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    int64_t p = rp[r];
    for (int o = -hb; o <= hb; ++o) {
        const int64_t c = r + o;
        if (c < 0 || c >= n) continue;
        ci[p] = (int)c;
        va[p] = (V)unit(hash3(3, r, o + hb));
        ++p;
    }
}
template <typename V>
__global__ void gen_lap3_fill(int64_t g, const int* rp, int* ci, V* va)
{
    const int64_t n = g * g * g;
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int64_t z = r % g, y = (r / g) % g, x = r / (g * g);
    int64_t p = rp[r];
    auto put = [&](int64_t c, double v) {
        ci[p] = (int)c;
        va[p] = (V)v;
        ++p;
    };
    if (x > 0) put(r - g * g, -1);
    if (y > 0) put(r - g, -1);
    if (z > 0) put(r - 1, -1);
    put(r, 6);
    if (z < g - 1) put(r + 1, -1);
    if (y < g - 1) put(r + g, -1);
    if (x < g - 1) put(r + g * g, -1);
}
template <typename V>
__global__ void gen_vec(int64_t n, V* x)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) x[i] = (V)unit(hash3(7, i, 0));
}

template <typename V>
struct Mat {
    int64_t n = 0, ncols = 0, nnz = 0;
    int *rp = nullptr, *ci = nullptr;
    V* va = nullptr;
    std::string name;
};

template <typename V>
Mat<V> make_matrix(const std::string& name)
{
    Mat<V> m;
    m.name = name;
    const int T = 256;
    if (name == "cfg2" || name == "cfg2h" || name == "cfg4") {
        // cfg2: n = 10M, 15/row over all columns; cfg2h: the same rows restricted to the first half
        // of the columns with ~half the entries (what one launch of the 2-block copy sees)
        m.n = name == "cfg4" ? 4000000 : 10000000;
        m.ncols = m.n;
        const int pr = name == "cfg4" ? 20 : (name == "cfg2h" ? 8 : 15);
        m.nnz = m.n * pr;
        CK(cudaMalloc(&m.rp, (m.n + 1) * sizeof(int)));
        CK(cudaMalloc(&m.ci, m.nnz * sizeof(int)));
        CK(cudaMalloc(&m.va, m.nnz * sizeof(V)));
        const int grid = (int)((m.n + 1 + T - 1) / T);
        if (pr == 15) gen_random<V, 15><<<grid, T>>>(m.n, m.ncols, 0, m.rp, m.ci, m.va, false);
        if (pr == 8) gen_random<V, 8><<<grid, T>>>(m.n, m.ncols / 2, 0, m.rp, m.ci, m.va, false);
        if (pr == 20) gen_random<V, 20><<<grid, T>>>(m.n, m.ncols, 0, m.rp, m.ci, m.va, false);
    } else if (name == "cfg2a") {
        m.n = m.ncols = 10000000;
        int* cnt;
        CK(cudaMalloc(&cnt, m.n * sizeof(int)));
        gen_random_half<V, 15><<<(int)((m.n + T - 1) / T), T>>>(m.n, m.ncols, nullptr, cnt, nullptr, nullptr);
        std::vector<int> h(m.n), rp(m.n + 1);
        CK(cudaMemcpy(h.data(), cnt, m.n * sizeof(int), cudaMemcpyDeviceToHost));
        int64_t p = 0;
        for (int64_t r = 0; r < m.n; ++r) {
            rp[r] = (int)p;
            p += h[r];
        }
        rp[m.n] = (int)p;
        m.nnz = p;
        CK(cudaMalloc(&m.rp, (m.n + 1) * sizeof(int)));
        CK(cudaMalloc(&m.ci, m.nnz * sizeof(int)));
        CK(cudaMalloc(&m.va, m.nnz * sizeof(V)));
        CK(cudaMemcpy(m.rp, rp.data(), (m.n + 1) * sizeof(int), cudaMemcpyHostToDevice));
        gen_random_half<V, 15><<<(int)((m.n + T - 1) / T), T>>>(m.n, m.ncols, m.rp, nullptr, m.ci, m.va);
        CK(cudaFree(cnt));
    } else if (name == "banded") {
        m.n = m.ncols = 10000000;
        const int hb = 7;
        std::vector<int> rp(m.n + 1);
        int64_t p = 0;
        for (int64_t r = 0; r < m.n; ++r) {
            rp[r] = (int)p;
            const int64_t lo = std::max<int64_t>(0, r - hb), hi = std::min<int64_t>(m.n - 1, r + hb);
            p += hi - lo + 1;
        }
        rp[m.n] = (int)p;
        m.nnz = p;
        CK(cudaMalloc(&m.rp, (m.n + 1) * sizeof(int)));
        CK(cudaMalloc(&m.ci, m.nnz * sizeof(int)));
        CK(cudaMalloc(&m.va, m.nnz * sizeof(V)));
        CK(cudaMemcpy(m.rp, rp.data(), (m.n + 1) * sizeof(int), cudaMemcpyHostToDevice));
        gen_band_fill<V><<<(int)((m.n + T - 1) / T), T>>>(m.n, hb, m.rp, m.ci, m.va);
    } else {  // cfg3
        const int64_t g = 200;
        m.n = m.ncols = g * g * g;
        std::vector<int> rp(m.n + 1);
        int64_t p = 0;
        for (int64_t r = 0; r < m.n; ++r) {
            rp[r] = (int)p;
            const int64_t z = r % g, y = (r / g) % g, x = r / (g * g);
            p += 1 + (x > 0) + (y > 0) + (z > 0) + (x < g - 1) + (y < g - 1) + (z < g - 1);
        }
        rp[m.n] = (int)p;
        m.nnz = p;
        CK(cudaMalloc(&m.rp, (m.n + 1) * sizeof(int)));
        CK(cudaMalloc(&m.ci, m.nnz * sizeof(int)));
        CK(cudaMalloc(&m.va, m.nnz * sizeof(V)));
        CK(cudaMemcpy(m.rp, rp.data(), (m.n + 1) * sizeof(int), cudaMemcpyHostToDevice));
        gen_lap3_fill<V><<<(int)((m.n + T - 1) / T), T>>>(g, m.rp, m.ci, m.va);
    }
    CK(cudaDeviceSynchronize());
    return m;
}

template <typename V>
__global__ void ref_spmv(int64_t n, const int* rp, const int* ci, const V* va, const V* x, V* y)
{
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    V acc = V(0);
    for (int64_t k = rp[r]; k < rp[r + 1]; ++k) acc += va[k] * x[ci[k]];
    y[r] = acc;
}
template <typename V>
__global__ void count_diff(int64_t n, const V* a, const V* b, unsigned long long* cnt)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool same;
    if (sizeof(V) == 8)
        same = reinterpret_cast<const unsigned long long*>(a)[i] == reinterpret_cast<const unsigned long long*>(b)[i];
    else
        same = reinterpret_cast<const unsigned int*>(a)[i] == reinterpret_cast<const unsigned int*>(b)[i];
    if (!same) atomicAdd(cnt, 1ull);
}

struct Timer {
    cudaEvent_t a, b;
    Timer()
    {
        cudaEventCreate(&a);
        cudaEventCreate(&b);
    }
    cudaStream_t stream = nullptr;  // the stream the timed work is launched on
    template <typename F>
    double ms(F f, int warm = 3, int reps = 20)
    {
        for (int i = 0; i < warm; ++i) f();
        CK(cudaDeviceSynchronize());
        CK(cudaEventRecord(a, stream));
        for (int i = 0; i < reps; ++i) f();
        CK(cudaEventRecord(b, stream));
        CK(cudaEventSynchronize(b));
        float t;
        cudaEventElapsedTime(&t, a, b);
        return t / reps;
    }
};

template <typename V>
double spmv_bytes(const Mat<V>& m)
{
    return (double)m.nnz * (sizeof(V) + 4) + (m.n + 1) * 4.0 + m.ncols * (double)sizeof(V) + m.n * (double)sizeof(V);
}

template <typename V>
struct Bench {
    Mat<V> m;
    V *x = nullptr, *y = nullptr, *yref = nullptr;
    unsigned long long* cnt = nullptr;
    b200_ctx* ctx = nullptr;
    Timer tm;
    void init(const std::string& name)
    {
        m = make_matrix<V>(name);
        CK(cudaMalloc(&x, m.ncols * sizeof(V)));
        CK(cudaMalloc(&y, m.n * sizeof(V)));
        CK(cudaMalloc(&yref, m.n * sizeof(V)));
        CK(cudaMalloc(&cnt, 8));
        gen_vec<V><<<(int)((m.ncols + 255) / 256), 256>>>(m.ncols, x);
        ref_spmv<V><<<(int)((m.n + 255) / 256), 256>>>(m.n, m.rp, m.ci, m.va, x, yref);
        CK(cudaDeviceSynchronize());
        if (b200_ctx_create(0, nullptr, &ctx) != B200_OK) {
            printf("ctx create failed\n");
            exit(2);
        }
        tm.stream = ctx->stream;
        printf("# matrix %s n=%lld nnz=%lld bytes=%.1f MB\n", name.c_str(), (long long)m.n, (long long)m.nnz,
               spmv_bytes(m) / 1e6);
    }
    template <typename F>
    void run(const char* label, F f)
    {
        if (const char* only = getenv("LAB_ONLY"))
            if (!strstr(label, only)) return;
        CK(cudaMemset(y, 0xff, m.n * sizeof(V)));
        CK(cudaMemset(cnt, 0, 8));
        f();
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            printf("%-44s FAILED: %s\n", label, cudaGetErrorString(e));
            exit(3);
        }
        count_diff<V><<<(int)((m.n + 255) / 256), 256>>>(m.n, y, yref, cnt);
        unsigned long long h = 0;
        CK(cudaMemcpy(&h, cnt, 8, cudaMemcpyDeviceToHost));
        const double t = tm.ms(f);
        const double gbs = spmv_bytes(m) / t / 1e6;
        printf("%-10s %-44s %8.4f ms  %7.1f GB/s  %5.1f%% of peak  %6.1f GFLOP/s  mismatching rows %llu\n",
               m.name.c_str(), label, t, gbs, 100 * gbs / kPeak, 2.0 * m.nnz / t / 1e6, h);
        fflush(stdout);
    }
};

// ------------------------------------------------------------------------------ group: base
template <typename V>
void group_base(const std::string& name)
{
    Bench<V> B;
    B.init(name);
    auto& m = B.m;
    const int64_t nt = num_tiles_for(m.n, m.nnz), nwt = num_wtiles_for(m.n, m.nnz);
    int64_t *tiles, *wtiles;
    CK(cudaMalloc(&tiles, 2 * (nt + 1) * 8));
    CK(cudaMalloc(&wtiles, 2 * (nwt + 1) * 8));
    fill_plan<int>(B.ctx, m.n, m.nnz, m.rp, nt, tiles, kTile);
    fill_plan<int>(B.ctx, m.n, m.nnz, m.rp, nwt, wtiles, kWTile);
    CK(cudaDeviceSynchronize());
    auto go = [&](Variant v) {
        launch_slab<V, int, false, false>(B.ctx, 1, v, nwt, wtiles, m.nnz, m.rp, m.ci, m.va, (const V*)nullptr, B.x,
                                          1, (const V*)nullptr, B.y, 1);
    };
    B.run("r01 warp_stream", [&] { go(csr::kWarp); });
    B.run("r01 warp_pipe", [&] { go(kPipe); });
    (void)nt;
    (void)tiles;
}

// ------------------------------------------------------------------------------ group: ring
template <typename V, int NW, int KB, bool GNA, int CAP, int STAGES, int NP>
void ring_case(Bench<V>& B, int64_t items = CAP - 512)
{
    auto& m = B.m;
    const int64_t nt = ceildiv(kRowW * m.n + m.nnz, items);
    int64_t* tiles;
    CK(cudaMalloc(&tiles, 2 * (nt + 1) * 8));
    fill_plan<int>(B.ctx, m.n, m.nnz, m.rp, nt, tiles, items);
    CK(cudaDeviceSynchronize());
    char label[128];
    snprintf(label, sizeof label, "ring NW=%d NP=%d KB=%d GNA=%d CAP=%d x%d items=%lld", NW, NP, KB, (int)GNA, CAP,
             STAGES, (long long)items);
    const int grid = (int)std::min<int64_t>(nt, B.ctx->num_sms);
    B.run(label, [&] {
        launch_ring<V, int, 1, false, false, NW, KB, GNA, CAP, STAGES, NP>(
            B.ctx, nt, tiles, m.nnz, m.n, m.rp, m.ci, m.va, (const V*)nullptr, B.x, 1, (const V*)nullptr, B.y, 1,
            DotArgs<V>{}, grid);
    });
    CK(cudaFree(tiles));
}

template <typename V>
void group_ring(const std::string& name)
{
    Bench<V> B;
    B.init(name);
    // deep rings (structured matrices)
    ring_case<V, 16, 8, false, 3584, 4, 1>(B);
    ring_case<V, 16, 8, false, 3584, 4, 2>(B);
    ring_case<V, 16, 8, false, 3584, 4, 4>(B);
    ring_case<V, 24, 8, false, 3584, 4, 2>(B);
    ring_case<V, 24, 8, false, 3584, 4, 4>(B);
    ring_case<V, 28, 8, false, 3584, 4, 4>(B);
    ring_case<V, 24, 8, false, 2560, 4, 4>(B);
    ring_case<V, 24, 8, false, 1792, 8, 4>(B);
    ring_case<V, 24, 8, false, 1792, 6, 2>(B);
    // shallower rings (scattered gathers: leave the SM's memory to L1)
    ring_case<V, 16, 8, true, 3584, 2, 2>(B);
    ring_case<V, 16, 8, false, 3584, 2, 2>(B);
    ring_case<V, 16, 8, true, 2560, 2, 2>(B);
    ring_case<V, 16, 8, true, 1792, 2, 2>(B);
    ring_case<V, 16, 8, true, 1792, 4, 4>(B);
    ring_case<V, 24, 8, true, 1792, 4, 4>(B);
    ring_case<V, 16, 16, true, 1792, 4, 4>(B);
    ring_case<V, 16, 8, true, 1024, 4, 4>(B);
    ring_case<V, 16, 8, true, 1024, 8, 4>(B);
    ring_case<V, 24, 8, true, 1024, 8, 4>(B);
}

// ------------------------------------------------------------------------------ group: micro
// M1: streaming read, 16 bytes per lane per load
__global__ void __launch_bounds__(512) stream_ldg(const int4* p, int64_t n16, int* out)
{
    int acc = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        int4 v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
            asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v[k].x), "=r"(v[k].y), "=r"(v[k].z), "=r"(v[k].w)
                         : "l"(p + i + k * stride));
#pragma unroll
        for (int k = 0; k < 4; ++k) acc ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
    }
    for (; i < n16; i += stride) acc ^= p[i].x;
    if (acc == 0x12345678) out[0] = acc;
}
// M1b: streaming read through the bulk-copy engine, 4-stage ring of CHUNK bytes per CTA, consumers only wait
template <int CHUNK, int STAGES>
__global__ void __launch_bounds__(128) stream_bulk(const unsigned char* p, int64_t bytes, int* out)
{
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ uint64_t full[STAGES];
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncthreads();
    const int64_t nchunks = bytes / CHUNK;
    const uint64_t pol = policy_evict_first();
    int acc = 0;
    int64_t c = blockIdx.x;
    // prologue
    if (threadIdx.x == 0)
        for (int s = 0; s < STAGES - 1; ++s) {
            const int64_t cc = c + (int64_t)s * gridDim.x;
            if (cc < nchunks) {
                mbar_arrive_expect_tx(&full[s], CHUNK);
                tma_load_1d(sm + (size_t)s * CHUNK, p + cc * CHUNK, CHUNK, &full[s], pol);
            }
        }
    int stage = 0;
    uint32_t ph = 0;
    for (; c < nchunks; c += gridDim.x) {
        __syncthreads();  // everybody is done with the stage that is refilled now
        if (threadIdx.x == 0) {
            const int64_t cc = c + (int64_t)(STAGES - 1) * gridDim.x;
            int ps = stage + STAGES - 1;
            if (ps >= STAGES) ps -= STAGES;
            if (cc < nchunks) {
                fence_proxy_async();
                mbar_arrive_expect_tx(&full[ps], CHUNK);
                tma_load_1d(sm + (size_t)ps * CHUNK, p + cc * CHUNK, CHUNK, &full[ps], pol);
            }
        }
        mbar_wait(&full[stage], ph);
        acc ^= reinterpret_cast<const int*>(sm + (size_t)stage * CHUNK)[threadIdx.x];
        if (++stage == STAGES) {
            stage = 0;
            ph ^= 1u;
        }
    }
    if (acc == 0x12345678) out[0] = acc;
}

// M2: 8-byte gathers through LSU: coalesced index stream (4 B) + gather from x[0..M)
template <int U, bool NA>
__global__ void __launch_bounds__(1024) gather_ldg(const int* idx, int64_t n, const double* x, double* out)
{
    const uint64_t pol = policy_evict_last();
    const uint64_t polf = policy_evict_first();
    double acc = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i + (U - 1) * stride < n; i += U * stride) {
        int c[U];
        double v[U];
#pragma unroll
        for (int k = 0; k < U; ++k) c[k] = ld_stream(idx + i + k * stride, polf);
#pragma unroll
        for (int k = 0; k < U; ++k) v[k] = NA ? ld_gather_na(x + c[k], pol) : ld_gather(x + c[k], pol);
#pragma unroll
        for (int k = 0; k < U; ++k) acc += v[k];
    }
    {  // tail: the last (n mod U*stride) indices
        const int64_t done = (n / (U * stride)) * (U * stride);
        for (int64_t i = done + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) acc += x[idx[i]];
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}
__global__ void gen_idx(int64_t n, int64_t M, int* idx)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (int)(hash3(11, i, 0) % (uint64_t)M);
}
__global__ void gen_xint(int64_t M, double* x)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < M) x[i] = (double)(i % 1021);
}

void group_micro()
{
    Timer tm;
    int* out;
    CK(cudaMalloc(&out, 64));
    {  // M1
        const int64_t bytes = 1800000000ll & ~int64_t(65535);
        unsigned char* p;
        CK(cudaMalloc(&p, bytes));
        CK(cudaMemset(p, 1, bytes));
        for (int ctas : {2, 3, 4}) {
            const double t = tm.ms([&] { stream_ldg<<<g_sms * ctas, 512>>>((const int4*)p, bytes / 16, out); });
            printf("micro stream_ldg  LDG.128 x4 unroll, %d CTAs/SM x 512 thr: %.4f ms  %.1f GB/s (%.1f%% of copy peak)\n",
                   ctas, t, bytes / t / 1e6, 100 * bytes / t / 1e6 / kPeak);
        }
        {
            constexpr int CH = 32768, ST = 4;
            auto k = stream_bulk<CH, ST>;
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, CH * ST));
            const double t = tm.ms([&] { k<<<g_sms, 128, CH * ST>>>(p, bytes, out); });
            printf("micro stream_bulk 32 KB chunks x 4 stages, 1 CTA/SM: %.4f ms  %.1f GB/s (%.1f%%)\n", t,
                   bytes / t / 1e6, 100 * bytes / t / 1e6 / kPeak);
        }
        {
            constexpr int CH = 16384, ST = 6;
            auto k = stream_bulk<CH, ST>;
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, CH * ST));
            const double t = tm.ms([&] { k<<<g_sms * 2, 128, CH * ST>>>(p, bytes, out); });
            printf("micro stream_bulk 16 KB chunks x 6 stages, 2 CTA/SM: %.4f ms  %.1f GB/s (%.1f%%)\n", t,
                   bytes / t / 1e6, 100 * bytes / t / 1e6 / kPeak);
        }
        {
            constexpr int CH = 49152, ST = 4;
            auto k = stream_bulk<CH, ST>;
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, CH * ST));
            const double t = tm.ms([&] { k<<<g_sms, 128, CH * ST>>>(p, bytes, out); });
            printf("micro stream_bulk 48 KB chunks x 4 stages, 1 CTA/SM: %.4f ms  %.1f GB/s (%.1f%%)\n", t,
                   bytes / t / 1e6, 100 * bytes / t / 1e6 / kPeak);
        }
        CK(cudaFree(p));
    }
    {  // M2
        const int64_t n = 75000000;
        int* idx;
        double *x, *dout;
        CK(cudaMalloc(&idx, n * 4));
        CK(cudaMalloc(&x, 10000000 * 8));
        CK(cudaMalloc(&dout, 8));
        gen_xint<<<(10000000 + 255) / 256, 256>>>(10000000, x);
        // x slices of 8 / 16 / 24 MB (one column part of cfg2 is 16 MB) and the whole 80 MB; 16 / 32 / 48
        // warps per SM in CTAs of 512 threads, 8 independent gathers per lane
        for (int64_t M : {1000000ll, 2000000ll, 3000000ll, 10000000ll}) {
            gen_idx<<<(int)((n + 255) / 256), 256>>>(n, M, idx);
            CK(cudaDeviceSynchronize());
            auto rep = [&](const char* l, double t) {
                printf("micro gather_ldg  %-34s x=%3lld MB: %.4f ms  %.1f G gathers/s  (150M gathers -> %.3f ms; "
                       "%.3f gathers/clk/SM at %.3f GHz)\n",
                       l, (long long)(M * 8 / 1000000), t, n / t / 1e6, 150e6 / (n / t / 1e6) / 1e6,
                       n / t / 1e6 / g_sms / g_ghz, g_ghz);
                fflush(stdout);
            };
            for (int ctas : {1, 2, 3}) {
                char l[64];
                snprintf(l, sizeof l, "U=8  %d warps/SM no_allocate", 16 * ctas);
                rep(l, tm.ms([&] { gather_ldg<8, true><<<g_sms * ctas, 512>>>(idx, n, x, dout); }));
            }
            rep("U=8  32 warps/SM L1 alloc", tm.ms([&] { gather_ldg<8, false><<<g_sms * 2, 512>>>(idx, n, x, dout); }));
        }
        CK(cudaFree(idx));
        CK(cudaFree(x));
    }
}


// ------------------------------------------------------------------------------ group: l1cap
// M4: the 8-byte gather rate against the shared-memory carve-out.  A pending L1 miss holds a 128-byte
// line of the unified L1 / shared-memory array, so every KB given to shared memory takes 8 outstanding
// gathers away: the budget a staging ring has on matrices with scattered columns.
void group_l1cap()
{
    Timer tm;
    const int64_t n = 75000000, M = 5000000;
    int* idx;
    double *x, *dout;
    CK(cudaMalloc(&idx, n * 4));
    CK(cudaMalloc(&x, M * 8));
    CK(cudaMalloc(&dout, 8));
    gen_xint<<<(int)((M + 255) / 256), 256>>>(M, x);
    gen_idx<<<(int)((n + 255) / 256), 256>>>(n, M, idx);
    CK(cudaDeviceSynchronize());
    auto k8 = gather_ldg<8, true>;
    auto k16 = gather_ldg<16, true>;
    CK(cudaFuncSetAttribute(k8, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CK(cudaFuncSetAttribute(k16, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    for (int kb : {0, 16, 32, 48, 64, 96, 128, 160, 192}) {
        for (int thr : {512, 1024}) {
            const double t8 = tm.ms([&] { k8<<<g_sms, thr, (size_t)kb * 1024>>>(idx, n, x, dout); });
            const double t16 = tm.ms([&] { k16<<<g_sms, thr, (size_t)kb * 1024>>>(idx, n, x, dout); });
            printf("micro l1cap  smem %3d KB/SM, 1 CTA x %4d thr: U=8 %.4f ms %.3f gathers/clk/SM | U=16 %.4f ms %.3f "
                   "gathers/clk/SM   (x = 40 MB, no_allocate)\n",
                   kb, thr, t8, n / t8 / 1e6 / g_sms / g_ghz, t16, n / t16 / 1e6 / g_sms / g_ghz);
            fflush(stdout);
        }
    }
    CK(cudaFree(idx));
    CK(cudaFree(x));
}

// ------------------------------------------------------------------------------ group: tma4
// M3: the same gathers through the TMA gather4 path: x viewed as a 2-D tensor of 16-byte rows
// {x[2i], x[2i+1]}; one cp.async.bulk.tensor.2d...tile::gather4 brings 4 rows (= 4 gathered
// elements' pairs) into shared memory, completion on an mbarrier.
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                             const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                             CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

__device__ __forceinline__ void tma_gather4(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int r0, int r1,
                                            int r2, int r3)
{
    // gather4 exists from sm_100 on; group_tma4 does not launch this on an sm_90a device
#if !defined(__CUDA_ARCH__) || __CUDA_ARCH__ >= 1000
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile::gather4.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
        : "memory");
#endif
}

constexpr int kG4Warps = 8, kG4Depth = 4, kG4Slot = 128;  // bytes of shared memory per (lane, batch)
__global__ void __launch_bounds__(kG4Warps * 32, 1)
    gather_tma4(const __grid_constant__ CUtensorMap map, const int* idx, int64_t n, double* out, int* bad,
                const double* x)
{
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ uint64_t bars[kG4Warps][kG4Depth];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        for (int d = 0; d < kG4Depth; ++d) mbar_init(&bars[warp][d], 1);
        fence_mbar_init();
    }
    __syncwarp();
    unsigned char* my = sm + (size_t)warp * kG4Depth * 32 * kG4Slot;
    // a batch = 128 indices per warp (4 per lane, one gather4 per lane)
    const int64_t nb = n / 128;
    const int64_t W = (int64_t)gridDim.x * kG4Warps;
    const int64_t b0 = (int64_t)blockIdx.x * kG4Warps + warp;
    int4 cur[kG4Depth];
    auto issue = [&](int64_t b, int d) {
        if (b >= nb) return;
        const int4 v = reinterpret_cast<const int4*>(idx)[b * 32 + lane];
        cur[d] = v;
        if (lane == 0) mbar_arrive_expect_tx(&bars[warp][d], 32 * 64);
        __syncwarp();
        tma_gather4(my + ((size_t)d * 32 + lane) * kG4Slot, &map, &bars[warp][d], 0, v.x >> 1, v.y >> 1, v.z >> 1,
                    v.w >> 1);
    };
#pragma unroll
    for (int d = 0; d < kG4Depth; ++d) issue(b0 + d * W, d);
    double acc = 0;
    uint32_t ph = 0;
    int nbad = 0;
    for (int64_t b = b0; b < nb; b += kG4Depth * W) {
#pragma unroll
        for (int d = 0; d < kG4Depth; ++d) {
            const int64_t bb = b + d * W;
            if (bb >= nb) break;
            mbar_wait(&bars[warp][d], ph);
            const double* s = reinterpret_cast<const double*>(my + ((size_t)d * 32 + lane) * kG4Slot);
            const int4 v = cur[d];
            const double g0 = s[0 + (v.x & 1)], g1 = s[2 + (v.y & 1)], g2 = s[4 + (v.z & 1)], g3 = s[6 + (v.w & 1)];
            if (bad && b == b0 && d == 0) {  // spot check of the first batch against direct loads
                nbad += (g0 != x[v.x]) + (g1 != x[v.y]) + (g2 != x[v.z]) + (g3 != x[v.w]);
            }
            acc += g0 + g1 + g2 + g3;
            __syncwarp();
            fence_proxy_async();
            issue(bb + kG4Depth * W, d);
        }
        ph ^= 1u;
    }
    acc = warp_sum(acc);
    if (lane == 0) atomicAdd(out, acc);
    if (bad && nbad) atomicAdd(bad, nbad);
}

void group_tma4()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    if (prop.major < 10) {
        printf("tma4: the TMA gather4 path needs compute capability 10.0 or later, skipped\n");
        return;
    }
    Timer tm;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn) {
        printf("tma4: no cuTensorMapEncodeTiled\n");
        return;
    }
    EncodeFn enc = (EncodeFn)fn;
    const int64_t n = 75000000;
    int* idx;
    double *x, *dout;
    int* bad;
    CK(cudaMalloc(&idx, n * 4));
    CK(cudaMalloc(&x, 10000000 * 8));
    CK(cudaMalloc(&dout, 16));
    CK(cudaMalloc(&bad, 4));
    gen_xint<<<(10000000 + 255) / 256, 256>>>(10000000, x);
    const size_t smem = (size_t)kG4Warps * kG4Depth * 32 * kG4Slot;
    CK(cudaFuncSetAttribute(gather_tma4, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int boxrows : {1, 4}) {
        for (int64_t M : {5000000ll, 10000000ll}) {
            CUtensorMap map;
            cuuint64_t gdim[2] = {2, (cuuint64_t)(M / 2)};
            cuuint64_t gstr[1] = {16};
            cuuint32_t box[2] = {2, (cuuint32_t)boxrows};
            cuuint32_t estr[2] = {1, 1};
            CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, x, gdim, gstr, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                printf("tma4: encode failed (box rows %d): %d\n", boxrows, (int)r);
                continue;
            }
            gen_idx<<<(int)((n + 255) / 256), 256>>>(n, M, idx);
            CK(cudaMemset(dout, 0, 16));
            CK(cudaMemset(bad, 0, 4));
            gather_tma4<<<g_sms, kG4Warps * 32, smem>>>(map, idx, n, dout, bad, x);
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) {
                printf("tma4: kernel failed (box rows %d): %s\n", boxrows, cudaGetErrorString(e));
                return;
            }
            double s_tma = 0, s_ldg = 0;
            int hb = 0;
            CK(cudaMemcpy(&s_tma, dout, 8, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(&hb, bad, 4, cudaMemcpyDeviceToHost));
            CK(cudaMemset(dout, 0, 16));
            gather_ldg<8, true><<<g_sms * 2, 1024>>>(idx, (n / 128) * 128, x, dout);
            CK(cudaDeviceSynchronize());
            CK(cudaMemcpy(&s_ldg, dout, 8, cudaMemcpyDeviceToHost));
            const double t = tm.ms([&] { gather_tma4<<<g_sms, kG4Warps * 32, smem>>>(map, idx, n, dout, nullptr, x); });
            printf("micro gather_tma4 box rows %d x=%3lld MB: %.4f ms  %.1f G gathers/s (150M -> %.3f ms)  sum %s "
                   "(tma %.0f ldg-ish %.0f) spot-check mismatches %d\n",
                   boxrows, (long long)(M * 8 / 1000000), t, n / t / 1e6, 150e6 / (n / t / 1e6) / 1e6,
                   s_tma == s_ldg ? "MATCH" : "differs", s_tma, s_ldg, hb);
            fflush(stdout);
        }
    }
}

// ------------------------------------------------------------------------------ group: san
// small matrices for compute-sanitizer (racecheck / memcheck / synccheck): every shipped CSR variant through
// a plan, incl. rows longer than a stage, rows split over CTAs, the fused dot and the advanced form
__global__ void gen_small(int64_t n, int64_t m, const int* rp, int* ci, double* va)
{
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int64_t len = rp[r + 1] - rp[r];
    for (int64_t k = 0; k < len; ++k) {
        const int64_t lo = k * m / len, hi = (k + 1) * m / len;
        ci[rp[r] + k] = (int)(lo + (int64_t)(hash3(5, r, k) % (uint64_t)(hi - lo)));
        va[rp[r] + k] = unit(hash3(6, r, k));
    }
}
void group_san()
{
    const int64_t n = 20011, m = 40000;
    std::vector<int> rp(n + 1);
    int64_t p = 0;
    for (int64_t r = 0; r < n; ++r) {
        rp[r] = (int)p;
        int64_t len = 3 + (r * 7) % 11;
        if (r == 17) len = 5000;      // longer than a stage
        if (r == 4242) len = 20000;   // split over CTAs (>= 16384)
        if (r == n - 1) len = 17001;  // split, last row
        if (r % 500 == 3) len = 0;
        p += len;
    }
    rp[n] = (int)p;
    const int64_t nnz = p;
    int *d_rp, *d_ci;
    double *d_va, *x, *y, *yref, *scal, *work;
    CK(cudaMalloc(&d_rp, (n + 1) * 4));
    CK(cudaMalloc(&d_ci, nnz * 4));
    CK(cudaMalloc(&d_va, nnz * 8));
    CK(cudaMalloc(&x, m * 8));
    CK(cudaMalloc(&y, n * 8));
    CK(cudaMalloc(&yref, n * 8));
    CK(cudaMalloc(&scal, 64));
    CK(cudaMemcpy(d_rp, rp.data(), (n + 1) * 4, cudaMemcpyHostToDevice));
    gen_small<<<(int)((n + 255) / 256), 256>>>(n, m, d_rp, d_ci, d_va);
    gen_vec<double><<<(int)((m + 255) / 256), 256>>>(m, x);
    ref_spmv<double><<<(int)((n + 255) / 256), 256>>>(n, d_rp, d_ci, d_va, x, yref);
    CK(cudaDeviceSynchronize());
    b200_ctx* ctx;
    if (b200_ctx_create(0, nullptr, &ctx) != B200_OK) exit(2);
    CK(cudaMalloc(&work, 8 * (size_t)b200_cg_fused_work_size_f64(ctx)));
    b200_csr_plan* plan;
    if (b200_csr_plan_create_f64_i32(ctx, n, nnz, d_rp, &plan) != B200_OK) exit(2);
    printf("san: n=%lld nnz=%lld long rows %lld\n", (long long)n, (long long)nnz,
           (long long)b200_csr_plan_num_long_rows(plan));
    const double ab[2] = {-1.5, 0.25};
    CK(cudaMemcpy(scal, ab, 16, cudaMemcpyHostToDevice));
    std::vector<double> h(n), hr(n);
    CK(cudaMemcpy(hr.data(), yref, n * 8, cudaMemcpyDeviceToHost));
    for (int v : {2, 4, 5}) {
        b200_csr_plan_set_variant(plan, v);
        CK(cudaMemset(y, 0, n * 8));
        if (b200_csr_spmv_f64_i32(ctx, plan, n, m, nnz, d_rp, d_ci, d_va, x, 1, 1, y, 1) != B200_OK) exit(3);
        if (b200_csr_advanced_spmv_f64_i32(ctx, plan, n, m, nnz, d_rp, d_ci, d_va, scal, x, 1, 1, scal + 1, y, 1) !=
            B200_OK)
            exit(3);
        if (b200_csr_spmv_dot_f64_i32(ctx, plan, n, n, nnz, d_rp, d_ci, d_va, x, y, scal + 4, work, nullptr) != B200_OK)
            exit(3);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(h.data(), y, n * 8, cudaMemcpyDeviceToHost));
        double worst = 0;
        for (int64_t r = 0; r < n; ++r) {
            const double d = fabs(h[r] - hr[r]) / (fabs(hr[r]) + 1e-300);
            if (d > worst && fabs(hr[r]) > 1e-12) worst = d;
        }
        printf("san: variant %d done, worst relative row difference to the reference kernel %.3e\n", v, worst);
    }
    b200_csr_plan_destroy(plan);
    printf("san: finished\n");
}

int main(int argc, char** argv)
{
    const std::string group = argc > 1 ? argv[1] : "micro";
    const std::string name = argc > 2 ? argv[2] : "cfg2";
    init_device();
    if (group == "micro") group_micro();
    if (group == "san") group_san();
    if (group == "tma4") group_tma4();
    if (group == "l1cap") group_l1cap();
    if (group == "base") {
        if (name == "cfg4")
            group_base<float>(name);
        else
            group_base<double>(name);
    }
    if (group == "ring") {
        if (name == "cfg4")
            group_ring<float>(name);
        else
            group_ring<double>(name);
    }
    return 0;
}
