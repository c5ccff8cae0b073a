/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused CG entry points for several
 * right-hand sides (ginkgo_b200/csrc/fused_cg_mrhs.cu: b200_cg_mrhs_*), so that
 * solver::Cg::try_fused_multi_rhs -- capture, replay, polling of the control block, the per-column
 * statuses -- runs on the CPU.  Every column's sums run over the rows in order, as the oracle's
 * compute_dot / compute_norm2 do, so this path and the kernel-by-kernel loop on the mock take the same
 * iterations and give the same bits.  The SpMV + dots (b200_csr_spmv_mdot_*) are in mock_spmv_dot.c. */
#include "mock.h"

#define MOCK_FUSED_MRHS(V, VT, SQRT, FABS)                                                              \
    static void mock_mrhs_step_p_##V(int64_t n, int64_t k, VT* p, const VT* z, const VT* sc,            \
                                     const uint8_t* status, const int32_t* ctl)                         \
    {                                                                                                   \
        if (ctl[0] != 0) return;                                                                        \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            if (status[j] & 0x3f) continue;                                                             \
            const VT rho = sc[j], prev = sc[k + j];                                                     \
            for (int64_t i = 0; i < n; ++i)                                                             \
                p[i * k + j] = prev == 0 ? z[i * k + j] : z[i * k + j] + (rho / prev) * p[i * k + j];   \
        }                                                                                               \
    }                                                                                                   \
    static void mock_mrhs_step_xr_##V(int init, int64_t n, int64_t k, VT* x, VT* r, const VT* p,        \
                                      const VT* q, VT* z, const VT* inv_diag, VT* sc, uint8_t* status,  \
                                      int32_t* ctl, int baseline, VT factor)                            \
    {                                                                                                   \
        if (!init && ctl[0] != 0) return;                                                               \
        const int32_t iter = ctl[1] + 1;                                                                \
        ctl[1] = iter;                                                                                  \
        int all_stopped = 1;                                                                            \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            uint8_t s = status[j];                                                                      \
            if (!(s & 0x3f)) {                                                                          \
                const VT pq = sc[2 * k + j];                                                            \
                const int update = !init && pq != 0;                                                    \
                const VT alpha = update ? sc[j] / pq : 0;                                               \
                VT s_rho = 0, s_rr = 0;                                                                 \
                for (int64_t i = 0; i < n; ++i) {                                                       \
                    const int64_t e = i * k + j;                                                        \
                    VT ri = r[e];                                                                       \
                    if (update) {                                                                       \
                        x[e] += alpha * p[e];                                                           \
                        ri -= alpha * q[e];                                                             \
                        r[e] = ri;                                                                      \
                    }                                                                                   \
                    const VT zi = inv_diag ? ri * inv_diag[i] : ri;                                     \
                    z[e] = zi;                                                                          \
                    s_rho += ri * zi;                                                                   \
                    s_rr += ri * ri;                                                                    \
                }                                                                                       \
                if (init) {                                                                             \
                    if (baseline == 1) sc[4 * k + j] = SQRT(s_rr);                                      \
                    if (baseline == 2) sc[4 * k + j] = 1;                                               \
                    sc[5 * k + j] = factor * sc[4 * k + j];                                             \
                }                                                                                       \
                sc[k + j] = sc[j];                                                                      \
                sc[j] = s_rho;                                                                          \
                sc[3 * k + j] = s_rr;                                                                   \
                const VT tau = ctl[3] == 1 ? SQRT(s_rr) : SQRT(FABS(s_rho));                            \
                status[j] = s = mock_criteria_status(iter, ctl, tau <= sc[5 * k + j], 0x40);            \
            }                                                                                           \
            if (!(s & 0x3f)) all_stopped = 0;                                                           \
        }                                                                                               \
        ctl[0] = all_stopped;                                                                           \
    }                                                                                                   \
    static b200_status replay_step_p_##V(b200_ctx* ctx, const mock_op* op)                              \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_mrhs_step_p_##V(op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4]);                         \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    static b200_status replay_step_xr_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_mrhs_step_xr_##V(0, op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7],    \
                              a[8], 0, 0);                                                              \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    int64_t b200_cg_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                                  \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        return 3 * k + 64;                                                                              \
    }                                                                                                   \
    b200_status b200_cg_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* z, VT* p,   \
                                      VT* q, const VT* inv_diag, VT* sc, uint8_t* status, int32_t* ctl, \
                                      VT* work, int64_t max_iters, int32_t res_kind,                    \
                                      int32_t iter_first, int32_t baseline, VT reduction_factor)        \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (ctx->capture) { mock_set_error("cg_mrhs_init inside a capture"); return B200_ERR_INVALID; } \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            sc[j] = 1; sc[k + j] = 1; sc[2 * k + j] = 0; sc[3 * k + j] = 0;                             \
            status[j] = 0;                                                                              \
        }                                                                                               \
        ctl[0] = 0; ctl[1] = -1;                                                                        \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                            \
        ctl[3] = res_kind; ctl[4] = iter_first;                                                         \
        memset(p, 0, sizeof(VT) * (size_t)(n * k));                                                     \
        memset(q, 0, sizeof(VT) * (size_t)(n * k));                                                     \
        mock_mrhs_step_xr_##V(1, n, k, NULL, (VT*)r, p, q, z, inv_diag, sc, status, ctl, baseline,      \
                              reduction_factor);                                                        \
        ctx->launches += 2;                                                                             \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_cg_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p, const VT* z,        \
                                        const VT* sc, const uint8_t* status, const int32_t* ctl)        \
    {                                                                                                   \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_step_p_##V);                                          \
            op->p[0] = p; op->p[1] = (void*)z; op->p[2] = (void*)sc; op->p[3] = (void*)status;          \
            op->p[4] = (void*)ctl; op->n[0] = n; op->n[1] = k;                                          \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_mrhs_step_p_##V(n, k, p, z, sc, status, ctl);                                              \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_cg_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* r,             \
                                         const VT* p, const VT* q, VT* z, const VT* inv_diag, VT* sc,   \
                                         uint8_t* status, int32_t* ctl, VT* work)                       \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_step_xr_##V);                                         \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)p; op->p[3] = (void*)q; op->p[4] = z;         \
            op->p[5] = (void*)inv_diag; op->p[6] = sc; op->p[7] = status; op->p[8] = ctl;               \
            op->n[0] = n; op->n[1] = k;                                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_mrhs_step_xr_##V(0, n, k, x, r, p, q, z, inv_diag, sc, status, ctl, 0, 0);                 \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_FUSED_MRHS(f64, double, sqrt, fabs)
MOCK_FUSED_MRHS(f32, float, sqrtf, fabsf)
