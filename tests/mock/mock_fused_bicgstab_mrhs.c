/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused BiCGStab entry points for several
 * right-hand sides (ginkgo_b200/csrc/fused_bicgstab_mrhs.cu: b200_bicgstab_mrhs_*), so that
 * solver::Bicgstab::try_fused_multi_rhs -- capture, replay, polling of the control block, the per-column
 * statuses, the finalize owed after a mid-iteration stop -- runs on the CPU.  Every column's sums run
 * over the rows in order, as the oracle's compute_dot / compute_norm2 do, so this path and the
 * kernel-by-kernel loop on the mock take the same iterations and give the same bits.  The SpMV + dots
 * (b200_csr_spmv_mdot2_*) are in mock_spmv_dot.c. */
#include "mock.h"

#define MOCK_FUSED_BM(V, VT, SQRT, FABS)                                                                \
    static void mock_bm_step_p_##V(int64_t n, int64_t k, VT* p, const VT* r, const VT* v, VT* y,        \
                                   const VT* d, const VT* sc, const uint8_t* status, const int32_t* ctl) \
    {                                                                                                   \
        if (ctl[0] != 0) return;                                                                        \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            if (STOPPED(status[j])) continue;                                                           \
            const VT rho = sc[j], prev = sc[k + j], alpha = sc[6 * k + j], omega = sc[7 * k + j];       \
            const int plain = !(prev * omega != 0);                                                     \
            const VT tmp = plain ? 0 : rho / prev * alpha / omega;                                      \
            for (int64_t i = 0; i < n; ++i) {                                                           \
                const int64_t e = i * k + j;                                                            \
                const VT pi = plain ? r[e] : r[e] + tmp * (p[e] - omega * v[e]);                        \
                p[e] = pi;                                                                              \
                y[e] = d ? pi * d[i] : pi;                                                              \
            }                                                                                           \
        }                                                                                               \
    }                                                                                                   \
    static void mock_bm_step_s_##V(int64_t n, int64_t k, const VT* r, const VT* v, VT* s, VT* z,        \
                                   const VT* d, VT* sc, uint8_t* status, int32_t* ctl)                  \
    {                                                                                                   \
        if (ctl[0] != 0) return;                                                                        \
        int all_stopped = 1, owed = 0;                                                                  \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            uint8_t st = status[j];                                                                     \
            if (!STOPPED(st)) {                                                                         \
                const VT beta = sc[2 * k + j];                                                          \
                const int update = beta != 0;                                                           \
                const VT alpha = update ? sc[j] / beta : 0;                                             \
                VT ss = 0;                                                                              \
                for (int64_t i = 0; i < n; ++i) {                                                       \
                    const int64_t e = i * k + j;                                                        \
                    const VT si = update ? r[e] - alpha * v[e] : r[e];                                  \
                    s[e] = si;                                                                          \
                    z[e] = d ? si * d[i] : si;                                                          \
                    ss += si * si;                                                                      \
                }                                                                                       \
                sc[6 * k + j] = alpha;                                                                  \
                sc[9 * k + j] = ss;                                                                     \
                const VT tau = ctl[3] == 1 ? SQRT(ss) : SQRT(FABS(sc[j]));                              \
                st = mock_criteria_status(ctl[1], ctl, tau <= sc[5 * k + j], 0);                        \
                if (st) {                                                                               \
                    status[j] = st;                                                                     \
                    owed = 1;                                                                           \
                }                                                                                       \
            }                                                                                           \
            if (!STOPPED(st)) all_stopped = 0;                                                          \
        }                                                                                               \
        if (owed) ctl[5] = 1;                                                                           \
        if (all_stopped) ctl[0] = 1;                                                                    \
    }                                                                                                   \
    static void mock_bm_step_xr_##V(int init, int64_t n, int64_t k, VT* x, VT* r, const VT* s,          \
                                    const VT* t, const VT* y, const VT* z, VT* rr, VT* sc,              \
                                    uint8_t* status, int32_t* ctl, int baseline, VT factor)             \
    {                                                                                                   \
        const int pending = !init && ctl[5] != 0, iterating = init || ctl[0] == 0;                      \
        if (!pending && !iterating) return;                                                             \
        const int32_t iter = iterating ? ctl[1] + 1 : ctl[1];                                           \
        if (iterating) ctl[1] = iter;                                                                   \
        int all_stopped = 1;                                                                            \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            uint8_t st = status[j];                                                                     \
            if (STOPPED(st)) {                                                                          \
                if (!init && !(st & 0x40)) { /* bicgstab::finalize */                                   \
                    const VT alpha = sc[6 * k + j];                                                     \
                    for (int64_t i = 0; i < n; ++i) x[i * k + j] += alpha * y[i * k + j];               \
                    status[j] = st = (uint8_t)(st | 0x40);                                              \
                }                                                                                       \
            } else if (iterating) {                                                                     \
                const VT beta = init ? 0 : sc[2 * k + j];                                               \
                const VT omega = init ? 0 : (beta != 0 ? sc[8 * k + j] / beta : 0);                     \
                const VT alpha = init ? 0 : sc[6 * k + j];                                              \
                VT rho = 0, rn = 0;                                                                     \
                for (int64_t i = 0; i < n; ++i) {                                                       \
                    const int64_t e = i * k + j;                                                        \
                    VT ri, rri;                                                                         \
                    if (init) {                                                                         \
                        ri = r[e];                                                                      \
                        rri = ri;                                                                       \
                        rr[e] = ri;                                                                     \
                    } else {                                                                            \
                        x[e] += alpha * y[e] + omega * z[e];                                            \
                        ri = s[e] - omega * t[e];                                                       \
                        r[e] = ri;                                                                      \
                        rri = rr[e];                                                                    \
                    }                                                                                   \
                    rho += rri * ri;                                                                    \
                    rn += ri * ri;                                                                      \
                }                                                                                       \
                if (init) {                                                                             \
                    if (baseline == 1) sc[4 * k + j] = (VT)sqrt(rn);                                    \
                    if (baseline == 2) sc[4 * k + j] = 1;                                               \
                    sc[5 * k + j] = factor * sc[4 * k + j];                                             \
                } else {                                                                                \
                    sc[7 * k + j] = omega;                                                              \
                }                                                                                       \
                sc[k + j] = sc[j];                                                                      \
                sc[j] = rho;                                                                            \
                sc[3 * k + j] = rn;                                                                     \
                const VT tau = ctl[3] == 1 ? SQRT(rn) : SQRT(FABS(rho));                                \
                status[j] = st = mock_criteria_status(iter, ctl, tau <= sc[5 * k + j], 0x40);           \
            }                                                                                           \
            if (!STOPPED(st)) all_stopped = 0;                                                          \
        }                                                                                               \
        ctl[5] = 0;                                                                                     \
        ctl[0] = all_stopped;                                                                           \
    }                                                                                                   \
    static b200_status replay_step_p_##V(b200_ctx* ctx, const mock_op* op)                              \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_bm_step_p_##V(op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);         \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    static b200_status replay_step_s_##V(b200_ctx* ctx, const mock_op* op)                              \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_bm_step_s_##V(op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);         \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    static b200_status replay_step_xr_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_bm_step_xr_##V(0, op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], \
                            a[9], 0, 0);                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    int64_t b200_bicgstab_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                            \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        return 4 * k + 64;                                                                              \
    }                                                                                                   \
    b200_status b200_bicgstab_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* rr,   \
                                            VT* p, VT* v, VT* y, VT* s, VT* t, VT* z, VT* sc,           \
                                            uint8_t* status, int32_t* ctl, VT* work, int64_t max_iters, \
                                            int32_t res_kind, int32_t iter_first, int32_t baseline,     \
                                            VT reduction_factor)                                        \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (ctx->capture) { mock_set_error("bicgstab_mrhs_init inside a capture"); return B200_ERR_INVALID; } \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            sc[j] = sc[k + j] = sc[2 * k + j] = sc[6 * k + j] = sc[7 * k + j] = sc[8 * k + j] = 1;      \
            sc[3 * k + j] = sc[9 * k + j] = 0;                                                          \
            status[j] = 0;                                                                              \
        }                                                                                               \
        ctl[0] = 0; ctl[1] = -1;                                                                        \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                            \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = 0;                                             \
        VT* zeroed[6] = {p, v, y, s, t, z};                                                             \
        for (int a = 0; a < 6; ++a) memset(zeroed[a], 0, sizeof(VT) * (size_t)(n * k));                 \
        mock_bm_step_xr_##V(1, n, k, NULL, (VT*)r, NULL, NULL, NULL, NULL, rr, sc, status, ctl,         \
                            baseline, reduction_factor);                                                \
        ctx->launches += 2;                                                                             \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_bicgstab_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p, const VT* r,  \
                                              const VT* v, VT* y, const VT* inv_diag, const VT* sc,     \
                                              const uint8_t* status, const int32_t* ctl)                \
    {                                                                                                   \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_step_p_##V);                                          \
            op->p[0] = p; op->p[1] = (void*)r; op->p[2] = (void*)v; op->p[3] = y;                       \
            op->p[4] = (void*)inv_diag; op->p[5] = (void*)sc; op->p[6] = (void*)status;                 \
            op->p[7] = (void*)ctl; op->n[0] = n; op->n[1] = k;                                          \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_bm_step_p_##V(n, k, p, r, v, y, inv_diag, sc, status, ctl);                                \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_bicgstab_mrhs_step_s_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r,         \
                                              const VT* v, VT* s, VT* z, const VT* inv_diag, VT* sc,    \
                                              uint8_t* status, int32_t* ctl, VT* work)                  \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_step_s_##V);                                          \
            op->p[0] = (void*)r; op->p[1] = (void*)v; op->p[2] = s; op->p[3] = z;                       \
            op->p[4] = (void*)inv_diag; op->p[5] = sc; op->p[6] = status; op->p[7] = ctl;               \
            op->n[0] = n; op->n[1] = k;                                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_bm_step_s_##V(n, k, r, v, s, z, inv_diag, sc, status, ctl);                                \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_bicgstab_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* r,       \
                                               const VT* s, const VT* t, const VT* y, const VT* z,      \
                                               const VT* rr, VT* sc, uint8_t* status, int32_t* ctl,     \
                                               VT* work)                                                \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_step_xr_##V);                                         \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)s; op->p[3] = (void*)t; op->p[4] = (void*)y;  \
            op->p[5] = (void*)z; op->p[6] = (void*)rr; op->p[7] = sc; op->p[8] = status;                \
            op->p[9] = ctl; op->n[0] = n; op->n[1] = k;                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_bm_step_xr_##V(0, n, k, x, r, s, t, y, z, (VT*)rr, sc, status, ctl, 0, 0);                 \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_FUSED_BM(f64, double, sqrt, fabs)
MOCK_FUSED_BM(f32, float, sqrtf, fabsf)
