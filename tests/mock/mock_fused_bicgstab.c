/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused BiCGStab entry points
 * (ginkgo_b200/csrc/fused_bicgstab.cu), so that solver::Bicgstab::try_fused -- capture, replay, polling
 * of the control block, the pending-finalize hand-over -- runs on the CPU.  The SpMV + dots
 * (b200_csr_spmv_dot2_*) are in mock_spmv_dot.c. */
#include "mock.h"

/* ---- fused BiCGStab (ginkgo_b200/csrc/fused_bicgstab.cu restated sequentially; sc / ctl layouts of the header) ---- */
#define MOCK_FUSED_BICGSTAB(V, VT, SQRT, FABS)                                                         \
    static void mock_bicgstab_step_p_##V(int64_t n, VT* p, const VT* r, const VT* v, VT* y,            \
                                         const VT* inv_diag, const VT* sc, const int32_t* ctl)         \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const VT rho = sc[0], prev = sc[1], alpha = sc[6], omega = sc[7];                              \
        const int plain = !(prev * omega != 0);                                                        \
        const VT tmp = plain ? 0 : rho / prev * alpha / omega;                                         \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            p[i] = plain ? r[i] : r[i] + tmp * (p[i] - omega * v[i]);                                  \
            y[i] = inv_diag ? p[i] * inv_diag[i] : p[i];                                               \
        }                                                                                              \
    }                                                                                                  \
    static void mock_bicgstab_step_s_##V(int64_t n, const VT* r, const VT* v, VT* s, VT* z,            \
                                         const VT* inv_diag, VT* sc, int32_t* ctl)                     \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const VT beta = sc[2];                                                                         \
        const VT alpha = beta != 0 ? sc[0] / beta : 0;                                                 \
        VT ss = 0;                                                                                     \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            s[i] = beta != 0 ? r[i] - alpha * v[i] : r[i];                                             \
            z[i] = inv_diag ? s[i] * inv_diag[i] : s[i];                                               \
            ss += s[i] * s[i];                                                                         \
        }                                                                                              \
        sc[6] = alpha;                                                                                 \
        sc[9] = ss;                                                                                    \
        const VT tau = ctl[3] == 1 ? SQRT(ss) : SQRT(FABS(sc[0]));                                     \
        const uint8_t status = mock_criteria_status(ctl[1], ctl, tau <= sc[5], 0x40);                  \
        if (status) {                                                                                  \
            ctl[0] = status;                                                                           \
            ctl[5] = 1;                                                                                \
        }                                                                                              \
    }                                                                                                  \
    static void mock_bicgstab_step_xr_##V(int init, int64_t n, VT* x, VT* r, const VT* s, const VT* t, \
                                          const VT* y, const VT* z, VT* rr, VT* sc, int32_t* ctl,      \
                                          int baseline, VT factor)                                     \
    {                                                                                                  \
        if (!init && ctl[5] != 0) {                                                                    \
            for (int64_t i = 0; i < n; ++i) x[i] += sc[6] * y[i];                                      \
            ctl[5] = 0;                                                                                \
            return;                                                                                    \
        }                                                                                              \
        if (!init && ctl[0] != 0) return;                                                              \
        const VT omega = init ? 0 : (sc[2] != 0 ? sc[8] / sc[2] : 0);                                  \
        const VT alpha = sc[6];                                                                        \
        VT s_rho = 0, s_rr = 0;                                                                        \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            if (init) {                                                                                \
                rr[i] = r[i];                                                                          \
            } else {                                                                                   \
                x[i] += alpha * y[i] + omega * z[i];                                                   \
                r[i] = s[i] - omega * t[i];                                                            \
            }                                                                                          \
            s_rho += rr[i] * r[i];                                                                     \
            s_rr += r[i] * r[i];                                                                       \
        }                                                                                              \
        if (init) {                                                                                    \
            if (baseline == 1) sc[4] = SQRT(s_rr);                                                     \
            if (baseline == 2) sc[4] = 1;                                                              \
            sc[5] = factor * sc[4];                                                                    \
        } else {                                                                                       \
            sc[7] = omega;                                                                             \
        }                                                                                              \
        mock_finish_scalars_##V(s_rho, s_rr, sc, ctl);                                                 \
    }                                                                                                  \
    static b200_status replay_step_p_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_bicgstab_step_p_##V(op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6]);                  \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_step_s_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_bicgstab_step_s_##V(op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6]);                  \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_step_xr_##V(b200_ctx* ctx, const mock_op* op)                            \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_bicgstab_step_xr_##V(0, op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], p[8], 0, 0); \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_bicgstab_fused_init_##V(b200_ctx* ctx, int64_t n, const VT* r, VT* rr, VT* p,     \
                                             VT* v, VT* y, VT* s, VT* t, VT* z, VT* sc, int32_t* ctl,  \
                                             VT* work, int64_t max_iters, int32_t res_kind,            \
                                             int32_t iter_first, int32_t baseline, VT reduction_factor) \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) { mock_set_error("fused_init inside a capture"); return B200_ERR_INVALID; }  \
        sc[0] = 1; sc[1] = 1; sc[2] = 1; sc[3] = 0; sc[6] = 1; sc[7] = 1; sc[8] = 1; sc[9] = 0;        \
        ctl[0] = 0; ctl[1] = -1;                                                                       \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                           \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = 0;                                            \
        VT* zeroed[6] = {p, v, y, s, t, z};                                                            \
        for (int k = 0; k < 6; ++k) memset(zeroed[k], 0, sizeof(VT) * (size_t)n);                      \
        mock_bicgstab_step_xr_##V(1, n, NULL, (VT*)r, NULL, NULL, NULL, NULL, rr, sc, ctl, baseline,   \
                                  reduction_factor);                                                   \
        ctx->launches += 8;                                                                            \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_bicgstab_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* r,           \
                                               const VT* v, VT* y, const VT* inv_diag, const VT* sc,   \
                                               const int32_t* ctl)                                     \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_step_p_##V);                                         \
            op->p[0] = p; op->p[1] = (void*)r; op->p[2] = (void*)v; op->p[3] = y;                      \
            op->p[4] = (void*)inv_diag; op->p[5] = (void*)sc; op->p[6] = (void*)ctl; op->n[0] = n;     \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_bicgstab_step_p_##V(n, p, r, v, y, inv_diag, sc, ctl);                                    \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_bicgstab_fused_step_s_##V(b200_ctx* ctx, int64_t n, const VT* r, const VT* v,     \
                                               VT* s, VT* z, const VT* inv_diag, VT* sc, int32_t* ctl, \
                                               VT* work)                                               \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_step_s_##V);                                         \
            op->p[0] = (void*)r; op->p[1] = (void*)v; op->p[2] = s; op->p[3] = z;                      \
            op->p[4] = (void*)inv_diag; op->p[5] = sc; op->p[6] = ctl; op->n[0] = n;                   \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_bicgstab_step_s_##V(n, r, v, s, z, inv_diag, sc, ctl);                                    \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_bicgstab_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r, const VT* s,   \
                                                const VT* t, const VT* y, const VT* z, const VT* rr,   \
                                                VT* sc, int32_t* ctl, VT* work)                        \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_step_xr_##V);                                        \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)s; op->p[3] = (void*)t; op->p[4] = (void*)y; \
            op->p[5] = (void*)z; op->p[6] = (void*)rr; op->p[7] = sc; op->p[8] = ctl; op->n[0] = n;    \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_bicgstab_step_xr_##V(0, n, x, r, s, t, y, z, (VT*)rr, sc, ctl, 0, 0);                     \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_FUSED_BICGSTAB(f64, double, sqrt, fabs)
MOCK_FUSED_BICGSTAB(f32, float, sqrtf, fabsf)
