/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused CG entry points
 * (ginkgo_b200/csrc/fused_cg.cu; sc / ctl layouts of the header), so that solver::Cg::try_fused --
 * capture, replay, polling of the control block -- runs on the CPU.  The SpMV + dot is in
 * mock_spmv_dot.c. */
#include "mock.h"

#define MOCK_FUSED(V, VT, SQRT)                                                                        \
    static void mock_step_xr_##V(int init, int64_t n, VT* x, VT* r, const VT* p, const VT* q, VT* z,   \
                                 const VT* inv_diag, VT* sc, int32_t* ctl, int finalize, int baseline, \
                                 VT factor)                                                            \
    {                                                                                                  \
        if (!init && ctl[0] != 0) return;                                                              \
        const VT pq = sc[2];                                                                           \
        const int update = !init && pq != 0;                                                           \
        const VT alpha = update ? sc[0] / pq : 0;                                                      \
        VT s_rho = 0, s_rr = 0;                                                                        \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            VT ri = r[i];                                                                              \
            if (update) {                                                                              \
                x[i] += alpha * p[i];                                                                  \
                ri -= alpha * q[i];                                                                    \
                r[i] = ri;                                                                             \
            }                                                                                          \
            const VT zi = inv_diag ? ri * inv_diag[i] : ri;                                            \
            z[i] = zi;                                                                                 \
            s_rho += ri * zi;                                                                          \
            s_rr += ri * ri;                                                                           \
        }                                                                                              \
        if (!finalize) {                                                                               \
            sc[6] = s_rho;                                                                             \
            sc[7] = s_rr;                                                                              \
            return;                                                                                    \
        }                                                                                              \
        if (init) {                                                                                    \
            if (baseline == 1) sc[4] = SQRT(s_rr);                                                     \
            if (baseline == 2) sc[4] = 1;                                                              \
            sc[5] = factor * sc[4];                                                                    \
        }                                                                                              \
        mock_finish_scalars_##V(s_rho, s_rr, sc, ctl);                                                 \
    }                                                                                                  \
    static void mock_step_p_##V(int64_t n, VT* p, const VT* z, const VT* sc, const int32_t* ctl)       \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const VT rho = sc[0], prev = sc[1];                                                            \
        for (int64_t i = 0; i < n; ++i) p[i] = prev == 0 ? z[i] : z[i] + (rho / prev) * p[i];          \
    }                                                                                                  \
    static void mock_finish_##V(VT* sc, int32_t* ctl, int init, int baseline, VT factor)               \
    {                                                                                                  \
        if (!init && ctl[0] != 0) return;                                                              \
        if (init) {                                                                                    \
            if (baseline == 1) sc[4] = SQRT(sc[7]);                                                    \
            if (baseline == 2) sc[4] = 1;                                                              \
            if (baseline == 3) sc[4] = SQRT(sc[4]);                                                    \
            sc[5] = factor * sc[4];                                                                    \
        }                                                                                              \
        mock_finish_scalars_##V(sc[6], sc[7], sc, ctl);                                                \
    }                                                                                                  \
    static b200_status replay_step_p_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        mock_step_p_##V(op->n[0], op->p[0], op->p[1], op->p[2], op->p[3]);                             \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_step_xr_##V(b200_ctx* ctx, const mock_op* op)                            \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_step_xr_##V(0, op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], op->i[0], 0, 0); \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_finish_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        mock_finish_##V(op->p[0], op->p[1], op->i[0], op->i[1], (VT)op->d);                            \
        return B200_OK;                                                                                \
    }                                                                                                  \
    int64_t b200_cg_fused_work_size_##V(const b200_ctx* ctx) { (void)ctx; return 64; }                 \
    b200_status b200_cg_fused_init_##V(b200_ctx* ctx, int64_t n, const VT* r, VT* z, VT* p, VT* q,     \
                                       const VT* inv_diag, VT* sc, int32_t* ctl, VT* work,             \
                                       int64_t max_iters, int32_t res_kind, int32_t iter_first,        \
                                       int32_t baseline, VT reduction_factor, int32_t finalize)        \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) { mock_set_error("fused_init inside a capture"); return B200_ERR_INVALID; }  \
        sc[0] = 1; sc[1] = 1; sc[2] = 0; sc[3] = 0; sc[6] = 0; sc[7] = 0;                              \
        ctl[0] = 0; ctl[1] = -1;                                                                       \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                           \
        ctl[3] = res_kind; ctl[4] = iter_first;                                                        \
        memset(p, 0, sizeof(VT) * (size_t)n);                                                          \
        memset(q, 0, sizeof(VT) * (size_t)n);                                                          \
        mock_step_xr_##V(1, n, NULL, (VT*)r, p, q, z, inv_diag, sc, ctl, finalize, baseline,           \
                         reduction_factor);                                                            \
        ctx->launches += 2;                                                                            \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_cg_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* z, const VT* sc,   \
                                         const int32_t* ctl)                                           \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_step_p_##V);                                         \
            op->p[0] = p; op->p[1] = (void*)z; op->p[2] = (void*)sc; op->p[3] = (void*)ctl;            \
            op->n[0] = n;                                                                              \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_step_p_##V(n, p, z, sc, ctl);                                                             \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_cg_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r, const VT* p,         \
                                          const VT* q, VT* z, const VT* inv_diag, VT* sc,              \
                                          int32_t* ctl, VT* work, int32_t finalize)                    \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_step_xr_##V);                                        \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)p; op->p[3] = (void*)q; op->p[4] = z;        \
            op->p[5] = (void*)inv_diag; op->p[6] = sc; op->p[7] = ctl;                                 \
            op->n[0] = n; op->i[0] = finalize;                                                         \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_step_xr_##V(0, n, x, r, p, q, z, inv_diag, sc, ctl, finalize, 0, 0);                      \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_cg_fused_finish_##V(b200_ctx* ctx, VT* sc, int32_t* ctl, int32_t init,            \
                                         int32_t baseline, VT reduction_factor)                        \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_finish_##V);                                         \
            op->p[0] = sc; op->p[1] = ctl; op->i[0] = init; op->i[1] = baseline;                       \
            op->d = (double)reduction_factor;                                                          \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_finish_##V(sc, ctl, init, baseline, reduction_factor);                                    \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_FUSED(f64, double, sqrt)
MOCK_FUSED(f32, float, sqrtf)
