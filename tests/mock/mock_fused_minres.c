/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused MINRES entry points
 * (ginkgo_b200/csrc/fused_minres.cu, b200_csr_spmv_sub_dot_*), so that solver::Minres::try_fused --
 * set-up, capture, replay, polling of the control block -- runs on the CPU.  The sums run in row order,
 * as the oracle's loop kernels run them, so the fused path and the loop give the same bits here. */
#include "mock.h"

/* sc / ctl layouts of the header; step_1 and step_2 in the oracle's expression order */
#define MOCK_FUSED_MINRES(V, VT, SQRT, FABS)                                                           \
    static VT mock_safe_divide_##V(VT a, VT b) { return b == 0 ? (VT)0 : a / b; }                      \
    static void mock_minres_lanczos_##V(int64_t n, VT* v, const VT* q, const VT* d, VT* sc,            \
                                        const int32_t* ctl)                                            \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const VT alpha = sc[0];                                                                        \
        VT beta = 0;                                                                                   \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            if (alpha != 0) v[i] -= alpha * q[i];                                                      \
            const VT zt = d ? v[i] * d[i] : v[i];                                                      \
            beta += v[i] * zt;                                                                         \
        }                                                                                              \
        /* minres::step_1 */                                                                           \
        sc[1] = SQRT(beta);                                                                            \
        sc[3] = sc[11] * sc[2];                                                                        \
        const VT tmp_d = sc[2], tmp_a = sc[0];                                                         \
        sc[2] = sc[9] * sc[10] * tmp_d + sc[12] * tmp_a;                                               \
        sc[0] = -sc[12] * sc[9] * tmp_d + sc[10] * tmp_a;                                              \
        VT t = sc[10]; sc[10] = sc[9]; sc[9] = t;                                                      \
        t = sc[12]; sc[12] = sc[11]; sc[11] = t;                                                       \
        if (sc[0] == 0) {                                                                              \
            sc[10] = 0;                                                                                \
            sc[12] = 1;                                                                                \
        } else {                                                                                       \
            const VT scale = FABS(sc[0]) + FABS(sc[1]);                                                \
            const VT hyp = scale * SQRT(FABS(sc[0] / scale) * FABS(sc[0] / scale) +                    \
                                        FABS(sc[1] / scale) * FABS(sc[1] / scale));                    \
            sc[10] = sc[0] / hyp;                                                                      \
            sc[12] = sc[1] / hyp;                                                                      \
        }                                                                                              \
        sc[0] = sc[10] * sc[0] + sc[12] * sc[1];                                                       \
        sc[6] = sc[12] * sc[12] * sc[6];                                                               \
        sc[7] = sc[8];                                                                                 \
        sc[8] = -sc[12] * sc[7];                                                                       \
    }                                                                                                  \
    static void mock_minres_update_##V(int64_t n, VT* x, VT* p0, VT* p1, VT* z, VT* q, VT* v,          \
                                       const VT* d, VT* sc, int32_t* ctl)                              \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const int32_t iter = ctl[1];                                                                   \
        VT* p = (iter & 1) ? p0 : p1;                                                                  \
        const VT* pp = (iter & 1) ? p1 : p0;                                                           \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            p[i] = mock_safe_divide_##V(z[i] - sc[2] * pp[i] - sc[3] * p[i], sc[0]);                   \
            x[i] = x[i] + sc[10] * sc[7] * p[i];                                                       \
            const VT vv = v[i], tmp = q[i];                                                            \
            q[i] = mock_safe_divide_##V(vv, sc[1]);                                                    \
            v[i] = tmp * sc[1];                                                                        \
            z[i] = mock_safe_divide_##V(d ? vv * d[i] : vv, sc[1]);                                    \
        }                                                                                              \
        const VT t = sc[1]; sc[1] = sc[2]; sc[2] = t;                                                  \
        ctl[1] = iter + 1;                                                                             \
        ctl[0] = mock_criteria_status(iter + 1, ctl, SQRT(FABS(sc[6])) <= sc[5], 0x40);                \
    }                                                                                                  \
    static b200_status replay_lanczos_##V(b200_ctx* ctx, const mock_op* op)                            \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_minres_lanczos_##V(op->n[0], p[0], p[1], p[2], p[3], p[4]);                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_update_##V(b200_ctx* ctx, const mock_op* op)                             \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_minres_update_##V(op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], p[8]);        \
        return B200_OK;                                                                                \
    }                                                                                                  \
    int64_t b200_minres_fused_work_size_##V(const b200_ctx* ctx)                                       \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        return 64;                                                                                     \
    }                                                                                                  \
    b200_status b200_minres_fused_init_##V(b200_ctx* ctx, VT* sc, int32_t* ctl, int64_t max_iters,     \
                                           int32_t res_kind, int32_t iter_first, int32_t baseline,     \
                                           VT reduction_factor)                                        \
    {                                                                                                  \
        if (ctx->capture) { mock_set_error("minres fused_init inside a capture"); return B200_ERR_INVALID; } \
        if (baseline == 2) sc[4] = 1;                                                                  \
        sc[5] = reduction_factor * sc[4];                                                              \
        ctl[1] = 0;                                                                                    \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                           \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = ctl[6] = ctl[7] = 0;                          \
        ctl[0] = mock_criteria_status(0, ctl, SQRT(FABS(sc[6])) <= sc[5], 0x40);                       \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_minres_fused_lanczos_##V(b200_ctx* ctx, int64_t n, VT* v, const VT* q,            \
                                              const VT* inv_diag, VT* sc, const int32_t* ctl,          \
                                              VT* work)                                                \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_lanczos_##V);                                        \
            op->p[0] = v; op->p[1] = (void*)q; op->p[2] = (void*)inv_diag; op->p[3] = sc;              \
            op->p[4] = (void*)ctl; op->n[0] = n;                                                       \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_minres_lanczos_##V(n, v, q, inv_diag, sc, ctl);                                           \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_minres_fused_update_##V(b200_ctx* ctx, int64_t n, VT* x, VT* p0, VT* p1, VT* z,   \
                                             VT* q, VT* v, const VT* inv_diag, VT* sc, int32_t* ctl)   \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_update_##V);                                         \
            op->p[0] = x; op->p[1] = p0; op->p[2] = p1; op->p[3] = z; op->p[4] = q; op->p[5] = v;      \
            op->p[6] = (void*)inv_diag; op->p[7] = sc; op->p[8] = ctl; op->n[0] = n;                   \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_minres_update_##V(n, x, p0, p1, z, q, v, inv_diag, sc, ctl);                              \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_FUSED_MINRES(f64, double, sqrt, fabs)
MOCK_FUSED_MINRES(f32, float, sqrtf, fabsf)

/* c = A b - c and *dot_out = c . b over the rows (the oracle's advanced SpMV with 1, -1); no-op
 * once the solver stopped */
#define MOCK_SPMV_SUB_DOT(V, VT, I, IT)                                                                \
    static void mock_spmv_sub_dot_##V##_##I(int64_t num_rows, const IT* rp, const IT* ci, const VT* va, \
                                            const VT* b, VT* c, VT* dot_out, const int32_t* ctl)       \
    {                                                                                                  \
        if (ctl && ctl[0] != 0) return;                                                                \
        const VT one = 1, neg_one = -1;                                                                \
        VT dot = 0;                                                                                    \
        for (int64_t r = 0; r < num_rows; ++r) {                                                       \
            VT sum = c[r] * neg_one;                                                                   \
            for (int64_t k = rp[r]; k < (int64_t)rp[r + 1]; ++k) sum += one * va[k] * b[ci[k]];        \
            c[r] = sum;                                                                                \
            dot += sum * b[r];                                                                         \
        }                                                                                              \
        *dot_out = dot;                                                                                \
    }                                                                                                  \
    static b200_status replay_spmv_sub_dot_##V##_##I(b200_ctx* ctx, const mock_op* op)                 \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_spmv_sub_dot_##V##_##I(op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6]);               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_csr_spmv_sub_dot_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan,              \
                                                int64_t num_rows, int64_t num_cols, int64_t nnz,       \
                                                const IT* row_ptrs, const IT* col_idxs,                \
                                                const VT* values, const VT* b, VT* c, VT* dot_out,     \
                                                VT* work, const int32_t* ctl)                          \
    {                                                                                                  \
        (void)plan; (void)num_cols; (void)nnz; (void)work;                                             \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_spmv_sub_dot_##V##_##I);                             \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;          \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = dot_out; op->p[6] = (void*)ctl;              \
            op->n[0] = num_rows;                                                                       \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_spmv_sub_dot_##V##_##I(num_rows, row_ptrs, col_idxs, values, b, c, dot_out, ctl);         \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_SPMV_SUB_DOT(f64, double, i32, int32_t)
MOCK_SPMV_SUB_DOT(f64, double, i64, int64_t)
MOCK_SPMV_SUB_DOT(f32, float, i32, int32_t)
MOCK_SPMV_SUB_DOT(f32, float, i64, int64_t)
