/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused MINRES entry points for several
 * right-hand sides (ginkgo_b200/csrc/fused_minres_mrhs.cu: b200_minres_mrhs_*, b200_csr_spmv_sub_mdot_*),
 * so that solver::Minres::try_fused_multi_rhs -- set-up, capture, replay, polling of the control block,
 * the per-column statuses -- runs on the CPU.  Every column's sums run over the rows in order, as the
 * oracle's compute_dot does, so this path and the kernel-by-kernel loop on the mock take the same
 * iterations and give the same bits. */
#include "mock.h"

/* sc[s k + j] with the slots of mock_fused_minres.c; step_1 and step_2 in the oracle's expression order,
 * skipped for a stopped column */
#define MOCK_FUSED_MINRES_MRHS(V, VT, SQRT, FABS)                                                       \
    static VT mock_mm_safe_divide_##V(VT a, VT b) { return b == 0 ? (VT)0 : a / b; }                    \
    static uint8_t mock_mm_status_##V(int32_t iter, const int32_t* ctl, const VT* sc, int64_t k, int64_t j) \
    {                                                                                                   \
        return mock_criteria_status(iter, ctl, SQRT(FABS(sc[6 * k + j])) <= sc[5 * k + j], 0x40);       \
    }                                                                                                   \
    static void mock_mm_lanczos_##V(int64_t n, int64_t k, VT* v, const VT* q, const VT* d, VT* sc,      \
                                    const uint8_t* status, const int32_t* ctl)                          \
    {                                                                                                   \
        if (ctl[0] != 0) return;                                                                        \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            if (STOPPED(status[j])) continue;                                                           \
            VT* s = sc + j;                                                                             \
            VT beta = 0;                                                                                \
            for (int64_t i = 0; i < n; ++i) {                                                           \
                const int64_t e = i * k + j;                                                            \
                v[e] -= s[0] * q[e];                                                                    \
                const VT zt = d ? v[e] * d[i] : v[e];                                                   \
                beta += v[e] * zt;                                                                      \
            }                                                                                           \
            s[k] = SQRT(beta);                                                                          \
            s[3 * k] = s[11 * k] * s[2 * k];                                                            \
            const VT tmp_d = s[2 * k], tmp_a = s[0];                                                    \
            s[2 * k] = s[9 * k] * s[10 * k] * tmp_d + s[12 * k] * tmp_a;                                \
            s[0] = -s[12 * k] * s[9 * k] * tmp_d + s[10 * k] * tmp_a;                                   \
            VT t = s[10 * k]; s[10 * k] = s[9 * k]; s[9 * k] = t;                                       \
            t = s[12 * k]; s[12 * k] = s[11 * k]; s[11 * k] = t;                                        \
            if (s[0] == 0) {                                                                            \
                s[10 * k] = 0;                                                                          \
                s[12 * k] = 1;                                                                          \
            } else {                                                                                    \
                const VT scale = FABS(s[0]) + FABS(s[k]);                                               \
                const VT hyp = scale * SQRT(FABS(s[0] / scale) * FABS(s[0] / scale) +                   \
                                            FABS(s[k] / scale) * FABS(s[k] / scale));                   \
                s[10 * k] = s[0] / hyp;                                                                 \
                s[12 * k] = s[k] / hyp;                                                                 \
            }                                                                                           \
            s[0] = s[10 * k] * s[0] + s[12 * k] * s[k];                                                 \
            s[6 * k] = s[12 * k] * s[12 * k] * s[6 * k];                                                \
            s[7 * k] = s[8 * k];                                                                        \
            s[8 * k] = -s[12 * k] * s[7 * k];                                                           \
        }                                                                                               \
    }                                                                                                   \
    static void mock_mm_update_##V(int64_t n, int64_t k, VT* x, VT* p0, VT* p1, VT* z, VT* q, VT* v,    \
                                   const VT* d, VT* sc, uint8_t* status, int32_t* ctl)                  \
    {                                                                                                   \
        if (ctl[0] != 0) return;                                                                        \
        const int32_t iter = ctl[1];                                                                    \
        VT* p = (iter & 1) ? p0 : p1;                                                                   \
        const VT* pp = (iter & 1) ? p1 : p0;                                                            \
        int all_stopped = 1;                                                                            \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            if (!STOPPED(status[j])) {                                                                  \
                VT* s = sc + j;                                                                         \
                for (int64_t i = 0; i < n; ++i) {                                                       \
                    const int64_t e = i * k + j;                                                        \
                    p[e] = mock_mm_safe_divide_##V(z[e] - s[2 * k] * pp[e] - s[3 * k] * p[e], s[0]);    \
                    x[e] = x[e] + s[10 * k] * s[7 * k] * p[e];                                          \
                    const VT vv = v[e], tmp = q[e];                                                     \
                    q[e] = mock_mm_safe_divide_##V(vv, s[k]);                                           \
                    v[e] = tmp * s[k];                                                                  \
                    z[e] = mock_mm_safe_divide_##V(d ? vv * d[i] : vv, s[k]);                           \
                }                                                                                       \
                const VT t = s[k]; s[k] = s[2 * k]; s[2 * k] = t;                                       \
                status[j] = mock_mm_status_##V(iter + 1, ctl, sc, k, j);                                \
            }                                                                                           \
            if (!STOPPED(status[j])) all_stopped = 0;                                                   \
        }                                                                                               \
        ctl[1] = iter + 1;                                                                              \
        ctl[0] = all_stopped;                                                                           \
    }                                                                                                   \
    static b200_status replay_mm_lanczos_##V(b200_ctx* ctx, const mock_op* op)                          \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_mm_lanczos_##V(op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5]);                    \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    static b200_status replay_mm_update_##V(b200_ctx* ctx, const mock_op* op)                           \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* a = op->p;                                                                         \
        mock_mm_update_##V(op->n[0], op->n[1], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8],    \
                           a[9]);                                                                       \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    int64_t b200_minres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                              \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        return 2 * k + 64;                                                                              \
    }                                                                                                   \
    b200_status b200_minres_mrhs_init_##V(b200_ctx* ctx, int64_t k, VT* sc, uint8_t* status,            \
                                          int32_t* ctl, int64_t max_iters, int32_t res_kind,            \
                                          int32_t iter_first, int32_t baseline, VT reduction_factor)    \
    {                                                                                                   \
        if (ctx->capture) { mock_set_error("minres_mrhs_init inside a capture"); return B200_ERR_INVALID; } \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        ctl[0] = 0; ctl[1] = 0;                                                                         \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                            \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = ctl[6] = ctl[7] = 0;                           \
        int all_stopped = 1;                                                                            \
        for (int64_t j = 0; j < k; ++j) {                                                               \
            if (baseline == 2) sc[4 * k + j] = 1;                                                       \
            sc[5 * k + j] = reduction_factor * sc[4 * k + j];                                           \
            status[j] = mock_mm_status_##V(0, ctl, sc, k, j);                                           \
            if (!STOPPED(status[j])) all_stopped = 0;                                                   \
        }                                                                                               \
        ctl[0] = all_stopped;                                                                           \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_minres_mrhs_lanczos_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v, const VT* q,   \
                                             const VT* inv_diag, VT* sc, const uint8_t* status,         \
                                             const int32_t* ctl, VT* work)                              \
    {                                                                                                   \
        (void)work;                                                                                     \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_mm_lanczos_##V);                                      \
            op->p[0] = v; op->p[1] = (void*)q; op->p[2] = (void*)inv_diag; op->p[3] = sc;               \
            op->p[4] = (void*)status; op->p[5] = (void*)ctl; op->n[0] = n; op->n[1] = k;                \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_mm_lanczos_##V(n, k, v, q, inv_diag, sc, status, ctl);                                     \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_minres_mrhs_update_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* p0, VT* p1, \
                                            VT* z, VT* q, VT* v, const VT* inv_diag, VT* sc,            \
                                            uint8_t* status, int32_t* ctl)                              \
    {                                                                                                   \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_mm_update_##V);                                       \
            op->p[0] = x; op->p[1] = p0; op->p[2] = p1; op->p[3] = z; op->p[4] = q; op->p[5] = v;       \
            op->p[6] = (void*)inv_diag; op->p[7] = sc; op->p[8] = status; op->p[9] = ctl;               \
            op->n[0] = n; op->n[1] = k;                                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_mm_update_##V(n, k, x, p0, p1, z, q, v, inv_diag, sc, status, ctl);                        \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_FUSED_MINRES_MRHS(f64, double, sqrt, fabs)
MOCK_FUSED_MINRES_MRHS(f32, float, sqrtf, fabsf)

/* c = A b - c for k columns (stride k), dots[j] = c_j . b_j over the rows (the oracle's advanced SpMV
 * with 1, -1); every column computed; no-op once every column stopped */
#define MOCK_SPMV_SUB_MDOT(V, VT, I, IT)                                                                \
    static void mock_spmv_sub_mdot_##V##_##I(int64_t num_rows, int64_t k, const IT* rp, const IT* ci,   \
                                             const VT* va, const VT* b, VT* c, VT* dots,                \
                                             const int32_t* ctl)                                        \
    {                                                                                                   \
        if (ctl && ctl[0] != 0) return;                                                                 \
        const VT one = 1, neg_one = -1;                                                                 \
        for (int64_t j = 0; j < k; ++j) dots[j] = 0;                                                    \
        for (int64_t r = 0; r < num_rows; ++r)                                                          \
            for (int64_t j = 0; j < k; ++j) {                                                           \
                VT sum = c[r * k + j] * neg_one;                                                        \
                for (int64_t e = rp[r]; e < (int64_t)rp[r + 1]; ++e) sum += one * va[e] * b[ci[e] * k + j]; \
                c[r * k + j] = sum;                                                                     \
                dots[j] += sum * b[r * k + j];                                                          \
            }                                                                                           \
    }                                                                                                   \
    static b200_status replay_spmv_sub_mdot_##V##_##I(b200_ctx* ctx, const mock_op* op)                 \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* p = op->p;                                                                         \
        mock_spmv_sub_mdot_##V##_##I(op->n[0], op->n[1], p[0], p[1], p[2], p[3], p[4], p[5], p[6]);     \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    b200_status b200_csr_spmv_sub_mdot_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,     \
                                                 int64_t nnz, const IT* row_ptrs, const IT* col_idxs,   \
                                                 const VT* values, const VT* b, int64_t k, VT* c,       \
                                                 VT* dots, VT* work, const int32_t* ctl)                \
    {                                                                                                   \
        (void)num_cols; (void)nnz; (void)work;                                                          \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, replay_spmv_sub_mdot_##V##_##I);                             \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;           \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = dots; op->p[6] = (void*)ctl;                  \
            op->n[0] = num_rows; op->n[1] = k;                                                          \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_spmv_sub_mdot_##V##_##I(num_rows, k, row_ptrs, col_idxs, values, b, c, dots, ctl);         \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_SPMV_SUB_MDOT(f64, double, i32, int32_t)
MOCK_SPMV_SUB_MDOT(f64, double, i64, int64_t)
MOCK_SPMV_SUB_MDOT(f32, float, i32, int32_t)
MOCK_SPMV_SUB_MDOT(f32, float, i64, int64_t)
