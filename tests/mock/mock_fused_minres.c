/* TEST INFRASTRUCTURE ONLY.  The host-memory mock of mock_base.c plus sequential restatements of the
 * fused MINRES entry points (ginkgo_b200/csrc/fused_minres.cu, b200_csr_spmv_sub_dot_*), so that
 * solver::Minres::try_fused -- set-up, capture, replay, polling of the control block -- runs on the
 * CPU.  mock_base.c is compiled as part of this file (its context and recorded graphs are file-local);
 * its b200_graph_launch is kept under another name and replays the operations it knows, one at a
 * time.  The sums run in row order, as the oracle's loop kernels run them, so the fused path and the
 * loop give the same bits here.  Built by tests/mock_minres_build.py. */
#define b200_graph_launch mock_base_graph_launch
#include "mock_base.c"
#undef b200_graph_launch

enum { OP_MINRES_LANCZOS = 200, OP_MINRES_UPDATE, OP_SPMV_SUB_DOT };

/* Iteration (ctl[2]) and ImplicitResidualNorm (ctl[3]) in the user's order (ctl[4]), ids 1 and 2 */
static uint8_t mock_minres_status(int32_t iter, const int32_t* ctl, int converged)
{
    const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];
    uint8_t status = 0, id = 1;
    for (int k = 0; k < 2 && status == 0; ++k) {
        const int is_it = (k == 0) == (iter_first != 0);
        if (is_it) {
            if (max_iters < 0) continue;
            if (iter >= max_iters) status = (uint8_t)((id & 0x3f) | 0x40);
            ++id;
        } else {
            if (!res_kind) continue;
            if (converged) status = (uint8_t)(0x80 | (id & 0x3f) | 0x40);
            ++id;
        }
    }
    return status;
}

/* sc / ctl layouts of the header; step_1 and step_2 in the oracle's expression order */
#define MOCK_FUSED_MINRES(V, VT, VID, SQRT, FABS)                                                      \
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
        ctl[0] = mock_minres_status(iter + 1, ctl, SQRT(FABS(sc[6])) <= sc[5]);                        \
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
        ctl[0] = mock_minres_status(0, ctl, SQRT(FABS(sc[6])) <= sc[5]);                               \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_minres_fused_lanczos_##V(b200_ctx* ctx, int64_t n, VT* v, const VT* q,            \
                                              const VT* inv_diag, VT* sc, const int32_t* ctl,          \
                                              VT* work)                                                \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, OP_MINRES_LANCZOS, VID);                                    \
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
            mock_op* op = mock_new_op(ctx, OP_MINRES_UPDATE, VID);                                     \
            op->p[0] = x; op->p[1] = p0; op->p[2] = p1; op->p[3] = z; op->p[4] = q; op->p[5] = v;      \
            op->p[6] = (void*)inv_diag; op->p[7] = sc; op->p[8] = ctl; op->n[0] = n;                   \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_minres_update_##V(n, x, p0, p1, z, q, v, inv_diag, sc, ctl);                              \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_FUSED_MINRES(f64, double, 0, sqrt, fabs)
MOCK_FUSED_MINRES(f32, float, 1, sqrtf, fabsf)

/* c = A b - c and *dot_out = c . b over the rows (the oracle's advanced SpMV with 1, -1); no-op
 * once the solver stopped */
#define MOCK_SPMV_SUB_DOT(V, VT, VID, I, IT, IID)                                                      \
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
    b200_status b200_csr_spmv_sub_dot_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan,             \
                                                int64_t num_rows, int64_t num_cols, int64_t nnz,       \
                                                const IT* row_ptrs, const IT* col_idxs,                \
                                                const VT* values, const VT* b, VT* c, VT* dot_out,     \
                                                VT* work, const int32_t* ctl)                          \
    {                                                                                                  \
        (void)plan; (void)num_cols; (void)nnz; (void)work;                                             \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, OP_SPMV_SUB_DOT, VID);                                      \
            op->it = IID;                                                                              \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;          \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = dot_out; op->p[6] = (void*)ctl;              \
            op->n[0] = num_rows;                                                                       \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_spmv_sub_dot_##V##_##I(num_rows, row_ptrs, col_idxs, values, b, c, dot_out, ctl);         \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_SPMV_SUB_DOT(f64, double, 0, i32, int32_t, 0)
MOCK_SPMV_SUB_DOT(f64, double, 0, i64, int64_t, 1)
MOCK_SPMV_SUB_DOT(f32, float, 1, i32, int32_t, 0)
MOCK_SPMV_SUB_DOT(f32, float, 1, i64, int64_t, 1)

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    for (int k = 0; k < graph->g.count; ++k) {
        mock_op* op = &graph->g.ops[k];
        const int f32 = op->vt == 1;
        void** p = op->p;
        switch (op->kind) {
        case OP_MINRES_LANCZOS:
            if (f32) mock_minres_lanczos_f32(op->n[0], (float*)p[0], (const float*)p[1], (const float*)p[2], (float*)p[3], (const int32_t*)p[4]);
            else mock_minres_lanczos_f64(op->n[0], (double*)p[0], (const double*)p[1], (const double*)p[2], (double*)p[3], (const int32_t*)p[4]);
            break;
        case OP_MINRES_UPDATE:
            if (f32) mock_minres_update_f32(op->n[0], (float*)p[0], (float*)p[1], (float*)p[2], (float*)p[3], (float*)p[4], (float*)p[5], (const float*)p[6], (float*)p[7], (int32_t*)p[8]);
            else mock_minres_update_f64(op->n[0], (double*)p[0], (double*)p[1], (double*)p[2], (double*)p[3], (double*)p[4], (double*)p[5], (const double*)p[6], (double*)p[7], (int32_t*)p[8]);
            break;
        case OP_SPMV_SUB_DOT:
            if (f32 && op->it == 0) mock_spmv_sub_dot_f32_i32(op->n[0], (const int32_t*)p[0], (const int32_t*)p[1], (const float*)p[2], (const float*)p[3], (float*)p[4], (float*)p[5], (const int32_t*)p[6]);
            else if (f32) mock_spmv_sub_dot_f32_i64(op->n[0], (const int64_t*)p[0], (const int64_t*)p[1], (const float*)p[2], (const float*)p[3], (float*)p[4], (float*)p[5], (const int32_t*)p[6]);
            else if (op->it == 0) mock_spmv_sub_dot_f64_i32(op->n[0], (const int32_t*)p[0], (const int32_t*)p[1], (const double*)p[2], (const double*)p[3], (double*)p[4], (double*)p[5], (const int32_t*)p[6]);
            else mock_spmv_sub_dot_f64_i64(op->n[0], (const int64_t*)p[0], (const int64_t*)p[1], (const double*)p[2], (const double*)p[3], (double*)p[4], (double*)p[5], (const int32_t*)p[6]);
            break;
        default: {  /* an operation of mock_base.c */
            b200_graph one;
            one.g.ops = op;
            one.g.count = one.g.cap = 1;
            b200_status st = mock_base_graph_launch(ctx, &one);
            if (st != B200_OK) return st;
            continue;
        }
        }
        ctx->launches++;
    }
    return B200_OK;
}
