/* TEST INFRASTRUCTURE ONLY.  The host-memory mock of mock_base.c plus sequential restatements of the
 * fused BiCGStab entry points (ginkgo_b200/csrc/fused_bicgstab.cu, b200_csr_spmv_dot2_*), so that
 * solver::Bicgstab::try_fused -- capture, replay, polling of the control block, the pending-finalize
 * hand-over -- runs on the CPU.  mock_base.c is compiled as part of this file (its context, recorded
 * graphs and finish_scalars are file-local); its b200_graph_launch is kept under another name and
 * replays the operations it knows, one at a time.  Built by tests/mock_bicgstab_build.py. */
#define b200_graph_launch mock_base_graph_launch
#include "mock_base.c"
#undef b200_graph_launch

enum { OP_BICGSTAB_STEP_P = 100, OP_BICGSTAB_STEP_S, OP_BICGSTAB_STEP_XR, OP_SPMV_DOT2 };

/* ---- fused BiCGStab (ginkgo_b200/csrc/fused_bicgstab.cu restated sequentially; sc / ctl layouts of the header) ---- */
#define MOCK_FUSED_BICGSTAB(V, VT, VID, SQRT, FABS)                                                    \
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
        const int32_t iter = ctl[1], max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];       \
        uint8_t status = 0, id = 1;                                                                    \
        for (int k = 0; k < 2 && status == 0; ++k) {                                                   \
            const int is_it = (k == 0) == (iter_first != 0);                                           \
            if (is_it) {                                                                               \
                if (max_iters < 0) continue;                                                           \
                if (iter >= max_iters) status = (uint8_t)((id & 0x3f) | 0x40);                         \
                ++id;                                                                                  \
            } else {                                                                                   \
                if (!res_kind) continue;                                                               \
                const VT tau = res_kind == 1 ? SQRT(ss) : SQRT(FABS(sc[0]));                           \
                if (tau <= sc[5]) status = (uint8_t)(0x80 | (id & 0x3f) | 0x40);                       \
                ++id;                                                                                  \
            }                                                                                          \
        }                                                                                              \
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
            mock_op* op = mock_new_op(ctx, OP_BICGSTAB_STEP_P, VID);                                   \
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
            mock_op* op = mock_new_op(ctx, OP_BICGSTAB_STEP_S, VID);                                   \
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
            mock_op* op = mock_new_op(ctx, OP_BICGSTAB_STEP_XR, VID);                                  \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)s; op->p[3] = (void*)t; op->p[4] = (void*)y; \
            op->p[5] = (void*)z; op->p[6] = (void*)rr; op->p[7] = sc; op->p[8] = ctl; op->n[0] = n;    \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_bicgstab_step_xr_##V(0, n, x, r, s, t, y, z, (VT*)rr, sc, ctl, 0, 0);                     \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_FUSED_BICGSTAB(f64, double, 0, sqrt, fabs)
MOCK_FUSED_BICGSTAB(f32, float, 1, sqrtf, fabsf)

/* c = A b, *dot_out = w . c and (dot2_out) *dot2_out = c . c over the rows; no-op once the solver stopped */
#define MOCK_SPMV_DOT2(V, VT, VID, I, IT, IID)                                                         \
    static void mock_spmv_dot2_##V##_##I(int64_t num_rows, const IT* rp, const IT* ci, const VT* va,   \
                                         const VT* b, VT* c, const VT* w, VT* dot_out, VT* dot2_out,   \
                                         const int32_t* ctl)                                           \
    {                                                                                                  \
        if (ctl && ctl[0] != 0) return;                                                                \
        VT dot = 0, dot2 = 0;                                                                          \
        for (int64_t r = 0; r < num_rows; ++r) {                                                       \
            VT sum = 0;                                                                                \
            for (int64_t k = rp[r]; k < (int64_t)rp[r + 1]; ++k) sum += va[k] * b[ci[k]];              \
            c[r] = sum;                                                                                \
            dot += w[r] * sum;                                                                         \
            dot2 += sum * sum;                                                                         \
        }                                                                                              \
        *dot_out = dot;                                                                                \
        if (dot2_out) *dot2_out = dot2;                                                                \
    }                                                                                                  \
    b200_status b200_csr_spmv_dot2_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan,                 \
                                             int64_t num_rows, int64_t num_cols, int64_t nnz,          \
                                             const IT* row_ptrs, const IT* col_idxs, const VT* values, \
                                             const VT* b, VT* c, const VT* w, VT* dot_out,             \
                                             VT* dot2_out, VT* work, const int32_t* ctl)               \
    {                                                                                                  \
        (void)plan; (void)num_cols; (void)nnz; (void)work;                                             \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, OP_SPMV_DOT2, VID);                                         \
            op->it = IID;                                                                              \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;          \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = (void*)w; op->p[6] = dot_out;                \
            op->p[7] = dot2_out; op->p[8] = (void*)ctl;                                                \
            op->n[0] = num_rows;                                                                       \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_spmv_dot2_##V##_##I(num_rows, row_ptrs, col_idxs, values, b, c, w, dot_out, dot2_out, ctl); \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }
MOCK_SPMV_DOT2(f64, double, 0, i32, int32_t, 0)
MOCK_SPMV_DOT2(f64, double, 0, i64, int64_t, 1)
MOCK_SPMV_DOT2(f32, float, 1, i32, int32_t, 0)
MOCK_SPMV_DOT2(f32, float, 1, i64, int64_t, 1)

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    for (int k = 0; k < graph->g.count; ++k) {
        mock_op* op = &graph->g.ops[k];
        const int f32 = op->vt == 1;
        switch (op->kind) {
        case OP_BICGSTAB_STEP_P:
            if (f32) mock_bicgstab_step_p_f32(op->n[0], (float*)op->p[0], (const float*)op->p[1], (const float*)op->p[2], (float*)op->p[3], (const float*)op->p[4], (const float*)op->p[5], (const int32_t*)op->p[6]);
            else mock_bicgstab_step_p_f64(op->n[0], (double*)op->p[0], (const double*)op->p[1], (const double*)op->p[2], (double*)op->p[3], (const double*)op->p[4], (const double*)op->p[5], (const int32_t*)op->p[6]);
            break;
        case OP_BICGSTAB_STEP_S:
            if (f32) mock_bicgstab_step_s_f32(op->n[0], (const float*)op->p[0], (const float*)op->p[1], (float*)op->p[2], (float*)op->p[3], (const float*)op->p[4], (float*)op->p[5], (int32_t*)op->p[6]);
            else mock_bicgstab_step_s_f64(op->n[0], (const double*)op->p[0], (const double*)op->p[1], (double*)op->p[2], (double*)op->p[3], (const double*)op->p[4], (double*)op->p[5], (int32_t*)op->p[6]);
            break;
        case OP_BICGSTAB_STEP_XR:
            if (f32) mock_bicgstab_step_xr_f32(0, op->n[0], (float*)op->p[0], (float*)op->p[1], (const float*)op->p[2], (const float*)op->p[3], (const float*)op->p[4], (const float*)op->p[5], (float*)op->p[6], (float*)op->p[7], (int32_t*)op->p[8], 0, 0);
            else mock_bicgstab_step_xr_f64(0, op->n[0], (double*)op->p[0], (double*)op->p[1], (const double*)op->p[2], (const double*)op->p[3], (const double*)op->p[4], (const double*)op->p[5], (double*)op->p[6], (double*)op->p[7], (int32_t*)op->p[8], 0, 0);
            break;
        case OP_SPMV_DOT2:
            if (f32 && op->it == 0) mock_spmv_dot2_f32_i32(op->n[0], (const int32_t*)op->p[0], (const int32_t*)op->p[1], (const float*)op->p[2], (const float*)op->p[3], (float*)op->p[4], (const float*)op->p[5], (float*)op->p[6], (float*)op->p[7], (const int32_t*)op->p[8]);
            else if (f32) mock_spmv_dot2_f32_i64(op->n[0], (const int64_t*)op->p[0], (const int64_t*)op->p[1], (const float*)op->p[2], (const float*)op->p[3], (float*)op->p[4], (const float*)op->p[5], (float*)op->p[6], (float*)op->p[7], (const int32_t*)op->p[8]);
            else if (op->it == 0) mock_spmv_dot2_f64_i32(op->n[0], (const int32_t*)op->p[0], (const int32_t*)op->p[1], (const double*)op->p[2], (const double*)op->p[3], (double*)op->p[4], (const double*)op->p[5], (double*)op->p[6], (double*)op->p[7], (const int32_t*)op->p[8]);
            else mock_spmv_dot2_f64_i64(op->n[0], (const int64_t*)op->p[0], (const int64_t*)op->p[1], (const double*)op->p[2], (const double*)op->p[3], (double*)op->p[4], (const double*)op->p[5], (double*)op->p[6], (double*)op->p[7], (const int32_t*)op->p[8]);
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
