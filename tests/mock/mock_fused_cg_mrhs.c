/* TEST INFRASTRUCTURE ONLY.  The host-memory mock of mock_base.c plus sequential restatements of the
 * fused CG entry points for several right-hand sides (ginkgo_b200/csrc/fused_cg_mrhs.cu:
 * b200_cg_mrhs_*, b200_csr_spmv_mdot_*), so that solver::Cg::try_fused_multi_rhs -- capture, replay,
 * polling of the control block, the per-column statuses -- runs on the CPU.  Every column's sums
 * run over the rows in order, as the oracle's compute_dot / compute_norm2 do, so this path and the
 * kernel-by-kernel loop on the mock take the same iterations and give the same bits.  mock_base.c is
 * compiled as part of this file; its b200_graph_launch is kept under another name and replays the
 * operations it knows.  Built by tests/mock_cg_mrhs_build.py. */
#define b200_graph_launch mock_base_graph_launch
#include "mock_base.c"
#undef b200_graph_launch

enum { OP_MRHS_STEP_P = 100, OP_MRHS_STEP_XR, OP_SPMV_MDOT };

#define MOCK_FUSED_MRHS(V, VT, VID, SQRT, FABS)                                                         \
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
                const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];               \
                uint8_t id = 1;                                                                         \
                for (int c = 0; c < 2 && s == 0; ++c) {                                                 \
                    const int is_it = (c == 0) == (iter_first != 0);                                    \
                    if (is_it) {                                                                        \
                        if (max_iters < 0) continue;                                                    \
                        if (iter >= max_iters) s = (uint8_t)((id & 0x3f) | 0x40);                       \
                        ++id;                                                                           \
                    } else {                                                                            \
                        if (!res_kind) continue;                                                        \
                        const VT tau = res_kind == 1 ? SQRT(s_rr) : SQRT(FABS(s_rho));                  \
                        if (tau <= sc[5 * k + j]) s = (uint8_t)(0x80 | (id & 0x3f) | 0x40);             \
                        ++id;                                                                           \
                    }                                                                                   \
                }                                                                                       \
                status[j] = s;                                                                          \
            }                                                                                           \
            if (!(s & 0x3f)) all_stopped = 0;                                                           \
        }                                                                                               \
        ctl[0] = all_stopped;                                                                           \
    }                                                                                                   \
    int64_t b200_cg_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                                  \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        return 3 * k + 64;                                                                              \
    }                                                                                                   \
    b200_status b200_cg_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* z, VT* p,  \
                                      VT* q, const VT* inv_diag, VT* sc, uint8_t* status, int32_t* ctl, \
                                      VT* work, int64_t max_iters, int32_t res_kind,                   \
                                      int32_t iter_first, int32_t baseline, VT reduction_factor)       \
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
            mock_op* op = mock_new_op(ctx, OP_MRHS_STEP_P, VID);                                        \
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
            mock_op* op = mock_new_op(ctx, OP_MRHS_STEP_XR, VID);                                       \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)p; op->p[3] = (void*)q; op->p[4] = z;         \
            op->p[5] = (void*)inv_diag; op->p[6] = sc; op->p[7] = status; op->p[8] = ctl;               \
            op->n[0] = n; op->n[1] = k;                                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_mrhs_step_xr_##V(0, n, k, x, r, p, q, z, inv_diag, sc, status, ctl, 0, 0);                 \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_FUSED_MRHS(f64, double, 0, sqrt, fabs)
MOCK_FUSED_MRHS(f32, float, 1, sqrtf, fabsf)

/* c = A b for k columns (stride k), dots[j] = b_j . c_j over the rows; no-op once every column stopped */
#define MOCK_SPMV_MDOT(V, VT, VID, I, IT, IID)                                                          \
    static void mock_spmv_mdot_##V##_##I(int64_t num_rows, int64_t k, const IT* rp, const IT* ci,       \
                                         const VT* va, const VT* b, VT* c, VT* dots, const int32_t* ctl) \
    {                                                                                                   \
        if (ctl && ctl[0] != 0) return;                                                                 \
        for (int64_t j = 0; j < k; ++j) dots[j] = 0;                                                    \
        for (int64_t r = 0; r < num_rows; ++r)                                                          \
            for (int64_t j = 0; j < k; ++j) {                                                           \
                VT sum = 0;                                                                             \
                for (int64_t e = rp[r]; e < (int64_t)rp[r + 1]; ++e) sum += va[e] * b[ci[e] * k + j];   \
                c[r * k + j] = sum;                                                                     \
                dots[j] += b[r * k + j] * sum;                                                          \
            }                                                                                           \
    }                                                                                                   \
    b200_status b200_csr_spmv_mdot_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,         \
                                             int64_t nnz, const IT* row_ptrs, const IT* col_idxs,       \
                                             const VT* values, const VT* b, int64_t k, VT* c, VT* dots, \
                                             VT* work, const int32_t* ctl)                              \
    {                                                                                                   \
        (void)num_cols; (void)nnz; (void)work;                                                          \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, OP_SPMV_MDOT, VID);                                          \
            op->it = IID;                                                                               \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;           \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = dots; op->p[6] = (void*)ctl;                  \
            op->n[0] = num_rows; op->n[1] = k;                                                          \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_spmv_mdot_##V##_##I(num_rows, k, row_ptrs, col_idxs, values, b, c, dots, ctl);             \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_SPMV_MDOT(f64, double, 0, i32, int32_t, 0)
MOCK_SPMV_MDOT(f64, double, 0, i64, int64_t, 1)
MOCK_SPMV_MDOT(f32, float, 1, i32, int32_t, 0)
MOCK_SPMV_MDOT(f32, float, 1, i64, int64_t, 1)

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    for (int k = 0; k < graph->g.count; ++k) {
        mock_op* op = &graph->g.ops[k];
        const int f32 = op->vt == 1;
        void** a = op->p;
        switch (op->kind) {
        case OP_MRHS_STEP_P:
            if (f32) mock_mrhs_step_p_f32(op->n[0], op->n[1], (float*)a[0], (const float*)a[1], (const float*)a[2], (const uint8_t*)a[3], (const int32_t*)a[4]);
            else mock_mrhs_step_p_f64(op->n[0], op->n[1], (double*)a[0], (const double*)a[1], (const double*)a[2], (const uint8_t*)a[3], (const int32_t*)a[4]);
            break;
        case OP_MRHS_STEP_XR:
            if (f32) mock_mrhs_step_xr_f32(0, op->n[0], op->n[1], (float*)a[0], (float*)a[1], (const float*)a[2], (const float*)a[3], (float*)a[4], (const float*)a[5], (float*)a[6], (uint8_t*)a[7], (int32_t*)a[8], 0, 0);
            else mock_mrhs_step_xr_f64(0, op->n[0], op->n[1], (double*)a[0], (double*)a[1], (const double*)a[2], (const double*)a[3], (double*)a[4], (const double*)a[5], (double*)a[6], (uint8_t*)a[7], (int32_t*)a[8], 0, 0);
            break;
        case OP_SPMV_MDOT:
            if (f32 && op->it == 0) mock_spmv_mdot_f32_i32(op->n[0], op->n[1], (const int32_t*)a[0], (const int32_t*)a[1], (const float*)a[2], (const float*)a[3], (float*)a[4], (float*)a[5], (const int32_t*)a[6]);
            else if (f32) mock_spmv_mdot_f32_i64(op->n[0], op->n[1], (const int64_t*)a[0], (const int64_t*)a[1], (const float*)a[2], (const float*)a[3], (float*)a[4], (float*)a[5], (const int32_t*)a[6]);
            else if (op->it == 0) mock_spmv_mdot_f64_i32(op->n[0], op->n[1], (const int32_t*)a[0], (const int32_t*)a[1], (const double*)a[2], (const double*)a[3], (double*)a[4], (double*)a[5], (const int32_t*)a[6]);
            else mock_spmv_mdot_f64_i64(op->n[0], op->n[1], (const int64_t*)a[0], (const int64_t*)a[1], (const double*)a[2], (const double*)a[3], (double*)a[4], (double*)a[5], (const int32_t*)a[6]);
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
