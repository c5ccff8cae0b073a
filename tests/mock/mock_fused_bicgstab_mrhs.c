/* TEST INFRASTRUCTURE ONLY.  The host-memory mock of mock_base.c plus sequential restatements of the
 * fused BiCGStab entry points for several right-hand sides (ginkgo_b200/csrc/fused_bicgstab_mrhs.cu:
 * b200_bicgstab_mrhs_*, b200_csr_spmv_mdot2_*), so that solver::Bicgstab::try_fused_multi_rhs --
 * capture, replay, polling of the control block, the per-column statuses, the finalize owed after a
 * mid-iteration stop -- runs on the CPU.  Every column's sums run over the rows in order, as the
 * oracle's compute_dot / compute_norm2 do, so this path and the kernel-by-kernel loop on the mock take
 * the same iterations and give the same bits.  mock_base.c is compiled as part of this file; its
 * b200_graph_launch is kept under another name and replays the operations it knows.  Built by
 * tests/mock_bicgstab_mrhs_build.py. */
#define b200_graph_launch mock_base_graph_launch
#include "mock_base.c"
#undef b200_graph_launch

enum { OP_BM_STEP_P = 110, OP_BM_STEP_S, OP_BM_STEP_XR, OP_SPMV_MDOT2 };

#define STOPPED(s) ((s) & 0x3f)

/* the criteria of fused::criteria_status for one column */
#define MOCK_CRITERIA(VT, SQRT, FABS)                                                                   \
    static uint8_t mock_bm_criteria_##VT(int32_t iter, const int32_t* ctl, VT ss, VT rho, VT threshold, \
                                         uint8_t finalized)                                             \
    {                                                                                                   \
        const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];                       \
        uint8_t s = 0, id = 1;                                                                          \
        for (int c = 0; c < 2 && s == 0; ++c) {                                                         \
            const int is_it = (c == 0) == (iter_first != 0);                                            \
            if (is_it) {                                                                                \
                if (max_iters < 0) continue;                                                            \
                if (iter >= max_iters) s = (uint8_t)((id & 0x3f) | finalized);                          \
                ++id;                                                                                   \
            } else {                                                                                    \
                if (!res_kind) continue;                                                                \
                const VT tau = res_kind == 1 ? SQRT(ss) : SQRT(FABS(rho));                              \
                if (tau <= threshold) s = (uint8_t)(0x80 | (id & 0x3f) | finalized);                    \
                ++id;                                                                                   \
            }                                                                                           \
        }                                                                                               \
        return s;                                                                                       \
    }
MOCK_CRITERIA(double, sqrt, fabs)
MOCK_CRITERIA(float, sqrtf, fabsf)

#define MOCK_FUSED_BM(V, VT, VID)                                                                       \
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
                st = mock_bm_criteria_##VT(ctl[1], ctl, ss, sc[j], sc[5 * k + j], 0);                   \
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
                status[j] = st = mock_bm_criteria_##VT(iter, ctl, rn, rho, sc[5 * k + j], 0x40);        \
            }                                                                                           \
            if (!STOPPED(st)) all_stopped = 0;                                                          \
        }                                                                                               \
        ctl[5] = 0;                                                                                     \
        ctl[0] = all_stopped;                                                                           \
    }                                                                                                   \
    int64_t b200_bicgstab_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k)                            \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        return 4 * k + 64;                                                                              \
    }                                                                                                   \
    b200_status b200_bicgstab_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* rr,   \
                                            VT* p, VT* v, VT* y, VT* s, VT* t, VT* z, VT* sc,           \
                                            uint8_t* status, int32_t* ctl, VT* work, int64_t max_iters,  \
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
        for (int a = 0; a < 6; ++a) memset(zeroed[a], 0, sizeof(VT) * (size_t)(n * k));                \
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
            mock_op* op = mock_new_op(ctx, OP_BM_STEP_P, VID);                                          \
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
            mock_op* op = mock_new_op(ctx, OP_BM_STEP_S, VID);                                          \
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
            mock_op* op = mock_new_op(ctx, OP_BM_STEP_XR, VID);                                         \
            op->p[0] = x; op->p[1] = r; op->p[2] = (void*)s; op->p[3] = (void*)t; op->p[4] = (void*)y;  \
            op->p[5] = (void*)z; op->p[6] = (void*)rr; op->p[7] = sc; op->p[8] = status;                \
            op->p[9] = ctl; op->n[0] = n; op->n[1] = k;                                                 \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_bm_step_xr_##V(0, n, k, x, r, s, t, y, z, (VT*)rr, sc, status, ctl, 0, 0);                 \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_FUSED_BM(f64, double, 0)
MOCK_FUSED_BM(f32, float, 1)

/* c = A b for k columns (stride k), dots[j] = w_j . c_j and dots2[j] = c_j . c_j over the rows; no-op
 * once every column stopped */
#define MOCK_SPMV_MDOT2(V, VT, VID, I, IT, IID)                                                         \
    static void mock_spmv_mdot2_##V##_##I(int64_t num_rows, int64_t k, const IT* rp, const IT* ci,      \
                                          const VT* va, const VT* b, VT* c, const VT* w, VT* dots,      \
                                          VT* dots2, const int32_t* ctl)                                \
    {                                                                                                   \
        if (ctl && ctl[0] != 0) return;                                                                 \
        VT d2[32];                                                                                      \
        for (int64_t j = 0; j < k; ++j) dots[j] = d2[j] = 0;                                            \
        for (int64_t r = 0; r < num_rows; ++r)                                                          \
            for (int64_t j = 0; j < k; ++j) {                                                           \
                VT sum = 0;                                                                             \
                for (int64_t e = rp[r]; e < (int64_t)rp[r + 1]; ++e) sum += va[e] * b[ci[e] * k + j];   \
                c[r * k + j] = sum;                                                                     \
                dots[j] += w[r * k + j] * sum;                                                          \
                d2[j] += sum * sum;                                                                     \
            }                                                                                           \
        if (dots2)                                                                                      \
            for (int64_t j = 0; j < k; ++j) dots2[j] = d2[j];                                           \
    }                                                                                                   \
    b200_status b200_csr_spmv_mdot2_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,        \
                                              int64_t nnz, const IT* row_ptrs, const IT* col_idxs,      \
                                              const VT* values, const VT* b, int64_t k, VT* c,          \
                                              const VT* w, VT* dots, VT* dots2, VT* work,               \
                                              const int32_t* ctl)                                       \
    {                                                                                                   \
        (void)num_cols; (void)nnz; (void)work;                                                          \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }       \
        if (ctx->capture) {                                                                             \
            mock_op* op = mock_new_op(ctx, OP_SPMV_MDOT2, VID);                                         \
            op->it = IID;                                                                               \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;           \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = (void*)w; op->p[6] = dots; op->p[7] = dots2;  \
            op->p[8] = (void*)ctl; op->n[0] = num_rows; op->n[1] = k;                                   \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_spmv_mdot2_##V##_##I(num_rows, k, row_ptrs, col_idxs, values, b, c, w, dots, dots2, ctl);  \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }
MOCK_SPMV_MDOT2(f64, double, 0, i32, int32_t, 0)
MOCK_SPMV_MDOT2(f64, double, 0, i64, int64_t, 1)
MOCK_SPMV_MDOT2(f32, float, 1, i32, int32_t, 0)
MOCK_SPMV_MDOT2(f32, float, 1, i64, int64_t, 1)

#define REPLAY_BM(V, VT)                                                                                          \
    static void replay_bm_##V(mock_op* op)                                                                        \
    {                                                                                                             \
        void** a = op->p;                                                                                         \
        const int64_t n = op->n[0], k = op->n[1];                                                                 \
        switch (op->kind) {                                                                                       \
        case OP_BM_STEP_P:                                                                                        \
            mock_bm_step_p_##V(n, k, (VT*)a[0], (const VT*)a[1], (const VT*)a[2], (VT*)a[3], (const VT*)a[4],     \
                               (const VT*)a[5], (const uint8_t*)a[6], (const int32_t*)a[7]);                      \
            break;                                                                                                \
        case OP_BM_STEP_S:                                                                                        \
            mock_bm_step_s_##V(n, k, (const VT*)a[0], (const VT*)a[1], (VT*)a[2], (VT*)a[3], (const VT*)a[4],     \
                               (VT*)a[5], (uint8_t*)a[6], (int32_t*)a[7]);                                        \
            break;                                                                                                \
        case OP_BM_STEP_XR:                                                                                       \
            mock_bm_step_xr_##V(0, n, k, (VT*)a[0], (VT*)a[1], (const VT*)a[2], (const VT*)a[3], (const VT*)a[4], \
                                (const VT*)a[5], (VT*)a[6], (VT*)a[7], (uint8_t*)a[8], (int32_t*)a[9], 0, 0);     \
            break;                                                                                                \
        default:                                                                                                  \
            if (op->it == 0)                                                                                      \
                mock_spmv_mdot2_##V##_i32(n, k, (const int32_t*)a[0], (const int32_t*)a[1], (const VT*)a[2],      \
                                          (const VT*)a[3], (VT*)a[4], (const VT*)a[5], (VT*)a[6], (VT*)a[7],      \
                                          (const int32_t*)a[8]);                                                  \
            else                                                                                                  \
                mock_spmv_mdot2_##V##_i64(n, k, (const int64_t*)a[0], (const int64_t*)a[1], (const VT*)a[2],      \
                                          (const VT*)a[3], (VT*)a[4], (const VT*)a[5], (VT*)a[6], (VT*)a[7],      \
                                          (const int32_t*)a[8]);                                                  \
        }                                                                                                         \
    }
REPLAY_BM(f64, double)
REPLAY_BM(f32, float)

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    for (int k = 0; k < graph->g.count; ++k) {
        mock_op* op = &graph->g.ops[k];
        if (op->kind >= OP_BM_STEP_P && op->kind <= OP_SPMV_MDOT2) {
            if (op->vt == 1) replay_bm_f32(op);
            else replay_bm_f64(op);
            ctx->launches++;
            continue;
        }
        /* an operation of mock_base.c */
        b200_graph one;
        one.g.ops = op;
        one.g.count = one.g.cap = 1;
        b200_status st = mock_base_graph_launch(ctx, &one);
        if (st != B200_OK) return st;
    }
    return B200_OK;
}
