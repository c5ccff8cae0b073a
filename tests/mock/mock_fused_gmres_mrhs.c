/* TEST INFRASTRUCTURE ONLY.  The host-memory mock of mock_base.c plus sequential restatements of the
 * fused GMRES entry points for several right-hand sides (ginkgo_b200/csrc/fused_gmres_mrhs.cu:
 * b200_gmres_mrhs_*, and b200_csr_spmv_mdot2_*), so that solver::Gmres::try_fused_multi_rhs -- capture,
 * replay of one graph per batch, polling of the control block, the per-column statuses, the host-issued
 * restart on all columns -- runs on the CPU.  Every column's sums run over the rows in order, as the
 * oracle's compute_dot / compute_norm2 / multi_dot do, so this path and the kernel-by-kernel loop on the
 * mock take the same iterations and give the same bits.  The Givens update is the oracle's masked
 * hessenberg_qr.  mock_base.c is compiled as part of this file; its b200_graph_launch is kept under
 * another name and replays the operations it knows.  Built by tests/mock_gmres_mrhs_build.py. */
#define b200_graph_launch mock_base_graph_launch
#include "mock_base.c"
#undef b200_graph_launch

void orc_common_gmres_hessenberg_qr_f64(int64_t, double*, int64_t, double*, int64_t, double*, double*, int64_t,
                                        double*, int64_t, int64_t, uint64_t*, const uint8_t*);
void orc_common_gmres_hessenberg_qr_f32(int64_t, float*, int64_t, float*, int64_t, float*, float*, int64_t,
                                        float*, int64_t, int64_t, uint64_t*, const uint8_t*);

enum { OP_GM_SCALE = 300, OP_GM_MGS, OP_GM_SUB, OP_GM_MDOT, OP_GM_SPMV_MDOT2 };

#define STOPPED(s) ((s) & 0x3f)

/* every argument of one captured operation (lives as long as the graph) */
typedef struct {
    int64_t n, k, i, j, first, nb;
    int32_t divide, it;
    void *w, *v, *z, *d, *krylov, *coef, *haux, *hcol, *gsin, *gcos, *rnorm, *rnc, *fin, *sc, *vp, *vi;
    void *rp, *ci, *va, *b, *dots;
    uint8_t* status;
    int32_t* ctl;
} gm_args;

/* the criteria of fused::criteria_status for one column, without the finalized bit */
static uint8_t mock_gm_criteria(int32_t iter, const int32_t* ctl, int converged)
{
    const int32_t max_iters = ctl[2], res_kind = ctl[3], iter_first = ctl[4];
    uint8_t s = 0, id = 1;
    for (int c = 0; c < 2 && s == 0; ++c) {
        const int is_it = (c == 0) == (iter_first != 0);
        if (is_it) {
            if (max_iters < 0) continue;
            if (iter >= max_iters) s = (uint8_t)(id & 0x3f);
            ++id;
        } else {
            if (!res_kind) continue;
            if (converged) s = (uint8_t)(0x80 | (id & 0x3f));
            ++id;
        }
    }
    return s;
}

static void mock_gm_raise(int64_t k, const uint8_t* status, int32_t* ctl)
{
    int all = 1;
    for (int64_t c = 0; c < k; ++c) all = all && STOPPED(status[c]);
    if (all) ctl[0] = 1;
}

#define MOCK_FUSED_GM(V, VT, VID, SQRT)                                                                  \
    static void mock_gm_run_##V(int kind, const gm_args* a)                                              \
    {                                                                                                    \
        const int64_t n = a->n, k = a->k;                                                                \
        uint8_t* status = a->status;                                                                     \
        int32_t* ctl = a->ctl;                                                                           \
        if (ctl[0] != 0) return;                                                                         \
        if (kind == OP_GM_SCALE) {                                                                       \
            VT *v = (VT*)a->v, *z = (VT*)a->z;                                                           \
            const VT *d = (const VT*)a->d, *sc = (const VT*)a->sc;                                       \
            for (int64_t c = 0; c < k; ++c) {                                                            \
                if (STOPPED(status[c])) continue;                                                        \
                for (int64_t r = 0; r < n; ++r) {                                                        \
                    const int64_t e = r * k + c;                                                         \
                    if (a->divide) v[e] = v[e] / sc[c];                                                  \
                    if (d) z[e] = v[e] * d[r];                                                           \
                }                                                                                        \
            }                                                                                            \
        } else if (kind == OP_GM_MGS) {                                                                  \
            VT *w = (VT*)a->w, *hcol = (VT*)a->hcol;                                                     \
            const VT *vp = (const VT*)a->vp, *vi = (const VT*)a->vi;                                     \
            for (int64_t c = 0; c < k; ++c) {                                                            \
                if (STOPPED(status[c])) continue;                                                        \
                const VT h = hcol[(a->i - 1) * k + c];                                                   \
                VT dot = 0;                                                                              \
                for (int64_t r = 0; r < n; ++r) {                                                        \
                    const int64_t e = r * k + c;                                                         \
                    if (h != 0) w[e] -= h * vp[e];                                                       \
                    dot += vi[e] * w[e];                                                                 \
                }                                                                                        \
                hcol[a->i * k + c] = dot;                                                                \
            }                                                                                            \
        } else if (kind == OP_GM_MDOT) {                                                                 \
            const VT *K = (const VT*)a->krylov, *w = (const VT*)a->w;                                    \
            VT* hcol = (VT*)a->hcol;                                                                     \
            for (int64_t c = 0; c < k; ++c) {                                                            \
                if (STOPPED(status[c])) continue;                                                        \
                for (int64_t i = 0; i < a->nb; ++i) {                                                    \
                    VT dot = 0;                                                                          \
                    for (int64_t r = 0; r < n; ++r) dot += K[(i * n + r) * k + c] * w[r * k + c];        \
                    hcol[i * k + c] = dot;                                                               \
                }                                                                                        \
            }                                                                                            \
        } else { /* OP_GM_SUB: the final pass when hcol != NULL */                                       \
            VT* w = (VT*)a->w;                                                                           \
            const VT *K = (const VT*)a->krylov, *coef = (const VT*)a->coef, *haux = (const VT*)a->haux;  \
            VT *hcol = (VT*)a->hcol, *sc = (VT*)a->sc, *rnorm = (VT*)a->rnorm;                           \
            const int64_t j = a->j;                                                                      \
            VT ss[32];                                                                                   \
            for (int64_t c = 0; c < k; ++c) {                                                            \
                ss[c] = 0;                                                                               \
                if (STOPPED(status[c])) continue;                                                        \
                for (int64_t r = 0; r < n; ++r) {                                                        \
                    const int64_t e = r * k + c;                                                         \
                    for (int64_t i = a->first; i <= j; ++i)                                              \
                        if (coef[i * k + c] != 0) w[e] -= coef[i * k + c] * K[i * n * k + e];            \
                    ss[c] += w[e] * w[e];                                                                \
                }                                                                                        \
            }                                                                                            \
            if (!hcol) return;                                                                           \
            for (int64_t c = 0; c < k; ++c) {                                                            \
                if (STOPPED(status[c])) continue;                                                        \
                if (haux)                                                                                \
                    for (int64_t i = 0; i <= j; ++i) hcol[i * k + c] += haux[i * k + c];                 \
                const VT nrm = SQRT(ss[c]);                                                              \
                hcol[(j + 1) * k + c] = nrm;                                                             \
                sc[c] = nrm;                                                                             \
            }                                                                                            \
            orc_common_gmres_hessenberg_qr_##V(k, (VT*)a->gsin, k, (VT*)a->gcos, k, rnorm, (VT*)a->rnc, k, \
                                               hcol, k, j, (uint64_t*)a->fin, status);                   \
            const int32_t iter = ++ctl[1];                                                               \
            for (int64_t c = 0; c < k; ++c)                                                              \
                if (!STOPPED(status[c])) status[c] = mock_gm_criteria(iter, ctl, rnorm[c] <= sc[2 * k + c]); \
            mock_gm_raise(k, status, ctl);                                                               \
        }                                                                                                \
    }                                                                                                    \
    static b200_status mock_gm_call_##V(b200_ctx* ctx, int kind, const gm_args* a)                       \
    {                                                                                                    \
        if (a->k < 2 || a->k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }  \
        if (ctx->capture) {                                                                              \
            mock_op* op = mock_new_op(ctx, kind, VID);                                                   \
            gm_args* keep = (gm_args*)malloc(sizeof(gm_args));                                           \
            *keep = *a;                                                                                  \
            op->p[0] = keep;                                                                             \
            return B200_OK;                                                                              \
        }                                                                                                \
        mock_gm_run_##V(kind, a);                                                                        \
        ctx->launches++;                                                                                 \
        return B200_OK;                                                                                  \
    }                                                                                                    \
    int64_t b200_gmres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k, int64_t krylov_dim)            \
    {                                                                                                    \
        (void)ctx; (void)k; (void)krylov_dim;                                                            \
        return 1;                                                                                        \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_init_##V(b200_ctx* ctx, int64_t k, const VT* rnorm, VT* sc, uint8_t* status, \
                                         int32_t* ctl, int64_t max_iters, int32_t res_kind, int32_t iter_first, \
                                         int32_t baseline, VT factor)                                    \
    {                                                                                                    \
        if (ctx->capture) { mock_set_error("gmres_mrhs_init inside a capture"); return B200_ERR_INVALID; } \
        ctl[0] = 0; ctl[1] = 0;                                                                          \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                             \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = ctl[6] = ctl[7] = 0;                            \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            if (baseline == 1) sc[k + c] = rnorm[c];                                                     \
            if (baseline == 2) sc[k + c] = 1;                                                            \
            sc[2 * k + c] = factor * sc[k + c];                                                          \
            sc[c] = 0;                                                                                   \
            status[c] = mock_gm_criteria(0, ctl, rnorm[c] <= sc[2 * k + c]);                             \
        }                                                                                                \
        mock_gm_raise(k, status, ctl);                                                                   \
        ctx->launches++;                                                                                 \
        return B200_OK;                                                                                  \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_scale_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v, VT* z,             \
                                          const VT* inv_diag, const VT* sc, const uint8_t* status,       \
                                          const int32_t* ctl, int32_t divide)                            \
    {                                                                                                    \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.v = v; a.z = z; a.d = (void*)inv_diag; a.sc = (void*)sc;                     \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl; a.divide = divide;                           \
        return mock_gm_call_##V(ctx, OP_GM_SCALE, &a);                                                   \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_mgs_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* v_prev, \
                                             const VT* v_i, VT* hcol, int64_t i, const uint8_t* status,  \
                                             const int32_t* ctl, VT* work)                               \
    {                                                                                                    \
        (void)work;                                                                                      \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.w = w; a.vp = (void*)v_prev; a.vi = (void*)v_i; a.hcol = hcol; a.i = i;      \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        return mock_gm_call_##V(ctx, OP_GM_MGS, &a);                                                     \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t k, int64_t num_bases,    \
                                              int64_t krylov_dim, const VT* krylov, const VT* w, VT* hcol, \
                                              const uint8_t* status, const int32_t* ctl, VT* work)       \
    {                                                                                                    \
        (void)work; (void)krylov_dim;                                                                    \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.nb = num_bases; a.krylov = (void*)krylov; a.w = (void*)w; a.hcol = hcol;     \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        return mock_gm_call_##V(ctx, OP_GM_MDOT, &a);                                                    \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_sub_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov, \
                                             const VT* coef, int64_t j, const uint8_t* status,           \
                                             const int32_t* ctl)                                         \
    {                                                                                                    \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.w = w; a.krylov = (void*)krylov; a.coef = (void*)coef; a.j = j;              \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        return mock_gm_call_##V(ctx, OP_GM_SUB, &a);                                                     \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_final_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov, \
                                               int64_t first, const VT* coef, const VT* haux, VT* hcol,  \
                                               int64_t j, VT* gsin, VT* gcos, VT* rnorm, VT* rnc,        \
                                               uint64_t* fin, uint8_t* status, VT* sc, int32_t* ctl,     \
                                               VT* work)                                                 \
    {                                                                                                    \
        (void)work;                                                                                      \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.w = w; a.krylov = (void*)krylov; a.first = first; a.coef = (void*)coef;      \
        a.haux = (void*)haux; a.hcol = hcol; a.j = j; a.gsin = gsin; a.gcos = gcos; a.rnorm = rnorm;     \
        a.rnc = rnc; a.fin = fin; a.status = status; a.sc = sc; a.ctl = ctl;                             \
        return mock_gm_call_##V(ctx, OP_GM_SUB, &a);                                                     \
    }
MOCK_FUSED_GM(f64, double, 0, sqrt)
MOCK_FUSED_GM(f32, float, 1, sqrtf)

/* c = A b for k columns (stride k), dots[j] = w_j . c_j and dots2[j] = c_j . c_j over the rows; no-op
 * once every column stopped */
#define MOCK_GM_SPMV_MDOT2(V, VT, I, IT)                                                                 \
    static void mock_gm_spmv_mdot2_##V##_##I(const gm_args* a)                                           \
    {                                                                                                    \
        const int64_t k = a->k;                                                                          \
        const IT *rp = (const IT*)a->rp, *ci = (const IT*)a->ci;                                         \
        const VT *va = (const VT*)a->va, *b = (const VT*)a->b, *w = (const VT*)a->w;                     \
        VT *c = (VT*)a->z, *dots = (VT*)a->dots, *dots2 = (VT*)a->haux;                                  \
        if (a->ctl && a->ctl[0] != 0) return;                                                            \
        VT d2[32];                                                                                       \
        for (int64_t j = 0; j < k; ++j) dots[j] = d2[j] = 0;                                             \
        for (int64_t r = 0; r < a->n; ++r)                                                               \
            for (int64_t j = 0; j < k; ++j) {                                                            \
                VT sum = 0;                                                                              \
                for (int64_t e = rp[r]; e < (int64_t)rp[r + 1]; ++e) sum += va[e] * b[ci[e] * k + j];    \
                c[r * k + j] = sum;                                                                      \
                dots[j] += w[r * k + j] * sum;                                                           \
                d2[j] += sum * sum;                                                                      \
            }                                                                                            \
        if (dots2)                                                                                       \
            for (int64_t j = 0; j < k; ++j) dots2[j] = d2[j];                                            \
    }                                                                                                    \
    b200_status b200_csr_spmv_mdot2_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,         \
                                              int64_t nnz, const IT* row_ptrs, const IT* col_idxs,       \
                                              const VT* values, const VT* b, int64_t k, VT* c,           \
                                              const VT* w, VT* dots, VT* dots2, VT* work,                \
                                              const int32_t* ctl)                                        \
    {                                                                                                    \
        (void)num_cols; (void)nnz; (void)work;                                                           \
        if (k < 2 || k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }        \
        gm_args a = {0};                                                                                 \
        a.n = num_rows; a.k = k; a.rp = (void*)row_ptrs; a.ci = (void*)col_idxs; a.va = (void*)values;   \
        a.b = (void*)b; a.z = c; a.w = (void*)w; a.dots = dots; a.haux = dots2; a.ctl = (int32_t*)ctl;   \
        a.it = sizeof(IT) == 8;                                                                          \
        if (ctx->capture) {                                                                              \
            mock_op* op = mock_new_op(ctx, OP_GM_SPMV_MDOT2, sizeof(VT) == 4);                           \
            gm_args* keep = (gm_args*)malloc(sizeof(gm_args));                                           \
            *keep = a;                                                                                   \
            op->p[0] = keep;                                                                             \
            return B200_OK;                                                                              \
        }                                                                                                \
        mock_gm_spmv_mdot2_##V##_##I(&a);                                                                \
        ctx->launches++;                                                                                 \
        return B200_OK;                                                                                  \
    }
MOCK_GM_SPMV_MDOT2(f64, double, i32, int32_t)
MOCK_GM_SPMV_MDOT2(f64, double, i64, int64_t)
MOCK_GM_SPMV_MDOT2(f32, float, i32, int32_t)
MOCK_GM_SPMV_MDOT2(f32, float, i64, int64_t)

b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph)
{
    for (int q = 0; q < graph->g.count; ++q) {
        mock_op* op = &graph->g.ops[q];
        if (op->kind >= OP_GM_SCALE && op->kind <= OP_GM_SPMV_MDOT2) {
            const gm_args* a = (const gm_args*)op->p[0];
            const int f32 = op->vt == 1;
            if (op->kind == OP_GM_SPMV_MDOT2) {
                if (f32) { if (a->it) mock_gm_spmv_mdot2_f32_i64(a); else mock_gm_spmv_mdot2_f32_i32(a); }
                else { if (a->it) mock_gm_spmv_mdot2_f64_i64(a); else mock_gm_spmv_mdot2_f64_i32(a); }
            } else if (f32) {
                mock_gm_run_f32(op->kind, a);
            } else {
                mock_gm_run_f64(op->kind, a);
            }
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
