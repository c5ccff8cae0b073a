/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused GMRES entry points for several
 * right-hand sides (ginkgo_b200/csrc/fused_gmres_mrhs.cu: b200_gmres_mrhs_*), so that
 * solver::Gmres::try_fused_multi_rhs -- capture, replay of one graph per batch, polling of the control
 * block, the per-column statuses, the host-issued restart on all columns -- runs on the CPU.  Every
 * column's sums run over the rows in order, as the oracle's compute_dot / compute_norm2 / multi_dot do,
 * so this path and the kernel-by-kernel loop on the mock take the same iterations and give the same
 * bits.  The Givens update is the oracle's masked hessenberg_qr.  The SpMV + dots
 * (b200_csr_spmv_mdot2_*) are in mock_spmv_dot.c. */
#include "mock.h"

/* every argument of one call and the restatement that runs it (a captured copy lives as long as the
 * graph) */
typedef struct gm_args gm_args;
struct gm_args {
    void (*run)(const gm_args* a);
    int64_t n, k, i, j, first, nb;
    int32_t divide;
    void *w, *v, *z, *d, *krylov, *coef, *haux, *hcol, *gsin, *gcos, *rnorm, *rnc, *fin, *sc, *vp, *vi;
    uint8_t* status;
    int32_t* ctl;
};

static void mock_gm_raise(int64_t k, const uint8_t* status, int32_t* ctl)
{
    int all = 1;
    for (int64_t c = 0; c < k; ++c) all = all && STOPPED(status[c]);
    if (all) ctl[0] = 1;
}

static b200_status replay_gm(b200_ctx* ctx, const mock_op* op)
{
    (void)ctx;
    const gm_args* a = op->keep;
    a->run(a);
    return B200_OK;
}

static b200_status mock_gm_call(b200_ctx* ctx, const gm_args* a)
{
    if (a->k < 2 || a->k > 32) { mock_set_error("k must be in [2, 32]"); return B200_ERR_INVALID; }
    if (ctx->capture) {
        mock_op* op = mock_new_op(ctx, replay_gm);
        gm_args* keep = (gm_args*)malloc(sizeof(gm_args));
        *keep = *a;
        op->keep = keep;
        return B200_OK;
    }
    a->run(a);
    ctx->launches++;
    return B200_OK;
}

#define MOCK_FUSED_GM(V, VT, SQRT)                                                                       \
    static void mock_gm_scale_##V(const gm_args* a)                                                      \
    {                                                                                                    \
        const int64_t n = a->n, k = a->k;                                                                \
        const uint8_t* status = a->status;                                                               \
        if (a->ctl[0] != 0) return;                                                                      \
        VT *v = (VT*)a->v, *z = (VT*)a->z;                                                               \
        const VT *d = (const VT*)a->d, *sc = (const VT*)a->sc;                                           \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            if (STOPPED(status[c])) continue;                                                            \
            for (int64_t r = 0; r < n; ++r) {                                                            \
                const int64_t e = r * k + c;                                                             \
                if (a->divide) v[e] = v[e] / sc[c];                                                      \
                if (d) z[e] = v[e] * d[r];                                                               \
            }                                                                                            \
        }                                                                                                \
    }                                                                                                    \
    static void mock_gm_mgs_##V(const gm_args* a)                                                        \
    {                                                                                                    \
        const int64_t n = a->n, k = a->k;                                                                \
        const uint8_t* status = a->status;                                                               \
        if (a->ctl[0] != 0) return;                                                                      \
        VT *w = (VT*)a->w, *hcol = (VT*)a->hcol;                                                         \
        const VT *vp = (const VT*)a->vp, *vi = (const VT*)a->vi;                                         \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            if (STOPPED(status[c])) continue;                                                            \
            const VT h = hcol[(a->i - 1) * k + c];                                                       \
            VT dot = 0;                                                                                  \
            for (int64_t r = 0; r < n; ++r) {                                                            \
                const int64_t e = r * k + c;                                                             \
                if (h != 0) w[e] -= h * vp[e];                                                           \
                dot += vi[e] * w[e];                                                                     \
            }                                                                                            \
            hcol[a->i * k + c] = dot;                                                                    \
        }                                                                                                \
    }                                                                                                    \
    static void mock_gm_mdot_##V(const gm_args* a)                                                       \
    {                                                                                                    \
        const int64_t n = a->n, k = a->k;                                                                \
        const uint8_t* status = a->status;                                                               \
        if (a->ctl[0] != 0) return;                                                                      \
        const VT *K = (const VT*)a->krylov, *w = (const VT*)a->w;                                        \
        VT* hcol = (VT*)a->hcol;                                                                         \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            if (STOPPED(status[c])) continue;                                                            \
            for (int64_t i = 0; i < a->nb; ++i) {                                                        \
                VT dot = 0;                                                                              \
                for (int64_t r = 0; r < n; ++r) dot += K[(i * n + r) * k + c] * w[r * k + c];            \
                hcol[i * k + c] = dot;                                                                   \
            }                                                                                            \
        }                                                                                                \
    }                                                                                                    \
    /* the sub pass; the final pass when hcol != NULL */                                                 \
    static void mock_gm_sub_##V(const gm_args* a)                                                        \
    {                                                                                                    \
        const int64_t n = a->n, k = a->k;                                                                \
        uint8_t* status = a->status;                                                                     \
        int32_t* ctl = a->ctl;                                                                           \
        if (ctl[0] != 0) return;                                                                         \
        VT* w = (VT*)a->w;                                                                               \
        const VT *K = (const VT*)a->krylov, *coef = (const VT*)a->coef, *haux = (const VT*)a->haux;      \
        VT *hcol = (VT*)a->hcol, *sc = (VT*)a->sc, *rnorm = (VT*)a->rnorm;                               \
        const int64_t j = a->j;                                                                          \
        VT ss[32];                                                                                       \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            ss[c] = 0;                                                                                   \
            if (STOPPED(status[c])) continue;                                                            \
            for (int64_t r = 0; r < n; ++r) {                                                            \
                const int64_t e = r * k + c;                                                             \
                for (int64_t i = a->first; i <= j; ++i)                                                  \
                    if (coef[i * k + c] != 0) w[e] -= coef[i * k + c] * K[i * n * k + e];                \
                ss[c] += w[e] * w[e];                                                                    \
            }                                                                                            \
        }                                                                                                \
        if (!hcol) return;                                                                               \
        for (int64_t c = 0; c < k; ++c) {                                                                \
            if (STOPPED(status[c])) continue;                                                            \
            if (haux)                                                                                    \
                for (int64_t i = 0; i <= j; ++i) hcol[i * k + c] += haux[i * k + c];                     \
            const VT nrm = SQRT(ss[c]);                                                                  \
            hcol[(j + 1) * k + c] = nrm;                                                                 \
            sc[c] = nrm;                                                                                 \
        }                                                                                                \
        orc_common_gmres_hessenberg_qr_##V(k, (VT*)a->gsin, k, (VT*)a->gcos, k, rnorm, (VT*)a->rnc, k,   \
                                           hcol, k, j, (uint64_t*)a->fin, status);                       \
        const int32_t iter = ++ctl[1];                                                                   \
        for (int64_t c = 0; c < k; ++c)                                                                  \
            if (!STOPPED(status[c]))                                                                     \
                status[c] = mock_criteria_status(iter, ctl, rnorm[c] <= sc[2 * k + c], 0);               \
        mock_gm_raise(k, status, ctl);                                                                   \
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
            status[c] = mock_criteria_status(0, ctl, rnorm[c] <= sc[2 * k + c], 0);                      \
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
        a.run = mock_gm_scale_##V;                                                                       \
        return mock_gm_call(ctx, &a);                                                                    \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_mgs_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* v_prev, \
                                             const VT* v_i, VT* hcol, int64_t i, const uint8_t* status,  \
                                             const int32_t* ctl, VT* work)                               \
    {                                                                                                    \
        (void)work;                                                                                      \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.w = w; a.vp = (void*)v_prev; a.vi = (void*)v_i; a.hcol = hcol; a.i = i;      \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        a.run = mock_gm_mgs_##V;                                                                         \
        return mock_gm_call(ctx, &a);                                                                    \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t k, int64_t num_bases,    \
                                              int64_t krylov_dim, const VT* krylov, const VT* w, VT* hcol, \
                                              const uint8_t* status, const int32_t* ctl, VT* work)       \
    {                                                                                                    \
        (void)work; (void)krylov_dim;                                                                    \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.nb = num_bases; a.krylov = (void*)krylov; a.w = (void*)w; a.hcol = hcol;     \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        a.run = mock_gm_mdot_##V;                                                                        \
        return mock_gm_call(ctx, &a);                                                                    \
    }                                                                                                    \
    b200_status b200_gmres_mrhs_sub_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov, \
                                             const VT* coef, int64_t j, const uint8_t* status,           \
                                             const int32_t* ctl)                                         \
    {                                                                                                    \
        gm_args a = {0};                                                                                 \
        a.n = n; a.k = k; a.w = w; a.krylov = (void*)krylov; a.coef = (void*)coef; a.j = j;              \
        a.status = (uint8_t*)status; a.ctl = (int32_t*)ctl;                                              \
        a.run = mock_gm_sub_##V;                                                                         \
        return mock_gm_call(ctx, &a);                                                                    \
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
        a.run = mock_gm_sub_##V;                                                                         \
        return mock_gm_call(ctx, &a);                                                                    \
    }
MOCK_FUSED_GM(f64, double, sqrt)
MOCK_FUSED_GM(f32, float, sqrtf)
