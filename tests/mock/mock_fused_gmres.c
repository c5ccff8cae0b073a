/* TEST INFRASTRUCTURE ONLY.  Sequential restatements of the fused GMRES entry points
 * (ginkgo_b200/csrc/fused_gmres.cu, b200_gmres_fused_multi_dot_*, b200_gmres_fused_block_apply_*), so
 * that solver::Gmres::try_fused -- capture, replay of one graph per batch, polling of the control block,
 * the host-issued restart -- runs on the CPU.  Sums run sequentially from row 0, as the oracle's, so the
 * fused path must give the loop's bits.  The Givens update, the multi-dot and the block-Jacobi apply call
 * what the loop calls (the oracle's hessenberg_qr, the mock's multi_dot and simple_apply).  The SpMV +
 * dots (b200_csr_spmv_dot2_*) are in mock_spmv_dot.c. */
#include "mock.h"

/* the criteria of fused_common.cuh, without the finalized bit; status into ctl[0] and the stop byte */
static void mock_gmres_check(int converged, int32_t* ctl, uint8_t* stop)
{
    const int32_t iter = ++ctl[1];
    const uint8_t status = mock_criteria_status(iter, ctl, converged, 0);
    if (status) {
        ctl[0] = status;
        stop[0] = status;
    }
}

#define MOCK_FUSED_GMRES(V, VT, SQRT)                                                                  \
    static void mock_g_scale_##V(int64_t n, VT* v, VT* z, const VT* d, const VT* sc, const int32_t* ctl, \
                                 int divide)                                                           \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        for (int64_t i = 0; i < n; ++i) {                                                              \
            if (divide) v[i] = v[i] / sc[0];                                                           \
            if (d) z[i] = v[i] * d[i];                                                                 \
        }                                                                                              \
    }                                                                                                  \
    static void mock_g_mgs_##V(int64_t n, VT* w, const VT* vp, const VT* vi, VT* hcol, int64_t i,      \
                               const int32_t* ctl)                                                     \
    {                                                                                                  \
        if (ctl[0] != 0) return;                                                                       \
        const VT h = hcol[i - 1];                                                                      \
        VT dot = 0;                                                                                    \
        for (int64_t r = 0; r < n; ++r) {                                                              \
            if (h != 0) w[r] -= h * vp[r];                                                             \
            dot += vi[r] * w[r];                                                                       \
        }                                                                                              \
        hcol[i] = dot;                                                                                 \
    }                                                                                                  \
    /* the final pass when hcol != NULL (the sub pass otherwise); p: w krylov coef haux hcol gsin gcos \
     * rnorm rnc fin stop sc ctl */                                                                    \
    static void mock_g_sub_##V(int64_t n, int64_t first, int64_t j, void* const* p)                    \
    {                                                                                                  \
        VT *w = (VT*)p[0], *hcol = (VT*)p[4], *sc = (VT*)p[11];                                        \
        const VT *K = (const VT*)p[1], *coef = (const VT*)p[2], *haux = (const VT*)p[3];               \
        int32_t* ctl = (int32_t*)p[12];                                                                \
        if (ctl[0] != 0) return;                                                                       \
        VT ss = 0;                                                                                     \
        for (int64_t r = 0; r < n; ++r) {                                                              \
            for (int64_t i = first; i <= j; ++i)                                                       \
                if (coef[i] != 0) w[r] -= coef[i] * K[i * n + r];                                      \
            ss += w[r] * w[r];                                                                         \
        }                                                                                              \
        if (!hcol) return;                                                                             \
        if (haux)                                                                                      \
            for (int64_t i = 0; i <= j; ++i) hcol[i] += haux[i];                                       \
        const VT nrm = SQRT(ss);                                                                       \
        hcol[j + 1] = nrm;                                                                             \
        sc[0] = nrm;                                                                                   \
        VT* rnorm = (VT*)p[7];                                                                         \
        orc_common_gmres_hessenberg_qr_##V(1, (VT*)p[5], 1, (VT*)p[6], 1, rnorm, (VT*)p[8], 1, hcol, 1, j, \
                                           (uint64_t*)p[9], (const uint8_t*)p[10]);                    \
        mock_gmres_check(rnorm[0] <= sc[2], ctl, (uint8_t*)p[10]);                                     \
    }                                                                                                  \
    static b200_status replay_scale_##V(b200_ctx* ctx, const mock_op* op)                              \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_g_scale_##V(op->n[0], p[0], p[1], p[2], p[3], p[4], op->i[0]);                            \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_mgs_##V(b200_ctx* ctx, const mock_op* op)                                \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_g_mgs_##V(op->n[0], p[0], p[1], p[2], p[3], op->n[1], p[4]);                              \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status replay_sub_##V(b200_ctx* ctx, const mock_op* op)                                \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        mock_g_sub_##V(op->n[0], op->n[1], op->n[2], op->p);                                           \
        return B200_OK;                                                                                \
    }                                                                                                  \
    int64_t b200_gmres_fused_work_size_##V(const b200_ctx* ctx, int64_t krylov_dim)                    \
    {                                                                                                  \
        (void)ctx; (void)krylov_dim;                                                                   \
        return 1;                                                                                      \
    }                                                                                                  \
    b200_status b200_gmres_fused_init_##V(b200_ctx* ctx, const VT* rnorm, VT* sc, int32_t* ctl,        \
                                          uint8_t* stop, int64_t max_iters, int32_t res_kind,          \
                                          int32_t iter_first, int32_t baseline, VT factor)             \
    {                                                                                                  \
        if (ctx->capture) { mock_set_error("fused_init inside a capture"); return B200_ERR_INVALID; }  \
        if (baseline == 1) sc[1] = rnorm[0];                                                           \
        if (baseline == 2) sc[1] = 1;                                                                  \
        sc[2] = factor * sc[1];                                                                        \
        sc[0] = 0;                                                                                     \
        ctl[0] = 0; ctl[1] = -1;                                                                       \
        ctl[2] = (int32_t)(max_iters > 0x7fffffff ? 0x7fffffff : max_iters);                           \
        ctl[3] = res_kind; ctl[4] = iter_first; ctl[5] = ctl[6] = ctl[7] = 0;                          \
        stop[0] = 0;                                                                                   \
        mock_gmres_check(rnorm[0] <= sc[2], ctl, stop);                                                \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_gmres_fused_scale_##V(b200_ctx* ctx, int64_t n, VT* v, VT* z, const VT* inv_diag, \
                                           const VT* sc, const int32_t* ctl, int32_t divide)           \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_scale_##V);                                          \
            op->p[0] = v; op->p[1] = z; op->p[2] = (void*)inv_diag; op->p[3] = (void*)sc;              \
            op->p[4] = (void*)ctl; op->n[0] = n; op->i[0] = divide;                                    \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_g_scale_##V(n, v, z, inv_diag, sc, ctl, divide);                                          \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_gmres_fused_mgs_pass_##V(b200_ctx* ctx, int64_t n, VT* w, const VT* v_prev,       \
                                              const VT* v_i, VT* hcol, int64_t i, const int32_t* ctl,  \
                                              VT* work)                                                \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_mgs_##V);                                            \
            op->p[0] = w; op->p[1] = (void*)v_prev; op->p[2] = (void*)v_i; op->p[3] = hcol;            \
            op->p[4] = (void*)ctl; op->n[0] = n; op->n[1] = i;                                         \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_g_mgs_##V(n, w, v_prev, v_i, hcol, i, ctl);                                               \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    static b200_status mock_g_sub_call_##V(b200_ctx* ctx, int64_t n, int64_t first, int64_t j,         \
                                           void* const* ptrs)                                          \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_sub_##V);                                            \
            memcpy(op->p, ptrs, 13 * sizeof(void*));                                                   \
            op->n[0] = n; op->n[1] = first; op->n[2] = j;                                              \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_g_sub_##V(n, first, j, ptrs);                                                             \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_gmres_fused_sub_pass_##V(b200_ctx* ctx, int64_t n, VT* w, const VT* krylov,       \
                                              const VT* coef, int64_t j, const int32_t* ctl)           \
    {                                                                                                  \
        void* p[13] = {w, (void*)krylov, (void*)coef, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL,  \
                       NULL, (void*)ctl};                                                              \
        return mock_g_sub_call_##V(ctx, n, 0, j, p);                                                   \
    }                                                                                                  \
    b200_status b200_gmres_fused_final_pass_##V(                                                       \
        b200_ctx* ctx, int64_t n, VT* w, const VT* krylov, int64_t first, const VT* coef,              \
        const VT* haux, VT* hcol, int64_t j, VT* gsin, VT* gcos, VT* rnorm, VT* rnc, uint64_t* fin,    \
        uint8_t* stop, VT* sc, int32_t* ctl, VT* work)                                                 \
    {                                                                                                  \
        (void)work;                                                                                    \
        void* p[13] = {w, (void*)krylov, (void*)coef, (void*)haux, hcol, gsin, gcos, rnorm, rnc, fin,  \
                       stop, sc, ctl};                                                                 \
        return mock_g_sub_call_##V(ctx, n, first, j, p);                                               \
    }                                                                                                  \
    static b200_status replay_multi_dot_##V(b200_ctx* ctx, const mock_op* op);                         \
    b200_status b200_gmres_fused_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t num_bases,            \
                                               const VT* krylov, const VT* w, VT* hcol,                \
                                               const int32_t* ctl, VT* work)                           \
    {                                                                                                  \
        (void)work;                                                                                    \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_multi_dot_##V);                                      \
            op->p[0] = (void*)krylov; op->p[1] = (void*)w; op->p[2] = hcol; op->p[3] = (void*)ctl;     \
            op->n[0] = n; op->n[1] = num_bases;                                                        \
            return B200_OK;                                                                            \
        }                                                                                              \
        if (ctl[0] != 0) return B200_OK;                                                               \
        return b200_gmres_multi_dot_##V(ctx, n, 1, num_bases, krylov, 1, w, 1, hcol, 1);               \
    }                                                                                                  \
    static b200_status replay_multi_dot_##V(b200_ctx* ctx, const mock_op* op)                          \
    {                                                                                                  \
        void* const* p = op->p;                                                                        \
        return b200_gmres_fused_multi_dot_##V(ctx, op->n[0], op->n[1], p[0], p[1], p[2], p[3], NULL);  \
    }
MOCK_FUSED_GMRES(f64, double, sqrt)
MOCK_FUSED_GMRES(f32, float, sqrtf)

/* the ctl-aware block-Jacobi apply: the mock's simple_apply (plain or adaptive) unless stopped */
#define MOCK_FUSED_GMRES_BLOCK(V, VT, I, IT)                                                           \
    static b200_status replay_block_apply_##V##_##I(b200_ctx* ctx, const mock_op* op);                 \
    b200_status b200_gmres_fused_block_apply_##V##_##I(                                                \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,               \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,                    \
        const IT* block_pointers, const VT* blocks, const VT* b, VT* x, const int32_t* ctl)            \
    {                                                                                                  \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_block_apply_##V##_##I);                              \
            op->p[0] = (void*)block_precisions; op->p[1] = (void*)block_pointers;                      \
            op->p[2] = (void*)blocks; op->p[3] = (void*)b; op->p[4] = x; op->p[5] = (void*)ctl;        \
            op->n[0] = num_blocks; op->n[1] = block_offset; op->n[2] = group_offset;                   \
            op->i[0] = max_block_size; op->i[1] = group_power;                                         \
            return B200_OK;                                                                            \
        }                                                                                              \
        if (ctl[0] != 0) return B200_OK;                                                               \
        if (block_precisions)                                                                          \
            return b200_jacobi_simple_apply_adaptive_##V##_##I(ctx, num_blocks, max_block_size,        \
                                                               block_offset, group_offset,             \
                                                               group_power, block_precisions,          \
                                                               block_pointers, blocks, b, 1, 1, x, 1); \
        return b200_jacobi_simple_apply_##V##_##I(ctx, num_blocks, max_block_size, block_offset,       \
                                                  group_offset, group_power, block_pointers, blocks,   \
                                                  b, 1, 1, x, 1);                                      \
    }                                                                                                  \
    static b200_status replay_block_apply_##V##_##I(b200_ctx* ctx, const mock_op* op)                  \
    {                                                                                                  \
        void* const* p = op->p;                                                                        \
        return b200_gmres_fused_block_apply_##V##_##I(ctx, op->n[0], op->i[0], op->n[1], op->n[2],     \
                                                      op->i[1], p[0], p[1], p[2], p[3], p[4], p[5]);   \
    }
MOCK_FUSED_GMRES_BLOCK(f64, double, i32, int32_t)
MOCK_FUSED_GMRES_BLOCK(f64, double, i64, int64_t)
MOCK_FUSED_GMRES_BLOCK(f32, float, i32, int32_t)
MOCK_FUSED_GMRES_BLOCK(f32, float, i64, int64_t)
