/* TEST INFRASTRUCTURE ONLY.  The CSR SpMV with dot products in its epilogue that the fused solver
 * paths share (b200_csr_spmv_dot_*, _dot2_*, _mdot_*, _mdot2_*), restated sequentially: every sum runs
 * over the rows in order, as the oracle's compute_dot / compute_norm2 do, so the fused paths on the
 * mock give the loop's bits.  The one-sum entry points are the two-sum ones with w = b and no second
 * sum; the first sum is the same term by term. */
#include "mock.h"

/* c = A b, *dot_out = w . c and (dot2_out) *dot2_out = c . c over the rows; no-op once the solver stopped */
#define MOCK_SPMV_DOT2(V, VT, I, IT)                                                                   \
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
    static b200_status replay_spmv_dot2_##V##_##I(b200_ctx* ctx, const mock_op* op)                    \
    {                                                                                                  \
        (void)ctx;                                                                                     \
        void* const* p = op->p;                                                                        \
        mock_spmv_dot2_##V##_##I(op->n[0], p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], p[8]);      \
        return B200_OK;                                                                                \
    }                                                                                                  \
    b200_status b200_csr_spmv_dot2_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan,                 \
                                             int64_t num_rows, int64_t num_cols, int64_t nnz,          \
                                             const IT* row_ptrs, const IT* col_idxs, const VT* values, \
                                             const VT* b, VT* c, const VT* w, VT* dot_out,             \
                                             VT* dot2_out, VT* work, const int32_t* ctl)               \
    {                                                                                                  \
        (void)plan; (void)num_cols; (void)nnz; (void)work;                                             \
        if (ctx->capture) {                                                                            \
            mock_op* op = mock_new_op(ctx, replay_spmv_dot2_##V##_##I);                                \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;          \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = (void*)w; op->p[6] = dot_out;                \
            op->p[7] = dot2_out; op->p[8] = (void*)ctl; op->n[0] = num_rows;                           \
            return B200_OK;                                                                            \
        }                                                                                              \
        mock_spmv_dot2_##V##_##I(num_rows, row_ptrs, col_idxs, values, b, c, w, dot_out, dot2_out, ctl); \
        ctx->launches++;                                                                               \
        return B200_OK;                                                                                \
    }                                                                                                  \
    /* c = A b, *dot_out = b . c */                                                                    \
    b200_status b200_csr_spmv_dot_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, \
                                            int64_t num_cols, int64_t nnz, const IT* row_ptrs,         \
                                            const IT* col_idxs, const VT* values, const VT* b, VT* c,  \
                                            VT* dot_out, VT* work, const int32_t* ctl)                 \
    {                                                                                                  \
        return b200_csr_spmv_dot2_##V##_##I(ctx, plan, num_rows, num_cols, nnz, row_ptrs, col_idxs,    \
                                            values, b, c, b, dot_out, NULL, work, ctl);                \
    }
MOCK_SPMV_DOT2(f64, double, i32, int32_t)
MOCK_SPMV_DOT2(f64, double, i64, int64_t)
MOCK_SPMV_DOT2(f32, float, i32, int32_t)
MOCK_SPMV_DOT2(f32, float, i64, int64_t)

/* c = A b for k columns (stride k), dots[j] = w_j . c_j and dots2[j] = c_j . c_j over the rows; no-op
 * once every column stopped */
#define MOCK_SPMV_MDOT2(V, VT, I, IT)                                                                   \
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
    static b200_status replay_spmv_mdot2_##V##_##I(b200_ctx* ctx, const mock_op* op)                    \
    {                                                                                                   \
        (void)ctx;                                                                                      \
        void* const* p = op->p;                                                                         \
        mock_spmv_mdot2_##V##_##I(op->n[0], op->n[1], p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7],   \
                                  p[8]);                                                                \
        return B200_OK;                                                                                 \
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
            mock_op* op = mock_new_op(ctx, replay_spmv_mdot2_##V##_##I);                                \
            op->p[0] = (void*)row_ptrs; op->p[1] = (void*)col_idxs; op->p[2] = (void*)values;           \
            op->p[3] = (void*)b; op->p[4] = c; op->p[5] = (void*)w; op->p[6] = dots; op->p[7] = dots2;  \
            op->p[8] = (void*)ctl; op->n[0] = num_rows; op->n[1] = k;                                   \
            return B200_OK;                                                                             \
        }                                                                                               \
        mock_spmv_mdot2_##V##_##I(num_rows, k, row_ptrs, col_idxs, values, b, c, w, dots, dots2, ctl);  \
        ctx->launches++;                                                                                \
        return B200_OK;                                                                                 \
    }                                                                                                   \
    /* c = A b for k columns, dots[j] = b_j . c_j */                                                    \
    b200_status b200_csr_spmv_mdot_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,         \
                                             int64_t nnz, const IT* row_ptrs, const IT* col_idxs,       \
                                             const VT* values, const VT* b, int64_t k, VT* c, VT* dots, \
                                             VT* work, const int32_t* ctl)                              \
    {                                                                                                   \
        return b200_csr_spmv_mdot2_##V##_##I(ctx, num_rows, num_cols, nnz, row_ptrs, col_idxs, values,  \
                                             b, k, c, b, dots, NULL, work, ctl);                        \
    }
MOCK_SPMV_MDOT2(f64, double, i32, int32_t)
MOCK_SPMV_MDOT2(f64, double, i64, int64_t)
MOCK_SPMV_MDOT2(f32, float, i32, int32_t)
MOCK_SPMV_MDOT2(f32, float, i64, int64_t)
