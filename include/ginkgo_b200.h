/*
 * ginkgo_b200.h -- the C ABI of the hand-written CUDA (sm_90a) SpMV + Krylov hot path.
 *
 * This is the drop-in boundary: every entry point below is what a
 * `gko::kernels::cuda::<ns>::<kernel>` wrapper (the reference's link-time
 * backend plug-in, SURVEY.md section 8b) would call after unpacking the
 * Ginkgo objects (matrix::Csr / Dense / array<>) into raw device pointers,
 * sizes and strides.  INTEGRATION.md shows that wrapper for each namespace.
 *
 * Conventions (all entry points):
 *   - `extern "C"`, POD arguments only; every data pointer is a DEVICE pointer
 *     owned by the caller (the Ginkgo object) and must stay valid until the
 *     stream reaches the call.  Scalars alpha/beta/rho/... are 1x1 or 1xncols
 *     Dense matrices IN DEVICE MEMORY, as in the reference.
 *   - Dense operands are row-major with an explicit row stride (elements),
 *     exactly `matrix::Dense::get_const_values()/get_stride()`
 *     (reference include/ginkgo/core/matrix/dense.hpp:861-912).
 *   - Every kernel is enqueued on the context's stream and returns without
 *     synchronising, except the calls documented as blocking (host copies and
 *     the two stopping-criterion checks that must hand a host `bool` back,
 *     reference core/stop/residual_norm.cpp:197-204).
 *   - Return value: B200_OK or an error code; no C++ exception crosses.
 *   - There is no CPU fallback: without a usable sm_90 (H100) device
 *     b200_ctx_create fails and nothing else can be called.
 *
 * Type suffixes: f32/f64 = value type (float/double), i32/i64 = index type.
 * `size_type` arrays of the reference (SELL-P slice_sets/slice_lengths, GMRES
 * final_iter_nums) are uint64_t here; `stopping_status` is one uint8_t per
 * right-hand side (bit7 converged, bit6 finalized, bits0-5 stopping id;
 * reference include/ginkgo/core/stop/stopping_status.hpp).
 */
#ifndef GINKGO_B200_H_
#define GINKGO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t b200_status;
enum {
    B200_OK = 0,
    B200_ERR_CUDA = 1,        /* a CUDA runtime call failed (-> gko::CudaError) */
    B200_ERR_INVALID = 2,     /* bad argument (-> gko::DimensionMismatch / BadDimension) */
    B200_ERR_UNSUPPORTED = 3, /* not implemented on this path (-> gko::NotSupported) */
    B200_ERR_ALLOC = 4,       /* device allocation failed (-> gko::AllocationError) */
    B200_ERR_COMM = 5         /* NCCL failure on the multi-GPU path */
};

typedef struct b200_ctx b200_ctx;           /* one per (device, stream): the CudaExecutor analogue */
typedef struct b200_csr_plan b200_csr_plan; /* cached row partition, the `srow` analogue */
typedef struct b200_coo_plan b200_coo_plan; /* cached row_idxs -> row_ptrs + row partition */

/* last error text of the calling thread ("" if none) */
const char* b200_last_error(void);
/* library version / build info string (contains "sm_90a") */
const char* b200_version(void);

/* ---------------------------------------------------------------------------
 * Executor glue: replaces CudaExecutor::{create, raw_alloc, raw_free,
 * raw_copy_to, synchronize, get_num_multiprocessor,...}
 * (reference cuda/base/executor.cpp; stubs core/device_hooks/cuda_hooks.cpp:19-250)
 * ------------------------------------------------------------------------- */
/* stream == NULL: the context creates and owns a non-blocking stream (the
 * legacy default stream is never used). */
b200_status b200_ctx_create(int32_t device_id, void* cuda_stream, b200_ctx** out);
void b200_ctx_destroy(b200_ctx* ctx);
void* b200_ctx_stream(const b200_ctx* ctx);
int32_t b200_ctx_device(const b200_ctx* ctx);
int32_t b200_ctx_num_sms(const b200_ctx* ctx);
int64_t b200_ctx_launch_count(const b200_ctx* ctx); /* kernels launched so far by this ctx */
/* stream-ordered on the context's stream (cudaMallocAsync / cudaFreeAsync, the reference's
 * CudaAsyncAllocator): memory may be used by work enqueued on that stream after the call;
 * free never synchronises and never fails loudly (cuda_hooks.cpp:113-118). */
b200_status b200_alloc(b200_ctx* ctx, size_t bytes, void** out);
b200_status b200_free(b200_ctx* ctx, void* ptr);
b200_status b200_copy_h2d(b200_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes); /* blocking */
b200_status b200_copy_d2h(b200_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes); /* blocking */
b200_status b200_copy_d2d(b200_ctx* ctx, void* dst_dev, const void* src_dev, size_t bytes);  /* async */
b200_status b200_synchronize(b200_ctx* ctx);
/* Stream-ordered snapshot of a few bytes (<= 256) of device memory: begin copies them, in stream order,
 * into slot 0 / 1 and on to pinned host memory on an auxiliary stream; end waits for THAT copy only and
 * hands the bytes out -- kernels enqueued after the begin keep running.  The fused device-resident
 * solvers poll their control block with it (one batch of iterations always queued ahead). */
b200_status b200_snapshot_begin(b200_ctx* ctx, int32_t slot, const void* src_dev, size_t bytes);
b200_status b200_snapshot_end(b200_ctx* ctx, int32_t slot, void* dst_host, size_t bytes);

/* Staging pipe for HOST-resident operands (the reference clones them onto the device inside
 * LinOp::apply: include/ginkgo/core/base/lin_op.hpp:129-215, make_temporary_clone).  Two
 * extra streams + events: the upload of call k+1, the kernels of call k and the download of
 * call k-1 overlap (PCIe is full duplex).  The caller owns b200_pipe_num_slots() pairs of
 * device staging buffers and cycles through the slots; host buffers should be pinned.
 *   upload(slot): after the compute that last read the slot's input
 *   begin_compute(slot) ... kernels on the context's stream ... end_compute(slot)
 *   download(slot): after end_compute(slot)
 *   join: the context's stream waits for all outstanding transfers. */
typedef struct b200_pipe b200_pipe;
b200_status b200_pipe_create(b200_ctx* ctx, b200_pipe** out);
void b200_pipe_destroy(b200_pipe* pipe);
int32_t b200_pipe_num_slots(void);
b200_status b200_pipe_upload(b200_pipe* pipe, int32_t slot, void* dst_dev, const void* src_host,
                             size_t bytes);
b200_status b200_pipe_begin_compute(b200_pipe* pipe, int32_t slot);
b200_status b200_pipe_end_compute(b200_pipe* pipe, int32_t slot);
b200_status b200_pipe_download(b200_pipe* pipe, int32_t slot, void* dst_host, const void* src_dev,
                               size_t bytes);
b200_status b200_pipe_join(b200_pipe* pipe);

/* ---------------------------------------------------------------------------
 * CSR  (reference core/matrix/csr_kernels.hpp:28-43; oracle
 * reference/matrix/csr_kernels.cpp:47-118; today's CUDA path
 * common/cuda_hip/matrix/csr_kernels.template.cpp:2353-2468)
 *   spmv:           c = A b
 *   advanced_spmv:  c = alpha A b + beta c      (beta == 0 never reads c)
 * `plan` may be NULL (the partition is then recomputed on the stream).
 * plan_tune (optional, set-up phase, synchronises, not capturable) times the kernel
 * variants on the matrix itself and records the faster one in the plan -- the analogue
 * of the reference's strategy selection (include/ginkgo/core/matrix/csr.hpp `automatical`,
 * which picks from nnz statistics); every variant sums rows in the same order, so the
 * choice never changes a result.  plan_variant returns the recorded choice (-1 untuned).
 * plan_tune decides from the matrix, not from a timing: the locality of its gathers (distinct
 * 128-byte lines of b per gathered element on a sample of row groups, plan_gather_lines), its size
 * and the size of b against L2 (B200_CSR_TUNE_TIMING=1 times the candidates instead).
 * COLUMN-BLOCKED COPY: for scattered gathers into a b larger than L2 keeps (> 3/8 of L2) with
 * column-sorted rows, tune can keep a copy of col_idxs / values split into parts of <= 5/16 of L2 of b,
 * applied in order (the row sums keep their exact left-to-right order: same bits).  The copy holds
 * VALUES, so it is built only for plans whose owner opted in with b200_csr_plan_allow_value_copy(plan, 1)
 * and thereby promises to call b200_csr_plan_refresh_values_* after changing values in place (the
 * C++ host layer and the Python harness do; a raw caller that never opts in cannot see stale
 * values).  It is used only for calls that pass the col_idxs / values pointers it was made from.
 * B200_CSR_REBLOCK=0 disables it, =N forces N parts.
 * ------------------------------------------------------------------------- */
#define B200_DECL_CSR(V, VT, I, IT)                                                          \
    b200_status b200_csr_plan_create_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t nnz, \
                                               const IT* row_ptrs, b200_csr_plan** out);     \
    b200_status b200_csr_plan_tune_##V##_##I(b200_ctx* ctx, b200_csr_plan* plan,             \
                                             int64_t num_rows, int64_t num_cols,             \
                                             int64_t nnz, const IT* row_ptrs,                \
                                             const IT* col_idxs, const VT* values);          \
    b200_status b200_csr_plan_refresh_values_##V##_##I(b200_ctx* ctx, b200_csr_plan* plan,   \
                                                       int64_t num_rows, const IT* row_ptrs, \
                                                       const VT* values);                    \
    /* column-blocked copy with GIVEN boundaries (parts + 1 ascending host values, 0 .. num_cols;  \
     * needs b200_csr_plan_allow_value_copy, at most 16 parts, column-sorted rows; plan parts == 0 \
     * afterwards if the matrix did not qualify) and the apply of ONE part: c = A_p b              \
     * (accumulate 0) or c += A_p b, optionally after *wait_flag >= wait_epoch (system-scope        \
     * acquire: the multi-GPU pipeline passes the arrival flag of the owner block the part         \
     * gathers from).  Parts applied in ascending order give the bits of the whole matrix; any     \
     * other order re-associates the row sums. */                                                  \
    b200_status b200_csr_plan_split_columns_##V##_##I(                                       \
        b200_ctx* ctx, b200_csr_plan* plan, int64_t num_rows, int64_t num_cols, int64_t nnz, \
        const IT* row_ptrs, const IT* col_idxs, const VT* values, int32_t parts,             \
        const int64_t* bounds_host);                                                         \
    b200_status b200_csr_spmv_part_##V##_##I(b200_ctx* ctx, const b200_csr_plan* plan,       \
                                             int32_t part, int32_t accumulate, const VT* b,  \
                                             int64_t b_stride, VT* c, int64_t c_stride,      \
                                             const uint64_t* wait_flag, uint64_t wait_epoch); \
    b200_status b200_csr_spmv_##V##_##I(                                                     \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,  \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride);                         \
    b200_status b200_csr_advanced_spmv_##V##_##I(                                            \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values,               \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, const VT* beta,     \
        VT* c, int64_t c_stride);
void b200_csr_plan_destroy(b200_csr_plan* plan);
int b200_csr_plan_variant(const b200_csr_plan* plan);
void b200_csr_plan_set_variant(b200_csr_plan* plan, int variant); /* 0 slab, 2 gather_pipe, 4 warp_pipe, 5 cta_ring */
void b200_csr_plan_allow_value_copy(b200_csr_plan* plan, int allow);
double b200_csr_plan_gather_lines(const b200_csr_plan* plan); /* -1 before tune */
int b200_csr_plan_parts(const b200_csr_plan* plan); /* > 1: a column-blocked copy is in use */
/* rows with >= 1024 entries: the plan splits them over CTAs (4096-entry chunks, chunk sums combined
 * in chunk order: deterministic) instead of leaving each to one warp / CTA -- the reference's
 * load-balance / merge-path kernels (common/cuda_hip/matrix/csr_kernels.template.cpp:208-505) */
int64_t b200_csr_plan_num_long_rows(const b200_csr_plan* plan);

/* ---------------------------------------------------------------------------
 * ELL (core/matrix/ell_kernels.hpp:21-35; reference/matrix/ell_kernels.cpp:29-120)
 * column-major storage: element (row, i) at values[row + i*ell_stride],
 * padding column index == -1 (invalid_index).
 * ------------------------------------------------------------------------- */
#define B200_DECL_ELL(V, VT, I, IT)                                                           \
    b200_status b200_ell_spmv_##V##_##I(                                                      \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t num_stored_per_row,        \
        int64_t ell_stride, const IT* col_idxs, const VT* values, const VT* b,                \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride);                          \
    b200_status b200_ell_advanced_spmv_##V##_##I(                                             \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t num_stored_per_row,        \
        int64_t ell_stride, const IT* col_idxs, const VT* values, const VT* alpha,            \
        const VT* b, int64_t b_stride, int64_t num_rhs, const VT* beta, VT* c,                \
        int64_t c_stride);

/* ---------------------------------------------------------------------------
 * SELL-P (core/matrix/sellp_kernels.hpp:21-32; reference/matrix/sellp_kernels.cpp:27-100)
 * element (row r of slice s, i) at (slice_sets[s] + i) * slice_size + r.
 * ------------------------------------------------------------------------- */
#define B200_DECL_SELLP(V, VT, I, IT)                                                        \
    b200_status b200_sellp_spmv_##V##_##I(                                                   \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t slice_size,               \
        const uint64_t* slice_sets, const uint64_t* slice_lengths, const IT* col_idxs,       \
        const VT* values, const VT* b, int64_t b_stride, int64_t num_rhs, VT* c,             \
        int64_t c_stride);                                                                   \
    b200_status b200_sellp_advanced_spmv_##V##_##I(                                          \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t slice_size,               \
        const uint64_t* slice_sets, const uint64_t* slice_lengths, const IT* col_idxs,       \
        const VT* values, const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs,   \
        const VT* beta, VT* c, int64_t c_stride);

/* ---------------------------------------------------------------------------
 * COO (core/matrix/coo_kernels.hpp:22-45; reference/matrix/coo_kernels.cpp:33-100)
 *   spmv: c = A b;  advanced_spmv: c = alpha A b + beta c;
 *   spmv2: c += A b;  advanced_spmv2: c += alpha A b.
 * Entries must be sorted by row (the reference's invariant).  A row-sorted COO
 * is a CSR whose row_ptrs have not been written down yet: the plan holds them
 * (components::convert_idxs_to_ptrs, reference/components/
 * format_conversion_kernels.cpp) plus the CSR row partition, so an apply streams
 * 12 B/nnz instead of 16 and needs no atomics.  `plan` may be NULL (then the
 * pointers are rebuilt on the stream for this call).
 * Hybrid::apply = ell_spmv then coo_spmv2 (core/matrix/hybrid.cpp:175-201).
 * ------------------------------------------------------------------------- */
#define B200_DECL_COO(V, VT, I, IT)                                                          \
    b200_status b200_coo_plan_create_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t nnz, \
                                               const IT* row_idxs, b200_coo_plan** out);     \
    b200_status b200_coo_spmv_##V##_##I(                                                     \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values, const VT* b,  \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride);                         \
    b200_status b200_coo_advanced_spmv_##V##_##I(                                            \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values,               \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, const VT* beta,     \
        VT* c, int64_t c_stride);                                                            \
    b200_status b200_coo_spmv2_##V##_##I(                                                    \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values, const VT* b,  \
        int64_t b_stride, int64_t num_rhs, VT* c, int64_t c_stride);                         \
    b200_status b200_coo_advanced_spmv2_##V##_##I(                                           \
        b200_ctx* ctx, const b200_coo_plan* plan, int64_t num_rows, int64_t num_cols,        \
        int64_t nnz, const IT* row_idxs, const IT* col_idxs, const VT* values,               \
        const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs, VT* c,              \
        int64_t c_stride);
void b200_coo_plan_destroy(b200_coo_plan* plan);

/* ---------------------------------------------------------------------------
 * Block-Jacobi apply (core/preconditioner/jacobi_kernels.hpp:47-74;
 * reference/preconditioner/jacobi_kernels.cpp:419-520).  Inverted blocks in
 * block_interleaved_storage_scheme (include/ginkgo/core/preconditioner/
 * jacobi.hpp:37-141): element (r,c) of block k at
 *   group_offset*(k >> group_power) + block_offset*(k & (2^group_power-1))
 *   + r + c*(block_offset << group_power).
 * The plain entry points read full-precision storage (block_precisions == NULL in the reference);
 * the *_adaptive ones take the reference's array<precision_reduction> (one byte per block).
 * ------------------------------------------------------------------------- */
#define B200_DECL_JACOBI_BLOCK(V, VT, I, IT)                                                  \
    b200_status b200_jacobi_simple_apply_##V##_##I(                                           \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,      \
        int64_t group_offset, int32_t group_power, const IT* block_pointers,                  \
        const VT* blocks, const VT* b, int64_t b_stride, int64_t num_rhs, VT* x,              \
        int64_t x_stride);                                                                    \
    b200_status b200_jacobi_apply_##V##_##I(                                                  \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,      \
        int64_t group_offset, int32_t group_power, const IT* block_pointers,                  \
        const VT* blocks, const VT* alpha, const VT* b, int64_t b_stride, int64_t num_rhs,    \
        const VT* beta, VT* x, int64_t x_stride);                                             \
    /* jacobi::generate, full precision (reference/preconditioner/jacobi_kernels.cpp:        \
     * 113-278, 320-410): extract each diagonal block, invert it with the reference's         \
     * pivoted Gauss-Jordan in the reference's operation order (bit-identical inverse), store \
     * it transposed + column-permuted.  Entries of a slot outside the bs x bs block are not  \
     * written.  A zero pivot leaves the block as the reference leaves it. */                 \
    b200_status b200_jacobi_generate_##V##_##I(                                               \
        b200_ctx* ctx, int64_t num_rows, const IT* row_ptrs, const IT* col_idxs,              \
        const VT* values, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,   \
        int64_t group_offset, int32_t group_power, const IT* block_pointers, VT* blocks);     \
    /* ---- adaptive precision (Jacobi `storage_optimization`, include/ginkgo/core/            \
     * preconditioner/jacobi.hpp:315-513).  block_precisions: gko::precision_reduction per     \
     * block, one byte = preserving << 4 | nonpreserving, 0xff = autodetect(); in/out for      \
     * generate.  jacobi::generate with conditioning + block_precisions                        \
     * (core/preconditioner/jacobi_kernels.hpp:28-40, reference/preconditioner/                \
     * jacobi_kernels.cpp:281-410): condition numbers (1-norm of block times 1-norm of its     \
     * inverse, the reference's compute_inf_norm on the row-major block), per-block detection  \
     * of the storage types that keep `accuracy` (core/preconditioner/jacobi_utils.hpp:        \
     * 100-189; reductions that narrow the exponent range are verified by inverting the        \
     * rounded inverse), ONE precision per storage group, blocks stored converted: float /     \
     * gko::half / truncated<double,2> / truncated<float,2> / truncated<double,4> for double,  \
     * gko::half / truncated<float,2> for float.  conditioning == NULL or block_precisions ==  \
     * NULL behave as in the reference (no detection / full precision).  Precisions,           \
     * condition numbers and stored bits are identical to the reference executor's. */        \
    b200_status b200_jacobi_generate_adaptive_##V##_##I(                                      \
        b200_ctx* ctx, int64_t num_rows, const IT* row_ptrs, const IT* col_idxs,              \
        const VT* values, int64_t num_blocks, int32_t max_block_size, double accuracy,        \
        int64_t block_offset, int64_t group_offset, int32_t group_power, VT* conditioning,    \
        uint8_t* block_precisions, const IT* block_pointers, VT* blocks);                     \
    /* jacobi::simple_apply / apply reading every block in its stored precision                \
     * (reference/preconditioner/jacobi_kernels.cpp:415-520) */                               \
    b200_status b200_jacobi_simple_apply_adaptive_##V##_##I(                                  \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,      \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,           \
        const IT* block_pointers, const VT* blocks, const VT* b, int64_t b_stride,            \
        int64_t num_rhs, VT* x, int64_t x_stride);                                            \
    b200_status b200_jacobi_apply_adaptive_##V##_##I(                                         \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,      \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,           \
        const IT* block_pointers, const VT* blocks, const VT* alpha, const VT* b,             \
        int64_t b_stride, int64_t num_rhs, const VT* beta, VT* x, int64_t x_stride);          \
    /* jacobi::transpose_jacobi with stored precisions (reference/...:597-627) */             \
    b200_status b200_jacobi_transpose_adaptive_##V##_##I(                                     \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,      \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,           \
        const IT* block_pointers, const VT* blocks, VT* out_blocks);

/* Block apply with many right-hand sides = a batch of small dense GEMMs: from 8 (fp32: 16) right-hand
 * sides on the blocks are applied on the fp64 tensor cores (mma.sync.m8n8k4.f64, fp32 operands widened;
 * agrees with the reference to r<T>), below that by the SIMT kernel whose sums have the reference's
 * order (bit-identical).  mode: -1 that default, 0 always SIMT, 1 always tensor cores.  Process-wide;
 * initial value from B200_JACOBI_MMA. */
void b200_jacobi_apply_mode(int mode);

/* jacobi::initialize_precisions (reference/preconditioner/jacobi_kernels.cpp:453-461):
 * precisions[i] = source[i % source_size] */
b200_status b200_jacobi_initialize_precisions(b200_ctx* ctx, const uint8_t* source, int64_t source_size,
                                              uint8_t* precisions, int64_t size);

/* jacobi::find_blocks (core/preconditioner/jacobi_kernels.hpp:19-26; reference/preconditioner/
 * jacobi_kernels.cpp:36-123): natural blocks = maximal runs of rows with identical column
 * patterns, cut at max_block_size, then greedy agglomeration of neighbours while the sum
 * stays <= max_block_size.  block_pointers needs num_rows + 1 entries; the number of blocks
 * comes back on the host (the call synchronises).  Integer-exact. */
b200_status b200_jacobi_find_blocks_i32(b200_ctx* ctx, int64_t num_rows, const int32_t* row_ptrs,
                                        const int32_t* col_idxs, int32_t max_block_size,
                                        int32_t* block_pointers, int64_t* num_blocks_host);
b200_status b200_jacobi_find_blocks_i64(b200_ctx* ctx, int64_t num_rows, const int64_t* row_ptrs,
                                        const int64_t* col_idxs, int32_t max_block_size,
                                        int64_t* block_pointers, int64_t* num_blocks_host);

/* ---------------------------------------------------------------------------
 * Dense BLAS-1 (core/matrix/dense_kernels.hpp:34-135;
 * reference/matrix/dense_kernels.cpp:95-437).  `result` is a 1 x cols device
 * row.  alpha is 1x1 (alpha_cols == 1) or 1 x cols (alpha_cols == cols).
 * Reductions are deterministic (fixed tree, no floating-point atomics).
 *
 * CG (core/solver/cg_kernels.hpp:25-50; reference/solver/cg_kernels.cpp:24-102)
 * BiCGStab (core/solver/bicgstab_kernels.hpp:25-74;
 *           reference/solver/bicgstab_kernels.cpp:25-178)
 * GMRES (core/solver/common_gmres_kernels.hpp:23-48, gmres_kernels.hpp:23-46;
 *        reference/solver/common_gmres_kernels.cpp:112-195, gmres_kernels.cpp:27-99)
 * Stopping criteria (core/stop/residual_norm_kernels.hpp:21-50;
 *        reference/stop/residual_norm_kernels.cpp:27-92)
 * Scalar Jacobi (core/preconditioner/jacobi_kernels.hpp:42-81;
 *        reference/preconditioner/jacobi_kernels.cpp:522-592)
 * ------------------------------------------------------------------------- */
#define B200_DECL_VALUE(V, VT)                                                                \
    b200_status b200_dense_compute_dot_##V(b200_ctx* ctx, int64_t rows, int64_t cols,         \
                                           const VT* x, int64_t x_stride, const VT* y,        \
                                           int64_t y_stride, VT* result);                     \
    b200_status b200_dense_compute_conj_dot_##V(b200_ctx* ctx, int64_t rows, int64_t cols,    \
                                                const VT* x, int64_t x_stride, const VT* y,   \
                                                int64_t y_stride, VT* result);                \
    b200_status b200_dense_compute_norm2_##V(b200_ctx* ctx, int64_t rows, int64_t cols,       \
                                             const VT* x, int64_t x_stride, VT* result);      \
    b200_status b200_dense_compute_squared_norm2_##V(b200_ctx* ctx, int64_t rows,             \
                                                     int64_t cols, const VT* x,               \
                                                     int64_t x_stride, VT* result);           \
    b200_status b200_dense_add_scaled_##V(b200_ctx* ctx, int64_t rows, int64_t cols,          \
                                          const VT* alpha, int64_t alpha_cols, const VT* x,   \
                                          int64_t x_stride, VT* y, int64_t y_stride);         \
    b200_status b200_dense_sub_scaled_##V(b200_ctx* ctx, int64_t rows, int64_t cols,          \
                                          const VT* alpha, int64_t alpha_cols, const VT* x,   \
                                          int64_t x_stride, VT* y, int64_t y_stride);         \
    b200_status b200_dense_scale_##V(b200_ctx* ctx, int64_t rows, int64_t cols,               \
                                     const VT* alpha, int64_t alpha_cols, VT* x,              \
                                     int64_t x_stride);                                       \
    b200_status b200_dense_inv_scale_##V(b200_ctx* ctx, int64_t rows, int64_t cols,           \
                                         const VT* alpha, int64_t alpha_cols, VT* x,          \
                                         int64_t x_stride);                                   \
    b200_status b200_dense_copy_##V(b200_ctx* ctx, int64_t rows, int64_t cols, const VT* in,  \
                                    int64_t in_stride, VT* out, int64_t out_stride);          \
    b200_status b200_dense_fill_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x,         \
                                    int64_t x_stride, VT value);                              \
                                                                                              \
    b200_status b200_cg_initialize_##V(                                                       \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* b, int64_t b_stride, VT* r,      \
        int64_t r_stride, VT* z, int64_t z_stride, VT* p, int64_t p_stride, VT* q,            \
        int64_t q_stride, VT* prev_rho, VT* rho, uint8_t* stop_status);                       \
    b200_status b200_cg_step_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* p,          \
                                   int64_t p_stride, const VT* z, int64_t z_stride,           \
                                   const VT* rho, const VT* prev_rho,                         \
                                   const uint8_t* stop_status);                               \
    b200_status b200_cg_step_2_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x,          \
                                   int64_t x_stride, VT* r, int64_t r_stride, const VT* p,    \
                                   int64_t p_stride, const VT* q, int64_t q_stride,           \
                                   const VT* beta, const VT* rho,                             \
                                   const uint8_t* stop_status);                               \
                                                                                              \
    /* FCG (core/solver/fcg_kernels.hpp; reference/solver/fcg_kernels.cpp:22-100) and CGS    \
     * (core/solver/cgs_kernels.hpp; reference/solver/cgs_kernels.cpp:22-140), SURVEY 8f-3 */ \
    b200_status b200_fcg_initialize_##V(                                                      \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* b, int64_t b_stride, VT* r,      \
        int64_t r_stride, VT* z, int64_t z_stride, VT* p, int64_t p_stride, VT* q,            \
        int64_t q_stride, VT* t, int64_t t_stride, VT* prev_rho, VT* rho, VT* rho_t,          \
        uint8_t* stop_status);                                                                \
    b200_status b200_fcg_step_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* p,         \
                                    int64_t p_stride, const VT* z, int64_t z_stride,          \
                                    const VT* rho_t, const VT* prev_rho,                      \
                                    const uint8_t* stop_status);                              \
    b200_status b200_fcg_step_2_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x,         \
                                    int64_t x_stride, VT* r, int64_t r_stride, VT* t,         \
                                    int64_t t_stride, const VT* p, int64_t p_stride,          \
                                    const VT* q, int64_t q_stride, const VT* beta,            \
                                    const VT* rho, const uint8_t* stop_status);               \
    b200_status b200_cgs_initialize_##V(                                                      \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* b, int64_t b_stride, VT* r,      \
        int64_t r_stride, VT* r_tld, int64_t r_tld_stride, VT* p, int64_t p_stride, VT* q,    \
        int64_t q_stride, VT* u, int64_t u_stride, VT* u_hat, int64_t u_hat_stride,           \
        VT* v_hat, int64_t v_hat_stride, VT* t, int64_t t_stride, VT* alpha, VT* beta,        \
        VT* gamma, VT* prev_rho, VT* rho, uint8_t* stop_status);                              \
    b200_status b200_cgs_step_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols, const VT* r,   \
                                    int64_t r_stride, VT* u, int64_t u_stride, VT* p,         \
                                    int64_t p_stride, const VT* q, int64_t q_stride,          \
                                    VT* beta, const VT* rho, const VT* prev_rho,              \
                                    const uint8_t* stop_status);                              \
    b200_status b200_cgs_step_2_##V(b200_ctx* ctx, int64_t rows, int64_t cols, const VT* u,   \
                                    int64_t u_stride, const VT* v_hat, int64_t v_hat_stride,  \
                                    VT* q, int64_t q_stride, VT* t, int64_t t_stride,         \
                                    VT* alpha, const VT* rho, const VT* gamma,                \
                                    const uint8_t* stop_status);                              \
    b200_status b200_cgs_step_3_##V(b200_ctx* ctx, int64_t rows, int64_t cols, const VT* t,   \
                                    int64_t t_stride, const VT* u_hat, int64_t u_hat_stride,  \
                                    VT* r, int64_t r_stride, VT* x, int64_t x_stride,         \
                                    const VT* alpha, const uint8_t* stop_status);             \
                                                                                              \
    /* Chebyshev (core/solver/chebyshev_kernels.hpp; reference/solver/chebyshev_kernels.cpp:   \
     * 15-66): alpha / beta by value, arithmetic in double for every value type */            \
    b200_status b200_chebyshev_init_update_##V(b200_ctx* ctx, int64_t rows, int64_t cols,     \
                                               double alpha, const VT* inner_sol,             \
                                               int64_t inner_stride, VT* update_sol,          \
                                               int64_t update_stride, VT* output,             \
                                               int64_t output_stride);                        \
    b200_status b200_chebyshev_update_##V(b200_ctx* ctx, int64_t rows, int64_t cols,          \
                                          double alpha, double beta, VT* inner_sol,           \
                                          int64_t inner_stride, VT* update_sol,               \
                                          int64_t update_stride, VT* output,                  \
                                          int64_t output_stride);                             \
                                                                                              \
    /* PipeCG (core/solver/pipe_cg_kernels.hpp; reference/solver/pipe_cg_kernels.cpp:24-160) */ \
    b200_status b200_pipe_cg_initialize_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols,      \
                                              const VT* b, int64_t b_stride, VT* r,           \
                                              int64_t r_stride, VT* prev_rho,                 \
                                              uint8_t* stop_status);                          \
    b200_status b200_pipe_cg_initialize_2_##V(                                                \
        b200_ctx* ctx, int64_t rows, int64_t cols, VT* p, int64_t p_stride, VT* q,            \
        int64_t q_stride, VT* f, int64_t f_stride, VT* g, int64_t g_stride, VT* beta,         \
        const VT* z, int64_t z_stride, const VT* w, int64_t w_stride, const VT* m,            \
        int64_t m_stride, const VT* n, int64_t n_stride, const VT* delta);                    \
    b200_status b200_pipe_cg_step_1_##V(                                                      \
        b200_ctx* ctx, int64_t rows, int64_t cols, VT* x, int64_t x_stride, VT* r,            \
        int64_t r_stride, VT* z1, int64_t z1_stride, VT* z2, int64_t z2_stride, VT* w,        \
        int64_t w_stride, const VT* p, int64_t p_stride, const VT* q, int64_t q_stride,       \
        const VT* f, int64_t f_stride, const VT* g, int64_t g_stride, const VT* rho,          \
        const VT* beta, const uint8_t* stop_status);                                          \
    b200_status b200_pipe_cg_step_2_##V(                                                      \
        b200_ctx* ctx, int64_t rows, int64_t cols, VT* beta, VT* p, int64_t p_stride, VT* q,  \
        int64_t q_stride, VT* f, int64_t f_stride, VT* g, int64_t g_stride, const VT* z,      \
        int64_t z_stride, const VT* w, int64_t w_stride, const VT* m, int64_t m_stride,       \
        const VT* n, int64_t n_stride, const VT* prev_rho, const VT* rho, const VT* delta,    \
        const uint8_t* stop_status);                                                          \
                                                                                              \
    /* GCR (core/solver/gcr_kernels.hpp; reference/solver/gcr_kernels.cpp:26-84) */           \
    b200_status b200_gcr_initialize_##V(b200_ctx* ctx, int64_t rows, int64_t cols,            \
                                        const VT* b, int64_t b_stride, VT* residual,          \
                                        int64_t residual_stride, uint8_t* stop_status);       \
    b200_status b200_gcr_restart_##V(b200_ctx* ctx, int64_t rows, int64_t cols,               \
                                     const VT* residual, int64_t residual_stride,             \
                                     const VT* a_residual, int64_t a_residual_stride,         \
                                     VT* p_bases, int64_t p_stride, VT* ap_bases,             \
                                     int64_t ap_stride, uint64_t* final_iter_nums);           \
    b200_status b200_gcr_step_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x,         \
                                    int64_t x_stride, VT* residual, int64_t residual_stride,  \
                                    const VT* p, int64_t p_stride, const VT* ap,              \
                                    int64_t ap_stride, const VT* ap_norm, const VT* rap,      \
                                    const uint8_t* stop_status);                              \
                                                                                              \
    /* MINRES (core/solver/minres_kernels.hpp; reference/solver/minres_kernels.cpp:26-150) */ \
    b200_status b200_minres_initialize_##V(                                                   \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* r, int64_t r_stride, VT* z,      \
        int64_t z_stride, VT* p, int64_t p_stride, VT* p_prev, int64_t p_prev_stride, VT* q,  \
        int64_t q_stride, VT* q_prev, int64_t q_prev_stride, VT* q_tilde,                     \
        int64_t q_tilde_stride, VT* beta, VT* gamma, VT* delta, VT* cos_prev, VT* cos_,       \
        VT* sin_prev, VT* sin_, VT* eta_next, VT* eta, uint8_t* stop_status);                 \
    b200_status b200_minres_step_1_##V(b200_ctx* ctx, int64_t cols, VT* alpha, VT* beta,      \
                                       VT* gamma, VT* delta, VT* cos_prev, VT* cos_,          \
                                       VT* sin_prev, VT* sin_, VT* eta, VT* eta_next,         \
                                       VT* tau, const uint8_t* stop_status);                  \
    b200_status b200_minres_step_2_##V(                                                       \
        b200_ctx* ctx, int64_t rows, int64_t cols, VT* x, int64_t x_stride, VT* p,            \
        int64_t p_stride, const VT* p_prev, int64_t p_prev_stride, VT* z, int64_t z_stride,   \
        const VT* z_tilde, int64_t z_tilde_stride, VT* q, int64_t q_stride, VT* q_prev,       \
        int64_t q_prev_stride, VT* v, int64_t v_stride, const VT* alpha, const VT* beta,      \
        const VT* gamma, const VT* delta, const VT* cos_, const VT* eta,                      \
        const uint8_t* stop_status);                                                          \
                                                                                              \
    b200_status b200_bicgstab_initialize_##V(                                                 \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* b, int64_t b_stride, VT* r,      \
        int64_t r_stride, VT* rr, int64_t rr_stride, VT* y, int64_t y_stride, VT* s,          \
        int64_t s_stride, VT* t, int64_t t_stride, VT* z, int64_t z_stride, VT* v,            \
        int64_t v_stride, VT* p, int64_t p_stride, VT* prev_rho, VT* rho, VT* alpha,          \
        VT* beta, VT* gamma, VT* omega, uint8_t* stop_status);                                \
    b200_status b200_bicgstab_step_1_##V(                                                     \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* r, int64_t r_stride, VT* p,      \
        int64_t p_stride, const VT* v, int64_t v_stride, const VT* rho, const VT* prev_rho,   \
        const VT* alpha, const VT* omega, const uint8_t* stop_status);                        \
    b200_status b200_bicgstab_step_2_##V(                                                     \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* r, int64_t r_stride, VT* s,      \
        int64_t s_stride, const VT* v, int64_t v_stride, const VT* rho, VT* alpha,            \
        const VT* beta, const uint8_t* stop_status);                                          \
    b200_status b200_bicgstab_step_3_##V(                                                     \
        b200_ctx* ctx, int64_t rows, int64_t cols, VT* x, int64_t x_stride, VT* r,            \
        int64_t r_stride, const VT* s, int64_t s_stride, const VT* t, int64_t t_stride,       \
        const VT* y, int64_t y_stride, const VT* z, int64_t z_stride, const VT* alpha,        \
        const VT* beta, const VT* gamma, VT* omega, const uint8_t* stop_status);              \
    b200_status b200_bicgstab_finalize_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x,  \
                                           int64_t x_stride, const VT* y, int64_t y_stride,   \
                                           const VT* alpha, uint8_t* stop_status);            \
                                                                                              \
    /* GMRES: krylov_bases is ((krylov_dim+1)*rows) x cols; hessenberg_iter is   */           \
    /* (iter+2) x cols with stride hess_stride; givens are krylov_dim x cols.     */           \
    b200_status b200_common_gmres_initialize_##V(                                             \
        b200_ctx* ctx, int64_t rows, int64_t cols, int64_t krylov_dim, const VT* b,           \
        int64_t b_stride, VT* residual, int64_t residual_stride, VT* givens_sin,              \
        int64_t sin_stride, VT* givens_cos, int64_t cos_stride, uint8_t* stop_status);        \
    b200_status b200_common_gmres_hessenberg_qr_##V(                                          \
        b200_ctx* ctx, int64_t cols, VT* givens_sin, int64_t sin_stride, VT* givens_cos,      \
        int64_t cos_stride, VT* residual_norm, VT* residual_norm_collection,                  \
        int64_t rnc_stride, VT* hessenberg_iter, int64_t hess_stride, int64_t iter,           \
        uint64_t* final_iter_nums, const uint8_t* stop_status);                               \
    b200_status b200_common_gmres_solve_krylov_##V(                                           \
        b200_ctx* ctx, int64_t cols, const VT* residual_norm_collection, int64_t rnc_stride,  \
        const VT* hessenberg, int64_t hess_stride, VT* y, int64_t y_stride,                   \
        const uint64_t* final_iter_nums, const uint8_t* stop_status);                         \
    b200_status b200_gmres_restart_##V(                                                       \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* residual,                        \
        int64_t residual_stride, const VT* residual_norm, VT* residual_norm_collection,       \
        VT* krylov_bases, int64_t krylov_stride, uint64_t* final_iter_nums);                  \
    b200_status b200_gmres_multi_axpy_##V(                                                    \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* krylov_bases,                    \
        int64_t krylov_stride, const VT* y, int64_t y_stride, VT* before_preconditioner,      \
        int64_t bp_stride, const uint64_t* final_iter_nums, uint8_t* stop_status);            \
    b200_status b200_gmres_multi_dot_##V(                                                     \
        b200_ctx* ctx, int64_t rows, int64_t cols, int64_t num_bases,                         \
        const VT* krylov_bases, int64_t krylov_stride, const VT* next_krylov,                 \
        int64_t next_stride, VT* hessenberg_col, int64_t hess_stride);                        \
                                                                                              \
    /* blocking: returns the two host bools of the reference signature */                     \
    b200_status b200_residual_norm_##V(                                                       \
        b200_ctx* ctx, int64_t cols, const VT* tau, const VT* orig_tau, VT rel_residual_goal, \
        uint8_t stopping_id, int32_t set_finalized, uint8_t* stop_status,                     \
        uint8_t* device_storage, int32_t* all_converged, int32_t* one_changed);               \
    b200_status b200_implicit_residual_norm_##V(                                              \
        b200_ctx* ctx, int64_t cols, const VT* tau, const VT* orig_tau, VT rel_residual_goal, \
        uint8_t stopping_id, int32_t set_finalized, uint8_t* stop_status,                     \
        uint8_t* device_storage, int32_t* all_converged, int32_t* one_changed);               \
                                                                                              \
    b200_status b200_jacobi_invert_diagonal_##V(b200_ctx* ctx, int64_t n, const VT* diag,     \
                                                VT* inv_diag);                                \
    b200_status b200_jacobi_simple_scalar_apply_##V(                                          \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* inv_diag, const VT* b,           \
        int64_t b_stride, VT* x, int64_t x_stride);                                           \
    b200_status b200_jacobi_scalar_apply_##V(                                                 \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* inv_diag, const VT* alpha,       \
        const VT* b, int64_t b_stride, const VT* beta, VT* x, int64_t x_stride);

/* ir::initialize (core/solver/ir_kernels.hpp; reference/solver/ir_kernels.cpp:17-24): reset */
b200_status b200_ir_initialize(b200_ctx* ctx, int64_t cols, uint8_t* stop_status);

/* set_all_statuses (core/stop/criterion_kernels.hpp:21; used by stop::Iteration) */
b200_status b200_set_all_statuses(b200_ctx* ctx, int64_t cols, uint8_t stopping_id,
                                  int32_t set_finalized, uint8_t* stop_status);

#define B200_DECL_VALUE_INDEX(V, VT, I, IT) \
    B200_DECL_CSR(V, VT, I, IT)             \
    B200_DECL_ELL(V, VT, I, IT)             \
    B200_DECL_SELLP(V, VT, I, IT)           \
    B200_DECL_COO(V, VT, I, IT)             \
    B200_DECL_JACOBI_BLOCK(V, VT, I, IT)

B200_DECL_VALUE(f64, double)
B200_DECL_VALUE(f32, float)
B200_DECL_VALUE_INDEX(f64, double, i32, int32_t)
B200_DECL_VALUE_INDEX(f64, double, i64, int64_t)
B200_DECL_VALUE_INDEX(f32, float, i32, int32_t)
B200_DECL_VALUE_INDEX(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused CG iteration (ginkgo_b200 extension behind solver::Cg::apply; it regroups the
 * loop body of core/solver/cg.cpp:142-180 into three launches per iteration with
 * every scalar produced and consumed on the device):
 *   step_p    p = z + (rho/prev_rho) p                        (cg::step_1)
 *   spmv_dot  q = A p, pq = p.q in the SpMV epilogue          (Csr::apply + compute_conj_dot)
 *   step_xr   x += (rho/pq) p; r -= (rho/pq) q; z = M^-1 r (scalar Jacobi or identity);
 *             rho' = r.z; rr = r.r; Iteration / (Implicit)ResidualNorm check
 *                                                             (cg::step_2 + jacobi apply + dot
 *                                                              + norm2 + criterion check)
 * sc:  VT[8]    0 rho, 1 prev_rho, 2 pq, 3 rr, 4 tau0, 5 threshold, 6/7 local partials
 * ctl: int32[8] 0 stopping_status byte (0 = running), 1 iterations, 2 max_iters,
 *               3 res_kind (0 none, 1 ResidualNorm, 2 ImplicitResidualNorm), 4 iter_first
 * Once ctl[0] != 0 every fused kernel is a no-op, so graphs of k iterations can be
 * replayed and the host polls ctl every k iterations.  finalize == 0 leaves the local
 * sums in sc[6..7] for a multi-GPU all-reduce followed by b200_cg_fused_finish.
 * baseline: 0 rhs_norm (caller stores ||b|| in sc[4] first), 1 initial_resnorm, 2 absolute.
 * ------------------------------------------------------------------------- */
typedef struct b200_graph b200_graph;
b200_status b200_graph_begin_capture(b200_ctx* ctx);
b200_status b200_graph_end_capture(b200_ctx* ctx, b200_graph** out);
b200_status b200_graph_launch(b200_ctx* ctx, b200_graph* graph);
void b200_graph_destroy(b200_graph* graph);

#define B200_DECL_FCG(V, VT)                                                                   \
    int64_t b200_cg_fused_work_size_##V(const b200_ctx* ctx);                                  \
    b200_status b200_cg_fused_init_##V(                                                        \
        b200_ctx* ctx, int64_t n, const VT* r, VT* z, VT* p, VT* q, const VT* inv_diag,        \
        VT* sc, int32_t* ctl, VT* work, int64_t max_iters, int32_t res_kind,                   \
        int32_t iter_first, int32_t baseline, VT reduction_factor, int32_t finalize);          \
    b200_status b200_cg_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* z,         \
                                         const VT* sc, const int32_t* ctl);                    \
    b200_status b200_cg_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r, const VT* p, \
                                          const VT* q, VT* z, const VT* inv_diag, VT* sc,      \
                                          int32_t* ctl, VT* work, int32_t finalize);           \
    b200_status b200_cg_fused_finish_##V(b200_ctx* ctx, VT* sc, int32_t* ctl, int32_t init,    \
                                         int32_t baseline, VT reduction_factor);
#define B200_DECL_SPMV_DOT(V, VT, I, IT)                                                       \
    b200_status b200_csr_spmv_dot_##V##_##I(                                                   \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,    \
        VT* c, VT* dot_out, VT* work, const int32_t* ctl);

B200_DECL_FCG(f64, double)
B200_DECL_FCG(f32, float)
B200_DECL_SPMV_DOT(f64, double, i32, int32_t)
B200_DECL_SPMV_DOT(f64, double, i64, int64_t)
B200_DECL_SPMV_DOT(f32, float, i32, int32_t)
B200_DECL_SPMV_DOT(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused BiCGStab iteration (ginkgo_b200 extension behind solver::Bicgstab::apply, single GPU;
 * it regroups the loop body of core/solver/bicgstab.cpp:95-233 into five launches per
 * iteration with every scalar produced and consumed on the device; d = inv_diag of a
 * scalar Jacobi preconditioner, NULL for Identity):
 *   step_p     p = r + (rho/prev_rho*alpha/omega)(p - omega v), p = r if prev_rho*omega == 0;
 *              y = d.p                                        (bicgstab::step_1 + jacobi apply)
 *   spmv_dot2  v = A y, beta = rr.v in the SpMV epilogue      (Csr::apply + compute_conj_dot)
 *   step_s     alpha = rho/beta (0 and s = r if beta == 0); s = r - alpha v; z = d.s; ||s||^2;
 *              the mid-iteration criterion check on s         (bicgstab::step_2 + norm2 +
 *                                                              criterion check + jacobi apply)
 *   spmv_dot2  t = A z, gamma = s.t and beta = t.t            (Csr::apply + 2 compute_conj_dot)
 *   step_xr    omega = gamma/beta (0 if beta == 0); x += alpha y + omega z; r = s - omega t;
 *              rho' = rr.r; ||r||^2; rho / prev_rho swapped; iteration count; the top-of-
 *              iteration criterion check on r                 (bicgstab::step_3 + dot + norm2 +
 *                                                              criterion check)
 *   init       r holds b - A x; rr = r; p = v = y = s = t = z = 0; rho = prev_rho = alpha = beta =
 *              gamma = omega = 1; rho = rr.r, ||r||^2, the baseline and the first check
 *                                                             (bicgstab::initialize + dot + check)
 * sc:  VT[16]   0 rho, 1 prev_rho, 2 beta (rr.v, then t.t), 3 ||r||^2, 4 tau0, 5 threshold,
 *               6 alpha, 7 omega, 8 gamma, 9 ||s||^2
 * ctl: int32[8] 0 stopping_status byte (0 = running), 1 iterations, 2 max_iters,
 *               3 res_kind (0 none, 1 ResidualNorm, 2 ImplicitResidualNorm), 4 iter_first,
 *               5 finalize pending
 * A stop at the mid check writes the (finalized) status to ctl[0] and sets ctl[5]; step_xr of
 * the same iteration then only applies bicgstab::finalize, x += alpha y, and clears ctl[5].
 * With ctl[0] != 0 and ctl[5] == 0 every kernel is a no-op, so graphs of k iterations can be
 * replayed and the host polls ctl every k iterations.  `work` has b200_cg_fused_work_size
 * elements; baseline as for the fused CG.
 *
 * b200_csr_spmv_dot2: c = A b, *dot_out = w . c and, unless dot2_out is NULL, *dot2_out = c . c
 * in the epilogue of the SpMV (w: one entry per row; A may be rectangular).  Plan, work, ctl and
 * alignment rules are those of b200_csr_spmv_dot.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FBICGSTAB(V, VT)                                                             \
    b200_status b200_bicgstab_fused_init_##V(                                                  \
        b200_ctx* ctx, int64_t n, const VT* r, VT* rr, VT* p, VT* v, VT* y, VT* s, VT* t,      \
        VT* z, VT* sc, int32_t* ctl, VT* work, int64_t max_iters, int32_t res_kind,            \
        int32_t iter_first, int32_t baseline, VT reduction_factor);                            \
    b200_status b200_bicgstab_fused_step_p_##V(b200_ctx* ctx, int64_t n, VT* p, const VT* r,   \
                                               const VT* v, VT* y, const VT* inv_diag,         \
                                               const VT* sc, const int32_t* ctl);              \
    b200_status b200_bicgstab_fused_step_s_##V(b200_ctx* ctx, int64_t n, const VT* r,          \
                                               const VT* v, VT* s, VT* z, const VT* inv_diag,  \
                                               VT* sc, int32_t* ctl, VT* work);                \
    b200_status b200_bicgstab_fused_step_xr_##V(b200_ctx* ctx, int64_t n, VT* x, VT* r,        \
                                                const VT* s, const VT* t, const VT* y,         \
                                                const VT* z, const VT* rr, VT* sc,             \
                                                int32_t* ctl, VT* work);
#define B200_DECL_SPMV_DOT2(V, VT, I, IT)                                                      \
    b200_status b200_csr_spmv_dot2_##V##_##I(                                                  \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,    \
        VT* c, const VT* w, VT* dot_out, VT* dot2_out, VT* work, const int32_t* ctl);

B200_DECL_FBICGSTAB(f64, double)
B200_DECL_FBICGSTAB(f32, float)
B200_DECL_SPMV_DOT2(f64, double, i32, int32_t)
B200_DECL_SPMV_DOT2(f64, double, i64, int64_t)
B200_DECL_SPMV_DOT2(f32, float, i32, int32_t)
B200_DECL_SPMV_DOT2(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused MINRES iteration (ginkgo_b200 extension behind solver::Minres::apply with with_fused(true),
 * single GPU; it regroups the loop body of core/solver/minres.cpp:199-285 into three launches per
 * iteration with every scalar produced and consumed on the device; d = inv_diag of a scalar
 * Jacobi preconditioner, NULL for Identity):
 *   spmv_sub_dot  v = A z - v, alpha = z.v in the SpMV epilogue
 *                                                   (Csr::apply(1, z, -1, v) + compute_conj_dot)
 *   lanczos       v -= alpha q (not when alpha == 0); beta = v.(d v); then in the last CTA
 *                 minres::step_1: beta = sqrt(beta), the two old rotations, the new Givens
 *                 rotation, tau, eta and eta_next   (sub_scaled + jacobi apply + compute_conj_dot
 *                                                    + minres::step_1)
 *   update        minres::step_2 with z~ = d v recomputed and q_prev not stored: p = (z - gamma
 *                 p_prev - delta p) / alpha; x += cos eta p; q = v / beta; v = q_old beta;
 *                 z = z~ / beta (0 for a zero divisor).  p / p_prev are p0 / p1 as the parity of
 *                 the iteration count says (iteration k writes p1 when k is even, p0 when odd).
 *                 The last CTA swaps gamma / beta, counts the iteration and runs the criterion
 *                 check of the next one       (std::swap(p, p_prev) + minres::step_2 + std::swap
 *                                              (gamma, beta) + criterion check)
 *   init          the first criterion check, after the host's minres::initialize; sc[4] holds
 *                 ||b|| (baseline 0) or ||r0|| (1) and is set to 1 for baseline 2
 * sc:  VT[16]   0 alpha, 1 beta, 2 gamma, 3 delta, 4 tau0, 5 threshold, 6 tau, 7 eta, 8 eta_next,
 *               9 cos_prev, 10 cos, 11 sin_prev, 12 sin
 * ctl: int32[8] 0 stopping_status byte (0 = running), 1 iterations, 2 max_iters (-1 none),
 *               3 res_kind (0 none, 2 ImplicitResidualNorm: sqrt|tau| <= threshold), 4 iter_first
 * With ctl[0] != 0 every kernel is a no-op, so graphs of k iterations can be replayed and the host
 * polls ctl every k iterations.  `work` has b200_minres_fused_work_size elements.
 *
 * b200_csr_spmv_sub_dot: c = A b - c and *dot_out = b . c in one launch (square A): the advanced
 * SpMV with alpha = 1, beta = -1, bit for bit b200_csr_advanced_spmv on a plan without column
 * parts.  Plan, work, ctl and alignment rules are those of b200_csr_spmv_dot.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FMINRES(V, VT)                                                               \
    int64_t b200_minres_fused_work_size_##V(const b200_ctx* ctx);                              \
    b200_status b200_minres_fused_init_##V(b200_ctx* ctx, VT* sc, int32_t* ctl,                \
                                           int64_t max_iters, int32_t res_kind,                \
                                           int32_t iter_first, int32_t baseline,               \
                                           VT reduction_factor);                               \
    b200_status b200_minres_fused_lanczos_##V(b200_ctx* ctx, int64_t n, VT* v, const VT* q,    \
                                              const VT* inv_diag, VT* sc, const int32_t* ctl,  \
                                              VT* work);                                       \
    b200_status b200_minres_fused_update_##V(b200_ctx* ctx, int64_t n, VT* x, VT* p0, VT* p1,  \
                                             VT* z, VT* q, VT* v, const VT* inv_diag, VT* sc,  \
                                             int32_t* ctl);
#define B200_DECL_SPMV_SUB_DOT(V, VT, I, IT)                                                   \
    b200_status b200_csr_spmv_sub_dot_##V##_##I(                                               \
        b200_ctx* ctx, const b200_csr_plan* plan, int64_t num_rows, int64_t num_cols,          \
        int64_t nnz, const IT* row_ptrs, const IT* col_idxs, const VT* values, const VT* b,    \
        VT* c, VT* dot_out, VT* work, const int32_t* ctl);

B200_DECL_FMINRES(f64, double)
B200_DECL_FMINRES(f32, float)
B200_DECL_SPMV_SUB_DOT(f64, double, i32, int32_t)
B200_DECL_SPMV_SUB_DOT(f64, double, i64, int64_t)
B200_DECL_SPMV_SUB_DOT(f32, float, i32, int32_t)
B200_DECL_SPMV_SUB_DOT(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused MINRES iteration for k = 2..32 right-hand sides (ginkgo_b200 extension behind
 * solver::Minres::apply with with_fused_multi_rhs(true), single GPU).  The regrouping of the fused
 * MINRES above with every vector n x k row-major (stride k) and every scalar per column; one matrix
 * pass per iteration serves all columns.  minres::step_1 / step_2 of a stopped column are skipped, as
 * the reference's kernels skip them by the column's stopping_status
 * (reference/solver/minres_kernels.cpp:64-150); d = inv_diag of a scalar Jacobi preconditioner, NULL
 * for Identity:
 *   spmv_sub_mdot  v = A z - v for all columns, alpha_j = z_j . v_j in the SpMV epilogue
 *                                     (Csr::apply(1, z, -1, v) with k columns + compute_conj_dot)
 *   lanczos        v_j -= alpha_j q_j (also for alpha_j == 0, as sub_scaled with a 1 x k alpha);
 *                  beta_j = v_j . (d v_j); then in the last CTA minres::step_1 of every running column
 *                               (sub_scaled + jacobi apply + compute_conj_dot + minres::step_1)
 *   update         minres::step_2 of every running column with z~ = d v recomputed and q_prev not
 *                  stored; p / p_prev are p0 / p1 as the parity of the shared iteration count says
 *                  (iteration i writes p1 when i is even, p0 when odd).  The last CTA swaps gamma /
 *                  beta and runs the criterion check of the next iteration on every running column
 *                  (std::swap(p, p_prev) + minres::step_2 + std::swap(gamma, beta) + criterion check)
 *   init           the first criterion check of every column, after the host's minres::initialize
 *                  with k columns; sc[4k + j] holds ||b_j|| (baseline 0) or ||r0_j|| (1) and is set to
 *                  1 for baseline 2
 * sc:     VT[16k]   sc[s*k + j]: s = 0 alpha, 1 beta, 2 gamma, 3 delta, 4 tau0, 5 threshold, 6 tau,
 *                   7 eta, 8 eta_next, 9 cos_prev, 10 cos, 11 sin_prev, 12 sin
 * status: uint8[k]  stopping_status byte of every column (0 = running)
 * ctl:    int32[8]  0 nonzero once every column has stopped, 1 iterations, 2 max_iters (-1 none),
 *                   3 res_kind (0 none, 2 ImplicitResidualNorm: sqrt|tau_j| <= threshold_j), 4 iter_first
 * Once ctl[0] != 0 every kernel is a no-op, so graphs of several iterations can be replayed and the
 * host polls ctl after each.  `work` has b200_minres_mrhs_work_size(k) elements.
 *
 * b200_csr_spmv_sub_mdot: c = A b - c for the k columns of the row-major b and c (stride k; square A,
 * b also the dot operand) and dots[j] = b_j . c_j.  c is bit-identical to b200_csr_advanced_spmv with
 * (alpha, beta) = (1, -1) and num_rhs = k; the dots are summed in a fixed order.  ctl may be NULL; with
 * num_rows == 0 the dots are 0.  No plan and no alignment are required.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FMINRESM(V, VT)                                                              \
    int64_t b200_minres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k);                    \
    b200_status b200_minres_mrhs_init_##V(b200_ctx* ctx, int64_t k, VT* sc, uint8_t* status,   \
                                          int32_t* ctl, int64_t max_iters, int32_t res_kind,   \
                                          int32_t iter_first, int32_t baseline,                \
                                          VT reduction_factor);                                \
    b200_status b200_minres_mrhs_lanczos_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v,       \
                                             const VT* q, const VT* inv_diag, VT* sc,          \
                                             const uint8_t* status, const int32_t* ctl,        \
                                             VT* work);                                        \
    b200_status b200_minres_mrhs_update_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x,        \
                                            VT* p0, VT* p1, VT* z, VT* q, VT* v,               \
                                            const VT* inv_diag, VT* sc, uint8_t* status,       \
                                            int32_t* ctl);
#define B200_DECL_SPMV_SUB_MDOT(V, VT, I, IT)                                                  \
    b200_status b200_csr_spmv_sub_mdot_##V##_##I(                                              \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t nnz, const IT* row_ptrs,    \
        const IT* col_idxs, const VT* values, const VT* b, int64_t k, VT* c, VT* dots,         \
        VT* work, const int32_t* ctl);

B200_DECL_FMINRESM(f64, double)
B200_DECL_FMINRESM(f32, float)
B200_DECL_SPMV_SUB_MDOT(f64, double, i32, int32_t)
B200_DECL_SPMV_SUB_MDOT(f64, double, i64, int64_t)
B200_DECL_SPMV_SUB_MDOT(f32, float, i32, int32_t)
B200_DECL_SPMV_SUB_MDOT(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused CG iteration for k = 2..32 right-hand sides (ginkgo_b200 extension behind solver::Cg::apply
 * with with_fused_multi_rhs(true), single GPU).  The regrouping of the fused CG above with every
 * vector n x k row-major (stride k) and every scalar per column; one matrix pass per iteration
 * serves all columns.  The element-wise steps of a stopped column are skipped, as the reference's
 * cg::step_1 / step_2 skip them by the column's stopping_status
 * (common/unified/solver/cg_kernels.cpp:74,99):
 *   step_p     p_j = z_j + (rho_j/prev_rho_j) p_j; p_j = z_j if prev_rho_j == 0   (cg::step_1)
 *   spmv_mdot  q = A p for all columns, pq_j = p_j . q_j in the SpMV epilogue
 *                                                (Csr::apply with k columns + compute_conj_dot)
 *   step_xr    alpha_j = rho_j/pq_j (no update if pq_j == 0); x_j += alpha_j p_j;
 *              r_j -= alpha_j q_j; z_j = M^-1 r_j (scalar Jacobi or identity); rho'_j = r_j . z_j;
 *              rr_j = r_j . r_j; the Iteration / (Implicit)ResidualNorm check of every running
 *              column                            (cg::step_2 + jacobi apply + dot + norm2 + check)
 *   init       r holds b - A x; p = q = 0; rho = prev_rho = 1; all columns running; z, rho, rr,
 *              each column's baseline and the first check        (cg::initialize + dot + check)
 * sc:     VT[6k]    sc[s*k + j]: s = 0 rho, 1 prev_rho, 2 pq, 3 rr, 4 tau0, 5 threshold
 * status: uint8[k]  stopping_status byte of every column (0 = running)
 * ctl:    int32[8]  0 nonzero once every column has stopped, 1 iterations, 2 max_iters,
 *                   3 res_kind (0 none, 1 ResidualNorm, 2 ImplicitResidualNorm), 4 iter_first
 * Once ctl[0] != 0 every kernel is a no-op, so graphs of several iterations can be replayed and the
 * host polls ctl after each.  `work` has b200_cg_mrhs_work_size(k) elements.  baseline: 0 rhs_norm
 * (caller stores ||b_j|| in sc[4k + j] first), 1 initial_resnorm, 2 absolute.
 *
 * b200_csr_spmv_mdot: c = A b for the k columns of the row-major b and c (stride k; square A, b
 * also the dot operand) and dots[j] = b_j . c_j.  c is bit-identical to b200_csr_spmv with
 * num_rhs = k; the dots are summed in a fixed order.  ctl may be NULL; with num_rows == 0 the dots
 * are 0.  No plan and no alignment are required.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FCGM(V, VT)                                                                  \
    int64_t b200_cg_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k);                        \
    b200_status b200_cg_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, VT* z, \
                                      VT* p, VT* q, const VT* inv_diag, VT* sc,                \
                                      uint8_t* status, int32_t* ctl, VT* work,                 \
                                      int64_t max_iters, int32_t res_kind, int32_t iter_first, \
                                      int32_t baseline, VT reduction_factor);                  \
    b200_status b200_cg_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p,            \
                                        const VT* z, const VT* sc, const uint8_t* status,      \
                                        const int32_t* ctl);                                   \
    b200_status b200_cg_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x, VT* r,    \
                                         const VT* p, const VT* q, VT* z, const VT* inv_diag,  \
                                         VT* sc, uint8_t* status, int32_t* ctl, VT* work);
#define B200_DECL_SPMV_MDOT(V, VT, I, IT)                                                      \
    b200_status b200_csr_spmv_mdot_##V##_##I(                                                  \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t nnz, const IT* row_ptrs,    \
        const IT* col_idxs, const VT* values, const VT* b, int64_t k, VT* c, VT* dots,         \
        VT* work, const int32_t* ctl);

B200_DECL_FCGM(f64, double)
B200_DECL_FCGM(f32, float)
B200_DECL_SPMV_MDOT(f64, double, i32, int32_t)
B200_DECL_SPMV_MDOT(f64, double, i64, int64_t)
B200_DECL_SPMV_MDOT(f32, float, i32, int32_t)
B200_DECL_SPMV_MDOT(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused BiCGStab iteration for k = 2..32 right-hand sides (ginkgo_b200 extension behind
 * solver::Bicgstab::apply with with_fused_multi_rhs(true), single GPU).  The regrouping of the fused
 * BiCGStab above with every vector n x k row-major (stride k) and every scalar per column; each SpMV
 * is one matrix pass for all columns.  The element-wise steps of a stopped column are skipped, as the
 * reference's bicgstab::step_1/2/3 skip them by the column's stopping_status
 * (reference/solver/bicgstab_kernels.cpp:65-178); d = inv_diag of a scalar Jacobi preconditioner,
 * NULL for Identity:
 *   step_p     p_j = r_j + (rho_j/prev_rho_j*alpha_j/omega_j)(p_j - omega_j v_j),
 *              p_j = r_j if prev_rho_j*omega_j == 0; y_j = d.p_j     (bicgstab::step_1 + jacobi apply)
 *   spmv_mdot2 v = A y for all columns, beta_j = rr_j . v_j        (Csr::apply + compute_conj_dot)
 *   step_s     alpha_j = rho_j/beta_j (0 and s_j = r_j if beta_j == 0); s_j = r_j - alpha_j v_j;
 *              z_j = d.s_j; ||s_j||^2; the mid-iteration check of every running column, which does
 *              not set the finalized bit     (bicgstab::step_2 + norm2 + criterion check + jacobi apply)
 *   spmv_mdot2 t = A z, gamma_j = s_j . t_j and beta_j = t_j . t_j (Csr::apply + 2 compute_conj_dot)
 *   step_xr    omega_j = gamma_j/beta_j (0 if beta_j == 0); x_j += alpha_j y_j + omega_j z_j;
 *              r_j = s_j - omega_j t_j; rho_j = rr_j . r_j; ||r_j||^2; rho / prev_rho shifted; the
 *              top-of-iteration check of every running column; a column stopped at this iteration's
 *              mid check gets only x_j += alpha_j y_j and its finalized bit
 *                                 (bicgstab::step_3 + finalize + dot + norm2 + criterion check)
 *   init       r holds b - A x; rr = r; p = v = y = s = t = z = 0; rho = prev_rho = alpha = beta =
 *              gamma = omega = 1; all columns running; rho, ||r||^2, each column's baseline and the
 *              first check                              (bicgstab::initialize + dot + norm2 + check)
 * sc:     VT[10k]   sc[s*k + j]: s = 0 rho, 1 prev_rho, 2 beta (rr.v, then t.t), 3 ||r||^2, 4 tau0,
 *                   5 threshold, 6 alpha, 7 omega, 8 gamma, 9 ||s||^2
 * status: uint8[k]  stopping_status byte of every column (0 = running)
 * ctl:    int32[8]  0 nonzero once every column has stopped, 1 iterations, 2 max_iters,
 *                   3 res_kind (0 none, 1 ResidualNorm, 2 ImplicitResidualNorm), 4 iter_first,
 *                   5 some column stopped at the mid check and owes its finalize
 * Once ctl[0] != 0 and ctl[5] == 0 every kernel is a no-op, so graphs of several iterations can be
 * replayed and the host polls ctl after each; every iteration ends with step_xr, which pays what a
 * mid-check stop owes.  `work` has b200_bicgstab_mrhs_work_size(k) elements.  baseline: 0 rhs_norm
 * (caller stores ||b_j|| in sc[4k + j] first), 1 initial_resnorm, 2 absolute.
 *
 * b200_csr_spmv_mdot2: c = A b for the k columns of the row-major b, c and w (stride k), dots[j] =
 * w_j . c_j and, unless dots2 is NULL, dots2[j] = c_j . c_j.  c is bit-identical to b200_csr_spmv
 * with num_rhs = k; the sums are added in a fixed order.  ctl may be NULL; with num_rows == 0 both
 * sums are 0.  No plan and no alignment are required.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FBICGSTABM(V, VT)                                                            \
    int64_t b200_bicgstab_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k);                  \
    b200_status b200_bicgstab_mrhs_init_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r,  \
                                            VT* rr, VT* p, VT* v, VT* y, VT* s, VT* t, VT* z,  \
                                            VT* sc, uint8_t* status, int32_t* ctl, VT* work,   \
                                            int64_t max_iters, int32_t res_kind,               \
                                            int32_t iter_first, int32_t baseline,              \
                                            VT reduction_factor);                              \
    b200_status b200_bicgstab_mrhs_step_p_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* p,      \
                                              const VT* r, const VT* v, VT* y,                 \
                                              const VT* inv_diag, const VT* sc,                \
                                              const uint8_t* status, const int32_t* ctl);      \
    b200_status b200_bicgstab_mrhs_step_s_##V(b200_ctx* ctx, int64_t n, int64_t k, const VT* r, \
                                              const VT* v, VT* s, VT* z, const VT* inv_diag,   \
                                              VT* sc, uint8_t* status, int32_t* ctl, VT* work); \
    b200_status b200_bicgstab_mrhs_step_xr_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* x,     \
                                               VT* r, const VT* s, const VT* t, const VT* y,   \
                                               const VT* z, const VT* rr, VT* sc,              \
                                               uint8_t* status, int32_t* ctl, VT* work);
#define B200_DECL_SPMV_MDOT2(V, VT, I, IT)                                                     \
    b200_status b200_csr_spmv_mdot2_##V##_##I(                                                 \
        b200_ctx* ctx, int64_t num_rows, int64_t num_cols, int64_t nnz, const IT* row_ptrs,    \
        const IT* col_idxs, const VT* values, const VT* b, int64_t k, VT* c, const VT* w,      \
        VT* dots, VT* dots2, VT* work, const int32_t* ctl);

B200_DECL_FBICGSTABM(f64, double)
B200_DECL_FBICGSTABM(f32, float)
B200_DECL_SPMV_MDOT2(f64, double, i32, int32_t)
B200_DECL_SPMV_MDOT2(f64, double, i64, int64_t)
B200_DECL_SPMV_MDOT2(f32, float, i32, int32_t)
B200_DECL_SPMV_MDOT2(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Fused GMRES iteration, modified Gram-Schmidt (ginkgo_b200 extension behind solver::Gmres::apply
 * with with_fused(true), single GPU; it regroups one iteration of core/solver/gmres.cpp:453-530 at
 * Krylov index j -- criterion check, preconditioner, SpMV, j+1 dots and sub_scaled, norm2,
 * inv_scale, hessenberg_qr -- into j + 3 launches (j + 4 with block Jacobi); every Hessenberg
 * entry, Givens rotation and residual estimate is produced and consumed on the device.  v_i is
 * Krylov basis i, w = basis j+1, hcol the Hessenberg column of iteration j (h_i = hcol[i]):
 *   scale        v_j = w / sc[0] if `divide` (the norm of the previous final pass: inv_scale);
 *                z = inv_diag . v_j unless inv_diag is NULL            (jacobi simple_scalar_apply)
 *   block_apply  z = M v_j for a block Jacobi M, SIMT kernel of b200_jacobi_simple_apply_* (and
 *                *_adaptive with block_precisions), one right-hand side, unit strides
 *   csr_spmv_dot2  w = A z, h_0 = v_0 . w                          (Csr::apply + compute_conj_dot)
 *   mgs_pass i   w -= h_{i-1} v_{i-1} (skipped for h == 0, as sub_scaled); h_i = v_i . w,
 *                i = 1..j                                     (sub_scaled + compute_conj_dot)
 *   final_pass   w -= coef[i] v_i for i = first..j in basis order (each as sub_scaled);
 *                h_{j+1} = ||w||, also kept in sc[0]; with haux != NULL first hcol[i] += haux[i],
 *                i <= j (add_scaled); the Givens update of b200_common_gmres_hessenberg_qr on hcol
 *                with iteration j (gsin, gcos, rnc, rnorm, fin, unit strides); then the criteria on
 *                tau = rnorm = |rnc[j+1]| for the top of iteration j+1.  MGS: first = j,
 *                coef = hcol                                  (sub_scaled + norm2 + hessenberg_qr
 *                                                              + criterion check)
 * CGS and CGS2 (krylov = v_0, bases at stride n):
 *   multi_dot    hcol[i] = v_i . w for i < num_bases, one pass (gmres multi_dot); CGS: bases
 *                1..j into hcol + 1 after the SpMV gave h_0
 *   final_pass   CGS: first = 0, coef = hcol (the loop's sub_all, then norm2 + hessenberg_qr)
 *   sub_pass     CGS2: w -= hcol[i] v_i, i = 0..j (sub_all), then multi_dot of bases 0..j into
 *                haux and final_pass with first = 0, coef = haux, haux = haux
 *   init         rnorm holds ||b - A x|| and v_0, rnc, fin, gsin, gcos are set by the loop's
 *                initialize / restart kernels; sets the baseline (sc[1] preset to ||b|| for
 *                rhs_norm), the threshold and runs the iteration-0 check
 * sc:  VT[8]    0 ||w|| of the last final pass, 1 tau0, 2 threshold = reduction_factor * tau0
 * ctl: int32[8] 0 stopping_status byte (0 = running), 1 iterations, 2 max_iters (-1 none),
 *               3 res_kind (0 none, 1 ResidualNorm), 4 iter_first
 * Stopping: Iteration and ResidualNorm in the user's order, ids 1 and 2, written WITHOUT the
 * finalized bit to ctl[0] and to the solver's stop_status byte `stop` (the final solve_krylov /
 * multi_axpy set it).  With ctl[0] != 0 every kernel above except init is a no-op.  `work` has
 * b200_gmres_fused_work_size elements; the passes share the ticket of the fused CG step kernels.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FGMRES(V, VT)                                                                \
    int64_t b200_gmres_fused_work_size_##V(const b200_ctx* ctx, int64_t krylov_dim);           \
    b200_status b200_gmres_fused_init_##V(b200_ctx* ctx, const VT* rnorm, VT* sc, int32_t* ctl, \
                                          uint8_t* stop, int64_t max_iters, int32_t res_kind,  \
                                          int32_t iter_first, int32_t baseline,                \
                                          VT reduction_factor);                                \
    b200_status b200_gmres_fused_scale_##V(b200_ctx* ctx, int64_t n, VT* v, VT* z,             \
                                           const VT* inv_diag, const VT* sc,                   \
                                           const int32_t* ctl, int32_t divide);                \
    b200_status b200_gmres_fused_mgs_pass_##V(b200_ctx* ctx, int64_t n, VT* w,                 \
                                              const VT* v_prev, const VT* v_i, VT* hcol,       \
                                              int64_t i, const int32_t* ctl, VT* work);        \
    b200_status b200_gmres_fused_sub_pass_##V(b200_ctx* ctx, int64_t n, VT* w,                 \
                                              const VT* krylov, const VT* coef, int64_t j,     \
                                              const int32_t* ctl);                             \
    b200_status b200_gmres_fused_final_pass_##V(                                               \
        b200_ctx* ctx, int64_t n, VT* w, const VT* krylov, int64_t first, const VT* coef,      \
        const VT* haux, VT* hcol, int64_t j, VT* gsin, VT* gcos, VT* rnorm, VT* rnc,           \
        uint64_t* fin, uint8_t* stop, VT* sc, int32_t* ctl, VT* work);                         \
    b200_status b200_gmres_fused_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t num_bases,    \
                                               const VT* krylov, const VT* w, VT* hcol,        \
                                               const int32_t* ctl, VT* work);
#define B200_DECL_FGMRES_BLOCK(V, VT, I, IT)                                                   \
    b200_status b200_gmres_fused_block_apply_##V##_##I(                                        \
        b200_ctx* ctx, int64_t num_blocks, int32_t max_block_size, int64_t block_offset,       \
        int64_t group_offset, int32_t group_power, const uint8_t* block_precisions,            \
        const IT* block_pointers, const VT* blocks, const VT* b, VT* x, const int32_t* ctl);

B200_DECL_FGMRES(f64, double)
B200_DECL_FGMRES(f32, float)

/* ---------------------------------------------------------------------------
 * Fused GMRES iteration for k = 2..32 right-hand sides (ginkgo_b200 extension behind
 * solver::Gmres::apply with with_fused_multi_rhs(true), single GPU): the entries above with every
 * vector n x k row-major (stride k) and every Hessenberg entry, Givens rotation and residual estimate
 * per column, in the loop's layout -- krylov n (kd+1) x k (basis i, column c at (i n + r) k + c),
 * hcol row j of the kd x (kd+1) k Hessenberg (h_i of column c at hcol[i k + c]), gsin, gcos, rnc,
 * haux, rnorm, fin of stride k -- so that the loop's initialize / restart / solve_krylov /
 * multi_axpy run on them with nrhs = k.  The SpMV is b200_csr_spmv_mdot2 with w = basis 0 and dots =
 * hcol (h_0), dots2 = NULL; it computes every column.  Every other kernel skips a stopped column:
 *   scale        v_j = w / sc[c] if `divide`; z = inv_diag . v_j unless inv_diag is NULL
 *   mgs_pass i   w -= h_{i-1} v_{i-1} (skipped for h == 0); h_i = v_i . w, i = 1..j
 *   multi_dot    hcol[i k + c] = v_i . w for i < num_bases (<= krylov_dim + 1), one pass over the
 *                bases for all columns
 *   sub_pass     w -= coef_i v_i, i = 0..j in basis order (CGS2's first subtraction)
 *   final_pass   w -= coef_i v_i for i = first..j; h_{j+1} = ||w||, kept in sc[c]; with haux !=
 *                NULL first h_i += haux_i, i <= j; the Givens update of hessenberg_qr for column c
 *                with iteration j; the criteria on tau_c = rnorm[c] = |rnc_c[j+1]| for the top of
 *                iteration j+1
 *   init         rnorm holds ||b_c - A x_c||; v_0, rnc, fin, gsin, gcos are set by the loop's
 *                initialize / restart; sets the baselines (sc[k + c] preset to ||b_c|| for
 *                rhs_norm), the thresholds, the statuses and runs the iteration-0 check
 * sc:     VT[3k]    sc[s*k + c]: s = 0 ||w|| of the last final pass, 1 tau0, 2 threshold
 * status: uint8[k]  stopping_status byte of every column (0 = running), WITHOUT the finalized bit
 * ctl:    int32[8]  0 nonzero once every column has stopped, 1 iterations, 2 max_iters (-1 none),
 *                   3 res_kind (0 none, 1 ResidualNorm), 4 iter_first
 * With ctl[0] != 0 every kernel but init is a no-op.  `work` has b200_gmres_mrhs_work_size(k,
 * krylov_dim) elements; the passes take ticket 2, the multi-dot ticket 3.
 * ------------------------------------------------------------------------- */
#define B200_DECL_FGMRESM(V, VT)                                                               \
    int64_t b200_gmres_mrhs_work_size_##V(const b200_ctx* ctx, int64_t k, int64_t krylov_dim); \
    b200_status b200_gmres_mrhs_init_##V(b200_ctx* ctx, int64_t k, const VT* rnorm, VT* sc,    \
                                         uint8_t* status, int32_t* ctl, int64_t max_iters,     \
                                         int32_t res_kind, int32_t iter_first,                 \
                                         int32_t baseline, VT reduction_factor);               \
    b200_status b200_gmres_mrhs_scale_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* v, VT* z,   \
                                          const VT* inv_diag, const VT* sc,                    \
                                          const uint8_t* status, const int32_t* ctl,           \
                                          int32_t divide);                                     \
    b200_status b200_gmres_mrhs_mgs_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w,       \
                                             const VT* v_prev, const VT* v_i, VT* hcol,        \
                                             int64_t i, const uint8_t* status,                 \
                                             const int32_t* ctl, VT* work);                    \
    b200_status b200_gmres_mrhs_multi_dot_##V(b200_ctx* ctx, int64_t n, int64_t k,             \
                                              int64_t num_bases, int64_t krylov_dim,           \
                                              const VT* krylov, const VT* w, VT* hcol,         \
                                              const uint8_t* status, const int32_t* ctl,       \
                                              VT* work);                                       \
    b200_status b200_gmres_mrhs_sub_pass_##V(b200_ctx* ctx, int64_t n, int64_t k, VT* w,       \
                                             const VT* krylov, const VT* coef, int64_t j,      \
                                             const uint8_t* status, const int32_t* ctl);       \
    b200_status b200_gmres_mrhs_final_pass_##V(                                                \
        b200_ctx* ctx, int64_t n, int64_t k, VT* w, const VT* krylov, int64_t first,           \
        const VT* coef, const VT* haux, VT* hcol, int64_t j, VT* gsin, VT* gcos, VT* rnorm,    \
        VT* rnc, uint64_t* fin, uint8_t* status, VT* sc, int32_t* ctl, VT* work);

B200_DECL_FGMRESM(f64, double)
B200_DECL_FGMRESM(f32, float)
B200_DECL_FGMRES_BLOCK(f64, double, i32, int32_t)
B200_DECL_FGMRES_BLOCK(f64, double, i64, int64_t)
B200_DECL_FGMRES_BLOCK(f32, float, i32, int32_t)
B200_DECL_FGMRES_BLOCK(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Integer-exact helpers either side of the SpMV path (SURVEY.md 8f rank 1):
 * components::convert_ptrs_to_idxs / convert_idxs_to_ptrs
 * (reference/components/format_conversion_kernels.cpp) and csr::extract_diagonal
 * (core/matrix/csr_kernels.hpp, reference/matrix/csr_kernels.cpp).
 * ------------------------------------------------------------------------- */
/* components::fill_array (core/components/fill_array_kernels.hpp:22-25): data[i] = *value_host
 * for n elements of elem_bytes (1, 2, 4, 8 or 16) bytes each; the value is read on the host
 * at call time. */
b200_status b200_fill_array(b200_ctx* ctx, void* data, int64_t n, const void* value_host,
                            int32_t elem_bytes);
#define B200_DECL_CONVERT_I(I, IT)                                                             \
    b200_status b200_convert_ptrs_to_idxs_##I(b200_ctx* ctx, const IT* ptrs, int64_t num_rows, \
                                              IT* idxs);                                       \
    b200_status b200_convert_idxs_to_ptrs_##I(b200_ctx* ctx, const IT* idxs, int64_t nnz,      \
                                              int64_t num_rows, IT* ptrs);
#define B200_DECL_EXTRACT_DIAG(V, VT, I, IT)                                                   \
    b200_status b200_csr_extract_diagonal_##V##_##I(b200_ctx* ctx, int64_t n,                  \
                                                    const IT* row_ptrs, const IT* col_idxs,    \
                                                    const VT* values, VT* diag);
B200_DECL_CONVERT_I(i32, int32_t)
B200_DECL_CONVERT_I(i64, int64_t)
B200_DECL_EXTRACT_DIAG(f64, double, i32, int32_t)
B200_DECL_EXTRACT_DIAG(f64, double, i64, int64_t)
B200_DECL_EXTRACT_DIAG(f32, float, i32, int32_t)
B200_DECL_EXTRACT_DIAG(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * CSR -> ELL / SELL-P / Hybrid on the device, and the in-row column sort (SURVEY.md 8f-1).
 * Bit-exact against the reference kernels:
 *   ell::compute_max_row_nnz (reference/matrix/ell_kernels.cpp:130-140; result on the host),
 *   csr::convert_to_ell (reference/matrix/csr_kernels.cpp:573-598),
 *   sellp::compute_slice_sets (reference/matrix/sellp_kernels.cpp:107-130; slice_sets has
 *   num_slices + 1 entries, slice_lengths num_slices, both size_type = uint64),
 *   csr::convert_to_sellp (reference/matrix/csr_kernels.cpp:528-567),
 *   csr::compute_hybrid_coo_row_ptrs + csr::convert_to_hybrid
 *   (core/matrix/csr.cpp:419-441, reference/matrix/csr_kernels.cpp:910-953; the ELL part is
 *   initialised for all ell_stride rows like the reference does),
 *   row_nnz_order_statistic: the sorted-row-length lookup of Hybrid's imbalance_limit
 *   strategy (include/ginkgo/core/matrix/hybrid.hpp:222-243),
 *   csr::sort_by_column_index (reference/matrix/csr_kernels.cpp:1272-1290; stable, i.e.
 *   identical to the reference for rows with distinct columns, which is all its unstable
 *   std::sort defines).
 * ------------------------------------------------------------------------- */
#define B200_DECL_CONVERT_FMT_I(I, IT)                                                         \
    b200_status b200_ell_compute_max_row_nnz_##I(b200_ctx* ctx, const IT* row_ptrs,            \
                                                 int64_t num_rows, int64_t* max_nnz_host);     \
    b200_status b200_sellp_compute_slice_sets_##I(                                             \
        b200_ctx* ctx, const IT* row_ptrs, int64_t num_rows, int64_t slice_size,               \
        int64_t stride_factor, uint64_t* slice_sets, uint64_t* slice_lengths);                 \
    b200_status b200_csr_compute_hybrid_coo_row_ptrs_##I(b200_ctx* ctx, const IT* row_ptrs,    \
                                                         int64_t num_rows, int64_t ell_lim,    \
                                                         int64_t* coo_row_ptrs);               \
    b200_status b200_csr_row_nnz_order_statistic_##I(b200_ctx* ctx, const IT* row_ptrs,        \
                                                     int64_t num_rows, int64_t k,              \
                                                     int64_t* value_host);
#define B200_DECL_CONVERT_FMT(V, VT, I, IT)                                                    \
    b200_status b200_csr_convert_to_ell_##V##_##I(                                             \
        b200_ctx* ctx, int64_t num_rows, const IT* row_ptrs, const IT* col_idxs,               \
        const VT* values, int64_t num_stored_per_row, int64_t ell_stride, IT* ell_col_idxs,    \
        VT* ell_values);                                                                       \
    b200_status b200_csr_convert_to_sellp_##V##_##I(                                           \
        b200_ctx* ctx, int64_t num_rows, int64_t slice_size, const uint64_t* slice_sets,       \
        const uint64_t* slice_lengths, const IT* row_ptrs, const IT* col_idxs,                 \
        const VT* values, IT* sellp_col_idxs, VT* sellp_values);                               \
    b200_status b200_csr_convert_to_hybrid_##V##_##I(                                          \
        b200_ctx* ctx, int64_t num_rows, const IT* row_ptrs, const IT* col_idxs,               \
        const VT* values, int64_t ell_lim, int64_t ell_stride, IT* ell_col_idxs,               \
        VT* ell_values, const int64_t* coo_row_ptrs, IT* coo_row_idxs, IT* coo_col_idxs,       \
        VT* coo_values);                                                                       \
    b200_status b200_csr_sort_by_column_index_##V##_##I(b200_ctx* ctx, int64_t num_rows,       \
                                                        const IT* row_ptrs, IT* col_idxs,      \
                                                        VT* values);
B200_DECL_CONVERT_FMT_I(i32, int32_t)
B200_DECL_CONVERT_FMT_I(i64, int64_t)
/* csr::is_sorted_by_column_index (core/matrix/csr_kernels.hpp; reference/matrix/csr_kernels.cpp):
 * *is_sorted_host = 1 iff every row's column indices are non-decreasing; blocking. */
b200_status b200_csr_is_sorted_by_column_index_i32(b200_ctx* ctx, int64_t num_rows,
                                                   const int32_t* row_ptrs, const int32_t* col_idxs,
                                                   int32_t* is_sorted_host);
b200_status b200_csr_is_sorted_by_column_index_i64(b200_ctx* ctx, int64_t num_rows,
                                                   const int64_t* row_ptrs, const int64_t* col_idxs,
                                                   int32_t* is_sorted_host);
B200_DECL_CONVERT_FMT(f64, double, i32, int32_t)
B200_DECL_CONVERT_FMT(f64, double, i64, int64_t)
B200_DECL_CONVERT_FMT(f32, float, i32, int32_t)
B200_DECL_CONVERT_FMT(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Multi-GPU (one process per GPU, 1-D row partition, NCCL over NVLink/NVSwitch):
 * the ginkgo_b200 replacement of the reference's MPI layer on this path --
 * experimental::distributed::Matrix::apply halo gather (core/distributed/matrix.cpp:450-509,
 * row_gatherer.cpp) and distributed::Vector reductions (core/distributed/vector.cpp:510-534).
 * All calls are enqueued on the context's stream and can be captured in CUDA graphs.
 * Extended vectors: [n_local owned entries | n_ghost received entries].
 * ------------------------------------------------------------------------- */
typedef struct b200_comm b200_comm;
typedef struct b200_halo b200_halo;
b200_status b200_comm_get_unique_id(uint8_t* id128); /* rank 0, then broadcast the 128 bytes */
b200_status b200_comm_create(b200_ctx* ctx, const uint8_t* id128, int32_t rank, int32_t nranks,
                             b200_comm** out);
void b200_comm_destroy(b200_comm* comm);
int32_t b200_comm_rank(const b200_comm* comm);
int32_t b200_comm_size(const b200_comm* comm);
b200_status b200_halo_create(b200_ctx* ctx, int32_t nranks, int64_t n_local, int64_t n_ghost,
                             const int64_t* send_counts, const int64_t* recv_counts,
                             const int32_t* send_idx_dev, int32_t value_bytes, b200_halo** out);
void b200_halo_destroy(b200_halo* halo);
int64_t b200_halo_num_ghost(const b200_halo* halo);
int64_t b200_halo_num_send(const b200_halo* halo);
/* Peer-memory data path (collective calls, set-up phase).  After enable_p2p the halo
 * exchange is two kernels -- pack+remote-store into the peers' landing slots over NVLink /
 * NVSwitch, and wait+unpack -- and all-reduces of <= 8 values are ONE single-CTA kernel that
 * stores into every peer's mailbox and sums in rank order (deterministic, identical bits on
 * every rank).  Windows are cudaMalloc blocks shared with cudaIpc*; synchronisation is by
 * epoch flags (st.release.sys / ld.acquire.sys), so everything stays CUDA-graph capturable.
 * Both return B200_ERR_COMM on EVERY rank alike when CUDA IPC is unavailable; the NCCL
 * send/recv + all-reduce path then remains in use.  p2p_error: 1 after a wait timed out.
 * Lifetime: the context outlives the communicator, the communicator outlives its halos
 * (exported blocks are only freed in b200_comm_destroy, after a barrier).
 * Slot reuse (two landing slots per halo) is safe when every exchanging pair of ranks sends in
 * both directions; b200_halo_enable_p2p checks the all-gathered counts and returns B200_ERR_COMM
 * (on every rank alike, the halo stays on NCCL) when some pair is coupled in one direction only. */
b200_status b200_comm_enable_p2p(b200_ctx* ctx, b200_comm* comm);
b200_status b200_halo_enable_p2p(b200_ctx* ctx, b200_comm* comm, b200_halo* halo);
int32_t b200_comm_p2p_enabled(const b200_comm* comm);
int32_t b200_halo_p2p_enabled(const b200_halo* halo);
b200_status b200_halo_exchange_staged_end(b200_ctx* ctx, b200_halo* halo);
b200_status b200_halo_counts(const b200_halo* halo, int64_t* recv_counts, int64_t* send_counts);
int32_t b200_comm_p2p_error(b200_ctx* ctx, const b200_comm* comm);
#define B200_DECL_COMM(V, VT)                                                                  \
    b200_status b200_comm_allreduce_sum_##V(b200_ctx* ctx, b200_comm* comm, VT* buf,           \
                                            int64_t count);                                    \
    b200_status b200_comm_allgather_##V(b200_ctx* ctx, b200_comm* comm, const VT* send,        \
                                        VT* recv, int64_t count_per_rank);                     \
    b200_status b200_halo_exchange_##V(b200_ctx* ctx, b200_comm* comm, b200_halo* halo,        \
                                       VT* x_ext, const int32_t* ctl);                         \
    /* the exchange without the landing-slot -> ghost-tail copy (peer memory, not capturable): */ \
    /* x_owned[0 .. n_local) goes to the peers (16-byte remote stores when every peer's send   */ \
    /* list is one contiguous run) and into this rank's extended vector inside the peer        */ \
    /* window; *x_ext_out = [owned | ghosts], valid until the exchange after the next one.     */ \
    /* B200_ERR_UNSUPPORTED without peer memory or after a captured exchange: use the call above */ \
    b200_status b200_halo_exchange_inplace_##V(b200_ctx* ctx, b200_comm* comm, b200_halo* halo, \
                                               const VT* x_owned, VT** x_ext_out);             \
    /* pipelined exchange (dense ghosts in contiguous runs, peer memory, not capturable): the push \
     * runs on its own stream in ring order (rank+1, rank+2, ...), flags[src] (device) reaches     \
     * *epoch_out when source src has landed in *x_ext_out; consume the owner blocks in arrival    \
     * order with b200_csr_spmv_part_*, then call b200_halo_exchange_staged_end */                 \
    b200_status b200_halo_exchange_staged_begin_##V(b200_ctx* ctx, b200_comm* comm, b200_halo* halo, \
                                                    const VT* x_owned, VT** x_ext_out,         \
                                                    const uint64_t** flags_out, uint64_t* epoch_out);
B200_DECL_COMM(f64, double)
B200_DECL_COMM(f32, float)
/* all-gather of raw device bytes (set-up exchanges of counts and index lists) */
b200_status b200_comm_allgather_bytes(b200_ctx* ctx, b200_comm* comm, const void* send, void* recv,
                                      int64_t bytes_per_rank);

/* dense::compute_sqrt (core/matrix/dense_kernels.hpp; reference/matrix/dense_kernels.cpp:440-448):
 * data = sqrt(data) element-wise -- the last step of a distributed norm2
 * (core/distributed/vector.cpp:520-534). */
b200_status b200_dense_compute_sqrt_f64(b200_ctx* ctx, int64_t rows, int64_t cols, double* data,
                                        int64_t stride);
b200_status b200_dense_compute_sqrt_f32(b200_ctx* ctx, int64_t rows, int64_t cols, float* data,
                                        int64_t stride);

/* ---------------------------------------------------------------------------
 * BiCG (SURVEY.md 8f rank 3) and the transposes it applies:
 *   bicg::initialize / step_1 / step_2   core/solver/bicg_kernels.hpp,
 *                                        reference/solver/bicg_kernels.cpp:25-118
 *   csr::transpose                       core/matrix/csr_kernels.hpp,
 *                                        reference/matrix/csr_kernels.cpp:694-731 (inside a row of
 *                                        the transpose: ordered by original row, then position)
 *   jacobi::transpose_jacobi             core/preconditioner/jacobi_kernels.hpp,
 *                                        reference/preconditioner/jacobi_kernels.cpp:597-627
 *                                        (full-precision storage; out_blocks has the layout of blocks)
 * ------------------------------------------------------------------------- */
#define B200_DECL_BICG(V, VT)                                                                            \
    b200_status b200_bicg_initialize_##V(                                                                \
        b200_ctx* ctx, int64_t rows, int64_t cols, const VT* b, int64_t bs, VT* r, int64_t rs, VT* z,    \
        int64_t zs, VT* p, int64_t ps, VT* q, int64_t qs, VT* prev_rho, VT* rho, VT* r2, int64_t r2s,    \
        VT* z2, int64_t z2s, VT* p2, int64_t p2s, VT* q2, int64_t q2s, uint8_t* stop);                   \
    b200_status b200_bicg_step_1_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* p, int64_t ps,       \
                                     const VT* z, int64_t zs, VT* p2, int64_t p2s, const VT* z2,         \
                                     int64_t z2s, const VT* rho, const VT* prev_rho,                     \
                                     const uint8_t* stop);                                               \
    b200_status b200_bicg_step_2_##V(b200_ctx* ctx, int64_t rows, int64_t cols, VT* x, int64_t xs,       \
                                     VT* r, int64_t rs, VT* r2, int64_t r2s, const VT* p, int64_t ps,    \
                                     const VT* q, int64_t qs, const VT* q2, int64_t q2s,                 \
                                     const VT* beta, const VT* rho, const uint8_t* stop);
B200_DECL_BICG(f64, double)
B200_DECL_BICG(f32, float)
#define B200_DECL_TRANSPOSE(V, VT, I, IT)                                                                \
    b200_status b200_csr_transpose_##V##_##I(b200_ctx* ctx, int64_t num_rows, int64_t num_cols,          \
                                             int64_t nnz, const IT* row_ptrs, const IT* col_idxs,        \
                                             const VT* values, IT* t_row_ptrs, IT* t_col_idxs,           \
                                             VT* t_values);                                              \
    b200_status b200_jacobi_transpose_##V##_##I(b200_ctx* ctx, int64_t num_blocks,                       \
                                                int32_t max_block_size, int64_t block_offset,            \
                                                int64_t group_offset, int32_t group_power,               \
                                                const IT* block_ptrs, const VT* blocks,                  \
                                                VT* out_blocks);
B200_DECL_TRANSPOSE(f64, double, i32, int32_t)
B200_DECL_TRANSPOSE(f64, double, i64, int64_t)
B200_DECL_TRANSPOSE(f32, float, i32, int32_t)
B200_DECL_TRANSPOSE(f32, float, i64, int64_t)

/* ---------------------------------------------------------------------------
 * Distributed set-up on the device (SURVEY.md 8f rank 4): what
 * experimental::distributed::Matrix::read_distributed runs before the first apply
 * (core/distributed/matrix.cpp:300-380).  G = global index type, L = local index type; the
 * (L, G) pairs are the reference's (int32, int32), (int32, int64), (int64, int64).  A partition
 * is passed as its arrays: range_bounds[num_ranges + 1], part_ids[num_ranges],
 * range_starting_indices[num_ranges], part_sizes[num_parts]
 * (include/ginkgo/core/distributed/partition.hpp:101-200).  `*_host` arguments are host
 * pointers, written after a stream synchronisation.  All results are bit-exact against the
 * reference kernels named below.
 *
 * partition:: (reference/distributed/partition_kernels.cpp)
 *   build_ranges_from_global_size :75-92   ranges[num_parts + 1], uniform split
 *   build_from_contiguous        :32-47   part_id_mapping may be NULL (part i owns range i)
 *   count_ranges / build_from_mapping :18-29, :52-70   one range per run of equal owners
 *   build_starting_indices       :97-113  local index of each range's first row + part sizes
 *   has_ordered_parts            :138-153
 * ------------------------------------------------------------------------- */
b200_status b200_partition_count_ranges(b200_ctx* ctx, int64_t n, const int32_t* mapping,
                                        int64_t* num_ranges_host);
b200_status b200_partition_has_ordered_parts(b200_ctx* ctx, int64_t num_ranges, const int32_t* part_ids,
                                             int32_t* result_host);
/* distributed_matrix::separate_local_nonlocal (reference/distributed/matrix_kernels.cpp:18-90)
 * in two steps.  classify_entries: cls[i] = 0 (row not owned by local_part), 1 (local column),
 * 2 (non-local column); local_rank / non_local_rank [nnz + 1] = exclusive counts, i.e. the
 * position of entry i in its output list (input order is kept, as in the reference);
 * num_local_host / num_non_local_host = their lengths.  separate_fill writes the reference's six arrays (rows
 * and local columns in local numbering, non-local columns still global); kept_fill writes all
 * entries of the owned rows in input order with global columns -- the input of a matrix in the
 * combined index space [local columns | remote columns].
 *
 * index_map (reference/distributed/index_map_kernels.cpp:20-105 build_mapping, :108-212
 * map_to_local).  The set of remote indices is a bitmap over the global index space
 * (global_size / 32 + 2 words) plus word_rank[words + 1], the number of set bits before each
 * word; the reference's "sort + unique by (part id, global index)" position of a connected
 * index g of range r is range_offsets[r] + (set bits of r below g).
 *   mark:  bit g set for every global_idxs[i]; skip_part >= 0 ignores indices that part owns
 *   rank:  word_rank, range_offsets[num_ranges], remote_sizes[num_parts] (entries received
 *          from each part), num_remote_host
 *   fill:  remote_global_idxs / remote_local_idxs (/ remote_part_ids, may be NULL), each
 *          num_remote long, ordered by (part id, global index)
 *   map_to_local: index_space 0 local, 1 non_local, 2 combined (non-local + local_size);
 *          -1 (invalid_index) where the reference returns it */
#define B200_DECL_DIST_G(G, GT)                                                                          \
    b200_status b200_partition_build_ranges_from_global_size_##G(b200_ctx* ctx, int32_t num_parts,       \
                                                                 int64_t global_size, GT* ranges);       \
    b200_status b200_partition_build_from_contiguous_##G(b200_ctx* ctx, int64_t num_ranges,              \
                                                         const GT* ranges,                               \
                                                         const int32_t* part_id_mapping,                 \
                                                         GT* range_bounds, int32_t* part_ids);           \
    b200_status b200_partition_build_from_mapping_##G(b200_ctx* ctx, int64_t n, const int32_t* mapping,  \
                                                      GT* range_bounds, int32_t* part_ids);              \
    b200_status b200_dist_classify_entries_##G(                                                          \
        b200_ctx* ctx, int64_t nnz, const GT* row_idxs, const GT* col_idxs, int64_t row_num_ranges,      \
        const GT* row_bounds, const int32_t* row_part_ids, int64_t col_num_ranges, const GT* col_bounds, \
        const int32_t* col_part_ids, int32_t local_part, uint8_t* cls, int64_t* local_rank,              \
        int64_t* non_local_rank, int64_t* num_local_host, int64_t* num_non_local_host);                  \
    b200_status b200_index_map_mark_##G(b200_ctx* ctx, int64_t global_size, int64_t num_ranges,          \
                                        const GT* bounds, const int32_t* part_ids, int32_t skip_part,    \
                                        int64_t m, const GT* global_idxs, uint32_t* bitmap);             \
    b200_status b200_index_map_rank_##G(b200_ctx* ctx, int64_t global_size, int64_t num_ranges,          \
                                        int32_t num_parts, const GT* bounds, const int32_t* part_ids,    \
                                        const uint32_t* bitmap, int64_t* word_rank,                      \
                                        int64_t* range_offsets, int64_t* remote_sizes,                   \
                                        int64_t* num_remote_host);
B200_DECL_DIST_G(i32, int32_t)
B200_DECL_DIST_G(i64, int64_t)
#define B200_DECL_DIST_LG(L, LT, G, GT)                                                                  \
    b200_status b200_partition_build_starting_indices_##L##_##G(                                         \
        b200_ctx* ctx, int64_t num_ranges, int32_t num_parts, const GT* range_bounds,                    \
        const int32_t* part_ids, LT* starting_indices, LT* part_sizes, int32_t* num_empty_parts_host);   \
    b200_status b200_index_map_fill_##L##_##G(                                                           \
        b200_ctx* ctx, int64_t global_size, int64_t num_ranges, const GT* bounds,                        \
        const int32_t* part_ids, const LT* starting, const uint32_t* bitmap, const int64_t* word_rank,   \
        const int64_t* range_offsets, GT* remote_global_idxs, LT* remote_local_idxs,                     \
        int32_t* remote_part_ids);                                                                       \
    b200_status b200_index_map_map_to_local_##L##_##G(                                                   \
        b200_ctx* ctx, int64_t global_size, int64_t num_ranges, const GT* bounds,                        \
        const int32_t* part_ids, const LT* starting, const uint32_t* bitmap, const int64_t* word_rank,   \
        const int64_t* range_offsets, int32_t rank, LT local_size, int32_t index_space, int64_t m,       \
        const GT* global_ids, LT* local_ids);
B200_DECL_DIST_LG(i32, int32_t, i32, int32_t)
B200_DECL_DIST_LG(i32, int32_t, i64, int64_t)
B200_DECL_DIST_LG(i64, int64_t, i64, int64_t)
#define B200_DECL_DIST_VLG(V, VT, L, LT, G, GT)                                                          \
    b200_status b200_dist_separate_fill_##V##_##L##_##G(                                                 \
        b200_ctx* ctx, int64_t nnz, const GT* row_idxs, const GT* col_idxs, const VT* values,            \
        int64_t row_num_ranges, const GT* row_bounds, const LT* row_starting, int64_t col_num_ranges,    \
        const GT* col_bounds, const LT* col_starting, const uint8_t* cls, const int64_t* local_rank,     \
        const int64_t* non_local_rank, LT* local_rows, LT* local_cols, VT* local_vals,                   \
        LT* non_local_rows, GT* non_local_cols, VT* non_local_vals);                                     \
    b200_status b200_dist_kept_fill_##V##_##L##_##G(                                                     \
        b200_ctx* ctx, int64_t nnz, const GT* row_idxs, const GT* col_idxs, const VT* values,            \
        int64_t row_num_ranges, const GT* row_bounds, const LT* row_starting, const uint8_t* cls,        \
        const int64_t* local_rank, const int64_t* non_local_rank, LT* rows, GT* cols, VT* vals);                                                                                                         \
    /* distributed_vector::build_local (reference/distributed/vector_kernels.cpp:15-40): scatter */     \
    /* the entries of local_part's rows into the pre-zeroed row-major local block; unique (row, */      \
    /* column) pairs, as for the reference's device backends */                                         \
    b200_status b200_dist_vector_build_local_##V##_##L##_##G(                                            \
        b200_ctx* ctx, int64_t nnz, const GT* row_idxs, const GT* col_idxs, const VT* values,            \
        int64_t num_ranges, const GT* bounds, const int32_t* part_ids, const LT* starting,               \
        int32_t local_part, VT* local_values, int64_t local_stride);
#define B200_DECL_DIST_VLG_ALL(V, VT)                     \
    B200_DECL_DIST_VLG(V, VT, i32, int32_t, i32, int32_t) \
    B200_DECL_DIST_VLG(V, VT, i32, int32_t, i64, int64_t) \
    B200_DECL_DIST_VLG(V, VT, i64, int64_t, i64, int64_t)
B200_DECL_DIST_VLG_ALL(f64, double)
B200_DECL_DIST_VLG_ALL(f32, float)

#ifdef __cplusplus
}
#endif
#endif /* GINKGO_B200_H_ */
