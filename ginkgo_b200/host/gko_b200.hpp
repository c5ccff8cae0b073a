// gko_b200.hpp -- C++ host side of the hand-written CUDA SpMV + Krylov hot path.
//
// Mirrors the reference's operator interface for this path (same class names,
// factory idiom, argument meaning and error behaviour) on top of the C ABI of
// include/ginkgo_b200.h:
//
//     auto exec = gko_b200::B200Executor::create(0);
//     auto A = gko_b200::matrix::Csr<double, int>::create(exec, dim2{n, n}, vals, cols, ptrs);
//     auto solver = gko_b200::solver::Cg<double>::build()
//                       .with_criteria(gko_b200::stop::Iteration::build().with_max_iters(1000u),
//                                      gko_b200::stop::ResidualNorm<double>::build()
//                                          .with_reduction_factor(1e-8))
//                       .with_preconditioner(gko_b200::preconditioner::Jacobi<double, int>::build()
//                                                .with_max_block_size(1u))
//                       .on(exec)->generate(A);
//     solver->apply(b, x);
//
// (`namespace gko = gko_b200;` makes reference user code read identically.)
// The solver loops are the reference's host loops (core/solver/{cg,bicgstab,gmres}.cpp),
// driving the drop-in step kernels; Cg additionally has the fused device-resident path
// (include/ginkgo_b200.h "Fused CG iteration").  Everything numerical happens in the
// CUDA library; this layer owns objects, workspaces and control flow only.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/ginkgo_b200.h"

#include "gko_b200_types.hpp"
#include "gko_b200_io.hpp"

namespace gko_b200 {

inline void check(b200_status st, const char* where)
{
    if (st == B200_OK) return;
    const std::string msg = std::string(where) + ": " + b200_last_error();
    switch (st) {
    case B200_ERR_ALLOC: throw AllocationError(msg);
    case B200_ERR_INVALID: throw BadDimension(msg);
    case B200_ERR_UNSUPPORTED: throw NotSupported(msg);
    default: throw CudaError(msg);
    }
}
#define GKOB_CALL(expr) ::gko_b200::check((expr), #expr)

// ---- C-ABI dispatch by value / index type ------------------------------------------------
template <typename V>
struct vabi;
template <typename V, typename I>
struct viabi;
#define GKOB_V(V, S)                                                                            \
    template <>                                                                                 \
    struct vabi<V> {                                                                            \
        static constexpr auto dot = b200_dense_compute_dot_##S;                                 \
        static constexpr auto conj_dot = b200_dense_compute_conj_dot_##S;                       \
        static constexpr auto norm2 = b200_dense_compute_norm2_##S;                             \
        static constexpr auto sqnorm2 = b200_dense_compute_squared_norm2_##S;                   \
        static constexpr auto add_scaled = b200_dense_add_scaled_##S;                           \
        static constexpr auto sub_scaled = b200_dense_sub_scaled_##S;                           \
        static constexpr auto scale = b200_dense_scale_##S;                                     \
        static constexpr auto inv_scale = b200_dense_inv_scale_##S;                             \
        static constexpr auto copy = b200_dense_copy_##S;                                       \
        static constexpr auto fill = b200_dense_fill_##S;                                       \
        static constexpr auto cg_initialize = b200_cg_initialize_##S;                           \
        static constexpr auto cg_step_1 = b200_cg_step_1_##S;                                   \
        static constexpr auto cg_step_2 = b200_cg_step_2_##S;                                   \
        static constexpr auto fcg_initialize = b200_fcg_initialize_##S;                         \
        static constexpr auto fcg_step_1 = b200_fcg_step_1_##S;                                 \
        static constexpr auto fcg_step_2 = b200_fcg_step_2_##S;                                 \
        static constexpr auto cgs_initialize = b200_cgs_initialize_##S;                         \
        static constexpr auto cgs_step_1 = b200_cgs_step_1_##S;                                 \
        static constexpr auto cgs_step_2 = b200_cgs_step_2_##S;                                 \
        static constexpr auto cgs_step_3 = b200_cgs_step_3_##S;                                 \
        static constexpr auto bicg_initialize = b200_bicg_initialize_##S;                       \
        static constexpr auto compute_sqrt = b200_dense_compute_sqrt_##S;                       \
        static constexpr auto bicg_step_1 = b200_bicg_step_1_##S;                               \
        static constexpr auto bicg_step_2 = b200_bicg_step_2_##S;                               \
        static constexpr auto pipe_cg_initialize_1 = b200_pipe_cg_initialize_1_##S;             \
        static constexpr auto pipe_cg_initialize_2 = b200_pipe_cg_initialize_2_##S;             \
        static constexpr auto pipe_cg_step_1 = b200_pipe_cg_step_1_##S;                         \
        static constexpr auto pipe_cg_step_2 = b200_pipe_cg_step_2_##S;                         \
        static constexpr auto gcr_initialize = b200_gcr_initialize_##S;                         \
        static constexpr auto gcr_restart = b200_gcr_restart_##S;                               \
        static constexpr auto gcr_step_1 = b200_gcr_step_1_##S;                                 \
        static constexpr auto minres_initialize = b200_minres_initialize_##S;                   \
        static constexpr auto minres_step_1 = b200_minres_step_1_##S;                           \
        static constexpr auto minres_step_2 = b200_minres_step_2_##S;                           \
        static constexpr auto chebyshev_init_update = b200_chebyshev_init_update_##S;           \
        static constexpr auto chebyshev_update = b200_chebyshev_update_##S;                     \
        static constexpr auto bicgstab_initialize = b200_bicgstab_initialize_##S;               \
        static constexpr auto bicgstab_step_1 = b200_bicgstab_step_1_##S;                       \
        static constexpr auto bicgstab_step_2 = b200_bicgstab_step_2_##S;                       \
        static constexpr auto bicgstab_step_3 = b200_bicgstab_step_3_##S;                       \
        static constexpr auto bicgstab_finalize = b200_bicgstab_finalize_##S;                   \
        static constexpr auto gmres_initialize = b200_common_gmres_initialize_##S;              \
        static constexpr auto gmres_hessenberg_qr = b200_common_gmres_hessenberg_qr_##S;        \
        static constexpr auto gmres_solve_krylov = b200_common_gmres_solve_krylov_##S;          \
        static constexpr auto gmres_restart = b200_gmres_restart_##S;                           \
        static constexpr auto gmres_multi_axpy = b200_gmres_multi_axpy_##S;                     \
        static constexpr auto gmres_multi_dot = b200_gmres_multi_dot_##S;                       \
        static constexpr auto residual_norm = b200_residual_norm_##S;                           \
        static constexpr auto implicit_residual_norm = b200_implicit_residual_norm_##S;         \
        static constexpr auto invert_diagonal = b200_jacobi_invert_diagonal_##S;                \
        static constexpr auto simple_scalar_apply = b200_jacobi_simple_scalar_apply_##S;        \
        static constexpr auto scalar_apply = b200_jacobi_scalar_apply_##S;                      \
        static constexpr auto fused_work_size = b200_cg_fused_work_size_##S;                    \
        static constexpr auto fused_init = b200_cg_fused_init_##S;                              \
        static constexpr auto fused_step_p = b200_cg_fused_step_p_##S;                          \
        static constexpr auto fused_step_xr = b200_cg_fused_step_xr_##S;                        \
        static constexpr auto fused_finish = b200_cg_fused_finish_##S;                          \
        static constexpr auto bicgstab_fused_init = b200_bicgstab_fused_init_##S;               \
        static constexpr auto bicgstab_fused_step_p = b200_bicgstab_fused_step_p_##S;           \
        static constexpr auto bicgstab_fused_step_s = b200_bicgstab_fused_step_s_##S;           \
        static constexpr auto bicgstab_fused_step_xr = b200_bicgstab_fused_step_xr_##S;         \
        static constexpr auto minres_fused_work_size = b200_minres_fused_work_size_##S;         \
        static constexpr auto minres_fused_init = b200_minres_fused_init_##S;                   \
        static constexpr auto minres_fused_lanczos = b200_minres_fused_lanczos_##S;             \
        static constexpr auto minres_fused_update = b200_minres_fused_update_##S;               \
        static constexpr auto minres_mrhs_work_size = b200_minres_mrhs_work_size_##S;           \
        static constexpr auto minres_mrhs_init = b200_minres_mrhs_init_##S;                     \
        static constexpr auto minres_mrhs_lanczos = b200_minres_mrhs_lanczos_##S;               \
        static constexpr auto minres_mrhs_update = b200_minres_mrhs_update_##S;                 \
        static constexpr auto gmres_fused_work_size = b200_gmres_fused_work_size_##S;           \
        static constexpr auto gmres_fused_init = b200_gmres_fused_init_##S;                     \
        static constexpr auto gmres_fused_scale = b200_gmres_fused_scale_##S;                   \
        static constexpr auto gmres_fused_mgs_pass = b200_gmres_fused_mgs_pass_##S;             \
        static constexpr auto gmres_fused_final_pass = b200_gmres_fused_final_pass_##S;         \
        static constexpr auto gmres_fused_sub_pass = b200_gmres_fused_sub_pass_##S;             \
        static constexpr auto gmres_fused_multi_dot = b200_gmres_fused_multi_dot_##S;           \
        static constexpr auto cg_mrhs_work_size = b200_cg_mrhs_work_size_##S;                   \
        static constexpr auto cg_mrhs_init = b200_cg_mrhs_init_##S;                             \
        static constexpr auto cg_mrhs_step_p = b200_cg_mrhs_step_p_##S;                         \
        static constexpr auto cg_mrhs_step_xr = b200_cg_mrhs_step_xr_##S;                       \
        static constexpr auto bicgstab_mrhs_work_size = b200_bicgstab_mrhs_work_size_##S;       \
        static constexpr auto bicgstab_mrhs_init = b200_bicgstab_mrhs_init_##S;                 \
        static constexpr auto bicgstab_mrhs_step_p = b200_bicgstab_mrhs_step_p_##S;             \
        static constexpr auto bicgstab_mrhs_step_s = b200_bicgstab_mrhs_step_s_##S;             \
        static constexpr auto bicgstab_mrhs_step_xr = b200_bicgstab_mrhs_step_xr_##S;           \
        static constexpr auto gmres_mrhs_work_size = b200_gmres_mrhs_work_size_##S;             \
        static constexpr auto gmres_mrhs_init = b200_gmres_mrhs_init_##S;                       \
        static constexpr auto gmres_mrhs_scale = b200_gmres_mrhs_scale_##S;                     \
        static constexpr auto gmres_mrhs_mgs_pass = b200_gmres_mrhs_mgs_pass_##S;               \
        static constexpr auto gmres_mrhs_multi_dot = b200_gmres_mrhs_multi_dot_##S;             \
        static constexpr auto gmres_mrhs_sub_pass = b200_gmres_mrhs_sub_pass_##S;               \
        static constexpr auto gmres_mrhs_final_pass = b200_gmres_mrhs_final_pass_##S;           \
    };
GKOB_V(double, f64)
GKOB_V(float, f32)
#define GKOB_VI(V, S, I, T)                                                                     \
    template <>                                                                                 \
    struct viabi<V, I> {                                                                        \
        static constexpr auto csr_plan_create = b200_csr_plan_create_##S##_##T;                 \
        static constexpr auto csr_plan_tune = b200_csr_plan_tune_##S##_##T;                     \
        static constexpr auto csr_plan_refresh_values = b200_csr_plan_refresh_values_##S##_##T; \
        static constexpr auto csr_plan_split_columns = b200_csr_plan_split_columns_##S##_##T;   \
        static constexpr auto csr_spmv_part = b200_csr_spmv_part_##S##_##T;                     \
        static constexpr auto csr_spmv = b200_csr_spmv_##S##_##T;                               \
        static constexpr auto csr_advanced_spmv = b200_csr_advanced_spmv_##S##_##T;             \
        static constexpr auto csr_spmv_dot = b200_csr_spmv_dot_##S##_##T;                       \
        static constexpr auto csr_spmv_dot2 = b200_csr_spmv_dot2_##S##_##T;                     \
        static constexpr auto csr_spmv_sub_dot = b200_csr_spmv_sub_dot_##S##_##T;               \
        static constexpr auto csr_spmv_mdot = b200_csr_spmv_mdot_##S##_##T;                     \
        static constexpr auto csr_spmv_sub_mdot = b200_csr_spmv_sub_mdot_##S##_##T;             \
        static constexpr auto csr_spmv_mdot2 = b200_csr_spmv_mdot2_##S##_##T;                   \
        static constexpr auto csr_extract_diagonal = b200_csr_extract_diagonal_##S##_##T;       \
        static constexpr auto csr_convert_to_ell = b200_csr_convert_to_ell_##S##_##T;           \
        static constexpr auto csr_convert_to_sellp = b200_csr_convert_to_sellp_##S##_##T;       \
        static constexpr auto csr_convert_to_hybrid = b200_csr_convert_to_hybrid_##S##_##T;     \
        static constexpr auto csr_sort_by_column_index = b200_csr_sort_by_column_index_##S##_##T; \
        static constexpr auto ell_compute_max_row_nnz = b200_ell_compute_max_row_nnz_##T;       \
        static constexpr auto sellp_compute_slice_sets = b200_sellp_compute_slice_sets_##T;     \
        static constexpr auto csr_compute_hybrid_coo_row_ptrs =                                 \
            b200_csr_compute_hybrid_coo_row_ptrs_##T;                                           \
        static constexpr auto csr_row_nnz_order_statistic = b200_csr_row_nnz_order_statistic_##T; \
        static constexpr auto convert_ptrs_to_idxs = b200_convert_ptrs_to_idxs_##T;             \
        static constexpr auto ell_spmv = b200_ell_spmv_##S##_##T;                               \
        static constexpr auto ell_advanced_spmv = b200_ell_advanced_spmv_##S##_##T;             \
        static constexpr auto sellp_spmv = b200_sellp_spmv_##S##_##T;                           \
        static constexpr auto sellp_advanced_spmv = b200_sellp_advanced_spmv_##S##_##T;         \
        static constexpr auto coo_plan_create = b200_coo_plan_create_##S##_##T;                 \
        static constexpr auto coo_spmv = b200_coo_spmv_##S##_##T;                               \
        static constexpr auto coo_advanced_spmv = b200_coo_advanced_spmv_##S##_##T;             \
        static constexpr auto coo_spmv2 = b200_coo_spmv2_##S##_##T;                             \
        static constexpr auto coo_advanced_spmv2 = b200_coo_advanced_spmv2_##S##_##T;           \
        static constexpr auto jacobi_simple_apply = b200_jacobi_simple_apply_##S##_##T;         \
        static constexpr auto jacobi_apply = b200_jacobi_apply_##S##_##T;                       \
        static constexpr auto jacobi_generate = b200_jacobi_generate_##S##_##T;                 \
        static constexpr auto jacobi_find_blocks = b200_jacobi_find_blocks_##T;                 \
        static constexpr auto csr_transpose = b200_csr_transpose_##S##_##T;                     \
        static constexpr auto jacobi_transpose = b200_jacobi_transpose_##S##_##T;               \
        static constexpr auto jacobi_generate_adaptive = b200_jacobi_generate_adaptive_##S##_##T; \
        static constexpr auto jacobi_simple_apply_adaptive =                                    \
            b200_jacobi_simple_apply_adaptive_##S##_##T;                                        \
        static constexpr auto jacobi_apply_adaptive = b200_jacobi_apply_adaptive_##S##_##T;     \
        static constexpr auto jacobi_transpose_adaptive =                                       \
            b200_jacobi_transpose_adaptive_##S##_##T;                                           \
        static constexpr auto gmres_fused_block_apply = b200_gmres_fused_block_apply_##S##_##T; \
    };
GKOB_VI(double, f64, int32, i32)
GKOB_VI(double, f64, int64, i64)
GKOB_VI(float, f32, int32, i32)
GKOB_VI(float, f32, int64, i64)

// ---- Executor (include/ginkgo/core/base/executor.hpp: CudaExecutor) ----------------------
class B200Executor : public std::enable_shared_from_this<B200Executor> {
public:
    static std::shared_ptr<B200Executor> create(int device_id = 0, void* cuda_stream = nullptr)
    {
        auto e = std::shared_ptr<B200Executor>(new B200Executor());
        GKOB_CALL(b200_ctx_create(device_id, cuda_stream, &e->ctx_));
        return e;
    }
    ~B200Executor() { b200_ctx_destroy(ctx_); }
    b200_ctx* ctx() const { return ctx_; }
    void* get_stream() const { return b200_ctx_stream(ctx_); }
    int get_device_id() const { return b200_ctx_device(ctx_); }
    int get_num_multiprocessor() const { return b200_ctx_num_sms(ctx_); }
    int64 launch_count() const { return b200_ctx_launch_count(ctx_); }
    void synchronize() const { GKOB_CALL(b200_synchronize(ctx_)); }
    template <typename T>
    T* alloc(size_type n) const
    {
        void* p = nullptr;
        GKOB_CALL(b200_alloc(ctx_, n * sizeof(T), &p));
        return static_cast<T*>(p);
    }
    void free(void* p) const noexcept { b200_free(ctx_, p); }
    template <typename T>
    void copy_from_host(T* dst, const T* src, size_type n) const
    {
        GKOB_CALL(b200_copy_h2d(ctx_, dst, src, n * sizeof(T)));
    }
    template <typename T>
    void copy_to_host(T* dst, const T* src, size_type n) const
    {
        GKOB_CALL(b200_copy_d2h(ctx_, dst, src, n * sizeof(T)));
    }
    template <typename T>
    void copy(T* dst, const T* src, size_type n) const
    {
        GKOB_CALL(b200_copy_d2d(ctx_, dst, src, n * sizeof(T)));
    }

private:
    B200Executor() = default;
    b200_ctx* ctx_ = nullptr;
};
using Executor = B200Executor;

// ---- array (include/ginkgo/core/base/array.hpp) ---------------------------------------------
template <typename T>
class array {
public:
    array() = default;
    array(std::shared_ptr<const Executor> exec, size_type n) : exec_(std::move(exec)), n_(n)
    {
        if (n) data_ = exec_->template alloc<T>(n);
        owns_ = true;
    }
    array(std::shared_ptr<const Executor> exec, const std::vector<T>& host) : array(exec, host.size())
    {
        if (n_) exec_->copy_from_host(data_, host.data(), n_);
    }
    static array view(std::shared_ptr<const Executor> exec, size_type n, T* device_ptr)
    {
        array a;
        a.exec_ = std::move(exec);
        a.n_ = n;
        a.data_ = device_ptr;
        a.owns_ = false;
        return a;
    }
    array(array&& o) noexcept { *this = std::move(o); }
    array& operator=(array&& o) noexcept
    {
        if (this != &o) {
            release();
            exec_ = std::move(o.exec_);
            data_ = o.data_;
            n_ = o.n_;
            owns_ = o.owns_;
            o.data_ = nullptr;
            o.n_ = 0;
            o.owns_ = false;
        }
        return *this;
    }
    array(const array&) = delete;
    array& operator=(const array&) = delete;
    ~array() { release(); }
    T* get_data() { return data_; }
    const T* get_const_data() const { return data_; }
    size_type get_size() const { return n_; }
    std::shared_ptr<const Executor> get_executor() const { return exec_; }
    std::vector<T> to_host() const
    {
        std::vector<T> h(n_);
        if (n_) exec_->copy_to_host(h.data(), data_, n_);
        return h;
    }

private:
    void release()
    {
        if (owns_ && data_ && exec_) exec_->free(data_);
        data_ = nullptr;
    }
    std::shared_ptr<const Executor> exec_;
    T* data_ = nullptr;
    size_type n_ = 0;
    bool owns_ = false;
};

// ---- LinOp (include/ginkgo/core/base/lin_op.hpp:129-215) ------------------------------------
class LinOp {
public:
    virtual ~LinOp() = default;
    const dim2& get_size() const { return size_; }
    std::shared_ptr<const Executor> get_executor() const { return exec_; }
    // include/ginkgo/core/base/lin_op.hpp `apply_uses_initial_guess`: true for the iterative
    // solvers (x is read as the starting point), false for matrices and preconditioners
    virtual bool apply_uses_initial_guess() const { return false; }
    // the operator whose rows this process holds: itself, or for a row-distributed operator its
    // local block [owned columns | ghost columns] (what a local preconditioner is generated from)
    virtual const LinOp* local_block() const { return this; }
    // x = op(b)
    void apply(const LinOp* b, LinOp* x) const
    {
        validate(b, x);
        apply_impl(b, x);
    }
    // x = alpha op(b) + beta x
    void apply(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const
    {
        validate(b, x);
        if (alpha->get_size().rows != 1 || alpha->get_size().cols != 1 ||
            beta->get_size().rows != 1 || beta->get_size().cols != 1)
            throw DimensionMismatch("apply: alpha and beta must be 1x1");
        apply_impl(alpha, b, beta, x);
    }
    // smart-pointer conveniences (std::unique_ptr / std::shared_ptr operands, as in the reference)
    template <typename P1, typename P2, typename = typename P1::element_type,
              typename = typename P2::element_type>
    void apply(const P1& b, const P2& x) const
    {
        apply(static_cast<const LinOp*>(b.get()), static_cast<LinOp*>(x.get()));
    }
    template <typename P0, typename P1, typename P2, typename P3,
              typename = typename P0::element_type, typename = typename P1::element_type,
              typename = typename P2::element_type, typename = typename P3::element_type>
    void apply(const P0& a, const P1& b, const P2& bt, const P3& x) const
    {
        apply(static_cast<const LinOp*>(a.get()), static_cast<const LinOp*>(b.get()),
              static_cast<const LinOp*>(bt.get()), static_cast<LinOp*>(x.get()));
    }

protected:
    LinOp(std::shared_ptr<const Executor> exec, dim2 size) : exec_(std::move(exec)), size_(size) {}
    virtual void apply_impl(const LinOp* b, LinOp* x) const = 0;
    virtual void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const = 0;
    void validate(const LinOp* b, const LinOp* x) const
    {
        if (size_.cols != b->get_size().rows || size_.rows != x->get_size().rows ||
            b->get_size().cols != x->get_size().cols)
            throw DimensionMismatch("LinOp::apply: operator " + std::to_string(size_.rows) + "x" +
                                    std::to_string(size_.cols) + ", b " +
                                    std::to_string(b->get_size().rows) + "x" +
                                    std::to_string(b->get_size().cols) + ", x " +
                                    std::to_string(x->get_size().rows) + "x" +
                                    std::to_string(x->get_size().cols));
    }
    std::shared_ptr<const Executor> exec_;
    dim2 size_;
};

// include/ginkgo/core/base/lin_op.hpp `Transposable` (real value types: conj_transpose == transpose)
class Transposable {
public:
    virtual ~Transposable() = default;
    virtual std::unique_ptr<LinOp> transpose() const = 0;
    virtual std::unique_ptr<LinOp> conj_transpose() const { return transpose(); }
};

class LinOpFactory {
public:
    virtual ~LinOpFactory() = default;
    virtual std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const = 0;
};

template <typename T, typename From>
const T* as(const From* p)
{
    auto r = dynamic_cast<const T*>(p);
    if (!r) throw NotSupported("operand has an unsupported type for this operation");
    return r;
}
template <typename T, typename From>
T* as(From* p)
{
    auto r = dynamic_cast<T*>(p);
    if (!r) throw NotSupported("operand has an unsupported type for this operation");
    return r;
}

namespace matrix {

// Sum over the ranks of a row-distributed vector: attached to a Dense that holds the LOCAL rows
// of a distributed vector (distributed::Vector), it completes compute_dot / compute_norm2 the way
// experimental::distributed::Vector does (core/distributed/vector.cpp:510-534: local kernel,
// all-reduce, square root).  Null for ordinary vectors.
template <typename V>
class reducer {
public:
    virtual ~reducer() = default;
    // in-place sum over all ranks of `count` device values (stream ordered)
    virtual void sum(V* device_values, size_type count) const = 0;
};

// ---- Dense (include/ginkgo/core/matrix/dense.hpp) ------------------------------------------
template <typename V>
class Dense : public LinOp {
public:
    using value_type = V;
    // a vector with `size` rows/cols on the same executor that reduces like this one
    // (Dense::create_with_config_of / create_with_type_of)
    std::unique_ptr<Dense> create_like(dim2 size) const
    {
        auto d = create(exec_, size);
        d->reducer_ = reducer_;
        return d;
    }
    void set_reducer(std::shared_ptr<const reducer<V>> r) { reducer_ = std::move(r); }
    const std::shared_ptr<const reducer<V>>& get_reducer() const { return reducer_; }
    static std::unique_ptr<Dense> create(std::shared_ptr<const Executor> exec, dim2 size = {},
                                         size_type stride = 0)
    {
        if (stride == 0) stride = size.cols;
        return std::unique_ptr<Dense>(
            new Dense(exec, size, array<V>(exec, size.rows * stride), stride));
    }
    static std::unique_ptr<Dense> create(std::shared_ptr<const Executor> exec, dim2 size,
                                         array<V> values, size_type stride)
    {
        return std::unique_ptr<Dense>(new Dense(exec, size, std::move(values), stride));
    }
    // non-owning view of device memory (array::view)
    static std::unique_ptr<Dense> create_view(std::shared_ptr<const Executor> exec, dim2 size,
                                              V* device_ptr, size_type stride)
    {
        return create(exec, size, array<V>::view(exec, size.rows * stride, device_ptr), stride);
    }
    static std::unique_ptr<Dense> create_from_host(std::shared_ptr<const Executor> exec, dim2 size,
                                                   const V* host_row_major)
    {
        auto d = create(exec, size);
        if (size.rows * size.cols != 0)
            exec->copy_from_host(d->get_values(), host_row_major, size.rows * size.cols);
        return d;
    }
    V* get_values() { return values_.get_data(); }
    const V* get_const_values() const { return values_.get_const_data(); }
    size_type get_stride() const { return stride_; }
    // ReadableFromMatrixData / WritableToMatrixData (core/matrix/dense.cpp `read`, :1074-1087
    // `write_impl`): zero-filled, entries scattered (later duplicates win); write lists the nonzeros
    template <typename I>
    void read(const matrix_data<V, I>& data)
    {
        std::vector<V> h(data.size.rows * data.size.cols, V(0));
        for (const auto& e : data.nonzeros) {
            if (e.row < 0 || (size_type)e.row >= data.size.rows || e.column < 0 ||
                (size_type)e.column >= data.size.cols)
                throw OutOfBounds("Dense::read: entry outside the matrix");
            h[(size_type)e.row * data.size.cols + (size_type)e.column] = e.value;
        }
        size_ = data.size;
        stride_ = data.size.cols;
        values_ = array<V>(exec_, h);
    }
    template <typename I>
    void write(matrix_data<V, I>& data) const
    {
        const auto h = to_host();
        data = matrix_data<V, I>(size_);
        for (size_type r = 0; r < size_.rows; ++r)
            for (size_type c = 0; c < size_.cols; ++c)
                if (h[r * size_.cols + c] != V(0)) data.nonzeros.push_back({(I)r, (I)c, h[r * size_.cols + c]});
    }
    std::vector<V> to_host() const
    {  // compact row-major copy
        std::vector<V> raw = values_.to_host();
        if (stride_ == size_.cols) return raw;
        std::vector<V> out(size_.rows * size_.cols);
        for (size_type i = 0; i < size_.rows; ++i)
            std::copy_n(raw.data() + i * stride_, size_.cols, out.data() + i * size_.cols);
        return out;
    }
    std::unique_ptr<Dense> clone() const
    {
        auto c = create(exec_, size_, stride_);
        c->reducer_ = reducer_;
        c->copy_from(this);
        return c;
    }
    // rows [r0, r1) as a view (create_submatrix with a full column span)
    std::unique_ptr<Dense> create_submatrix_rows(size_type r0, size_type r1)
    {
        auto v = create_view(exec_, dim2{r1 - r0, size_.cols}, get_values() + r0 * stride_, stride_);
        v->reducer_ = reducer_;
        return v;
    }
    std::unique_ptr<const Dense> create_submatrix_rows(size_type r0, size_type r1) const
    {
        auto v = create_view(exec_, dim2{r1 - r0, size_.cols},
                             const_cast<V*>(get_const_values()) + r0 * stride_, stride_);
        v->reducer_ = reducer_;
        return v;
    }
    void copy_from(const Dense* o)
    {
        require_same(o);
        GKOB_CALL(vabi<V>::copy(exec_->ctx(), size_.rows, size_.cols, o->get_const_values(),
                                o->get_stride(), get_values(), stride_));
    }
    void fill(V v)
    {
        GKOB_CALL(vabi<V>::fill(exec_->ctx(), size_.rows, size_.cols, get_values(), stride_, v));
    }
    void scale(const Dense* alpha)
    {
        GKOB_CALL(vabi<V>::scale(exec_->ctx(), size_.rows, size_.cols, alpha->get_const_values(),
                                 alpha_cols(alpha), get_values(), stride_));
    }
    void inv_scale(const Dense* alpha)
    {
        GKOB_CALL(vabi<V>::inv_scale(exec_->ctx(), size_.rows, size_.cols,
                                     alpha->get_const_values(), alpha_cols(alpha), get_values(),
                                     stride_));
    }
    void add_scaled(const Dense* alpha, const Dense* b)
    {
        require_same(b);
        GKOB_CALL(vabi<V>::add_scaled(exec_->ctx(), size_.rows, size_.cols,
                                      alpha->get_const_values(), alpha_cols(alpha),
                                      b->get_const_values(), b->get_stride(), get_values(), stride_));
    }
    void sub_scaled(const Dense* alpha, const Dense* b)
    {
        require_same(b);
        GKOB_CALL(vabi<V>::sub_scaled(exec_->ctx(), size_.rows, size_.cols,
                                      alpha->get_const_values(), alpha_cols(alpha),
                                      b->get_const_values(), b->get_stride(), get_values(), stride_));
    }
    void compute_dot(const Dense* b, Dense* result) const
    {
        require_same(b);
        require_row(result);
        GKOB_CALL(vabi<V>::dot(exec_->ctx(), size_.rows, size_.cols, get_const_values(), stride_,
                               b->get_const_values(), b->get_stride(), result->get_values()));
        if (reducer_) reducer_->sum(result->get_values(), size_.cols);
    }
    void compute_conj_dot(const Dense* b, Dense* result) const
    {
        require_same(b);
        require_row(result);
        GKOB_CALL(vabi<V>::conj_dot(exec_->ctx(), size_.rows, size_.cols, get_const_values(),
                                    stride_, b->get_const_values(), b->get_stride(),
                                    result->get_values()));
        if (reducer_) reducer_->sum(result->get_values(), size_.cols);
    }
    void compute_norm2(Dense* result) const
    {
        require_row(result);
        if (reducer_) {  // local squared norms, sum over the ranks, square root
            compute_squared_norm2(result);
            GKOB_CALL(vabi<V>::compute_sqrt(exec_->ctx(), 1, size_.cols, result->get_values(),
                                            result->get_stride()));
            return;
        }
        GKOB_CALL(vabi<V>::norm2(exec_->ctx(), size_.rows, size_.cols, get_const_values(), stride_,
                                 result->get_values()));
    }
    void compute_squared_norm2(Dense* result) const
    {
        require_row(result);
        GKOB_CALL(vabi<V>::sqnorm2(exec_->ctx(), size_.rows, size_.cols, get_const_values(),
                                   stride_, result->get_values()));
        if (reducer_) reducer_->sum(result->get_values(), size_.cols);
    }

protected:
    Dense(std::shared_ptr<const Executor> exec, dim2 size, array<V> values, size_type stride)
        : LinOp(std::move(exec), size), values_(std::move(values)), stride_(stride)
    {
        if (stride_ < size_.cols) throw BadDimension("Dense: stride smaller than the column count");
    }
    void apply_impl(const LinOp*, LinOp*) const override
    {
        throw NotSupported("Dense::apply (GEMM) is outside the SpMV + Krylov hot path");
    }
    void apply_impl(const LinOp*, const LinOp*, const LinOp*, LinOp*) const override
    {
        throw NotSupported("Dense::apply (GEMM) is outside the SpMV + Krylov hot path");
    }

private:
    int64 alpha_cols(const Dense* alpha) const
    {
        if (alpha->get_size().rows != 1 ||
            (alpha->get_size().cols != 1 && alpha->get_size().cols != size_.cols))
            throw DimensionMismatch("scaling factor must be 1x1 or 1xcols");
        return (int64)alpha->get_size().cols;
    }
    void require_same(const Dense* o) const
    {
        if (!(o->get_size() == size_)) throw DimensionMismatch("Dense: operand sizes differ");
    }
    void require_row(const Dense* r) const
    {
        if (r->get_size().rows != 1 || r->get_size().cols != size_.cols)
            throw DimensionMismatch("Dense: result must be 1 x cols");
    }
    array<V> values_;
    size_type stride_;
    std::shared_ptr<const reducer<V>> reducer_;
};

template <typename V>
std::unique_ptr<Dense<V>> initialize(std::initializer_list<V> vals,
                                     std::shared_ptr<const Executor> exec)
{
    std::vector<V> h(vals);
    return Dense<V>::create_from_host(exec, dim2{h.size(), 1}, h.data());
}
template <typename V>
std::unique_ptr<Dense<V>> scalar(V v, std::shared_ptr<const Executor> exec)
{
    return Dense<V>::create_from_host(exec, dim2{1, 1}, &v);
}

// ---- Csr (include/ginkgo/core/matrix/csr.hpp) ------------------------------------------------
template <typename V, typename I>
class Ell;
template <typename V, typename I>
class Sellp;
template <typename V, typename I>
class Coo;
template <typename V, typename I>
class Hybrid;

template <typename V, typename I>
class Csr : public LinOp, public Transposable {
public:
    using value_type = V;
    using index_type = I;
    static std::unique_ptr<Csr> create(std::shared_ptr<const Executor> exec, dim2 size,
                                       array<V> values, array<I> col_idxs, array<I> row_ptrs)
    {
        return std::unique_ptr<Csr>(new Csr(exec, size, std::move(values), std::move(col_idxs),
                                            std::move(row_ptrs)));
    }
    static std::unique_ptr<Csr> create_from_host(std::shared_ptr<const Executor> exec, dim2 size,
                                                 const std::vector<V>& values,
                                                 const std::vector<I>& col_idxs,
                                                 const std::vector<I>& row_ptrs)
    {
        return create(exec, size, array<V>(exec, values), array<I>(exec, col_idxs),
                      array<I>(exec, row_ptrs));
    }
    ~Csr() override { b200_csr_plan_destroy(plan_); }
    const V* get_const_values() const { return values_.get_const_data(); }
    // mutable access: the plan may hold a column-blocked copy of the values, refreshed on the next use
    V* get_values()
    {
        values_dirty_ = true;
        return values_.get_data();
    }
    const I* get_const_col_idxs() const { return col_idxs_.get_const_data(); }
    const I* get_const_row_ptrs() const { return row_ptrs_.get_const_data(); }
    size_type get_num_stored_elements() const { return values_.get_size(); }
    // the cached row partition (the reference's srow / strategy->process())
    const b200_csr_plan* get_plan() const
    {
        if (!plan_) {
            GKOB_CALL((viabi<V, I>::csr_plan_create(exec_->ctx(), size_.rows, values_.get_size(),
                                                    row_ptrs_.get_const_data(), &plan_)));
            // this class sees every mutable access to the values (get_values), so the plan may keep
            // its column-blocked value copy
            b200_csr_plan_allow_value_copy(plan_, 1);
            // strategy selection (reference: csr.hpp `automatical`), a function of the matrix
            GKOB_CALL((viabi<V, I>::csr_plan_tune(
                exec_->ctx(), plan_, size_.rows, size_.cols, values_.get_size(),
                row_ptrs_.get_const_data(), col_idxs_.get_const_data(), values_.get_const_data())));
            values_dirty_ = false;
        } else if (values_dirty_) {
            GKOB_CALL((viabi<V, I>::csr_plan_refresh_values(exec_->ctx(), plan_, size_.rows,
                                                            row_ptrs_.get_const_data(),
                                                            values_.get_const_data())));
            values_dirty_ = false;
        }
        return plan_;
    }
    // empty matrix, to be filled by read()
    static std::unique_ptr<Csr> create(std::shared_ptr<const Executor> exec)
    {
        return create(exec, dim2{}, array<V>(exec, 0), array<I>(exec, 0),
                      array<I>(exec, std::vector<I>{I(0)}));
    }
    // ReadableFromMatrixData / WritableToMatrixData (core/matrix/csr.cpp:558-582, :633-650):
    // `data` must be in row-major order (read_raw and friends deliver it that way)
    void read(const matrix_data<V, I>& data)
    {
        std::vector<V> va;
        std::vector<I> ci, rp;
        csr_arrays_from_matrix_data(data, rp, ci, va);
        b200_csr_plan_destroy(plan_);
        plan_ = nullptr;
        size_ = data.size;
        values_ = array<V>(exec_, va);
        col_idxs_ = array<I>(exec_, ci);
        row_ptrs_ = array<I>(exec_, rp);
    }
    void write(matrix_data<V, I>& data) const
    {
        data = matrix_data_from_csr_arrays(size_, row_ptrs_.to_host(), col_idxs_.to_host(),
                                           values_.to_host());
    }
    // Csr::convert_to(Ell|Sellp|Coo|Hybrid) and sort_by_column_index on the device
    // (core/matrix/csr.cpp:285-300, :419-530, :1402); defined in gko_b200_convert.hpp
    void convert_to(Ell<V, I>* result) const;
    void convert_to(Sellp<V, I>* result) const;
    void convert_to(Coo<V, I>* result) const;
    void convert_to(Hybrid<V, I>* result) const;
    void sort_by_column_index();
    // Csr::transpose (core/matrix/csr.cpp:1097-1107): rows of the result ordered like the
    // reference's (by original row, then position), on the device
    std::unique_ptr<LinOp> transpose() const override
    {
        const size_type nnz = get_num_stored_elements();
        array<V> tv(exec_, nnz);
        array<I> tc(exec_, nnz), tr(exec_, size_.cols + 1);
        GKOB_CALL((viabi<V, I>::csr_transpose(exec_->ctx(), size_.rows, size_.cols, nnz, get_const_row_ptrs(),
                                              get_const_col_idxs(), get_const_values(), tr.get_data(),
                                              tc.get_data(), tv.get_data())));
        return create(exec_, dim2{size_.cols, size_.rows}, std::move(tv), std::move(tc), std::move(tr));
    }
    std::unique_ptr<Dense<V>> extract_diagonal() const
    {
        auto d = Dense<V>::create(exec_, dim2{std::min(size_.rows, size_.cols), 1});
        GKOB_CALL((viabi<V, I>::csr_extract_diagonal(exec_->ctx(), d->get_size().rows,
                                                     get_const_row_ptrs(), get_const_col_idxs(),
                                                     get_const_values(), d->get_values())));
        return d;
    }

protected:
    Csr(std::shared_ptr<const Executor> exec, dim2 size, array<V> values, array<I> col_idxs,
        array<I> row_ptrs)
        : LinOp(std::move(exec), size),
          values_(std::move(values)),
          col_idxs_(std::move(col_idxs)),
          row_ptrs_(std::move(row_ptrs))
    {
        if (row_ptrs_.get_size() != size_.rows + 1 || values_.get_size() != col_idxs_.get_size())
            throw BadDimension("Csr: inconsistent array sizes");
    }
    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::csr_spmv(exec_->ctx(), get_plan(), size_.rows, size_.cols,
                                         values_.get_size(), get_const_row_ptrs(),
                                         get_const_col_idxs(), get_const_values(),
                                         db->get_const_values(), db->get_stride(),
                                         db->get_size().cols, dx->get_values(), dx->get_stride())));
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::csr_advanced_spmv(
            exec_->ctx(), get_plan(), size_.rows, size_.cols, values_.get_size(),
            get_const_row_ptrs(), get_const_col_idxs(), get_const_values(),
            as<Dense<V>>(alpha)->get_const_values(), db->get_const_values(), db->get_stride(),
            db->get_size().cols, as<Dense<V>>(beta)->get_const_values(), dx->get_values(),
            dx->get_stride())));
    }

private:
    array<V> values_;
    array<I> col_idxs_;
    array<I> row_ptrs_;
    mutable b200_csr_plan* plan_ = nullptr;
    mutable bool values_dirty_ = false;
};

// ---- Ell / Sellp / Coo / Hybrid: device arrays in the reference's layouts ---------------------
template <typename V, typename I>
class Ell : public LinOp {
public:
    using value_type = V;
    using index_type = I;
    // ReadableFromMatrixData / WritableToMatrixData (gko_b200_convert.hpp): read = Csr::read +
    // Csr::convert_to on the device, write = the stored entries in row-major order
    void read(const matrix_data<V, I>& data);
    void write(matrix_data<V, I>& data) const;
    static std::unique_ptr<Ell> create(std::shared_ptr<const Executor> exec, dim2 size,
                                       size_type num_stored_per_row, size_type stride,
                                       array<V> values, array<I> col_idxs)
    {
        return std::unique_ptr<Ell>(new Ell(exec, size, num_stored_per_row, stride,
                                            std::move(values), std::move(col_idxs)));
    }
    // empty matrix, to be filled by Csr::convert_to
    static std::unique_ptr<Ell> create(std::shared_ptr<const Executor> exec)
    {
        return std::unique_ptr<Ell>(new Ell(exec, dim2{}, 0, 0, array<V>(exec, 0), array<I>(exec, 0)));
    }
    size_type get_num_stored_elements_per_row() const { return width_; }
    size_type get_stride() const { return stride_; }
    const V* get_const_values() const { return values_.get_const_data(); }
    const I* get_const_col_idxs() const { return col_idxs_.get_const_data(); }
    size_type get_num_stored_elements() const { return values_.get_size(); }

protected:
    friend class Csr<V, I>;
    friend class Hybrid<V, I>;
    Ell(std::shared_ptr<const Executor> exec, dim2 size, size_type w, size_type stride, array<V> v,
        array<I> c)
        : LinOp(std::move(exec), size), width_(w), stride_(stride), values_(std::move(v)),
          col_idxs_(std::move(c))
    {}
    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::ell_spmv(exec_->ctx(), size_.rows, size_.cols, width_, stride_,
                                         col_idxs_.get_const_data(), values_.get_const_data(),
                                         db->get_const_values(), db->get_stride(),
                                         db->get_size().cols, dx->get_values(), dx->get_stride())));
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::ell_advanced_spmv(
            exec_->ctx(), size_.rows, size_.cols, width_, stride_, col_idxs_.get_const_data(),
            values_.get_const_data(), as<Dense<V>>(alpha)->get_const_values(),
            db->get_const_values(), db->get_stride(), db->get_size().cols,
            as<Dense<V>>(beta)->get_const_values(), dx->get_values(), dx->get_stride())));
    }

private:
    size_type width_, stride_;
    array<V> values_;
    array<I> col_idxs_;
};

template <typename V, typename I>
class Sellp : public LinOp {
public:
    using value_type = V;
    using index_type = I;
    // ReadableFromMatrixData / WritableToMatrixData (gko_b200_convert.hpp): read = Csr::read +
    // Csr::convert_to on the device, write = the stored entries in row-major order
    void read(const matrix_data<V, I>& data);
    void write(matrix_data<V, I>& data) const;
    static std::unique_ptr<Sellp> create(std::shared_ptr<const Executor> exec, dim2 size,
                                         size_type slice_size, array<std::uint64_t> slice_sets,
                                         array<std::uint64_t> slice_lengths, array<V> values,
                                         array<I> col_idxs)
    {
        return std::unique_ptr<Sellp>(new Sellp(exec, size, slice_size, std::move(slice_sets),
                                                std::move(slice_lengths), std::move(values),
                                                std::move(col_idxs)));
    }
    // empty matrix with the reference's defaults (slice_size 64, stride_factor 1:
    // include/ginkgo/core/matrix/sellp.hpp), to be filled by Csr::convert_to
    static std::unique_ptr<Sellp> create(std::shared_ptr<const Executor> exec,
                                         size_type slice_size = 64, size_type stride_factor = 1)
    {
        auto r = std::unique_ptr<Sellp>(new Sellp(exec, dim2{}, slice_size,
                                                  array<std::uint64_t>(exec, 1),
                                                  array<std::uint64_t>(exec, 0), array<V>(exec, 0),
                                                  array<I>(exec, 0)));
        r->stride_factor_ = stride_factor;
        return r;
    }
    size_type get_slice_size() const { return slice_size_; }
    size_type get_stride_factor() const { return stride_factor_; }
    const std::uint64_t* get_const_slice_sets() const { return sets_.get_const_data(); }
    const std::uint64_t* get_const_slice_lengths() const { return lens_.get_const_data(); }
    const V* get_const_values() const { return values_.get_const_data(); }
    const I* get_const_col_idxs() const { return col_idxs_.get_const_data(); }
    size_type get_num_stored_elements() const { return values_.get_size(); }

protected:
    friend class Csr<V, I>;
    Sellp(std::shared_ptr<const Executor> exec, dim2 size, size_type ss, array<std::uint64_t> sets,
          array<std::uint64_t> lens, array<V> v, array<I> c)
        : LinOp(std::move(exec), size), slice_size_(ss), sets_(std::move(sets)),
          lens_(std::move(lens)), values_(std::move(v)), col_idxs_(std::move(c))
    {}
    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::sellp_spmv(
            exec_->ctx(), size_.rows, size_.cols, slice_size_, sets_.get_const_data(),
            lens_.get_const_data(), col_idxs_.get_const_data(), values_.get_const_data(),
            db->get_const_values(), db->get_stride(), db->get_size().cols, dx->get_values(),
            dx->get_stride())));
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        GKOB_CALL((viabi<V, I>::sellp_advanced_spmv(
            exec_->ctx(), size_.rows, size_.cols, slice_size_, sets_.get_const_data(),
            lens_.get_const_data(), col_idxs_.get_const_data(), values_.get_const_data(),
            as<Dense<V>>(alpha)->get_const_values(), db->get_const_values(), db->get_stride(),
            db->get_size().cols, as<Dense<V>>(beta)->get_const_values(), dx->get_values(),
            dx->get_stride())));
    }

private:
    size_type slice_size_;
    size_type stride_factor_ = 1;
    array<std::uint64_t> sets_, lens_;
    array<V> values_;
    array<I> col_idxs_;
};

template <typename V, typename I>
class Coo : public LinOp {
public:
    using value_type = V;
    using index_type = I;
    // ReadableFromMatrixData / WritableToMatrixData (gko_b200_convert.hpp): read = Csr::read +
    // Csr::convert_to on the device, write = the stored entries in row-major order
    void read(const matrix_data<V, I>& data);
    void write(matrix_data<V, I>& data) const;
    static std::unique_ptr<Coo> create(std::shared_ptr<const Executor> exec, dim2 size,
                                       array<V> values, array<I> col_idxs, array<I> row_idxs)
    {
        return std::unique_ptr<Coo>(
            new Coo(exec, size, std::move(values), std::move(col_idxs), std::move(row_idxs)));
    }
    static std::unique_ptr<Coo> create(std::shared_ptr<const Executor> exec)
    {
        return std::unique_ptr<Coo>(
            new Coo(exec, dim2{}, array<V>(exec, 0), array<I>(exec, 0), array<I>(exec, 0)));
    }
    ~Coo() override { b200_coo_plan_destroy(plan_); }
    const V* get_const_values() const { return values_.get_const_data(); }
    const I* get_const_col_idxs() const { return col_idxs_.get_const_data(); }
    const I* get_const_row_idxs() const { return row_idxs_.get_const_data(); }
    size_type get_num_stored_elements() const { return values_.get_size(); }
    // x += A b   /   x += alpha A b   (Coo::apply2, used by Hybrid)
    void apply2(const LinOp* b, LinOp* x) const { run(2, nullptr, b, nullptr, x); }
    void apply2(const LinOp* alpha, const LinOp* b, LinOp* x) const { run(3, alpha, b, nullptr, x); }

protected:
    friend class Csr<V, I>;
    friend class Hybrid<V, I>;
    Coo(std::shared_ptr<const Executor> exec, dim2 size, array<V> v, array<I> c, array<I> r)
        : LinOp(std::move(exec), size), values_(std::move(v)), col_idxs_(std::move(c)),
          row_idxs_(std::move(r))
    {}
    void apply_impl(const LinOp* b, LinOp* x) const override { run(0, nullptr, b, nullptr, x); }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        run(1, alpha, b, beta, x);
    }

private:
    void run(int mode, const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const
    {
        auto db = as<Dense<V>>(b);
        auto dx = as<Dense<V>>(x);
        const int64 nnz = values_.get_size();
        if (!plan_)
            GKOB_CALL((viabi<V, I>::coo_plan_create(exec_->ctx(), size_.rows, nnz,
                                                    row_idxs_.get_const_data(), &plan_)));
        auto ctx = exec_->ctx();
        const I* ri = row_idxs_.get_const_data();
        const I* ci = col_idxs_.get_const_data();
        const V* va = values_.get_const_data();
        const V* al = alpha ? as<Dense<V>>(alpha)->get_const_values() : nullptr;
        const V* be = beta ? as<Dense<V>>(beta)->get_const_values() : nullptr;
        const int64 nrhs = db->get_size().cols;
        switch (mode) {
        case 0:
            GKOB_CALL((viabi<V, I>::coo_spmv(ctx, plan_, size_.rows, size_.cols, nnz, ri, ci, va,
                                             db->get_const_values(), db->get_stride(), nrhs,
                                             dx->get_values(), dx->get_stride())));
            break;
        case 1:
            GKOB_CALL((viabi<V, I>::coo_advanced_spmv(ctx, plan_, size_.rows, size_.cols, nnz, ri,
                                                      ci, va, al, db->get_const_values(),
                                                      db->get_stride(), nrhs, be, dx->get_values(),
                                                      dx->get_stride())));
            break;
        case 2:
            GKOB_CALL((viabi<V, I>::coo_spmv2(ctx, plan_, size_.rows, size_.cols, nnz, ri, ci, va,
                                              db->get_const_values(), db->get_stride(), nrhs,
                                              dx->get_values(), dx->get_stride())));
            break;
        default:
            GKOB_CALL((viabi<V, I>::coo_advanced_spmv2(ctx, plan_, size_.rows, size_.cols, nnz, ri,
                                                       ci, va, al, db->get_const_values(),
                                                       db->get_stride(), nrhs, dx->get_values(),
                                                       dx->get_stride())));
        }
    }
    array<V> values_;
    array<I> col_idxs_, row_idxs_;
    mutable b200_coo_plan* plan_ = nullptr;
};

// Hybrid = ELL part + COO part (core/matrix/hybrid.cpp:175-201)
template <typename V, typename I>
class Hybrid : public LinOp {
public:
    using value_type = V;
    using index_type = I;
    // ReadableFromMatrixData / WritableToMatrixData (gko_b200_convert.hpp): read = Csr::read +
    // Csr::convert_to on the device, write = the stored entries in row-major order
    void read(const matrix_data<V, I>& data);
    void write(matrix_data<V, I>& data) const;
    static std::unique_ptr<Hybrid> create(std::shared_ptr<const Executor> exec,
                                          std::unique_ptr<Ell<V, I>> ell,
                                          std::unique_ptr<Coo<V, I>> coo)
    {
        return std::unique_ptr<Hybrid>(new Hybrid(exec, std::move(ell), std::move(coo)));
    }
    // How many entries per row go into the ELL part (include/ginkgo/core/matrix/
    // hybrid.hpp:188-352).  The sorted-row-length lookup of imbalance_limit is one device
    // order statistic instead of the reference's host std::sort.
    struct strategy_type {
        enum kind_t { column_limit_k, imbalance_limit_k, imbalance_bounded_limit_k } kind;
        size_type columns;
        double percent, ratio;
        size_type compute_ell_num_stored_elements_per_row(const Executor* exec, const I* row_ptrs,
                                                          size_type num_rows) const
        {
            if (kind == column_limit_k) return columns;
            if (num_rows == 0) return 0;
            const double pct = std::min(std::max(percent, 0.0), 1.0);
            const int64 k = pct < 1 ? (int64)(size_type)(num_rows * pct) : (int64)num_rows - 1;
            int64 v = 0;
            GKOB_CALL((viabi<V, I>::csr_row_nnz_order_statistic(exec->ctx(), row_ptrs, num_rows, k, &v)));
            if (kind == imbalance_bounded_limit_k)
                return std::min((size_type)v, (size_type)(num_rows * ratio));
            return (size_type)v;
        }
    };
    static strategy_type column_limit(size_type num_columns = 0)
    {
        return {strategy_type::column_limit_k, num_columns, 0.0, 0.0};
    }
    static strategy_type imbalance_limit(double percent = 0.8)
    {
        return {strategy_type::imbalance_limit_k, 0, percent, 0.0};
    }
    static strategy_type imbalance_bounded_limit(double percent = 0.8, double ratio = 0.0001)
    {
        return {strategy_type::imbalance_bounded_limit_k, 0, percent, ratio};
    }
    static strategy_type minimal_storage_limit()
    {
        return imbalance_limit(static_cast<double>(sizeof(I)) / (sizeof(V) + 2 * sizeof(I)));
    }
    static strategy_type automatic() { return imbalance_bounded_limit(1.0 / 3.0, 0.001); }
    // empty matrix, to be filled by Csr::convert_to
    static std::unique_ptr<Hybrid> create(std::shared_ptr<const Executor> exec,
                                          strategy_type strategy = automatic())
    {
        auto r = std::unique_ptr<Hybrid>(new Hybrid(exec, Ell<V, I>::create(exec), Coo<V, I>::create(exec)));
        r->strategy_ = strategy;
        return r;
    }
    const Ell<V, I>* get_ell() const { return ell_.get(); }
    const Coo<V, I>* get_coo() const { return coo_.get(); }
    size_type get_ell_num_stored_elements_per_row() const { return ell_->get_num_stored_elements_per_row(); }
    size_type get_ell_stride() const { return ell_->get_stride(); }
    size_type get_coo_num_stored_elements() const { return coo_->get_num_stored_elements(); }
    const strategy_type& get_strategy() const { return strategy_; }

protected:
    friend class Csr<V, I>;
    Hybrid(std::shared_ptr<const Executor> exec, std::unique_ptr<Ell<V, I>> ell,
           std::unique_ptr<Coo<V, I>> coo)
        : LinOp(std::move(exec), ell->get_size()), ell_(std::move(ell)), coo_(std::move(coo))
    {}
    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        ell_->apply(b, x);
        coo_->apply2(b, x);
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        ell_->apply(alpha, b, beta, x);
        coo_->apply2(alpha, b, x);
    }

private:
    std::unique_ptr<Ell<V, I>> ell_;
    std::unique_ptr<Coo<V, I>> coo_;
    strategy_type strategy_ = automatic();
};

// matrix::Identity: apply == copy (default preconditioner of the solvers)
template <typename V>
class Identity : public LinOp, public Transposable {
public:
    static std::unique_ptr<Identity> create(std::shared_ptr<const Executor> exec, size_type n)
    {
        return std::unique_ptr<Identity>(new Identity(exec, n));
    }
    std::unique_ptr<LinOp> transpose() const override { return create(exec_, size_.rows); }

protected:
    Identity(std::shared_ptr<const Executor> exec, size_type n) : LinOp(std::move(exec), dim2{n, n}) {}
    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        as<Dense<V>>(x)->copy_from(as<Dense<V>>(b));
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        auto dx = as<Dense<V>>(x);
        dx->scale(as<Dense<V>>(beta));
        dx->add_scaled(as<Dense<V>>(alpha), as<Dense<V>>(b));
    }
};

}  // namespace matrix

template <typename V>
using Vec = matrix::Dense<V>;

// ---- small conveniences of the reference's user code -------------------------------------------
// gko::share (include/ginkgo/core/base/utils_helper.hpp): unique -> shared ownership
template <typename T>
std::shared_ptr<T> share(std::unique_ptr<T>&& p)
{
    return std::shared_ptr<T>(std::move(p));
}
// gko::clone of a vector
template <typename V>
std::unique_ptr<matrix::Dense<V>> clone(const matrix::Dense<V>* v)
{
    return v->clone();
}
template <typename V>
std::unique_ptr<matrix::Dense<V>> clone(const std::unique_ptr<matrix::Dense<V>>& v)
{
    return v->clone();
}
// gko::initialize<Matrix>({...}, exec) (include/ginkgo/core/matrix/dense.hpp `initialize`): a column
// vector from a flat list, a matrix from a list of rows; sparse formats drop the zeros like the
// reference's Dense -> format conversion does
namespace detail {
template <typename M>
struct is_dense : std::false_type {};
template <typename V>
struct is_dense<matrix::Dense<V>> : std::true_type {};
template <typename M>
struct index_of {
    using type = typename M::index_type;
};
template <typename V>
struct index_of<matrix::Dense<V>> {
    using type = int32;
};
}  // namespace detail
template <typename Matrix>
std::unique_ptr<Matrix> initialize(
    std::initializer_list<std::initializer_list<typename Matrix::value_type>> rows,
    std::shared_ptr<const Executor> exec)
{
    using V = typename Matrix::value_type;
    const size_type nr = rows.size(), nc = nr ? rows.begin()->size() : 0;
    std::vector<V> flat;
    flat.reserve(nr * nc);
    for (const auto& r : rows) {
        if (r.size() != nc) throw BadDimension("initialize: rows of different length");
        flat.insert(flat.end(), r.begin(), r.end());
    }
    if constexpr (detail::is_dense<Matrix>::value) {
        return Matrix::create_from_host(exec, dim2{nr, nc}, flat.data());
    } else {
        using I = typename detail::index_of<Matrix>::type;
        matrix_data<V, I> data(dim2{nr, nc});
        for (size_type i = 0; i < nr; ++i)
            for (size_type j = 0; j < nc; ++j)
                if (flat[i * nc + j] != V(0)) data.nonzeros.push_back({(I)i, (I)j, flat[i * nc + j]});
        auto m = Matrix::create(exec);
        m->read(data);
        return m;
    }
}
template <typename Matrix>
std::unique_ptr<Matrix> initialize(std::initializer_list<typename Matrix::value_type> column,
                                   std::shared_ptr<const Executor> exec)
{
    using V = typename Matrix::value_type;
    static_assert(detail::is_dense<Matrix>::value, "a flat list initialises a column vector");
    std::vector<V> h(column);
    return Matrix::create_from_host(exec, dim2{h.size(), 1}, h.data());
}

// gko::read / read_binary / read_generic / write / write_binary
// (include/ginkgo/core/base/mtx_io.hpp:150-320) for Dense and the five sparse formats
template <typename MatrixType, typename StreamType>
std::unique_ptr<MatrixType> read(StreamType&& is, std::shared_ptr<const Executor> exec)
{
    auto mtx = MatrixType::create(std::move(exec));
    mtx->read(read_raw<typename MatrixType::value_type, typename detail::index_of<MatrixType>::type>(is));
    return mtx;
}
template <typename MatrixType, typename StreamType>
std::unique_ptr<MatrixType> read_binary(StreamType&& is, std::shared_ptr<const Executor> exec)
{
    auto mtx = MatrixType::create(std::move(exec));
    mtx->read(read_binary_raw<typename MatrixType::value_type, typename detail::index_of<MatrixType>::type>(is));
    return mtx;
}
template <typename MatrixType, typename StreamType>
std::unique_ptr<MatrixType> read_generic(StreamType&& is, std::shared_ptr<const Executor> exec)
{
    auto mtx = MatrixType::create(std::move(exec));
    mtx->read(read_generic_raw<typename MatrixType::value_type, typename detail::index_of<MatrixType>::type>(is));
    return mtx;
}
template <typename MatrixType, typename StreamType>
void write(StreamType&& os, const MatrixType* mtx, layout_type layout = layout_type::coordinate)
{
    matrix_data<typename MatrixType::value_type, typename detail::index_of<MatrixType>::type> data;
    mtx->write(data);
    write_raw(os, data, layout);
}
template <typename MatrixType, typename StreamType>
void write_binary(StreamType&& os, const MatrixType* mtx)
{
    matrix_data<typename MatrixType::value_type, typename detail::index_of<MatrixType>::type> data;
    mtx->write(data);
    write_binary_raw(os, data);
}

}  // namespace gko_b200

#include "gko_b200_convert.hpp"
#include "gko_b200_staging.hpp"
#include "gko_b200_solvers.hpp"
