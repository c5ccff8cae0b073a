// gko_b200_solvers.hpp -- preconditioner::Jacobi, stop::*, solver::{Cg,Bicgstab,Gmres}.
// Included by gko_b200.hpp.
#pragma once

#include <chrono>
#include <functional>

namespace gko_b200 {

// =============================================================================================
// stop:: criteria (include/ginkgo/core/stop/*.hpp, core/stop/*.cpp)
// =============================================================================================
namespace stop {

enum class mode { absolute, initial_resnorm, rhs_norm };

struct CriterionArgs {
    std::shared_ptr<const LinOp> system_matrix;
    const LinOp* b = nullptr;
    const LinOp* x = nullptr;
    const LinOp* initial_residual = nullptr;
};

// what Criterion::Updater carries (include/ginkgo/core/stop/criterion.hpp)
struct Updater {
    size_type num_iterations = 0;
    const LinOp* residual = nullptr;
    const LinOp* residual_norm = nullptr;
    const LinOp* implicit_sq_residual_norm = nullptr;
    const LinOp* solution = nullptr;
    // core/stop/criterion.hpp `ignore_residual_check`: a ResidualNorm criterion that is handed
    // no residual norm reports "not converged" instead of computing one
    bool ignore_residual_check = false;
};

class Criterion {
public:
    virtual ~Criterion() = default;
    // returns true if all right-hand sides have stopped
    virtual bool check(uint8 stopping_id, bool set_finalized, array<uint8>* stop_status,
                       bool* one_changed, const Updater& u) = 0;
};

class CriterionFactory {
public:
    virtual ~CriterionFactory() = default;
    virtual std::unique_ptr<Criterion> generate(std::shared_ptr<const Executor> exec,
                                                const CriterionArgs& args) const = 0;
    // description used by the fused solver paths
    virtual int kind() const = 0;  // 0 iteration, 1 residual norm, 2 implicit residual norm
    virtual size_type max_iters() const { return 0; }
    virtual double reduction_factor() const { return 0; }
    virtual mode baseline() const { return mode::rhs_norm; }
};

// core/stop/iteration.cpp:14-24
class Iteration : public Criterion {
public:
    struct Factory : CriterionFactory {
        size_type max_iters_ = 0;
        Factory& with_max_iters(size_type n)
        {
            max_iters_ = n;
            return *this;
        }
        std::shared_ptr<const CriterionFactory> on(std::shared_ptr<const Executor>) const
        {
            return std::make_shared<Factory>(*this);
        }
        std::unique_ptr<Criterion> generate(std::shared_ptr<const Executor> exec,
                                            const CriterionArgs&) const override
        {
            return std::unique_ptr<Criterion>(new Iteration(exec, max_iters_));
        }
        int kind() const override { return 0; }
        size_type max_iters() const override { return max_iters_; }
    };
    static Factory build() { return Factory{}; }
    bool check(uint8 id, bool set_finalized, array<uint8>* stop_status, bool* one_changed,
               const Updater& u) override
    {
        const bool result = u.num_iterations >= max_iters_;
        if (result) {
            GKOB_CALL(b200_set_all_statuses(exec_->ctx(), stop_status->get_size(), id,
                                            set_finalized, stop_status->get_data()));
            *one_changed = true;
        }
        return result;
    }

private:
    Iteration(std::shared_ptr<const Executor> exec, size_type n) : exec_(exec), max_iters_(n) {}
    std::shared_ptr<const Executor> exec_;
    size_type max_iters_;
};

// core/stop/time.cpp:17-27, include/ginkgo/core/stop/time.hpp:24-58: wall-clock limit, the clock
// starts when the criterion is generated (i.e. at the beginning of a solve)
class Time : public Criterion {
public:
    using clock = std::chrono::steady_clock;
    struct Factory : CriterionFactory {
        std::chrono::nanoseconds time_limit_{10000000000LL};
        Factory& with_time_limit(std::chrono::nanoseconds t)
        {
            time_limit_ = t;
            return *this;
        }
        std::shared_ptr<const CriterionFactory> on(std::shared_ptr<const Executor>) const
        {
            return std::make_shared<Factory>(*this);
        }
        std::unique_ptr<Criterion> generate(std::shared_ptr<const Executor> exec,
                                            const CriterionArgs&) const override
        {
            return std::unique_ptr<Criterion>(new Time(exec, time_limit_));
        }
        int kind() const override { return 3; }  // host-side only: keeps the solver off the fused path
    };
    static Factory build() { return Factory{}; }
    bool check(uint8 id, bool set_finalized, array<uint8>* stop_status, bool* one_changed,
               const Updater&) override
    {
        const bool result = clock::now() - start_ >= time_limit_;
        if (result) {
            GKOB_CALL(b200_set_all_statuses(exec_->ctx(), stop_status->get_size(), id, set_finalized,
                                            stop_status->get_data()));
            *one_changed = true;
        }
        return result;
    }

private:
    Time(std::shared_ptr<const Executor> exec, std::chrono::nanoseconds limit)
        : exec_(exec), time_limit_(limit), start_(clock::now())
    {}
    std::shared_ptr<const Executor> exec_;
    std::chrono::nanoseconds time_limit_;
    clock::time_point start_;
};

// core/stop/residual_norm.cpp:91-228
template <typename V, bool IMPLICIT>
class ResidualNormBase : public Criterion {
public:
    struct Factory : CriterionFactory {
        double factor_ = 5 * std::numeric_limits<V>::epsilon();
        mode baseline_ = mode::rhs_norm;
        Factory& with_reduction_factor(double f)
        {
            factor_ = f;
            return *this;
        }
        Factory& with_baseline(mode m)
        {
            baseline_ = m;
            return *this;
        }
        std::shared_ptr<const CriterionFactory> on(std::shared_ptr<const Executor>) const
        {
            return std::make_shared<Factory>(*this);
        }
        std::unique_ptr<Criterion> generate(std::shared_ptr<const Executor> exec,
                                            const CriterionArgs& args) const override
        {
            return std::unique_ptr<Criterion>(new ResidualNormBase(exec, args, (V)factor_, baseline_));
        }
        int kind() const override { return IMPLICIT ? 2 : 1; }
        double reduction_factor() const override { return factor_; }
        mode baseline() const override { return baseline_; }
    };
    static Factory build() { return Factory{}; }

    bool check(uint8 id, bool set_finalized, array<uint8>* stop_status, bool* one_changed,
               const Updater& u) override
    {
        using Dense = matrix::Dense<V>;
        const Dense* tau = nullptr;
        if (IMPLICIT) {
            if (!u.implicit_sq_residual_norm) throw NotSupported("ImplicitResidualNorm needs rho");
            tau = as<Dense>(u.implicit_sq_residual_norm);
        } else if (u.residual_norm) {
            tau = as<Dense>(u.residual_norm);
        } else if (u.ignore_residual_check) {
            return false;  // core/stop/residual_norm.cpp:172-175
        } else if (u.residual) {
            as<Dense>(u.residual)->compute_norm2(u_tau_.get());
            tau = u_tau_.get();
        } else if (u.solution && system_matrix_ && b_) {
            auto r = as<Dense>(b_)->clone();
            system_matrix_->apply(neg_one_.get(), u.solution, one_.get(), r.get());
            r->compute_norm2(u_tau_.get());
            tau = u_tau_.get();
        } else {
            throw NotSupported("ResidualNorm: no residual information");
        }
        int32 all_conv = 0, changed = 0;
        auto fn = IMPLICIT ? vabi<V>::implicit_residual_norm : vabi<V>::residual_norm;
        GKOB_CALL(fn(exec_->ctx(), tau->get_size().cols, tau->get_const_values(),
                     starting_tau_->get_const_values(), factor_, id, set_finalized,
                     stop_status->get_data(), device_storage_.get_data(), &all_conv, &changed));
        *one_changed = changed != 0;
        return all_conv != 0;
    }

private:
    ResidualNormBase(std::shared_ptr<const Executor> exec, const CriterionArgs& args, V factor,
                     mode baseline)
        : exec_(exec), factor_(factor), device_storage_(exec, 2), system_matrix_(args.system_matrix),
          b_(args.b)
    {
        using Dense = matrix::Dense<V>;
        one_ = matrix::scalar<V>(V(1), exec);
        neg_one_ = matrix::scalar<V>(V(-1), exec);
        if (!args.b) throw NotSupported("ResidualNorm needs b");
        const size_type cols = args.b->get_size().cols;
        starting_tau_ = Dense::create(exec, dim2{1, cols});
        u_tau_ = Dense::create(exec, dim2{1, cols});
        switch (baseline) {
        case mode::initial_resnorm:
            if (args.initial_residual) {
                as<Dense>(args.initial_residual)->compute_norm2(starting_tau_.get());
            } else {
                if (!args.system_matrix || !args.x) throw NotSupported("initial_resnorm needs A, x");
                auto r = as<Dense>(args.b)->clone();
                args.system_matrix->apply(neg_one_.get(), args.x, one_.get(), r.get());
                r->compute_norm2(starting_tau_.get());
            }
            break;
        case mode::rhs_norm:
            as<Dense>(args.b)->compute_norm2(starting_tau_.get());
            break;
        case mode::absolute:
            starting_tau_->fill(V(1));
            break;
        }
    }
    std::shared_ptr<const Executor> exec_;
    V factor_;
    array<uint8> device_storage_;
    std::shared_ptr<const LinOp> system_matrix_;
    const LinOp* b_;
    std::unique_ptr<matrix::Dense<V>> starting_tau_, u_tau_, one_, neg_one_;
};
template <typename V>
using ResidualNorm = ResidualNormBase<V, false>;
template <typename V>
using ImplicitResidualNorm = ResidualNormBase<V, true>;

// core/stop/combined.cpp:33-52: ids 1, 2, ... in order, first converged criterion wins
class Combined : public Criterion {
public:
    explicit Combined(std::vector<std::unique_ptr<Criterion>> c) : criteria_(std::move(c)) {}
    bool check(uint8, bool set_finalized, array<uint8>* stop_status, bool* one_changed,
               const Updater& u) override
    {
        bool one_converged = false;
        uint8 ids = 1;
        *one_changed = false;
        for (auto& c : criteria_) {
            bool local = false;
            one_converged |= c->check(ids, set_finalized, stop_status, &local, u);
            *one_changed |= local;
            if (one_converged) break;
            ids++;
        }
        return one_converged;
    }

private:
    std::vector<std::unique_ptr<Criterion>> criteria_;
};

inline std::unique_ptr<Criterion> combine_and_generate(
    const std::vector<std::shared_ptr<const CriterionFactory>>& factories,
    std::shared_ptr<const Executor> exec, const CriterionArgs& args)
{
    if (factories.empty()) throw NotSupported("a solver needs at least one stopping criterion");
    if (factories.size() == 1) return factories[0]->generate(exec, args);
    std::vector<std::unique_ptr<Criterion>> c;
    for (auto& f : factories) c.push_back(f->generate(exec, args));
    return std::unique_ptr<Criterion>(new Combined(std::move(c)));
}

}  // namespace stop

// =============================================================================================
// preconditioner::Jacobi (include/ginkgo/core/preconditioner/jacobi.hpp, core/preconditioner/
// jacobi.cpp).  apply and generate run on the device; generate: scalar = extract_diagonal +
// invert_diagonal kernels; block = b200_jacobi_generate_* (the reference's pivoted
// Gauss-Jordan, reference/preconditioner/jacobi_kernels.cpp:113-410, in the reference's
// operation order); block pointers are user-supplied or detected by b200_jacobi_find_blocks_*
// (reference/preconditioner/jacobi_kernels.cpp:36-123).
// =============================================================================================
// gko::precision_reduction (include/ginkgo/core/base/types.hpp:239-350): how far the storage of a
// Jacobi block may be reduced -- `preserving` steps keep the exponent range (truncation), `nonpreserving`
// steps switch to the next smaller IEEE type; one byte, preserving << 4 | nonpreserving.
class precision_reduction {
public:
    constexpr precision_reduction() noexcept : data_(0) {}
    constexpr precision_reduction(uint8 preserving, uint8 nonpreserving) noexcept
        : data_((uint8)((preserving << 4) | nonpreserving))
    {}
    constexpr operator uint8() const noexcept { return data_; }
    constexpr uint8 get_preserving() const noexcept { return (uint8)(data_ >> 4); }
    constexpr uint8 get_nonpreserving() const noexcept { return (uint8)(data_ & 0xf); }
    static constexpr precision_reduction autodetect() noexcept { return from_byte(0xff); }
    static constexpr precision_reduction from_byte(uint8 b) noexcept
    {
        precision_reduction p;
        p.data_ = b;
        return p;
    }

private:
    uint8 data_;
};

namespace preconditioner {

template <typename I>
struct block_interleaved_storage_scheme {
    I block_offset = 0, group_offset = 0;
    uint32 group_power = 0;
    I get_group_size() const { return I(1) << group_power; }
    I get_stride() const { return block_offset << group_power; }
    I get_global_block_offset(I k) const
    {
        return group_offset * (k >> group_power) + block_offset * (k & (get_group_size() - 1));
    }
    size_type compute_storage_space(size_type num_blocks) const
    {
        const size_type gs = get_group_size();
        return (num_blocks + gs - 1) / gs * group_offset;
    }
};

template <typename V, typename I>
class Jacobi : public LinOp, public Transposable {
public:
    struct Factory : LinOpFactory {
        uint32 max_block_size_ = 32;
        std::vector<I> block_pointers_;
        // storage_optimization (jacobi.hpp:391-485): one reduction for all blocks, or block-wise
        // (replicated cyclically over the blocks, jacobi::initialize_precisions)
        bool so_block_wise_ = false;
        precision_reduction so_all_{};
        std::vector<precision_reduction> so_blocks_;
        double accuracy_ = 1e-1;  // jacobi.hpp:513
        std::shared_ptr<const Executor> exec_;
        Factory& with_storage_optimization(precision_reduction p)
        {
            so_block_wise_ = false;
            so_all_ = p;
            return *this;
        }
        Factory& with_storage_optimization(std::vector<precision_reduction> block_wise)
        {
            so_block_wise_ = true;
            so_blocks_ = std::move(block_wise);
            return *this;
        }
        Factory& with_accuracy(double a)
        {
            accuracy_ = a;
            return *this;
        }
        Factory& with_max_block_size(uint32 s)
        {
            max_block_size_ = s;
            return *this;
        }
        Factory& with_block_pointers(std::vector<I> p)
        {
            block_pointers_ = std::move(p);
            return *this;
        }
        std::shared_ptr<const LinOpFactory> on(std::shared_ptr<const Executor> exec) const
        {
            auto f = std::make_shared<Factory>(*this);
            f->exec_ = exec;
            return f;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            return std::unique_ptr<LinOp>(new Jacobi(exec_, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

    uint32 get_max_block_size() const { return max_block_size_; }
    size_type get_num_blocks() const { return num_blocks_; }
    const V* get_blocks() const { return blocks_.get_const_data(); }
    const I* get_const_block_pointers() const { return block_pointers_.get_const_data(); }
    const block_interleaved_storage_scheme<I>& get_storage_scheme() const { return scheme_; }
    // adaptive precision: condition numbers (device, num_blocks; nullptr without storage
    // optimisation, jacobi.hpp:254) and the precision every block was stored in (device bytes)
    const V* get_conditioning() const { return conditioning_.get_size() ? conditioning_.get_const_data() : nullptr; }
    const uint8* get_block_precisions() const
    {
        return precisions_.get_size() ? precisions_.get_const_data() : nullptr;
    }
    size_type get_num_stored_elements() const { return blocks_.get_size(); }
    // Jacobi::transpose (core/preconditioner/jacobi.cpp:261-283): same scheme and block
    // pointers, every inverted block transposed (a scalar Jacobi is its own transpose)
    std::unique_ptr<LinOp> transpose() const override
    {
        auto res = std::unique_ptr<Jacobi>(new Jacobi(exec_, size_, max_block_size_));
        res->num_blocks_ = num_blocks_;
        res->scheme_ = scheme_;
        res->blocks_ = array<V>(exec_, blocks_.get_size());
        if (max_block_size_ == 1) {
            if (blocks_.get_size())
                exec_->copy(res->blocks_.get_data(), blocks_.get_const_data(), blocks_.get_size());
            return res;
        }
        res->block_pointers_ = array<I>(exec_, block_pointers_.get_size());
        exec_->copy(res->block_pointers_.get_data(), block_pointers_.get_const_data(),
                    block_pointers_.get_size());
        GKOB_CALL(vabi<V>::fill(exec_->ctx(), blocks_.get_size(), 1, res->blocks_.get_data(), 1, V(0)));
        if (precisions_.get_size()) {
            res->precisions_ = array<uint8>(exec_, precisions_.get_size());
            exec_->copy(res->precisions_.get_data(), precisions_.get_const_data(), precisions_.get_size());
            res->conditioning_ = array<V>(exec_, conditioning_.get_size());
            exec_->copy(res->conditioning_.get_data(), conditioning_.get_const_data(), conditioning_.get_size());
            GKOB_CALL((viabi<V, I>::jacobi_transpose_adaptive(
                exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset, scheme_.group_offset,
                scheme_.group_power, precisions_.get_const_data(), block_pointers_.get_const_data(),
                blocks_.get_const_data(), res->blocks_.get_data())));
            return res;
        }
        GKOB_CALL((viabi<V, I>::jacobi_transpose(exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset,
                                                 scheme_.group_offset, scheme_.group_power,
                                                 block_pointers_.get_const_data(), blocks_.get_const_data(),
                                                 res->blocks_.get_data())));
        return res;
    }

protected:
    Jacobi(std::shared_ptr<const Executor> exec, dim2 size, uint32 max_block_size)
        : LinOp(exec, size), max_block_size_(max_block_size)
    {}
    // op: square, or the local block [owned columns | ghost columns] of a distributed matrix, whose
    // diagonal blocks lie in the owned columns
    Jacobi(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : LinOp(exec, dim2{op->get_size().rows, op->get_size().rows}), max_block_size_(f.max_block_size_)
    {
        if (op->local_block()->get_size().cols < op->get_size().rows)
            throw BadDimension("Jacobi: the matrix has fewer columns than rows");
        if (max_block_size_ < 1 || max_block_size_ > 32)
            throw NotSupported("Jacobi: max_block_size must be in [1, 32]");
        auto csr = as<matrix::Csr<V, I>>(op->local_block());
        const size_type n = size_.rows;
        if (max_block_size_ == 1) {
            auto diag = csr->extract_diagonal();
            blocks_ = array<V>(exec, n);
            GKOB_CALL(vabi<V>::invert_diagonal(exec->ctx(), n, diag->get_const_values(),
                                               blocks_.get_data()));
            num_blocks_ = n;
            return;
        }
        std::vector<I> ptrs = f.block_pointers_;
        if (ptrs.empty()) {
            // jacobi::find_blocks on the device (natural blocks + agglomeration)
            array<I> dev_ptrs(exec, n + 1);
            int64 nb = 0;
            GKOB_CALL((viabi<V, I>::jacobi_find_blocks(exec->ctx(), n, csr->get_const_row_ptrs(),
                                                       csr->get_const_col_idxs(),
                                                       (int32)max_block_size_, dev_ptrs.get_data(),
                                                       &nb)));
            ptrs.resize(nb + 1);
            exec->copy_to_host(ptrs.data(), dev_ptrs.get_const_data(), nb + 1);
        }
        num_blocks_ = ptrs.size() - 1;
        // compute_storage_scheme (jacobi.hpp:589-625)
        uint32 pow2 = 1;
        while (pow2 < max_block_size_) pow2 *= 2;
        const uint32 group_size = 32 / pow2;
        scheme_.block_offset = (I)max_block_size_;
        scheme_.group_offset = (I)(max_block_size_ * group_size * max_block_size_);
        scheme_.group_power = 0;
        while ((1u << scheme_.group_power) < group_size) ++scheme_.group_power;
        // extract + invert every diagonal block on the device (jacobi::generate)
        for (size_type k = 0; k < num_blocks_; ++k) {
            const I bs = ptrs[k + 1] - ptrs[k];
            if (bs < 1 || (uint32)bs > max_block_size_)
                throw BadDimension("Jacobi: block larger than max_block_size");
        }
        if ((size_type)ptrs.back() != n) throw BadDimension("Jacobi: block pointers do not cover the rows");
        const size_type space = scheme_.compute_storage_space(num_blocks_);
        blocks_ = array<V>(exec, space);
        GKOB_CALL(vabi<V>::fill(exec->ctx(), space, 1, blocks_.get_data(), 1, V(0)));
        block_pointers_ = array<I>(exec, ptrs);
        // adaptive variant (core/preconditioner/jacobi.cpp:380-401): the precision array is replicated
        // to one entry per block and the condition numbers are kept
        if (f.so_block_wise_ || (uint8)f.so_all_ != 0) {
            std::vector<uint8> src;
            if (f.so_block_wise_)
                for (auto p : f.so_blocks_) src.push_back((uint8)p);
            else
                src.push_back((uint8)f.so_all_);
            if (src.empty()) throw BadDimension("Jacobi: empty block-wise storage optimization");
            array<uint8> dsrc(exec, src);
            precisions_ = array<uint8>(exec, num_blocks_);
            GKOB_CALL(b200_jacobi_initialize_precisions(exec->ctx(), dsrc.get_const_data(), (int64)src.size(),
                                                        precisions_.get_data(), (int64)num_blocks_));
            conditioning_ = array<V>(exec, num_blocks_);
            GKOB_CALL((viabi<V, I>::jacobi_generate_adaptive(
                exec->ctx(), n, csr->get_const_row_ptrs(), csr->get_const_col_idxs(), csr->get_const_values(),
                num_blocks_, max_block_size_, f.accuracy_, scheme_.block_offset, scheme_.group_offset,
                scheme_.group_power, conditioning_.get_data(), precisions_.get_data(),
                block_pointers_.get_const_data(), blocks_.get_data())));
            return;
        }
        GKOB_CALL((viabi<V, I>::jacobi_generate(
            exec->ctx(), n, csr->get_const_row_ptrs(), csr->get_const_col_idxs(),
            csr->get_const_values(), num_blocks_, max_block_size_, scheme_.block_offset,
            scheme_.group_offset, scheme_.group_power, block_pointers_.get_const_data(),
            blocks_.get_data())));
    }

    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        auto db = as<matrix::Dense<V>>(b);
        auto dx = as<matrix::Dense<V>>(x);
        if (max_block_size_ == 1) {
            GKOB_CALL(vabi<V>::simple_scalar_apply(exec_->ctx(), size_.rows, db->get_size().cols,
                                                   blocks_.get_const_data(), db->get_const_values(),
                                                   db->get_stride(), dx->get_values(),
                                                   dx->get_stride()));
        } else if (precisions_.get_size()) {
            GKOB_CALL((viabi<V, I>::jacobi_simple_apply_adaptive(
                exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset, scheme_.group_offset,
                scheme_.group_power, precisions_.get_const_data(), block_pointers_.get_const_data(),
                blocks_.get_const_data(), db->get_const_values(), db->get_stride(), db->get_size().cols,
                dx->get_values(), dx->get_stride())));
        } else {
            GKOB_CALL((viabi<V, I>::jacobi_simple_apply(
                exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset,
                scheme_.group_offset, scheme_.group_power, block_pointers_.get_const_data(),
                blocks_.get_const_data(), db->get_const_values(), db->get_stride(),
                db->get_size().cols, dx->get_values(), dx->get_stride())));
        }
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        auto db = as<matrix::Dense<V>>(b);
        auto dx = as<matrix::Dense<V>>(x);
        const V* al = as<matrix::Dense<V>>(alpha)->get_const_values();
        const V* be = as<matrix::Dense<V>>(beta)->get_const_values();
        if (max_block_size_ == 1) {
            GKOB_CALL(vabi<V>::scalar_apply(exec_->ctx(), size_.rows, db->get_size().cols,
                                            blocks_.get_const_data(), al, db->get_const_values(),
                                            db->get_stride(), be, dx->get_values(),
                                            dx->get_stride()));
        } else if (precisions_.get_size()) {
            GKOB_CALL((viabi<V, I>::jacobi_apply_adaptive(
                exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset, scheme_.group_offset,
                scheme_.group_power, precisions_.get_const_data(), block_pointers_.get_const_data(),
                blocks_.get_const_data(), al, db->get_const_values(), db->get_stride(), db->get_size().cols, be,
                dx->get_values(), dx->get_stride())));
        } else {
            GKOB_CALL((viabi<V, I>::jacobi_apply(
                exec_->ctx(), num_blocks_, max_block_size_, scheme_.block_offset,
                scheme_.group_offset, scheme_.group_power, block_pointers_.get_const_data(),
                blocks_.get_const_data(), al, db->get_const_values(), db->get_stride(),
                db->get_size().cols, be, dx->get_values(), dx->get_stride())));
        }
    }

private:
    uint32 max_block_size_;
    size_type num_blocks_ = 0;
    block_interleaved_storage_scheme<I> scheme_;
    array<V> blocks_;
    array<I> block_pointers_;
    array<uint8> precisions_;  // adaptive variant only: one precision_reduction byte per block
    array<V> conditioning_;    // adaptive variant only
};

}  // namespace preconditioner

// =============================================================================================
// solver:: Cg / Bicgstab / Gmres (core/solver/{cg,bicgstab,gmres}.cpp)
// =============================================================================================
namespace solver {

namespace gmres {
enum class ortho_method { mgs, cgs, cgs2 };
}

// include/ginkgo/core/solver/solver_base.hpp:33-46: what a solver assumes about the x it is given
enum class initial_guess_mode { zero, rhs, provided };

template <typename V>
class SolverBase : public LinOp {
public:
    // what log::Convergence reports in the reference
    size_type get_num_iterations() const { return num_iterations_; }
    uint8 get_stop_status(size_type col = 0) const { return col < status_.size() ? status_[col] : 0; }
    bool has_converged() const
    {
        for (auto s : status_)
            if (!(s & 0x80)) return false;
        return !status_.empty();
    }
    std::shared_ptr<const LinOp> get_system_matrix() const { return system_matrix_; }
    std::shared_ptr<const LinOp> get_preconditioner() const { return preconditioner_; }
    bool apply_uses_initial_guess() const override { return true; }

protected:
    using Dense = matrix::Dense<V>;
    // core/solver/update_residual.hpp:20-73 (IR, Chebyshev): iteration 0 checks the residual it
    // is given; later iterations first ask the criteria with the residual check switched off,
    // then recompute residual = b - A x and check again
    bool update_residual(stop::Criterion* crit, int64 iter, const Dense* b, Dense* x, Dense* residual,
                         const Dense*& residual_ptr, array<uint8>* stop_status) const
    {
        bool one_changed = false;
        stop::Updater u;
        u.num_iterations = iter;
        u.solution = x;
        if (iter == 0) {
            u.residual = residual_ptr;
            return crit->check(1, true, stop_status, &one_changed, u);
        }
        u.ignore_residual_check = true;
        if (crit->check(1, false, stop_status, &one_changed, u)) return true;
        residual_ptr = residual;
        residual->copy_from(b);
        system_matrix_->apply(neg_one_.get(), x, one_.get(), residual);
        stop::Updater u2;
        u2.num_iterations = iter;
        u2.solution = x;
        u2.residual = residual_ptr;
        return crit->check(1, true, stop_status, &one_changed, u2);
    }
    template <typename FactoryT>
    SolverBase(std::shared_ptr<const Executor> exec, const FactoryT& f,
               std::shared_ptr<const LinOp> op)
        : LinOp(exec, op->get_size()), system_matrix_(std::move(op)), criteria_(f.criteria_)
    {
        if (size_.rows != size_.cols) throw DimensionMismatch("solver needs a square operator");
        if (f.generated_preconditioner_)
            preconditioner_ = f.generated_preconditioner_;
        else if (f.preconditioner_)
            preconditioner_ = f.preconditioner_->generate(system_matrix_);
        else
            preconditioner_ = matrix::Identity<V>::create(exec, size_.rows);
        one_ = matrix::scalar<V>(V(1), exec);
        neg_one_ = matrix::scalar<V>(V(-1), exec);
    }
    void apply_impl(const LinOp* alpha, const LinOp* b, const LinOp* beta, LinOp* x) const override
    {
        // x = alpha * solve(b) + beta * x   (core/solver/cg.cpp:184-200)
        auto dx = as<Dense>(x);
        auto x_clone = dx->clone();
        static_cast<const LinOp*>(this)->apply(b, static_cast<LinOp*>(x_clone.get()));
        dx->scale(as<Dense>(beta));
        dx->add_scaled(as<Dense>(alpha), x_clone.get());
    }
    void record(size_type iters, const array<uint8>& stop) const
    {
        num_iterations_ = iters;
        status_ = stop.to_host();
    }
    // What the fused device-resident iterations (Cg, Bicgstab, Gmres, Minres) take: a Csr matrix with
    // 16-byte-aligned arrays, 1..max_cols right-hand sides stored without gaps (stride == columns)
    // and no reducer (rows of a distributed vector take the loop with its all-reduces), and one or
    // two criteria out of Iteration / (Implicit)ResidualNorm.  Which preconditioners each takes is
    // its own rule; every caller but Cg's several-column path accepts one column.
    template <typename I>
    struct FusedProblem {
        const matrix::Csr<V, I>* A = nullptr;
        const V* inv_diag = nullptr;
        int64 max_iters = -1;
        int32 res_kind = 0, iter_first = 1, baseline = 0;
        double factor = 0;
    };
    // Cg and Bicgstab fold the preconditioner into their element-wise steps: Identity, or scalar
    // Jacobi with its inverted diagonal in f.inv_diag
    template <typename I>
    bool fused_scalar_preconditioner(FusedProblem<I>& f) const
    {
        if (auto J = dynamic_cast<const preconditioner::Jacobi<V, I>*>(preconditioner_.get())) {
            if (J->get_max_block_size() != 1) return false;
            f.inv_diag = J->get_blocks();
            return true;
        }
        return dynamic_cast<const matrix::Identity<V>*>(preconditioner_.get()) != nullptr;
    }
    template <typename I>
    bool fused_problem(const Dense* b, const Dense* x, FusedProblem<I>& f, size_type max_cols = 1) const
    {
        f = FusedProblem<I>{};
        f.A = dynamic_cast<const matrix::Csr<V, I>*>(system_matrix_.get());
        const size_type cols = b->get_size().cols;
        if (!f.A || cols < 1 || cols > max_cols || b->get_stride() != cols || x->get_stride() != cols)
            return false;
        if (b->get_reducer()) return false;
        if (criteria_.empty() || criteria_.size() > 2) return false;
        for (size_type k = 0; k < criteria_.size(); ++k) {
            auto& c = criteria_[k];
            if (c->kind() < 0 || c->kind() > 2) return false;  // e.g. stop::Time: host-side criterion
            if (c->kind() == 0) {
                if (f.max_iters >= 0) return false;
                f.max_iters = (int64)c->max_iters();
                if (k == 1) f.iter_first = 0;
            } else {
                if (f.res_kind) return false;
                f.res_kind = c->kind();
                f.factor = c->reduction_factor();
                f.baseline = c->baseline() == stop::mode::rhs_norm
                                 ? 0
                                 : c->baseline() == stop::mode::initial_resnorm ? 1 : 2;
            }
        }
        return !((((std::uintptr_t)f.A->get_const_col_idxs()) | ((std::uintptr_t)f.A->get_const_values())) & 15);
    }
    // What a fused path's graphs bake in besides their launch sequence.  Each path fills in what its
    // own graphs hold and leaves the rest null.  pre is the preconditioner's storage: the Jacobi blocks
    // (the inverted diagonal when scalar), their precisions and block pointers.  The index arrays are
    // untyped pointers (int32 or int64).
    struct FusedKey {
        int64 k = 0, nnz = -1;
        const V* ws = nullptr;
        const V* x = nullptr;
        const void* pre[3] = {};
        const void* row_ptrs = nullptr;
        const void* col_idxs = nullptr;
        const V* values = nullptr;
        const void* plan = nullptr;
        bool operator==(const FusedKey& o) const
        {
            return k == o.k && nnz == o.nnz && ws == o.ws && x == o.x && std::equal(pre, pre + 3, o.pre) &&
                   row_ptrs == o.row_ptrs && col_idxs == o.col_idxs && values == o.values && plan == o.plan;
        }
    };
    // A fused path's workspace, control block and graphs, kept across applies: the graphs bake in the
    // workspace's pointers
    struct FusedState {
        std::unique_ptr<Dense> ws;
        array<V> sc, work;
        array<uint8> status;
        array<int32> ctl;
        int64 n = -1, k = 0;
        std::vector<b200_graph*> graphs;
        FusedKey key;
        ~FusedState() { drop(); }
        void drop()
        {
            for (auto g : graphs) b200_graph_destroy(g);
            graphs.clear();
            key = FusedKey{};
        }
        // alloc() (re)allocates the workspace for n rows and k columns when either changed; the graphs
        // hold the pointers it frees
        template <typename Alloc>
        void reshape(int64 rows, int64 cols, Alloc alloc)
        {
            if (n == rows && k == cols) return;
            drop();
            alloc();
            n = rows;
            k = cols;
        }
        // Unless the cached graphs were captured for this key, capture `batches` new ones; enqueue(i)
        // enqueues batch i.  Whatever the capture bakes in must exist before it: a Csr's plan comes from
        // get_plan() before, never inside, begin_capture.
        template <typename Enqueue>
        void capture(b200_ctx* ctx, const FusedKey& new_key, int64 batches, Enqueue enqueue)
        {
            if (!graphs.empty() && key == new_key) return;
            drop();
            for (int64 i = 0; i < batches; ++i) {
                b200_graph* g = nullptr;
                GKOB_CALL(b200_graph_begin_capture(ctx));
                enqueue(i);
                GKOB_CALL(b200_graph_end_capture(ctx, &g));
                graphs.push_back(g);
            }
            key = new_key;
        }
        // One GPU: launch the graph next() names (next() also does the host work between batches), read
        // the control block, launch the next, until ctl[0] is set; returns (ctl[0], ctl[1]), the stop
        // flags and the iteration count.  (The distributed solver keeps a batch queued ahead through
        // b200_snapshot_* because there every rank's GPU waits for the slowest HOST; on one GPU the two
        // loops measure the same -- 3400 vs 3394 it/s on cfg3 -- so the simple one stays.)
        template <typename Next>
        std::pair<int32, int32> poll(const Executor& exec, const char* path, Next next) const
        {
            int32 h[8] = {0};
            exec.copy_to_host(h, ctl.get_const_data(), 8);
            while (h[0] == 0) {
                const size_type g = next();
                const int32 before = h[1];
                GKOB_CALL(b200_graph_launch(exec.ctx(), graphs[g]));
                exec.copy_to_host(h, ctl.get_const_data(), 8);
                if (h[0] == 0 && h[1] == before)
                    throw Error(std::string(path) + ": the device iteration made no progress");
            }
            return {h[0], h[1]};
        }
    };
    std::shared_ptr<const LinOp> system_matrix_;
    std::shared_ptr<const LinOp> preconditioner_;
    std::vector<std::shared_ptr<const stop::CriterionFactory>> criteria_;
    std::unique_ptr<Dense> one_, neg_one_;
    mutable size_type num_iterations_ = 0;
    mutable std::vector<uint8> status_;
};

// common factory parameters (GKO_CREATE_FACTORY_PARAMETERS idiom)
template <typename Derived>
struct SolverFactoryBase : LinOpFactory {
    std::vector<std::shared_ptr<const stop::CriterionFactory>> criteria_;
    std::shared_ptr<const LinOpFactory> preconditioner_;
    std::shared_ptr<const LinOp> generated_preconditioner_;
    std::shared_ptr<const Executor> exec_;
    template <typename... F>
    Derived& with_criteria(const F&... f)
    {
        criteria_.clear();
        (criteria_.push_back(to_shared(f)), ...);
        return static_cast<Derived&>(*this);
    }
    Derived& with_criteria(std::vector<std::shared_ptr<const stop::CriterionFactory>> v)
    {
        criteria_ = std::move(v);
        return static_cast<Derived&>(*this);
    }
    template <typename PF>
    Derived& with_preconditioner(const PF& pf)
    {
        preconditioner_ = to_shared_lo(pf);
        return static_cast<Derived&>(*this);
    }
    Derived& with_generated_preconditioner(std::shared_ptr<const LinOp> p)
    {
        generated_preconditioner_ = std::move(p);
        return static_cast<Derived&>(*this);
    }
    std::shared_ptr<const Derived> on(std::shared_ptr<const Executor> exec) const
    {
        auto f = std::make_shared<Derived>(static_cast<const Derived&>(*this));
        f->exec_ = exec;
        // deferred factories (criteria / preconditioner built without .on(exec))
        return f;
    }

private:
    static std::shared_ptr<const stop::CriterionFactory> to_shared(
        std::shared_ptr<const stop::CriterionFactory> p)
    {
        return p;
    }
    template <typename F>
    static std::shared_ptr<const stop::CriterionFactory> to_shared(const F& f)
    {
        return std::make_shared<F>(f);  // deferred_factory_parameter: no .on(exec) needed
    }
    static std::shared_ptr<const LinOpFactory> to_shared_lo(std::shared_ptr<const LinOpFactory> p)
    {
        return p;
    }
    template <typename F>
    static std::shared_ptr<const LinOpFactory> to_shared_lo(const F& f)
    {
        return std::make_shared<F>(f);
    }
};

// ---------------------------------------------------------------------------------------------
// Cg (core/solver/cg.cpp:93-181)
// ---------------------------------------------------------------------------------------------
template <typename V>
class Cg : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        bool fused_ = true;
        bool fused_multi_rhs_ = false;
        int check_every_ = 16;
        // ginkgo_b200 extension: device-resident fused iteration (default on where applicable)
        Factory& with_fused(bool f)
        {
            fused_ = f;
            return *this;
        }
        // ginkgo_b200 extension: the device-resident iteration for 2..32 right-hand sides, one
        // matrix pass per iteration for all columns (opt-in)
        Factory& with_fused_multi_rhs(bool f)
        {
            fused_multi_rhs_ = f;
            return *this;
        }
        Factory& with_check_every(int k)
        {
            check_every_ = k;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Cg(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    bool used_fused_path() const { return used_fused_; }

protected:
    Cg(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), fused_(f.fused_), fused_multi_rhs_(f.fused_multi_rhs_),
          check_every_(std::max(1, f.check_every_))
    {}
    using Base::apply_impl;

    void apply_impl(const LinOp* b, LinOp* x) const override
    {
        auto db = as<Dense>(b);
        auto dx = as<Dense>(x);
        if (fused_ && try_fused<int32>(db, dx)) return;
        if (fused_ && try_fused<int64>(db, dx)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int32>(db, dx)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int64>(db, dx)) return;
        used_fused_ = false;
        apply_dense_impl(db, dx);
    }

    // the reference's loop, kernel for kernel
    void apply_dense_impl(const Dense* b, Dense* x) const
    {
        auto exec = this->exec_;
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto r = b->create_like(sz), z = b->create_like(sz), p = b->create_like(sz), q = b->create_like(sz);
        auto beta = Dense::create(exec, dim2{1, nrhs}), prev_rho = Dense::create(exec, dim2{1, nrhs}),
             rho = Dense::create(exec, dim2{1, nrhs});
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        auto ctx = exec->ctx();
        GKOB_CALL(vabi<V>::cg_initialize(ctx, sz.rows, nrhs, b->get_const_values(), b->get_stride(),
                                         r->get_values(), r->get_stride(), z->get_values(),
                                         z->get_stride(), p->get_values(), p->get_stride(),
                                         q->get_values(), q->get_stride(), prev_rho->get_values(),
                                         rho->get_values(), stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 iter = -1;
        while (true) {
            this->preconditioner_->apply(r.get(), z.get());
            r->compute_conj_dot(z.get(), rho.get());
            ++iter;
            stop::Updater u;
            u.num_iterations = iter;
            u.residual = r.get();
            u.implicit_sq_residual_norm = rho.get();
            u.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, u)) break;
            GKOB_CALL(vabi<V>::cg_step_1(ctx, sz.rows, nrhs, p->get_values(), p->get_stride(),
                                         z->get_const_values(), z->get_stride(),
                                         rho->get_const_values(), prev_rho->get_const_values(),
                                         stop_status.get_const_data()));
            this->system_matrix_->apply(p.get(), q.get());
            p->compute_conj_dot(q.get(), beta.get());
            GKOB_CALL(vabi<V>::cg_step_2(ctx, sz.rows, nrhs, x->get_values(), x->get_stride(),
                                         r->get_values(), r->get_stride(), p->get_const_values(),
                                         p->get_stride(), q->get_const_values(), q->get_stride(),
                                         beta->get_const_values(), rho->get_const_values(),
                                         stop_status.get_const_data()));
            std::swap(prev_rho, rho);
        }
        this->record(iter, stop_status);
    }

    // Fused device-resident path: Csr matrix, one right-hand side, Identity or scalar-Jacobi
    // preconditioner, criteria made of Iteration / (Implicit)ResidualNorm.
    template <typename I>
    bool try_fused(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (!this->template fused_problem<I>(b, x, f) || !this->template fused_scalar_preconditioner<I>(f))
            return false;
        const auto A = f.A;
        const V* inv_diag = f.inv_diag;
        const int64 max_iters = f.max_iters;
        const int32 res_kind = f.res_kind, iter_first = f.iter_first, baseline = f.baseline;
        const double factor = f.factor;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 nnz = A->get_num_stored_elements();
        auto& s = single_;
        s.reshape(n, 1, [&] {
            s.ws = Dense::create(exec, dim2{(size_type)(4 * n), 1});
            s.sc = array<V>(exec, 8);
            s.ctl = array<int32>(exec, 8);
            s.work = array<V>(exec, (size_type)vabi<V>::fused_work_size(ctx));
        });
        V* r = s.ws->get_values();
        V* z = r + n;
        V* p = z + n;
        V* q = p + n;
        V* xv = x->get_values();
        V* sc = s.sc.get_data();
        int32* ctl = s.ctl.get_data();
        V* work = s.work.get_data();
        // r = b - A x
        exec->copy(r, b->get_const_values(), n);
        auto rview = Dense::create_view(exec, dim2{(size_type)n, 1}, r, 1);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rview.get());
        if (baseline == 0)  // ||b|| into sc[4]
            GKOB_CALL(vabi<V>::norm2(ctx, n, 1, b->get_const_values(), 1, sc + 4));
        GKOB_CALL(vabi<V>::fused_init(ctx, n, r, z, p, q, inv_diag, sc, ctl, work, max_iters, res_kind,
                                      iter_first, baseline, (V)factor, 1));
        const FusedKey key{1, nnz, r, xv, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values(), A->get_plan()};
        s.capture(ctx, key, 1, [&](int64) {
            for (int k = 0; k < check_every_; ++k) {
                GKOB_CALL(vabi<V>::fused_step_p(ctx, n, p, z, sc, ctl));
                GKOB_CALL((viabi<V, I>::csr_spmv_dot(ctx, A->get_plan(), n, n, nnz, A->get_const_row_ptrs(),
                                                     A->get_const_col_idxs(), A->get_const_values(), p, q,
                                                     sc + 2, work, ctl)));
                GKOB_CALL(vabi<V>::fused_step_xr(ctx, n, xv, r, p, q, z, inv_diag, sc, ctl, work, 1));
            }
        });
        const auto [flags, iters] = s.poll(*exec, "fused CG", [] { return 0; });
        this->num_iterations_ = (size_type)iters;
        this->status_.assign(1, (uint8)flags);
        used_fused_ = true;
        return true;
    }

    // Fused device-resident path for k = 2..32 right-hand sides (csrc/fused_cg_mrhs.cu): the same
    // admission as try_fused but with b and x of k columns stored without gaps.  Every column stops
    // on its own; the device keeps a stopped column's x, r and p as the loop's masked steps leave
    // them, and the host reads all k statuses at the end.
    template <typename I>
    bool try_fused_multi_rhs(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (b->get_size().cols < 2 || !this->template fused_problem<I>(b, x, f, 32) ||
            !this->template fused_scalar_preconditioner<I>(f))
            return false;
        const auto A = f.A;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 k = (int64)b->get_size().cols;
        const int64 nnz = A->get_num_stored_elements();
        auto& m = mrhs_;
        // workspace r, z, p, q (n x k each), per-column scalars, statuses, control block, partials
        m.reshape(n, k, [&] {
            m.ws = Dense::create(exec, dim2{(size_type)(4 * n * k), 1});
            m.sc = array<V>(exec, (size_type)(6 * k));
            m.status = array<uint8>(exec, (size_type)k);
            m.ctl = array<int32>(exec, 8);
            m.work = array<V>(exec, (size_type)vabi<V>::cg_mrhs_work_size(ctx, k));
        });
        V* r = m.ws->get_values();
        V* z = r + n * k;
        V* p = z + n * k;
        V* q = p + n * k;
        V* xv = x->get_values();
        V* sc = m.sc.get_data();
        // r = b - A x
        exec->copy(r, b->get_const_values(), n * k);
        auto rview = Dense::create_view(exec, dim2{(size_type)n, (size_type)k}, r, (size_type)k);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rview.get());
        if (f.baseline == 0)  // ||b_j|| into sc[4k + j]
            GKOB_CALL(vabi<V>::norm2(ctx, n, k, b->get_const_values(), k, sc + 4 * k));
        GKOB_CALL(vabi<V>::cg_mrhs_init(ctx, n, k, r, z, p, q, f.inv_diag, sc, m.status.get_data(),
                                        m.ctl.get_data(), m.work.get_data(), f.max_iters, f.res_kind,
                                        f.iter_first, f.baseline, (V)f.factor));
        const FusedKey key{k, nnz, r, xv, {f.inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values()};
        m.capture(ctx, key, 1, [&](int64) {
            for (int it = 0; it < check_every_; ++it) {
                GKOB_CALL(vabi<V>::cg_mrhs_step_p(ctx, n, k, p, z, sc, m.status.get_const_data(),
                                                  m.ctl.get_const_data()));
                GKOB_CALL((viabi<V, I>::csr_spmv_mdot(ctx, n, n, nnz, A->get_const_row_ptrs(),
                                                      A->get_const_col_idxs(), A->get_const_values(), p, k,
                                                      q, sc + 2 * k, m.work.get_data(),
                                                      m.ctl.get_const_data())));
                GKOB_CALL(vabi<V>::cg_mrhs_step_xr(ctx, n, k, xv, r, p, q, z, f.inv_diag, sc,
                                                   m.status.get_data(), m.ctl.get_data(),
                                                   m.work.get_data()));
            }
        });
        this->record(m.poll(*exec, "fused CG (several right-hand sides)", [] { return 0; }).second, m.status);
        used_fused_ = true;
        return true;
    }

private:
    bool fused_;
    bool fused_multi_rhs_;
    int check_every_;
    mutable bool used_fused_ = false;
    using FusedKey = typename Base::FusedKey;
    mutable typename Base::FusedState single_, mrhs_;
};

// ---------------------------------------------------------------------------------------------
// Bicgstab (core/solver/bicgstab.cpp:95-233)
// ---------------------------------------------------------------------------------------------
// solver::Fcg (core/solver/fcg.cpp:93-188): flexible CG, one more vector (t = r_new - r_old)
// and one more dot per iteration than CG.  SURVEY.md 8f-3.
// ---------------------------------------------------------------------------------------------
#define GKOB_VS(d) (d)->get_values(), (d)->get_stride()
#define GKOB_CVS(d) (d)->get_const_values(), (d)->get_stride()
template <typename V>
class Fcg : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Fcg(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

protected:
    Fcg(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), z = mk(), p = mk(), q = mk(), t = mk();
        auto beta = sc(), prev_rho = sc(), rho = sc(), rho_t = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::fcg_initialize(ctx, sz.rows, nrhs, GKOB_CVS(b), GKOB_VS(r), GKOB_VS(z),
                                          GKOB_VS(p), GKOB_VS(q), GKOB_VS(t), prev_rho->get_values(),
                                          rho->get_values(), rho_t->get_values(),
                                          stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 iter = -1;
        while (true) {
            this->preconditioner_->apply(r.get(), z.get());
            r->compute_conj_dot(z.get(), rho.get());
            t->compute_conj_dot(z.get(), rho_t.get());
            ++iter;
            stop::Updater u;
            u.num_iterations = iter;
            u.residual = r.get();
            u.implicit_sq_residual_norm = rho.get();
            u.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, u)) break;
            GKOB_CALL(vabi<V>::fcg_step_1(ctx, sz.rows, nrhs, GKOB_VS(p), GKOB_CVS(z),
                                          rho_t->get_const_values(), prev_rho->get_const_values(),
                                          stop_status.get_const_data()));
            this->system_matrix_->apply(p.get(), q.get());
            p->compute_conj_dot(q.get(), beta.get());
            GKOB_CALL(vabi<V>::fcg_step_2(ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_VS(r), GKOB_VS(t),
                                          GKOB_CVS(p), GKOB_CVS(q), beta->get_const_values(),
                                          rho->get_const_values(), stop_status.get_const_data()));
            std::swap(prev_rho, rho);
        }
        this->record(iter, stop_status);
    }
};

// ---------------------------------------------------------------------------------------------
// solver::Cgs (core/solver/cgs.cpp:93-205): two SpMVs and two preconditioner applications per
// iteration, no transpose.  SURVEY.md 8f-3.
// ---------------------------------------------------------------------------------------------
template <typename V>
class Cgs : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Cgs(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

protected:
    Cgs(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), r_tld = mk(), p = mk(), q = mk(), u = mk(), u_hat = mk(), v_hat = mk(),
             t = mk();
        auto alpha = sc(), beta = sc(), gamma = sc(), prev_rho = sc(), rho = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::cgs_initialize(
            ctx, sz.rows, nrhs, GKOB_CVS(b), GKOB_VS(r), GKOB_VS(r_tld), GKOB_VS(p), GKOB_VS(q),
            GKOB_VS(u), GKOB_VS(u_hat), GKOB_VS(v_hat), GKOB_VS(t), alpha->get_values(),
            beta->get_values(), gamma->get_values(), prev_rho->get_values(), rho->get_values(),
            stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        r_tld->copy_from(r.get());
        int64 iter = -1;
        while (true) {
            r->compute_conj_dot(r_tld.get(), rho.get());
            ++iter;
            stop::Updater up;
            up.num_iterations = iter;
            up.residual = r.get();
            up.implicit_sq_residual_norm = rho.get();
            up.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, up)) break;
            GKOB_CALL(vabi<V>::cgs_step_1(ctx, sz.rows, nrhs, GKOB_CVS(r), GKOB_VS(u), GKOB_VS(p),
                                          GKOB_CVS(q), beta->get_values(), rho->get_const_values(),
                                          prev_rho->get_const_values(),
                                          stop_status.get_const_data()));
            this->preconditioner_->apply(p.get(), t.get());
            this->system_matrix_->apply(t.get(), v_hat.get());
            r_tld->compute_conj_dot(v_hat.get(), gamma.get());
            GKOB_CALL(vabi<V>::cgs_step_2(ctx, sz.rows, nrhs, GKOB_CVS(u), GKOB_CVS(v_hat),
                                          GKOB_VS(q), GKOB_VS(t), alpha->get_values(),
                                          rho->get_const_values(), gamma->get_const_values(),
                                          stop_status.get_const_data()));
            this->preconditioner_->apply(t.get(), u_hat.get());
            this->system_matrix_->apply(u_hat.get(), t.get());
            GKOB_CALL(vabi<V>::cgs_step_3(ctx, sz.rows, nrhs, GKOB_CVS(t), GKOB_CVS(u_hat),
                                          GKOB_VS(r), GKOB_VS(x), alpha->get_const_values(),
                                          stop_status.get_const_data()));
            std::swap(prev_rho, rho);
        }
        this->record(iter, stop_status);
    }
};
// ---------------------------------------------------------------------------------------------
// solver::Bicg (core/solver/bicg.cpp:113-232): two coupled recurrences, one with A and M, one
// with their transposes (Transposable::conj_transpose of the system matrix and the
// preconditioner, built once per apply like the reference does).
// ---------------------------------------------------------------------------------------------
template <typename V>
class Bicg : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Bicg(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

protected:
    Bicg(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), z = mk(), p = mk(), q = mk(), r2 = mk(), z2 = mk(), p2 = mk(), q2 = mk();
        auto beta = sc(), prev_rho = sc(), rho = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::bicg_initialize(ctx, sz.rows, nrhs, GKOB_CVS(b), GKOB_VS(r), GKOB_VS(z), GKOB_VS(p),
                                           GKOB_VS(q), prev_rho->get_values(), rho->get_values(), GKOB_VS(r2),
                                           GKOB_VS(z2), GKOB_VS(p2), GKOB_VS(q2), stop_status.get_data()));
        auto trans_A = dynamic_cast<const Transposable*>(this->system_matrix_.get());
        auto trans_M = dynamic_cast<const Transposable*>(this->preconditioner_.get());
        if (!trans_A) throw NotSupported("Bicg: the system matrix is not Transposable");
        if (!trans_M) throw NotSupported("Bicg: the preconditioner is not Transposable");
        auto conj_trans_A = trans_A->conj_transpose();
        auto conj_trans_M = trans_M->conj_transpose();
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        r2->copy_from(r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 iter = -1;
        while (true) {
            this->preconditioner_->apply(r.get(), z.get());
            conj_trans_M->apply(r2.get(), z2.get());
            z->compute_conj_dot(r2.get(), rho.get());
            ++iter;
            stop::Updater up;
            up.num_iterations = iter;
            up.residual = r.get();
            up.implicit_sq_residual_norm = rho.get();
            up.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, up)) break;
            GKOB_CALL(vabi<V>::bicg_step_1(ctx, sz.rows, nrhs, GKOB_VS(p), GKOB_CVS(z), GKOB_VS(p2), GKOB_CVS(z2),
                                           rho->get_const_values(), prev_rho->get_const_values(),
                                           stop_status.get_const_data()));
            this->system_matrix_->apply(p.get(), q.get());
            conj_trans_A->apply(p2.get(), q2.get());
            p2->compute_conj_dot(q.get(), beta.get());
            GKOB_CALL(vabi<V>::bicg_step_2(ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_VS(r), GKOB_VS(r2), GKOB_CVS(p),
                                           GKOB_CVS(q), GKOB_CVS(q2), beta->get_const_values(),
                                           rho->get_const_values(), stop_status.get_const_data()));
            std::swap(prev_rho, rho);
        }
        this->record(iter, stop_status);
    }
};
// ---------------------------------------------------------------------------------------------
// solver::PipeCg (core/solver/pipe_cg.cpp:95-285): pipelined CG, one reduction point per
// iteration (rho = r.z and delta = w.z together).  The reference stores (r | w), (z1 | z2)
// side by side to get both with ONE compute_conj_dot; every column of that dot is an
// independent sum, so the two dots issued here return the same values.
// ---------------------------------------------------------------------------------------------
template <typename V>
class PipeCg : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new PipeCg(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

protected:
    PipeCg(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), w = mk(), z1 = mk(), z2 = mk(), p = mk(), m = mk(), n = mk(), q = mk(), f = mk(),
             g = mk();
        auto rho = sc(), delta = sc(), beta = sc(), prev_rho = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::pipe_cg_initialize_1(ctx, sz.rows, nrhs, GKOB_CVS(b), GKOB_VS(r),
                                                prev_rho->get_values(), stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        this->preconditioner_->apply(r.get(), z1.get());
        z2->copy_from(z1.get());
        this->system_matrix_->apply(z1.get(), w.get());
        this->preconditioner_->apply(w.get(), m.get());
        this->system_matrix_->apply(m.get(), n.get());
        r->compute_conj_dot(z1.get(), rho.get());
        w->compute_conj_dot(z2.get(), delta.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 iter = 0;
        auto check = [&] {
            stop::Updater u;
            u.num_iterations = iter;
            u.residual = r.get();
            u.implicit_sq_residual_norm = rho.get();
            u.solution = x;
            return crit->check(1, true, &stop_status, &one_changed, u);
        };
        if (!check()) {
            GKOB_CALL(vabi<V>::pipe_cg_initialize_2(
                ctx, sz.rows, nrhs, GKOB_VS(p), GKOB_VS(q), GKOB_VS(f), GKOB_VS(g), beta->get_values(),
                GKOB_CVS(z1), GKOB_CVS(w), GKOB_CVS(m), GKOB_CVS(n), delta->get_const_values()));
            while (true) {
                GKOB_CALL(vabi<V>::pipe_cg_step_1(
                    ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_VS(r), GKOB_VS(z1), GKOB_VS(z2), GKOB_VS(w),
                    GKOB_CVS(p), GKOB_CVS(q), GKOB_CVS(f), GKOB_CVS(g), rho->get_const_values(),
                    beta->get_const_values(), stop_status.get_const_data()));
                this->preconditioner_->apply(w.get(), m.get());
                this->system_matrix_->apply(m.get(), n.get());
                prev_rho->copy_from(rho.get());
                r->compute_conj_dot(z1.get(), rho.get());
                w->compute_conj_dot(z2.get(), delta.get());
                ++iter;
                if (check()) break;
                GKOB_CALL(vabi<V>::pipe_cg_step_2(
                    ctx, sz.rows, nrhs, beta->get_values(), GKOB_VS(p), GKOB_VS(q), GKOB_VS(f),
                    GKOB_VS(g), GKOB_CVS(z1), GKOB_CVS(w), GKOB_CVS(m), GKOB_CVS(n),
                    prev_rho->get_const_values(), rho->get_const_values(),
                    delta->get_const_values(), stop_status.get_const_data()));
            }
        }
        this->record(iter, stop_status);
    }
};

// ---------------------------------------------------------------------------------------------
// solver::Gcr (core/solver/gcr.cpp:99-292): generalised conjugate residual with restarts; the
// modified Gram-Schmidt on the A p_i bases is built from the Dense kernels as in the reference.
// ---------------------------------------------------------------------------------------------
template <typename V>
class Gcr : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        size_type krylov_dim_ = 100;  // gcr_default_krylov_dim (include/ginkgo/core/solver/gcr.hpp)
        Factory& with_krylov_dim(size_type k)
        {
            krylov_dim_ = k;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Gcr(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    size_type get_krylov_dim() const { return krylov_dim_; }

protected:
    Gcr(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), krylov_dim_(f.krylov_dim_ ? f.krylov_dim_ : 100)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type n = sz.rows, nrhs = sz.cols, kd = krylov_dim_;
        auto residual = b->create_like(sz), precon_residual = b->create_like(sz),
             a_precon_residual = b->create_like(sz);
        auto p_bases = b->create_like(dim2{n * (kd + 1), nrhs});
        auto ap_bases = b->create_like(dim2{n * (kd + 1), nrhs});
        auto tmp_rap = Dense::create(exec, dim2{1, nrhs}), tmp_minus_beta = Dense::create(exec, dim2{1, nrhs}),
             residual_norm = Dense::create(exec, dim2{1, nrhs});
        auto ap_norms = Dense::create(exec, dim2{kd + 1, nrhs});
        array<std::uint64_t> final_iter_nums(exec, nrhs);
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::gcr_initialize(ctx, n, nrhs, GKOB_CVS(b), GKOB_VS(residual),
                                          stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        this->preconditioner_->apply(residual.get(), precon_residual.get());
        this->system_matrix_->apply(precon_residual.get(), a_precon_residual.get());
        auto restart = [&] {
            GKOB_CALL(vabi<V>::gcr_restart(ctx, n, nrhs, GKOB_CVS(precon_residual),
                                           GKOB_CVS(a_precon_residual), GKOB_VS(p_bases),
                                           GKOB_VS(ap_bases), final_iter_nums.get_data()));
        };
        restart();
        stop::CriterionArgs args{this->system_matrix_, b, x, residual.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 total_iter = -1;
        size_type restart_iter = 0;
        while (true) {
            ++total_iter;
            residual->compute_norm2(residual_norm.get());
            stop::Updater u;
            u.num_iterations = total_iter;
            u.residual = residual.get();
            u.residual_norm = residual_norm.get();
            u.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, u)) break;
            if (restart_iter == kd) {
                restart();
                restart_iter = 0;
            }
            auto ap = ap_bases->create_submatrix_rows(n * restart_iter, n * (restart_iter + 1));
            auto p = p_bases->create_submatrix_rows(n * restart_iter, n * (restart_iter + 1));
            residual->compute_conj_dot(ap.get(), tmp_rap.get());
            auto ap_norm = ap_norms->create_submatrix_rows(restart_iter, restart_iter + 1);
            ap->compute_squared_norm2(ap_norm.get());
            GKOB_CALL(vabi<V>::gcr_step_1(ctx, n, nrhs, GKOB_VS(x), GKOB_VS(residual), GKOB_CVS(p),
                                          GKOB_CVS(ap), ap_norm->get_const_values(),
                                          tmp_rap->get_const_values(), stop_status.get_const_data()));
            this->preconditioner_->apply(residual.get(), precon_residual.get());
            this->system_matrix_->apply(precon_residual.get(), a_precon_residual.get());
            auto next_ap = ap_bases->create_submatrix_rows(n * (restart_iter + 1), n * (restart_iter + 2));
            auto next_p = p_bases->create_submatrix_rows(n * (restart_iter + 1), n * (restart_iter + 2));
            next_ap->copy_from(a_precon_residual.get());
            next_p->copy_from(precon_residual.get());
            for (size_type i = 0; i <= restart_iter; ++i) {
                auto api = ap_bases->create_submatrix_rows(n * i, n * (i + 1));
                auto pi = p_bases->create_submatrix_rows(n * i, n * (i + 1));
                auto ni = ap_norms->create_submatrix_rows(i, i + 1);
                a_precon_residual->compute_conj_dot(api.get(), tmp_minus_beta.get());
                tmp_minus_beta->inv_scale(ni.get());
                next_ap->sub_scaled(tmp_minus_beta.get(), api.get());
                next_p->sub_scaled(tmp_minus_beta.get(), pi.get());
            }
            ++restart_iter;
        }
        this->record(total_iter, stop_status);
    }

private:
    size_type krylov_dim_;
};

// ---------------------------------------------------------------------------------------------
// solver::Minres (core/solver/minres.cpp:114-286): symmetric (possibly indefinite) systems; the
// residual norm is tracked by a recurrence (tau), the criteria receive it as the implicit
// squared norm and no residual vector.
// ---------------------------------------------------------------------------------------------
template <typename V>
class Minres : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        bool fused_ = false;
        bool fused_multi_rhs_ = false;
        int check_every_ = 16;
        // ginkgo_b200 extension: device-resident fused iteration where applicable (default off)
        Factory& with_fused(bool f)
        {
            fused_ = f;
            return *this;
        }
        // ginkgo_b200 extension: the device-resident iteration for 2..32 right-hand sides, one
        // matrix pass per iteration for all columns (opt-in, independent of with_fused)
        Factory& with_fused_multi_rhs(bool f)
        {
            fused_multi_rhs_ = f;
            return *this;
        }
        // iterations per graph launch (and per read of the control block) on the fused paths
        Factory& with_check_every(int k)
        {
            check_every_ = k;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Minres(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    bool used_fused_path() const { return used_fused_; }

protected:
    Minres(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), fused_(f.fused_), fused_multi_rhs_(f.fused_multi_rhs_),
          check_every_(std::max(1, f.check_every_))
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        if (fused_ && try_fused<int32>(b, x)) return;
        if (fused_ && try_fused<int64>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int32>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int64>(b, x)) return;
        used_fused_ = false;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), z = mk(), p = mk(), q = mk(), v = mk(), z_tilde = mk(), p_prev = mk(), q_prev = mk();
        auto alpha = sc(), beta = sc(), gamma = sc(), delta = sc(), eta_next = sc(), eta = sc(), tau = sc(),
             cos_prev = sc(), cos = sc(), sin_prev = sc(), sin = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        r->copy_from(b);
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        this->preconditioner_->apply(r.get(), z.get());
        r->compute_conj_dot(z.get(), beta.get());
        z->compute_conj_dot(z.get(), tau.get());
        GKOB_CALL(vabi<V>::minres_initialize(
            ctx, sz.rows, nrhs, GKOB_CVS(r), GKOB_VS(z), GKOB_VS(p), GKOB_VS(p_prev), GKOB_VS(q),
            GKOB_VS(q_prev), GKOB_VS(v), beta->get_values(), gamma->get_values(), delta->get_values(),
            cos_prev->get_values(), cos->get_values(), sin_prev->get_values(), sin->get_values(),
            eta_next->get_values(), eta->get_values(), stop_status.get_data()));
        int64 iter = -1;
        while (true) {
            ++iter;
            stop::Updater u;
            u.num_iterations = iter;
            u.implicit_sq_residual_norm = tau.get();
            u.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, u)) break;
            this->system_matrix_->apply(this->one_.get(), z.get(), this->neg_one_.get(), v.get());
            v->compute_conj_dot(z.get(), alpha.get());
            v->sub_scaled(alpha.get(), q.get());
            this->preconditioner_->apply(v.get(), z_tilde.get());
            v->compute_conj_dot(z_tilde.get(), beta.get());
            GKOB_CALL(vabi<V>::minres_step_1(
                ctx, nrhs, alpha->get_values(), beta->get_values(), gamma->get_values(),
                delta->get_values(), cos_prev->get_values(), cos->get_values(), sin_prev->get_values(),
                sin->get_values(), eta->get_values(), eta_next->get_values(), tau->get_values(),
                stop_status.get_const_data()));
            std::swap(p, p_prev);
            GKOB_CALL(vabi<V>::minres_step_2(
                ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_VS(p), GKOB_CVS(p_prev), GKOB_VS(z),
                GKOB_CVS(z_tilde), GKOB_VS(q), GKOB_VS(q_prev), GKOB_VS(v), alpha->get_const_values(),
                beta->get_const_values(), gamma->get_const_values(), delta->get_const_values(),
                cos->get_const_values(), eta->get_const_values(), stop_status.get_const_data()));
            std::swap(gamma, beta);
        }
        this->record(iter, stop_status);
    }

    // Fused device-resident path (csrc/fused_minres.cu): three launches per iteration, a graph of
    // check_every iterations per read of the control block.  The set-up is the loop's own calls.
    // ResidualNorm recomputes b - A x from the solution at every check, so it keeps the loop.
    template <typename I>
    bool try_fused(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (!this->template fused_problem<I>(b, x, f) || !this->template fused_scalar_preconditioner<I>(f) ||
            f.res_kind == 1)
            return false;
        const auto A = f.A;
        const V* inv_diag = f.inv_diag;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 nnz = A->get_num_stored_elements();
        auto& s = single_;
        s.reshape(n, 1, [&] {
            s.ws = Dense::create(exec, dim2{(size_type)(6 * n), 1});
            s.sc = array<V>(exec, 16);
            s.ctl = array<int32>(exec, 8);
            s.status = array<uint8>(exec, 1);
            s.work = array<V>(exec, (size_type)vabi<V>::minres_fused_work_size(ctx));
        });
        V* r = s.ws->get_values();
        V *z = r + n, *q = r + 2 * n, *v = r + 3 * n, *p0 = r + 4 * n, *p1 = r + 5 * n;
        V* xv = x->get_values();
        V* sc = s.sc.get_data();
        int32* ctl = s.ctl.get_data();
        V* work = s.work.get_data();
        auto view = [&](V* d, int64 rows) { return Dense::create_view(exec, dim2{(size_type)rows, 1}, d, 1); };
        auto rv = view(r, n), zv = view(z, n);
        // the loop's set-up: r = b - A x, z = M r, beta = r.z, tau = z.z, minres::initialize (q_prev
        // is not kept: its zeros go to v, which initialize zeroes as well)
        exec->copy(r, b->get_const_values(), n);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rv.get());
        this->preconditioner_->apply(rv.get(), zv.get());
        rv->compute_conj_dot(zv.get(), view(sc + 1, 1).get());
        zv->compute_conj_dot(zv.get(), view(sc + 6, 1).get());
        GKOB_CALL(vabi<V>::minres_initialize(ctx, n, 1, r, 1, z, 1, p0, 1, p1, 1, q, 1, v, 1, v, 1, sc + 1,
                                             sc + 2, sc + 3, sc + 9, sc + 10, sc + 11, sc + 12, sc + 8, sc + 7,
                                             s.status.get_data()));
        if (f.baseline == 0) b->compute_norm2(view(sc + 4, 1).get());
        if (f.baseline == 1) rv->compute_norm2(view(sc + 4, 1).get());
        GKOB_CALL(vabi<V>::minres_fused_init(ctx, sc, ctl, f.max_iters, f.res_kind, f.iter_first, f.baseline,
                                             (V)f.factor));
        const FusedKey key{1, nnz, r, xv, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values(), A->get_plan()};
        s.capture(ctx, key, 1, [&](int64) {
            for (int k = 0; k < check_every_; ++k) {
                GKOB_CALL((viabi<V, I>::csr_spmv_sub_dot(ctx, A->get_plan(), n, n, nnz, A->get_const_row_ptrs(),
                                                         A->get_const_col_idxs(), A->get_const_values(), z, v, sc,
                                                         work, ctl)));
                GKOB_CALL(vabi<V>::minres_fused_lanczos(ctx, n, v, q, inv_diag, sc, ctl, work));
                GKOB_CALL(vabi<V>::minres_fused_update(ctx, n, xv, p0, p1, z, q, v, inv_diag, sc, ctl));
            }
        });
        const auto [flags, iters] = s.poll(*exec, "fused MINRES", [] { return 0; });
        this->num_iterations_ = (size_type)iters;
        this->status_.assign(1, (uint8)flags);
        used_fused_ = true;
        return true;
    }

    // Fused device-resident path for k = 2..32 right-hand sides (csrc/fused_minres_mrhs.cu): try_fused's
    // admission with b and x of k columns stored without gaps, and its set-up on the n x k views.  Every
    // column stops on its own; the device keeps a stopped column's scalars, x, p, q, v and z as the
    // loop's masked steps leave them, and the host reads all k statuses at the end.
    template <typename I>
    bool try_fused_multi_rhs(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (b->get_size().cols < 2 || !this->template fused_problem<I>(b, x, f, 32) ||
            !this->template fused_scalar_preconditioner<I>(f) || f.res_kind == 1)
            return false;
        const auto A = f.A;
        const V* inv_diag = f.inv_diag;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 k = (int64)b->get_size().cols;
        const int64 nnz = A->get_num_stored_elements();
        auto& m = mrhs_;
        // workspace r, z, q, v, p0, p1 (n x k each), per-column scalars, statuses, control block, partials
        m.reshape(n, k, [&] {
            m.ws = Dense::create(exec, dim2{(size_type)(6 * n * k), 1});
            m.sc = array<V>(exec, (size_type)(16 * k));
            m.status = array<uint8>(exec, (size_type)k);
            m.ctl = array<int32>(exec, 8);
            m.work = array<V>(exec, (size_type)vabi<V>::minres_mrhs_work_size(ctx, k));
        });
        V* r = m.ws->get_values();
        V *z = r + n * k, *q = r + 2 * n * k, *v = r + 3 * n * k, *p0 = r + 4 * n * k, *p1 = r + 5 * n * k;
        V* xv = x->get_values();
        V* sc = m.sc.get_data();
        uint8* status = m.status.get_data();
        int32* ctl = m.ctl.get_data();
        V* work = m.work.get_data();
        auto view = [&](V* d, int64 rows) {
            return Dense::create_view(exec, dim2{(size_type)rows, (size_type)k}, d, (size_type)k);
        };
        auto rv = view(r, n), zv = view(z, n);
        // the loop's set-up on k columns, its per-column scalars straight into slots sc[s k + .]
        exec->copy(r, b->get_const_values(), n * k);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rv.get());
        this->preconditioner_->apply(rv.get(), zv.get());
        rv->compute_conj_dot(zv.get(), view(sc + k, 1).get());
        zv->compute_conj_dot(zv.get(), view(sc + 6 * k, 1).get());
        GKOB_CALL(vabi<V>::minres_initialize(ctx, n, k, r, k, z, k, p0, k, p1, k, q, k, v, k, v, k, sc + k,
                                             sc + 2 * k, sc + 3 * k, sc + 9 * k, sc + 10 * k, sc + 11 * k,
                                             sc + 12 * k, sc + 8 * k, sc + 7 * k, status));
        if (f.baseline == 0) b->compute_norm2(view(sc + 4 * k, 1).get());
        if (f.baseline == 1) rv->compute_norm2(view(sc + 4 * k, 1).get());
        GKOB_CALL(vabi<V>::minres_mrhs_init(ctx, k, sc, status, ctl, f.max_iters, f.res_kind, f.iter_first,
                                            f.baseline, (V)f.factor));
        // the k-wide SpMV uses no plan
        const FusedKey key{k, nnz, r, xv, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values()};
        m.capture(ctx, key, 1, [&](int64) {
            for (int it = 0; it < check_every_; ++it) {
                GKOB_CALL((viabi<V, I>::csr_spmv_sub_mdot(ctx, n, n, nnz, A->get_const_row_ptrs(),
                                                          A->get_const_col_idxs(), A->get_const_values(), z, k,
                                                          v, sc, work, ctl)));
                GKOB_CALL(vabi<V>::minres_mrhs_lanczos(ctx, n, k, v, q, inv_diag, sc, status, ctl, work));
                GKOB_CALL(vabi<V>::minres_mrhs_update(ctx, n, k, xv, p0, p1, z, q, v, inv_diag, sc, status, ctl));
            }
        });
        this->record(m.poll(*exec, "fused MINRES (several right-hand sides)", [] { return 0; }).second, m.status);
        used_fused_ = true;
        return true;
    }

private:
    using FusedKey = typename Base::FusedKey;
    bool fused_;
    bool fused_multi_rhs_;
    int check_every_;
    mutable bool used_fused_ = false;
    mutable typename Base::FusedState single_, mrhs_;
};

// ---------------------------------------------------------------------------------------------
// solver::Ir (core/solver/ir.cpp:192-258): x += relaxation_factor * inner_solver(b - A x).
// The inner solver is the `with_solver` / preconditioner slot of the factory (Identity by
// default, which gives Richardson iteration).  default_initial_guess = provided.
// ---------------------------------------------------------------------------------------------
template <typename V>
class Ir : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        V relaxation_factor_ = V(1);
        initial_guess_mode default_initial_guess_ = initial_guess_mode::provided;
        Factory& with_relaxation_factor(V w)
        {
            relaxation_factor_ = w;
            return *this;
        }
        // zero / rhs: x is overwritten before the first iteration (needed when the Ir is itself a
        // preconditioner or smoother: a fixed number of sweeps from a fixed start is a fixed operator)
        Factory& with_default_initial_guess(initial_guess_mode m)
        {
            default_initial_guess_ = m;
            return *this;
        }
        // the reference's name for the inner-solver slot
        Factory& with_solver(std::shared_ptr<const LinOpFactory> f) { return this->with_preconditioner(std::move(f)); }
        Factory& with_generated_solver(std::shared_ptr<const LinOp> s)
        {
            return this->with_generated_preconditioner(std::move(s));
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Ir(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    std::shared_ptr<const LinOp> get_solver() const { return this->preconditioner_; }

protected:
    Ir(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), relaxation_(matrix::scalar<V>(f.relaxation_factor_, exec)),
          guess_(f.default_initial_guess_)
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        const dim2 sz = b->get_size();
        auto residual = b->create_like(sz);
        std::unique_ptr<Dense> inner_solution;
        array<uint8> stop_status(exec, sz.cols);
        GKOB_CALL(b200_ir_initialize(exec->ctx(), sz.cols, stop_status.get_data()));
        // core/solver/ir.cpp:177-217: prepare the guess; from zero the first residual is b itself
        if (guess_ == initial_guess_mode::zero) x->fill(V(0));
        if (guess_ == initial_guess_mode::rhs) x->copy_from(b);
        if (guess_ != initial_guess_mode::zero) {
            residual->copy_from(b);
            this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        }
        const Dense* residual_ptr = guess_ == initial_guess_mode::zero ? b : residual.get();
        stop::CriterionArgs args{this->system_matrix_, b, x, residual_ptr};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        auto inner = this->preconditioner_.get();
        int64 iter = -1;
        while (true) {
            ++iter;
            if (this->update_residual(crit.get(), iter, b, x, residual.get(), residual_ptr, &stop_status))
                break;
            if (inner->apply_uses_initial_guess()) {
                if (!inner_solution) inner_solution = b->create_like(sz);
                inner_solution->copy_from(residual_ptr);
                inner->apply(residual_ptr, inner_solution.get());
                x->add_scaled(relaxation_.get(), inner_solution.get());
            } else {
                inner->apply(relaxation_.get(), residual_ptr, this->one_.get(), x);
            }
        }
        this->record(iter, stop_status);
    }

private:
    std::unique_ptr<Dense> relaxation_;
    initial_guess_mode guess_;
};

// ---------------------------------------------------------------------------------------------
// solver::Chebyshev (core/solver/chebyshev.cpp:85-97, :201-296): no inner products; `foci` =
// the interval that contains the spectrum of the preconditioned operator.
// ---------------------------------------------------------------------------------------------
template <typename V>
class Chebyshev : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        std::pair<double, double> foci_{0.0, 1.0};
        Factory& with_foci(double lo, double hi)
        {
            foci_ = {lo, hi};
            return *this;
        }
        Factory& with_foci(std::pair<double, double> f)
        {
            foci_ = f;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Chebyshev(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }

protected:
    Chebyshev(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op),
          center_((f.foci_.first + f.foci_.second) / 2.0),
          foci_direction_((f.foci_.second - f.foci_.first) / 2.0)
    {
        if (!(f.foci_.first <= f.foci_.second) || center_ == 0.0)
            throw BadDimension("Chebyshev: foci must satisfy lo <= hi and lo + hi != 0");
    }
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        auto residual = b->create_like(sz), inner_solution = b->create_like(sz),
             update_solution = b->create_like(sz);
        double alpha_host = 1.0 / center_;
        double beta_host = 0.5 * (foci_direction_ * alpha_host) * (foci_direction_ * alpha_host);
        array<uint8> stop_status(exec, sz.cols);
        GKOB_CALL(b200_ir_initialize(ctx, sz.cols, stop_status.get_data()));
        residual->copy_from(b);
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        const Dense* residual_ptr = residual.get();
        stop::CriterionArgs args{this->system_matrix_, b, x, residual_ptr};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        int64 iter = -1;
        while (true) {
            ++iter;
            if (this->update_residual(crit.get(), iter, b, x, residual.get(), residual_ptr, &stop_status))
                break;
            if (this->preconditioner_->apply_uses_initial_guess()) inner_solution->copy_from(residual_ptr);
            this->preconditioner_->apply(residual_ptr, inner_solution.get());
            if (iter == 0) {
                GKOB_CALL(vabi<V>::chebyshev_init_update(
                    ctx, sz.rows, sz.cols, alpha_host, GKOB_CVS(inner_solution), GKOB_VS(update_solution),
                    GKOB_VS(x)));
                continue;
            }
            if (iter > 1)
                beta_host = (foci_direction_ * alpha_host / 2.0) * (foci_direction_ * alpha_host / 2.0);
            alpha_host = 1.0 / (center_ - beta_host / alpha_host);
            GKOB_CALL(vabi<V>::chebyshev_update(ctx, sz.rows, sz.cols, alpha_host, beta_host,
                                                GKOB_VS(inner_solution), GKOB_VS(update_solution),
                                                GKOB_VS(x)));
        }
        this->record(iter, stop_status);
    }

private:
    double center_, foci_direction_;
};
#undef GKOB_VS
#undef GKOB_CVS

// ---------------------------------------------------------------------------------------------
template <typename V>
class Bicgstab : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        bool fused_ = false;
        bool fused_multi_rhs_ = false;
        int check_every_ = 16;
        // ginkgo_b200 extension: device-resident fused iteration where applicable (default off)
        Factory& with_fused(bool f)
        {
            fused_ = f;
            return *this;
        }
        // ginkgo_b200 extension: the device-resident iteration for 2..32 right-hand sides, one
        // matrix pass per SpMV for all columns (opt-in)
        Factory& with_fused_multi_rhs(bool f)
        {
            fused_multi_rhs_ = f;
            return *this;
        }
        Factory& with_check_every(int k)
        {
            check_every_ = k;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Bicgstab(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    bool used_fused_path() const { return used_fused_; }

protected:
    Bicgstab(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), fused_(f.fused_), fused_multi_rhs_(f.fused_multi_rhs_),
          check_every_(std::max(1, f.check_every_))
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        if (fused_ && try_fused<int32>(b, x)) return;
        if (fused_ && try_fused<int64>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int32>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int64>(b, x)) return;
        used_fused_ = false;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type nrhs = sz.cols;
        auto mk = [&] { return b->create_like(sz); };  // reduces like b (distributed vectors)
        auto sc = [&] { return Dense::create(exec, dim2{1, nrhs}); };
        auto r = mk(), z = mk(), y = mk(), v = mk(), s = mk(), t = mk(), p = mk(), rr = mk();
        auto alpha = sc(), beta = sc(), gamma = sc(), prev_rho = sc(), rho = sc(), omega = sc();
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
#define GKOB_VS(d) (d)->get_values(), (d)->get_stride()
#define GKOB_CVS(d) (d)->get_const_values(), (d)->get_stride()
        GKOB_CALL(vabi<V>::bicgstab_initialize(
            ctx, sz.rows, nrhs, GKOB_CVS(b), GKOB_VS(r), GKOB_VS(rr), GKOB_VS(y), GKOB_VS(s),
            GKOB_VS(t), GKOB_VS(z), GKOB_VS(v), GKOB_VS(p), prev_rho->get_values(),
            rho->get_values(), alpha->get_values(), beta->get_values(), gamma->get_values(),
            omega->get_values(), stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), r.get());
        stop::CriterionArgs args{this->system_matrix_, b, x, r.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        rr->copy_from(r.get());
        int64 iter = -1;
        while (true) {
            ++iter;
            rr->compute_conj_dot(r.get(), rho.get());
            stop::Updater u;
            u.num_iterations = iter;
            u.residual = r.get();
            u.implicit_sq_residual_norm = rho.get();
            u.solution = x;
            if (crit->check(1, true, &stop_status, &one_changed, u)) break;
            GKOB_CALL(vabi<V>::bicgstab_step_1(ctx, sz.rows, nrhs, GKOB_CVS(r), GKOB_VS(p),
                                               GKOB_CVS(v), rho->get_const_values(),
                                               prev_rho->get_const_values(),
                                               alpha->get_const_values(), omega->get_const_values(),
                                               stop_status.get_const_data()));
            this->preconditioner_->apply(p.get(), y.get());
            this->system_matrix_->apply(y.get(), v.get());
            rr->compute_conj_dot(v.get(), beta.get());
            GKOB_CALL(vabi<V>::bicgstab_step_2(ctx, sz.rows, nrhs, GKOB_CVS(r), GKOB_VS(s),
                                               GKOB_CVS(v), rho->get_const_values(),
                                               alpha->get_values(), beta->get_const_values(),
                                               stop_status.get_const_data()));
            stop::Updater u2;
            u2.num_iterations = iter;
            u2.residual = s.get();
            u2.implicit_sq_residual_norm = rho.get();
            const bool all_stopped = crit->check(1, false, &stop_status, &one_changed, u2);
            if (one_changed)
                GKOB_CALL(vabi<V>::bicgstab_finalize(ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_CVS(y),
                                                     alpha->get_const_values(),
                                                     stop_status.get_data()));
            if (all_stopped) break;
            this->preconditioner_->apply(s.get(), z.get());
            this->system_matrix_->apply(z.get(), t.get());
            s->compute_conj_dot(t.get(), gamma.get());
            t->compute_conj_dot(t.get(), beta.get());
            GKOB_CALL(vabi<V>::bicgstab_step_3(
                ctx, sz.rows, nrhs, GKOB_VS(x), GKOB_VS(r), GKOB_CVS(s), GKOB_CVS(t), GKOB_CVS(y),
                GKOB_CVS(z), alpha->get_const_values(), beta->get_const_values(),
                gamma->get_const_values(), omega->get_values(), stop_status.get_const_data()));
            std::swap(prev_rho, rho);
        }
        this->record(iter, stop_status);
    }

    // Fused device-resident path (csrc/fused_bicgstab.cu): five launches per iteration, a graph of
    // check_every iterations per read of the control block.
    template <typename I>
    bool try_fused(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (!this->template fused_problem<I>(b, x, f) || !this->template fused_scalar_preconditioner<I>(f))
            return false;
        const auto A = f.A;
        const V* inv_diag = f.inv_diag;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 nnz = A->get_num_stored_elements();
        auto& st = single_;
        st.reshape(n, 1, [&] {
            st.ws = Dense::create(exec, dim2{(size_type)(8 * n), 1});
            st.sc = array<V>(exec, 16);
            st.ctl = array<int32>(exec, 8);
            st.work = array<V>(exec, (size_type)vabi<V>::fused_work_size(ctx));
        });
        V* r = st.ws->get_values();
        V *rr = r + n, *p = r + 2 * n, *v = r + 3 * n, *y = r + 4 * n, *s = r + 5 * n, *t = r + 6 * n,
          *z = r + 7 * n;
        V* xv = x->get_values();
        V* sc = st.sc.get_data();
        int32* ctl = st.ctl.get_data();
        V* work = st.work.get_data();
        // r = b - A x
        exec->copy(r, b->get_const_values(), n);
        auto rview = Dense::create_view(exec, dim2{(size_type)n, 1}, r, 1);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rview.get());
        if (f.baseline == 0)  // ||b|| into sc[4]
            GKOB_CALL(vabi<V>::norm2(ctx, n, 1, b->get_const_values(), 1, sc + 4));
        GKOB_CALL(vabi<V>::bicgstab_fused_init(ctx, n, r, rr, p, v, y, s, t, z, sc, ctl, work, f.max_iters,
                                               f.res_kind, f.iter_first, f.baseline, (V)f.factor));
        auto spmv_dot2 = [&](const V* in, V* out, const V* w, V* dot, V* dot2) {
            GKOB_CALL((viabi<V, I>::csr_spmv_dot2(ctx, A->get_plan(), n, n, nnz, A->get_const_row_ptrs(),
                                                  A->get_const_col_idxs(), A->get_const_values(), in, out,
                                                  w, dot, dot2, work, ctl)));
        };
        const FusedKey key{1, nnz, r, xv, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values(), A->get_plan()};
        st.capture(ctx, key, 1, [&](int64) {
            for (int k = 0; k < check_every_; ++k) {
                GKOB_CALL(vabi<V>::bicgstab_fused_step_p(ctx, n, p, r, v, y, inv_diag, sc, ctl));
                spmv_dot2(y, v, rr, sc + 2, nullptr);
                GKOB_CALL(vabi<V>::bicgstab_fused_step_s(ctx, n, r, v, s, z, inv_diag, sc, ctl, work));
                spmv_dot2(z, t, s, sc + 8, sc + 2);
                GKOB_CALL(vabi<V>::bicgstab_fused_step_xr(ctx, n, xv, r, s, t, y, z, rr, sc, ctl, work));
            }
        });
        // every captured iteration ends with step_xr, so a stop read here has its finalize applied
        const auto [flags, iters] = st.poll(*exec, "fused BiCGStab", [] { return 0; });
        this->num_iterations_ = (size_type)iters;
        this->status_.assign(1, (uint8)flags);
        used_fused_ = true;
        return true;
    }

    // Fused device-resident path for k = 2..32 right-hand sides (csrc/fused_bicgstab_mrhs.cu): the
    // admission of try_fused with b and x of k columns stored without gaps.  Every column stops on
    // its own, at the top or the mid-iteration check; the device keeps a stopped column's x, r and p
    // as the loop's masked steps leave them, and the host reads all k statuses at the end.
    template <typename I>
    bool try_fused_multi_rhs(const Dense* b, Dense* x) const
    {
        typename Base::template FusedProblem<I> f;
        if (b->get_size().cols < 2 || !this->template fused_problem<I>(b, x, f, 32) ||
            !this->template fused_scalar_preconditioner<I>(f))
            return false;
        const auto A = f.A;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows;
        const int64 k = (int64)b->get_size().cols;
        const int64 nnz = A->get_num_stored_elements();
        auto& m = mrhs_;
        // workspace r, rr, p, v, y, s, t, z (n x k each), per-column scalars, statuses, control block,
        // partials
        m.reshape(n, k, [&] {
            m.ws = Dense::create(exec, dim2{(size_type)(8 * n * k), 1});
            m.sc = array<V>(exec, (size_type)(10 * k));
            m.status = array<uint8>(exec, (size_type)k);
            m.ctl = array<int32>(exec, 8);
            m.work = array<V>(exec, (size_type)vabi<V>::bicgstab_mrhs_work_size(ctx, k));
        });
        const int64 nk = n * k;
        V* r = m.ws->get_values();
        V *rr = r + nk, *p = r + 2 * nk, *v = r + 3 * nk, *y = r + 4 * nk, *s = r + 5 * nk, *t = r + 6 * nk,
          *z = r + 7 * nk;
        V* xv = x->get_values();
        V* sc = m.sc.get_data();
        uint8* status = m.status.get_data();
        int32* ctl = m.ctl.get_data();
        V* work = m.work.get_data();
        const V* inv_diag = f.inv_diag;
        // r = b - A x
        exec->copy(r, b->get_const_values(), nk);
        auto rview = Dense::create_view(exec, dim2{(size_type)n, (size_type)k}, r, (size_type)k);
        A->apply(this->neg_one_.get(), x, this->one_.get(), rview.get());
        if (f.baseline == 0)  // ||b_j|| into sc[4k + j]
            GKOB_CALL(vabi<V>::norm2(ctx, n, k, b->get_const_values(), k, sc + 4 * k));
        GKOB_CALL(vabi<V>::bicgstab_mrhs_init(ctx, n, k, r, rr, p, v, y, s, t, z, sc, status, ctl, work,
                                              f.max_iters, f.res_kind, f.iter_first, f.baseline, (V)f.factor));
        auto spmv_mdot2 = [&](const V* in, V* out, const V* w, V* dots, V* dots2) {
            GKOB_CALL((viabi<V, I>::csr_spmv_mdot2(ctx, n, n, nnz, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                                                   A->get_const_values(), in, k, out, w, dots, dots2, work,
                                                   ctl)));
        };
        const FusedKey key{k, nnz, r, xv, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values()};
        m.capture(ctx, key, 1, [&](int64) {
            for (int it = 0; it < check_every_; ++it) {
                GKOB_CALL(vabi<V>::bicgstab_mrhs_step_p(ctx, n, k, p, r, v, y, inv_diag, sc, status, ctl));
                spmv_mdot2(y, v, rr, sc + 2 * k, nullptr);
                GKOB_CALL(vabi<V>::bicgstab_mrhs_step_s(ctx, n, k, r, v, s, z, inv_diag, sc, status, ctl, work));
                spmv_mdot2(z, t, s, sc + 8 * k, sc + 2 * k);
                GKOB_CALL(vabi<V>::bicgstab_mrhs_step_xr(ctx, n, k, xv, r, s, t, y, z, rr, sc, status, ctl,
                                                         work));
            }
        });
        // every captured iteration ends with step_xr, so a stop read here has its finalizes paid
        this->record(m.poll(*exec, "fused BiCGStab (several right-hand sides)", [] { return 0; }).second,
                     m.status);
        used_fused_ = true;
        return true;
    }

private:
    bool fused_;
    bool fused_multi_rhs_;
    int check_every_;
    mutable bool used_fused_ = false;
    using FusedKey = typename Base::FusedKey;
    mutable typename Base::FusedState single_, mrhs_;
};

// ---------------------------------------------------------------------------------------------
// Gmres (core/solver/gmres.cpp:321-626, non-flexible)
// ---------------------------------------------------------------------------------------------
template <typename V>
class Gmres : public SolverBase<V> {
    using Base = SolverBase<V>;
    using Dense = matrix::Dense<V>;

public:
    struct Factory : SolverFactoryBase<Factory> {
        size_type krylov_dim_ = 100;  // include/ginkgo/core/solver/gmres.hpp:32
        gmres::ortho_method ortho_ = gmres::ortho_method::mgs;
        Factory& with_krylov_dim(size_type d)
        {
            krylov_dim_ = d;
            return *this;
        }
        Factory& with_ortho_method(gmres::ortho_method m)
        {
            ortho_ = m;
            return *this;
        }
        bool fused_ = false;
        int check_every_ = 16;  // DESIGN.md 4.5: 8 to 16 are equally fast on an H100, 1 is up to 25 % slower
        // ginkgo_b200 extension: device-resident fused iteration where applicable (default off)
        Factory& with_fused(bool f)
        {
            fused_ = f;
            return *this;
        }
        bool fused_multi_rhs_ = false;
        // ginkgo_b200 extension: the device-resident iteration for 2..32 right-hand sides, one matrix
        // pass per SpMV for all columns (opt-in, independent of with_fused)
        Factory& with_fused_multi_rhs(bool f)
        {
            fused_multi_rhs_ = f;
            return *this;
        }
        // iterations per graph launch (and per read of the control block) on the fused paths
        Factory& with_check_every(int k)
        {
            check_every_ = k;
            return *this;
        }
        std::unique_ptr<LinOp> generate(std::shared_ptr<const LinOp> op) const override
        {
            auto exec = this->exec_ ? this->exec_ : op->get_executor();
            return std::unique_ptr<LinOp>(new Gmres(exec, *this, op));
        }
    };
    static Factory build() { return Factory{}; }
    bool used_fused_path() const { return used_fused_; }

protected:
    Gmres(std::shared_ptr<const Executor> exec, const Factory& f, std::shared_ptr<const LinOp> op)
        : Base(exec, f, op), krylov_dim_(f.krylov_dim_), ortho_(f.ortho_), fused_(f.fused_),
          fused_multi_rhs_(f.fused_multi_rhs_), check_every_(std::max(1, f.check_every_))
    {}
    using Base::apply_impl;
    void apply_impl(const LinOp* lb, LinOp* lx) const override
    {
        auto b = as<Dense>(lb);
        auto x = as<Dense>(lx);
        if (fused_ && try_fused<int32>(b, x)) return;
        if (fused_ && try_fused<int64>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int32>(b, x)) return;
        if (fused_multi_rhs_ && try_fused_multi_rhs<int64>(b, x)) return;
        used_fused_ = false;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const dim2 sz = b->get_size();
        const size_type n = sz.rows, nrhs = sz.cols, kd = krylov_dim_;
        auto residual = b->create_like(sz), precv = b->create_like(sz), before = b->create_like(sz),
             after = b->create_like(sz);
        auto krylov = b->create_like(dim2{n * (kd + 1), nrhs});
        auto hess = Dense::create(exec, dim2{kd, (kd + 1) * nrhs});
        hess->fill(V(0));
        std::unique_ptr<Dense> hess_aux;
        if (ortho_ == gmres::ortho_method::cgs2) {
            hess_aux = Dense::create(exec, dim2{kd + 1, nrhs});
            hess_aux->fill(V(0));
        }
        auto gsin = Dense::create(exec, dim2{kd, nrhs}), gcos = Dense::create(exec, dim2{kd, nrhs});
        auto rnc = Dense::create(exec, dim2{kd + 1, nrhs});
        rnc->fill(V(0));
        auto rnorm = Dense::create(exec, dim2{1, nrhs});
        auto y = Dense::create(exec, dim2{kd, nrhs});
        y->fill(V(0));
        array<std::uint64_t> fin(exec, nrhs);
        array<uint8> stop_status(exec, nrhs);
        bool one_changed = false;
        GKOB_CALL(vabi<V>::gmres_initialize(ctx, n, nrhs, kd, GKOB_CVS(b), GKOB_VS(residual),
                                            GKOB_VS(gsin), GKOB_VS(gcos), stop_status.get_data()));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        residual->compute_norm2(rnorm.get());
        auto restart = [&] {
            GKOB_CALL(vabi<V>::gmres_restart(ctx, n, nrhs, GKOB_CVS(residual),
                                             rnorm->get_const_values(), rnc->get_values(),
                                             GKOB_VS(krylov), fin.get_data()));
        };
        restart();
        stop::CriterionArgs args{this->system_matrix_, b, x, residual.get()};
        auto crit = stop::combine_and_generate(this->criteria_, exec, args);
        auto solve_and_update = [&] {
            GKOB_CALL(vabi<V>::gmres_solve_krylov(ctx, nrhs, GKOB_CVS(rnc), GKOB_CVS(hess),
                                                  GKOB_VS(y), fin.get_const_data(),
                                                  stop_status.get_const_data()));
            GKOB_CALL(vabi<V>::gmres_multi_axpy(ctx, n, nrhs, GKOB_CVS(krylov), GKOB_CVS(y),
                                                GKOB_VS(before), fin.get_const_data(),
                                                stop_status.get_data()));
            this->preconditioner_->apply(before.get(), after.get());
            x->add_scaled(this->one_.get(), after.get());
        };
        int64 total_iter = -1;
        size_type restart_iter = 0;
        while (true) {
            ++total_iter;
            stop::Updater u;
            u.num_iterations = total_iter;
            u.residual = residual.get();
            u.residual_norm = rnorm.get();
            u.solution = x;
            if (crit->check(1, false, &stop_status, &one_changed, u)) break;
            if (restart_iter == kd) {
                solve_and_update();
                residual->copy_from(b);
                this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(),
                                            residual.get());
                residual->compute_norm2(rnorm.get());
                restart();
                restart_iter = 0;
            }
            auto this_k = krylov->create_submatrix_rows(n * restart_iter, n * (restart_iter + 1));
            auto next_k = krylov->create_submatrix_rows(n * (restart_iter + 1), n * (restart_iter + 2));
            this->preconditioner_->apply(this_k.get(), precv.get());
            // hessenberg_iter = (restart_iter + 2) x nrhs view of row restart_iter
            auto hiter = Dense::create_view(exec, dim2{restart_iter + 2, nrhs},
                                            hess->get_values() + restart_iter * hess->get_stride(),
                                            nrhs);
            this->system_matrix_->apply(precv.get(), next_k.get());
            auto sub_all = [&](Dense* h) {
                for (size_type i = 0; i <= restart_iter; ++i) {
                    auto hi = h->create_submatrix_rows(i, i + 1);
                    auto ki = krylov->create_submatrix_rows(n * i, n * (i + 1));
                    next_k->sub_scaled(hi.get(), ki.get());
                }
            };
            if (ortho_ == gmres::ortho_method::mgs) {
                for (size_type i = 0; i <= restart_iter; ++i) {
                    auto hi = hiter->create_submatrix_rows(i, i + 1);
                    auto ki = krylov->create_submatrix_rows(n * i, n * (i + 1));
                    ki->compute_conj_dot(next_k.get(), hi.get());
                    next_k->sub_scaled(hi.get(), ki.get());
                }
            } else {
                GKOB_CALL(vabi<V>::gmres_multi_dot(ctx, n, nrhs, restart_iter + 1, GKOB_CVS(krylov),
                                                   GKOB_CVS(next_k), GKOB_VS(hiter)));
                if (b->get_reducer()) b->get_reducer()->sum(hiter->get_values(), (restart_iter + 1) * nrhs);
                sub_all(hiter.get());
                if (ortho_ == gmres::ortho_method::cgs2) {
                    auto haux = hess_aux->create_submatrix_rows(0, restart_iter + 2);
                    GKOB_CALL(vabi<V>::gmres_multi_dot(ctx, n, nrhs, restart_iter + 1,
                                                       GKOB_CVS(krylov), GKOB_CVS(next_k),
                                                       GKOB_VS(haux)));
                    if (b->get_reducer())
                        b->get_reducer()->sum(haux->get_values(), (restart_iter + 1) * nrhs);
                    sub_all(haux.get());
                    hiter->add_scaled(this->one_.get(), haux.get());
                }
            }
            auto hnorm = hiter->create_submatrix_rows(restart_iter + 1, restart_iter + 2);
            next_k->compute_norm2(hnorm.get());
            next_k->inv_scale(hnorm.get());
            GKOB_CALL(vabi<V>::gmres_hessenberg_qr(ctx, nrhs, GKOB_VS(gsin), GKOB_VS(gcos),
                                                   rnorm->get_values(), GKOB_VS(rnc), GKOB_VS(hiter),
                                                   restart_iter, fin.get_data(),
                                                   stop_status.get_const_data()));
            restart_iter++;
        }
        solve_and_update();
        this->record(total_iter, stop_status);
#undef GKOB_VS
#undef GKOB_CVS
    }

    // Fused device-resident path (csrc/fused_gmres.cu): at Krylov index j, MGS takes j + 3 launches, CGS 4
    // and CGS2 6 (one more with block Jacobi); the Hessenberg column, the Givens rotations and the stopping
    // check stay on the device.  One graph per batch of check_every iterations, a batch never crosses a
    // restart; the host reads the 32-byte control block after each batch.  The initial residual, the
    // restart and the final update are the loop's kernels, issued by the host.
    template <typename I>
    bool try_fused(const Dense* b, Dense* x) const
    {
        if (krylov_dim_ == 0) return false;
        typename Base::template FusedProblem<I> f;
        // ImplicitResidualNorm: the loop reports NotSupported, and so must this solver
        if (!this->template fused_problem<I>(b, x, f) || f.res_kind == 2) return false;
        // any Jacobi (of either index type): scalar (its inverted diagonal), block with given or detected
        // blocks, adaptive storage
        const V* inv_diag = nullptr;
        bool block = false;
        const void* pre_key[3] = {nullptr, nullptr, nullptr};
        std::function<void(const V*, V*, const int32*)> block_apply;
        auto take_jacobi = [&](auto* J) {
            pre_key[0] = J->get_blocks();
            pre_key[1] = J->get_block_precisions();
            if (J->get_max_block_size() == 1) {
                inv_diag = J->get_blocks();
                return;
            }
            using JI = std::remove_cv_t<std::remove_pointer_t<decltype(J->get_const_block_pointers())>>;
            pre_key[2] = J->get_const_block_pointers();
            block = true;
            block_apply = [J, this](const V* in, V* out, const int32* ctl) {
                const auto& s = J->get_storage_scheme();
                GKOB_CALL((viabi<V, JI>::gmres_fused_block_apply(
                    this->exec_->ctx(), (int64)J->get_num_blocks(), (int32)J->get_max_block_size(), s.block_offset,
                    s.group_offset, (int32)s.group_power, J->get_block_precisions(), J->get_const_block_pointers(),
                    J->get_blocks(), in, out, ctl)));
            };
        };
        const LinOp* pre = this->preconditioner_.get();
        if (auto J = dynamic_cast<const preconditioner::Jacobi<V, int32>*>(pre))
            take_jacobi(J);
        else if (auto J = dynamic_cast<const preconditioner::Jacobi<V, int64>*>(pre))
            take_jacobi(J);
        else if (!dynamic_cast<const matrix::Identity<V>*>(pre))
            return false;
        const auto A = f.A;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows, kd = (int64)krylov_dim_;
        const int64 nnz = A->get_num_stored_elements();
        auto& st = single_;
        st.reshape(n, 1, [&] {
            fkrylov_ = Dense::create(exec, dim2{(size_type)(n * (kd + 1)), 1});
            fvec_ = Dense::create(exec, dim2{(size_type)(4 * n), 1});  // residual | z | before | after
            fhess_ = Dense::create(exec, dim2{(size_type)kd, (size_type)(kd + 1)});
            st.sc = array<V>(exec, (size_type)(5 * kd + 11));
            st.work = array<V>(exec, (size_type)vabi<V>::gmres_fused_work_size(ctx, kd));
            ffin_ = array<std::uint64_t>(exec, 1);
            st.status = array<uint8>(exec, 1);
            st.ctl = array<int32>(exec, 8);
        });
        V* K = fkrylov_->get_values();
        // x is not baked in: the host's final update applies it
        const FusedKey key{1, nnz, K, nullptr, {pre_key[0], pre_key[1], pre_key[2]}, A->get_const_row_ptrs(),
                           A->get_const_col_idxs(), A->get_const_values(), A->get_plan()};
        auto col = [&](int c) {
            return Dense::create_view(exec, dim2{(size_type)n, 1}, fvec_->get_values() + c * n, 1);
        };
        auto residual = col(0), z = col(1), before = col(2), after = col(3);
        V* hess = fhess_->get_values();
        const int64 hs = fhess_->get_stride();
        V *sc = st.sc.get_data(), *gsin = sc + 8, *gcos = gsin + kd, *rnc = gcos + kd, *y = rnc + kd + 1,
          *rnorm = y + kd, *haux = rnorm + 1;
        auto rnorm_view = Dense::create_view(exec, dim2{1, 1}, rnorm, 1);
        std::uint64_t* fin = ffin_.get_data();
        uint8* stop = st.status.get_data();
        int32* ctl = st.ctl.get_data();
        V* work = st.work.get_data();
        // the loop's start: fresh Hessenberg, rnc and y; initialize; r = b - A x; ||r||; restart
        fhess_->fill(V(0));
        GKOB_CALL(vabi<V>::fill(ctx, 2 * kd + 1, 1, rnc, 1, V(0)));
        GKOB_CALL(vabi<V>::gmres_initialize(ctx, n, 1, kd, b->get_const_values(), 1, residual->get_values(), 1,
                                            gsin, 1, gcos, 1, stop));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        residual->compute_norm2(rnorm_view.get());
        auto restart = [&] {
            GKOB_CALL(vabi<V>::gmres_restart(ctx, n, 1, residual->get_const_values(), 1, rnorm, rnc, K, 1, fin));
        };
        restart();
        if (f.baseline == 0)  // ||b|| into sc[1]
            GKOB_CALL(vabi<V>::norm2(ctx, n, 1, b->get_const_values(), 1, sc + 1));
        GKOB_CALL(vabi<V>::gmres_fused_init(ctx, rnorm, sc, ctl, stop, f.max_iters, f.res_kind, f.iter_first,
                                            f.baseline, (V)f.factor));
        auto solve_and_update = [&] {
            GKOB_CALL(vabi<V>::gmres_solve_krylov(ctx, 1, rnc, 1, hess, hs, y, 1, fin, stop));
            GKOB_CALL(vabi<V>::gmres_multi_axpy(ctx, n, 1, K, 1, y, 1, before->get_values(), 1, fin, stop));
            this->preconditioner_->apply(before.get(), after.get());
            x->add_scaled(this->one_.get(), after.get());
        };
        auto enqueue_iteration = [&](int64 j) {
            V *vj = K + j * n, *w = vj + n, *hcol = hess + j * hs;
            V* in = vj;
            if (block) {
                if (j > 0) GKOB_CALL(vabi<V>::gmres_fused_scale(ctx, n, vj, nullptr, nullptr, sc, ctl, 1));
                block_apply(vj, z->get_values(), ctl);
                in = z->get_values();
            } else if (inv_diag) {
                GKOB_CALL(vabi<V>::gmres_fused_scale(ctx, n, vj, z->get_values(), inv_diag, sc, ctl, j > 0));
                in = z->get_values();
            } else if (j > 0) {
                GKOB_CALL(vabi<V>::gmres_fused_scale(ctx, n, vj, nullptr, nullptr, sc, ctl, 1));
            }
            GKOB_CALL((viabi<V, I>::csr_spmv_dot2(ctx, A->get_plan(), n, n, nnz, A->get_const_row_ptrs(),
                                                  A->get_const_col_idxs(), A->get_const_values(), in, w, K,
                                                  hcol, nullptr, work, ctl)));
            auto final_pass = [&](int64 first, const V* coef, const V* add) {
                GKOB_CALL(vabi<V>::gmres_fused_final_pass(ctx, n, w, K, first, coef, add, hcol, j, gsin, gcos, rnorm,
                                                          rnc, fin, stop, sc, ctl, work));
            };
            if (ortho_ == gmres::ortho_method::mgs) {
                for (int64 i = 1; i <= j; ++i)
                    GKOB_CALL(vabi<V>::gmres_fused_mgs_pass(ctx, n, w, K + (i - 1) * n, K + i * n, hcol, i, ctl,
                                                            work));
                final_pass(j, hcol, nullptr);
                return;
            }
            // CGS: h_1..h_j in one pass (h_0 came with the SpMV), one subtract pass over all bases
            if (j > 0) GKOB_CALL(vabi<V>::gmres_fused_multi_dot(ctx, n, j, K + n, w, hcol + 1, ctl, work));
            if (ortho_ == gmres::ortho_method::cgs) {
                final_pass(0, hcol, nullptr);
                return;
            }
            // CGS2: subtract, re-orthogonalise against all bases into haux, subtract again; h += haux
            GKOB_CALL(vabi<V>::gmres_fused_sub_pass(ctx, n, w, K, hcol, j, ctl));
            GKOB_CALL(vabi<V>::gmres_fused_multi_dot(ctx, n, j + 1, K, w, haux, ctl, work));
            final_pass(0, haux, haux);
        };
        // batches start at Krylov index 0, c, 2c, ... and end at the restart
        const int64 ce = std::min<int64>(check_every_, kd);
        st.capture(ctx, key, (kd + ce - 1) / ce, [&](int64 i) {
            for (int64 j = i * ce; j < std::min((i + 1) * ce, kd); ++j) enqueue_iteration(j);
        });
        int64 j = 0;
        auto next_batch = [&] {
            // the loop's restart, only once the check at the top of iteration krylov_dim said "running"
            if (j == kd) {
                solve_and_update();
                residual->copy_from(b);
                this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
                residual->compute_norm2(rnorm_view.get());
                restart();
                j = 0;
            }
            const int64 i = j / ce;
            j = std::min(j + ce, kd);
            return i;
        };
        const int32 iters = st.poll(*exec, "fused GMRES", next_batch).second;
        solve_and_update();
        this->record((size_type)iters, st.status);
        used_fused_ = true;
        return true;
    }

    // Fused device-resident path for k = 2..32 right-hand sides (csrc/fused_gmres_mrhs.cu): at Krylov
    // index j, MGS takes j + 3 launches, CGS 4 and CGS2 6, and the k-wide SpMV is one matrix pass for all
    // columns.  Every array the restart block shares with the loop kernels has the loop's layout, so the
    // initial residual, the restart and the final update are the loop's own calls on all k columns.  Each
    // column stops on its own; a batch of check_every iterations per graph never crosses a restart.
    template <typename I>
    bool try_fused_multi_rhs(const Dense* b, Dense* x) const
    {
        if (krylov_dim_ == 0) return false;
        typename Base::template FusedProblem<I> f;
        // ImplicitResidualNorm: the loop reports NotSupported, and so must this solver
        if (b->get_size().cols < 2 || !this->template fused_problem<I>(b, x, f, 32) || f.res_kind == 2)
            return false;
        // Identity or scalar Jacobi of either index type.  Block Jacobi is the loop's: its k-column apply
        // switches to a tensor-core kernel whose bits a SIMT apply would not reproduce.
        const V* inv_diag = nullptr;
        const LinOp* pre = this->preconditioner_.get();
        if (auto J = dynamic_cast<const preconditioner::Jacobi<V, int32>*>(pre)) {
            if (J->get_max_block_size() != 1) return false;
            inv_diag = J->get_blocks();
        } else if (auto J = dynamic_cast<const preconditioner::Jacobi<V, int64>*>(pre)) {
            if (J->get_max_block_size() != 1) return false;
            inv_diag = J->get_blocks();
        } else if (!dynamic_cast<const matrix::Identity<V>*>(pre)) {
            return false;
        }
        const auto A = f.A;
        auto exec = this->exec_;
        auto ctx = exec->ctx();
        const int64 n = this->size_.rows, kd = (int64)krylov_dim_;
        const int64 k = (int64)b->get_size().cols, nk = n * k;
        const int64 nnz = A->get_num_stored_elements();
        auto& m = mrhs_;
        // basis n (kd+1) x k; residual, z, before, after n x k each; the Hessenberg kd x (kd+1) k;
        // sc[3k], gsin, gcos, y (kd x k), rnc, haux ((kd+1) x k), rnorm
        m.reshape(n, k, [&] {
            m.ws = Dense::create(exec, dim2{(size_type)(nk * (kd + 5)), 1});
            mhess_ = Dense::create(exec, dim2{(size_type)kd, (size_type)((kd + 1) * k)});
            m.sc = array<V>(exec, (size_type)(k * (5 * kd + 6)));
            m.status = array<uint8>(exec, (size_type)k);
            m.ctl = array<int32>(exec, 8);
            m.work = array<V>(exec, (size_type)vabi<V>::gmres_mrhs_work_size(ctx, k, kd));
            mfin_ = array<std::uint64_t>(exec, (size_type)k);
        });
        V* K = m.ws->get_values();
        auto vec = [&](int c) {
            return Dense::create_view(exec, dim2{(size_type)n, (size_type)k}, K + nk * (kd + 1 + c), (size_type)k);
        };
        auto residual = vec(0), z = vec(1), before = vec(2), after = vec(3);
        V* hess = mhess_->get_values();
        const int64 hs = mhess_->get_stride();
        V *sc = m.sc.get_data(), *gsin = sc + 3 * k, *gcos = gsin + kd * k, *rnc = gcos + kd * k,
          *y = rnc + (kd + 1) * k, *rnorm = y + kd * k, *haux = rnorm + k;
        auto rnorm_view = Dense::create_view(exec, dim2{1, (size_type)k}, rnorm, (size_type)k);
        std::uint64_t* fin = mfin_.get_data();
        uint8* status = m.status.get_data();
        int32* ctl = m.ctl.get_data();
        V* work = m.work.get_data();
        // the loop's start: fresh Hessenberg, rnc, y and haux; initialize; r = b - A x; ||r||; restart
        mhess_->fill(V(0));
        GKOB_CALL(vabi<V>::fill(ctx, (3 * kd + 3) * k, 1, rnc, 1, V(0)));
        GKOB_CALL(vabi<V>::gmres_initialize(ctx, n, k, kd, b->get_const_values(), k, residual->get_values(), k, gsin,
                                            k, gcos, k, status));
        this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
        residual->compute_norm2(rnorm_view.get());
        auto restart = [&] {
            GKOB_CALL(vabi<V>::gmres_restart(ctx, n, k, residual->get_const_values(), k, rnorm, rnc, K, k, fin));
        };
        restart();
        if (f.baseline == 0)  // ||b_c|| into sc[k + c]
            GKOB_CALL(vabi<V>::norm2(ctx, n, k, b->get_const_values(), k, sc + k));
        GKOB_CALL(vabi<V>::gmres_mrhs_init(ctx, k, rnorm, sc, status, ctl, f.max_iters, f.res_kind, f.iter_first,
                                           f.baseline, (V)f.factor));
        // before keeps a finalized column's last correction, as the loop's does
        auto solve_and_update = [&] {
            GKOB_CALL(vabi<V>::gmres_solve_krylov(ctx, k, rnc, k, hess, hs, y, k, fin, status));
            GKOB_CALL(vabi<V>::gmres_multi_axpy(ctx, n, k, K, k, y, k, before->get_values(), k, fin, status));
            this->preconditioner_->apply(before.get(), after.get());
            x->add_scaled(this->one_.get(), after.get());
        };
        auto enqueue_iteration = [&](int64 j) {
            V *vj = K + j * nk, *w = vj + nk, *hcol = hess + j * hs;
            V* in = vj;
            if (inv_diag) {
                GKOB_CALL(vabi<V>::gmres_mrhs_scale(ctx, n, k, vj, z->get_values(), inv_diag, sc, status, ctl, j > 0));
                in = z->get_values();
            } else if (j > 0) {
                GKOB_CALL(vabi<V>::gmres_mrhs_scale(ctx, n, k, vj, nullptr, nullptr, sc, status, ctl, 1));
            }
            GKOB_CALL((viabi<V, I>::csr_spmv_mdot2(ctx, n, n, nnz, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                                                   A->get_const_values(), in, k, w, K, hcol, nullptr, work, ctl)));
            auto final_pass = [&](int64 first, const V* coef, const V* add) {
                GKOB_CALL(vabi<V>::gmres_mrhs_final_pass(ctx, n, k, w, K, first, coef, add, hcol, j, gsin, gcos,
                                                         rnorm, rnc, fin, status, sc, ctl, work));
            };
            if (ortho_ == gmres::ortho_method::mgs) {
                for (int64 i = 1; i <= j; ++i)
                    GKOB_CALL(vabi<V>::gmres_mrhs_mgs_pass(ctx, n, k, w, K + (i - 1) * nk, K + i * nk, hcol, i,
                                                           status, ctl, work));
                final_pass(j, hcol, nullptr);
                return;
            }
            // CGS: h_1..h_j in one pass (h_0 came with the SpMV), one subtract pass over all bases
            if (j > 0)
                GKOB_CALL(vabi<V>::gmres_mrhs_multi_dot(ctx, n, k, j, kd, K + nk, w, hcol + k, status, ctl, work));
            if (ortho_ == gmres::ortho_method::cgs) {
                final_pass(0, hcol, nullptr);
                return;
            }
            // CGS2: subtract, re-orthogonalise against all bases into haux, subtract again; h += haux
            GKOB_CALL(vabi<V>::gmres_mrhs_sub_pass(ctx, n, k, w, K, hcol, j, status, ctl));
            GKOB_CALL(vabi<V>::gmres_mrhs_multi_dot(ctx, n, k, j + 1, kd, K, w, haux, status, ctl, work));
            final_pass(0, haux, haux);
        };
        // x is not baked in: the host's final update applies it.  Batches start at Krylov index 0, c,
        // 2c, ... and end at the restart.
        const FusedKey key{k, nnz, K, nullptr, {inv_diag}, A->get_const_row_ptrs(), A->get_const_col_idxs(),
                           A->get_const_values()};
        const int64 ce = std::min<int64>(check_every_, kd);
        m.capture(ctx, key, (kd + ce - 1) / ce, [&](int64 i) {
            for (int64 j = i * ce; j < std::min((i + 1) * ce, kd); ++j) enqueue_iteration(j);
        });
        int64 j = 0;
        auto next_batch = [&] {
            // the loop's restart on all k columns, only once the check at the top of iteration krylov_dim
            // said "running"
            if (j == kd) {
                solve_and_update();
                residual->copy_from(b);
                this->system_matrix_->apply(this->neg_one_.get(), x, this->one_.get(), residual.get());
                residual->compute_norm2(rnorm_view.get());
                restart();
                j = 0;
            }
            const int64 i = j / ce;
            j = std::min(j + ce, kd);
            return i;
        };
        const int32 iters = m.poll(*exec, "fused GMRES (several right-hand sides)", next_batch).second;
        solve_and_update();
        this->record((size_type)iters, m.status);
        used_fused_ = true;
        return true;
    }

private:
    size_type krylov_dim_;
    gmres::ortho_method ortho_;
    bool fused_;
    bool fused_multi_rhs_;
    int check_every_;
    mutable bool used_fused_ = false;
    using FusedKey = typename Base::FusedKey;
    // the one-column path: sc, work, status and ctl in single_, the basis, vectors, Hessenberg and fin here
    mutable typename Base::FusedState single_;
    mutable std::unique_ptr<Dense> fkrylov_, fvec_, fhess_;
    mutable array<std::uint64_t> ffin_;
    // the several-column path: workspace and control block in mrhs_, Hessenberg and fin here
    mutable typename Base::FusedState mrhs_;
    mutable std::unique_ptr<Dense> mhess_;
    mutable array<std::uint64_t> mfin_;
};

}  // namespace solver
}  // namespace gko_b200
