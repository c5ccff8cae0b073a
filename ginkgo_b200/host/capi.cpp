// capi.cpp -- a C handle API over the C++ host layer (gko_b200.hpp) so that the Python
// harness (tests, bench.py) drives the SAME host code a C++ user links: executor, Csr, Dense
// views, preconditioner::Jacobi, stop criteria, solver::{Cg,Bicgstab,Gmres}.
#include <cstdio>
#include <fstream>
#include <iomanip>
#include <string>

#include "gko_b200_dist.hpp"

using namespace gko_b200;

namespace {
thread_local std::string g_err;
struct Handle {
    std::shared_ptr<Executor> exec;
    std::shared_ptr<LinOp> op;
};
template <typename F>
int guarded(F f)
{
    try {
        f();
        return 0;
    } catch (const DimensionMismatch& e) {
        g_err = std::string("DimensionMismatch: ") + e.what();
        return 2;
    } catch (const NotSupported& e) {
        g_err = std::string("NotSupported: ") + e.what();
        return 3;
    } catch (const std::exception& e) {
        g_err = e.what();
        return 1;
    }
}

// extra parameters of solver kinds 5 (Ir) and 6 (Chebyshev), set by gkob_solver_params
double g_relaxation = 1.0, g_foci_lo = 0.0, g_foci_hi = 1.0;
int g_ir_guess = 0;  // kind 5: 0 provided, 1 zero, 2 rhs (gkob_solver_guess)
// a generated preconditioner for the next gkob_solver_create_* (gkob_solver_preconditioner)
std::shared_ptr<const LinOp> g_generated_pre;

template <typename V>
std::unique_ptr<LinOp> make_solver(std::shared_ptr<Executor> exec, int kind,
                                   std::shared_ptr<LinOp> A, int precond_max_bs,
                                   const int32* block_ptrs, int64 nblocks, int64 max_iters,
                                   int res_kind, int baseline, double reduction, int iter_first,
                                   int krylov_dim, int ortho, int fused, int check_every,
                                   std::shared_ptr<const LinOp> generated_pre = nullptr)
{
    std::vector<std::shared_ptr<const stop::CriterionFactory>> crit;
    std::shared_ptr<const stop::CriterionFactory> it_c, res_c;
    if (max_iters >= 0) it_c = stop::Iteration::build().with_max_iters((size_type)max_iters).on(exec);
    auto mode = baseline == 0   ? stop::mode::rhs_norm
                : baseline == 1 ? stop::mode::initial_resnorm
                                : stop::mode::absolute;
    if (res_kind == 1)
        res_c = stop::ResidualNorm<V>::build().with_baseline(mode).with_reduction_factor(reduction).on(exec);
    else if (res_kind == 2)
        res_c = stop::ImplicitResidualNorm<V>::build()
                    .with_baseline(mode)
                    .with_reduction_factor(reduction)
                    .on(exec);
    if (iter_first) {
        if (it_c) crit.push_back(it_c);
        if (res_c) crit.push_back(res_c);
    } else {
        if (res_c) crit.push_back(res_c);
        if (it_c) crit.push_back(it_c);
    }
    std::shared_ptr<const LinOpFactory> pre;
    if (precond_max_bs > 0) {
        auto pb = preconditioner::Jacobi<V, int32>::build();
        pb.with_max_block_size((uint32)precond_max_bs);
        if (block_ptrs && precond_max_bs > 1)
            pb.with_block_pointers(std::vector<int32>(block_ptrs, block_ptrs + nblocks + 1));
        pre = pb.on(exec);
    }
    auto set_pre = [&](auto& f) {
        if (generated_pre)
            f.with_generated_preconditioner(generated_pre);
        else if (pre)
            f.with_preconditioner(pre);
    };
    if (generated_pre && kind == 5) throw NotSupported("make_solver: Ir takes a solver factory");
    if (kind == 0) {
        auto f = solver::Cg<V>::build();
        f.with_criteria(crit).with_fused((fused & 1) != 0).with_check_every(check_every);
        // bit 3 of `fused`: the fused iteration for several right-hand sides is opt-in
        f.with_fused_multi_rhs((fused & 8) != 0);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 1) {
        auto f = solver::Bicgstab<V>::build();
        // bit 1 of `fused`: the fused BiCGStab iteration is opt-in, bit 0 keeps meaning Cg's
        f.with_criteria(crit).with_fused((fused & 2) != 0).with_check_every(check_every);
        // bit 4 of `fused`: its iteration for several right-hand sides, opt-in as well
        f.with_fused_multi_rhs((fused & 16) != 0);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 10) {
        auto f = solver::Bicg<V>::build();
        f.with_criteria(crit);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 9) {
        auto f = solver::Minres<V>::build();
        // bit 6 of `fused`: the fused MINRES iteration is opt-in, as BiCGStab's and GMRES's
        f.with_criteria(crit).with_fused((fused & 64) != 0).with_check_every(check_every);
        // bit 7: its iteration for 2..32 right-hand sides, opt-in and independent of bit 6
        f.with_fused_multi_rhs((fused & 128) != 0);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 8) {
        auto f = solver::Gcr<V>::build();
        f.with_criteria(crit).with_krylov_dim((size_type)krylov_dim);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 7) {
        auto f = solver::PipeCg<V>::build();
        f.with_criteria(crit);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 5) {
        auto f = solver::Ir<V>::build();
        f.with_criteria(crit).with_relaxation_factor((V)g_relaxation);
        f.with_default_initial_guess(g_ir_guess == 1   ? solver::initial_guess_mode::zero
                                     : g_ir_guess == 2 ? solver::initial_guess_mode::rhs
                                                       : solver::initial_guess_mode::provided);
        if (pre) f.with_solver(pre);
        return f.on(exec)->generate(A);
    }
    if (kind == 6) {
        auto f = solver::Chebyshev<V>::build();
        f.with_criteria(crit).with_foci(g_foci_lo, g_foci_hi);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 3) {
        auto f = solver::Fcg<V>::build();
        f.with_criteria(crit);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    if (kind == 4) {
        auto f = solver::Cgs<V>::build();
        f.with_criteria(crit);
        set_pre(f);
        return f.on(exec)->generate(A);
    }
    auto f = solver::Gmres<V>::build();
    f.with_criteria(crit).with_krylov_dim((size_type)krylov_dim);
    // bit 2 of `fused`: the fused GMRES iteration is opt-in, as BiCGStab's
    f.with_fused((fused & 4) != 0).with_check_every(check_every);
    // bit 5: the fused GMRES iteration for 2..32 right-hand sides, opt-in and independent of bit 2
    f.with_fused_multi_rhs((fused & 32) != 0);
    f.with_ortho_method(ortho == 0   ? solver::gmres::ortho_method::mgs
                        : ortho == 1 ? solver::gmres::ortho_method::cgs
                                     : solver::gmres::ortho_method::cgs2);
    set_pre(f);
    return f.on(exec)->generate(A);
}
}  // namespace

// Csr::convert_to on the device: fmt = "ell" | "sellp" (p0 slice_size, p1 stride_factor) |
// "coo" | "hybrid" (p0: 0 automatic, 1 column_limit(p1), 2 imbalance_limit(pd),
// 3 imbalance_bounded_limit(pd, pd2), 4 minimal_storage_limit).  Returns a new LinOp handle.
template <typename V>
static std::shared_ptr<LinOp> convert_csr(const matrix::Csr<V, int32>* a, const std::string& f,
                                          long long p0, long long p1, double pd, double pd2)
{
    auto e = a->get_executor();
    if (f == "ell") {
        auto t = matrix::Ell<V, int32>::create(e);
        a->convert_to(t.get());
        return std::shared_ptr<LinOp>(std::move(t));
    }
    if (f == "sellp") {
        auto t = matrix::Sellp<V, int32>::create(e, (size_type)p0, (size_type)p1);
        a->convert_to(t.get());
        return std::shared_ptr<LinOp>(std::move(t));
    }
    if (f == "coo") {
        auto t = matrix::Coo<V, int32>::create(e);
        a->convert_to(t.get());
        return std::shared_ptr<LinOp>(std::move(t));
    }
    if (f == "hybrid") {
        using H = matrix::Hybrid<V, int32>;
        auto st = p0 == 1   ? H::column_limit((size_type)p1)
                  : p0 == 2 ? H::imbalance_limit(pd)
                  : p0 == 3 ? H::imbalance_bounded_limit(pd, pd2)
                  : p0 == 4 ? H::minimal_storage_limit()
                            : H::automatic();
        auto t = H::create(e, st);
        a->convert_to(t.get());
        return std::shared_ptr<LinOp>(std::move(t));
    }
    throw NotSupported("gkob_csr_convert: unknown format");
}


// preconditioner::Jacobi as an object of its own (generate, storage optimisation, transpose):
//   so_kind 0 none, 1 one precision_reduction byte for all blocks (so[0]), 2 block-wise so[0 .. so_len);
//   a byte 0xff is autodetect().  vt 0 double, 1 float.
template <typename V>
static std::shared_ptr<LinOp> make_jacobi(std::shared_ptr<Executor> exec, std::shared_ptr<LinOp> A, int max_bs,
                                          const int32* block_ptrs, long long nblocks, int so_kind,
                                          const unsigned char* so, long long so_len, double accuracy)
{
    auto pb = preconditioner::Jacobi<V, int32>::build();
    pb.with_max_block_size((uint32)max_bs);
    pb.with_accuracy(accuracy);
    if (block_ptrs && max_bs > 1) pb.with_block_pointers(std::vector<int32>(block_ptrs, block_ptrs + nblocks + 1));
    if (so_kind == 1) pb.with_storage_optimization(precision_reduction::from_byte(so[0]));
    if (so_kind == 2) {
        std::vector<precision_reduction> v;
        for (long long i = 0; i < so_len; ++i) v.push_back(precision_reduction::from_byte(so[i]));
        pb.with_storage_optimization(v);
    }
    return std::shared_ptr<LinOp>(pb.on(exec)->generate(A));
}
template <typename V>
static int jacobi_get(Handle* h, long long* meta, void* blocks, int32* ptrs, unsigned char* prec, void* cond)
{
    auto J = dynamic_cast<const preconditioner::Jacobi<V, int32>*>(h->op.get());
    if (!J) throw NotSupported("gkob_jacobi_get: not a Jacobi of this value type");
    auto e = J->get_executor();
    const auto& sch = J->get_storage_scheme();
    const long long nb = (long long)J->get_num_blocks();
    meta[0] = sch.block_offset;
    meta[1] = sch.group_offset;
    meta[2] = sch.group_power;
    meta[3] = nb;
    meta[4] = (long long)J->get_num_stored_elements();
    meta[5] = J->get_block_precisions() ? 1 : 0;
    if (blocks && meta[4]) e->copy_to_host((V*)blocks, J->get_blocks(), (size_type)meta[4]);
    if (ptrs && J->get_max_block_size() > 1) e->copy_to_host(ptrs, J->get_const_block_pointers(), (size_type)nb + 1);
    if (prec && J->get_block_precisions()) e->copy_to_host(prec, J->get_block_precisions(), (size_type)nb);
    if (cond && J->get_conditioning()) e->copy_to_host((V*)cond, J->get_conditioning(), (size_type)nb);
    return 0;
}

extern "C" {

void* gkob_jacobi_create(void* exec, int vt, void* matrix, int max_bs, const int* block_ptrs, long long nblocks,
                         int so_kind, const unsigned char* so, long long so_len, double accuracy)
{
    Handle* h = new Handle();
    auto e = static_cast<Handle*>(exec)->exec;
    auto A = static_cast<Handle*>(matrix)->op;
    if (guarded([&] {
            h->exec = e;
            h->op = vt == 0 ? make_jacobi<double>(e, A, max_bs, block_ptrs, nblocks, so_kind, so, so_len, accuracy)
                            : make_jacobi<float>(e, A, max_bs, block_ptrs, nblocks, so_kind, so, so_len, accuracy);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}
// meta: block_offset, group_offset, group_power, num_blocks, stored elements, has precisions;
// blocks (raw storage as the value type) / block pointers / precisions / condition numbers -> host
int gkob_jacobi_get(void* jacobi, int vt, long long* meta, void* blocks, int* ptrs, unsigned char* prec, void* cond)
{
    return guarded([&] {
        auto h = static_cast<Handle*>(jacobi);
        vt == 0 ? jacobi_get<double>(h, meta, blocks, ptrs, prec, cond)
                : jacobi_get<float>(h, meta, blocks, ptrs, prec, cond);
    });
}
// Jacobi::transpose()
void* gkob_jacobi_transpose(void* jacobi)
{
    Handle* src = static_cast<Handle*>(jacobi);
    Handle* h = new Handle();
    if (guarded([&] {
            auto t = dynamic_cast<const Transposable*>(src->op.get());
            if (!t) throw NotSupported("gkob_jacobi_transpose: not transposable");
            h->exec = src->exec;
            h->op = std::shared_ptr<LinOp>(t->transpose());
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

}  // extern "C"


extern "C" {

const char* gkob_last_error() { return g_err.c_str(); }

void* gkob_exec_create(int device, void* stream)
{
    Handle* h = new Handle();
    if (guarded([&] { h->exec = B200Executor::create(device, stream); })) {
        delete h;
        return nullptr;
    }
    return h;
}

void gkob_destroy(void* handle) { delete static_cast<Handle*>(handle); }

long long gkob_launch_count(void* exec) { return static_cast<Handle*>(exec)->exec->launch_count(); }

void* gkob_csr_convert(void* csr, const char* fmt, long long p0, long long p1, double pd, double pd2)
{
    auto src = static_cast<Handle*>(csr);
    Handle* h = new Handle{src->exec, nullptr};
    if (guarded([&] {
            auto op = src->op.get();
            if (auto a = dynamic_cast<const matrix::Csr<double, int32>*>(op))
                h->op = convert_csr<double>(a, fmt, p0, p1, pd, pd2);
            else if (auto a = dynamic_cast<const matrix::Csr<float, int32>*>(op))
                h->op = convert_csr<float>(a, fmt, p0, p1, pd, pd2);
            else
                throw NotSupported("gkob_csr_convert: handle is not a Csr<double|float, int32>");
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

// Csr::sort_by_column_index in place (the handle's arrays, i.e. the caller's views)
int gkob_csr_sort_by_column_index(void* csr)
{
    return guarded([&] {
        auto op = static_cast<Handle*>(csr)->op.get();
        if (auto a = dynamic_cast<matrix::Csr<double, int32>*>(op))
            a->sort_by_column_index();
        else if (auto a = dynamic_cast<matrix::Csr<float, int32>*>(op))
            a->sort_by_column_index();
        else
            throw NotSupported("gkob_csr_sort_by_column_index: not a Csr<double|float, int32>");
    });
}

// Transposable::transpose of a Csr<double|float, int32> handle -> new handle
void* gkob_csr_transpose(void* csr)
{
    auto src = static_cast<Handle*>(csr);
    auto h = new Handle{src->exec, nullptr};
    if (guarded([&] {
            auto t = dynamic_cast<const Transposable*>(src->op.get());
            if (!t) throw NotSupported("gkob_csr_transpose: the operator is not Transposable");
            h->op = t->transpose();
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

// staged_apply<V> over a LinOp handle: apply with HOST vectors, pipelined (gko_b200_staging.hpp)
struct StagedHandle {
    std::shared_ptr<Executor> exec;
    std::unique_ptr<staged_apply<double>> f64;
    std::unique_ptr<staged_apply<float>> f32;
};
void* gkob_staged_create(void* op, int vt, long long nrhs)
{
    auto src = static_cast<Handle*>(op);
    auto h = new StagedHandle();
    h->exec = src->exec;
    if (guarded([&] {
            if (vt == 0)
                h->f64.reset(new staged_apply<double>(src->op, (size_type)nrhs));
            else
                h->f32.reset(new staged_apply<float>(src->op, (size_type)nrhs));
        })) {
        delete h;
        return nullptr;
    }
    return h;
}
int gkob_staged_apply(void* staged, const void* b_host, void* x_host)
{
    return guarded([&] {
        auto h = static_cast<StagedHandle*>(staged);
        if (h->f64)
            h->f64->apply((const double*)b_host, (double*)x_host);
        else
            h->f32->apply((const float*)b_host, (float*)x_host);
    });
}
int gkob_staged_join(void* staged)
{
    return guarded([&] {
        auto h = static_cast<StagedHandle*>(staged);
        h->f64 ? h->f64->join() : h->f32->join();
    });
}
int gkob_staged_wait(void* staged)
{
    return guarded([&] {
        auto h = static_cast<StagedHandle*>(staged);
        h->f64 ? h->f64->wait() : h->f32->wait();
    });
}
void gkob_staged_destroy(void* staged) { delete static_cast<StagedHandle*>(staged); }

// number of column blocks the tuned plan of a Csr handle applies (0 / 1: the original arrays)
int gkob_csr_plan_parts(void* csr)
{
    int v = 0;
    guarded([&] {
        auto op = static_cast<Handle*>(csr)->op.get();
        if (auto a = dynamic_cast<const matrix::Csr<double, int32>*>(op))
            v = b200_csr_plan_parts(a->get_plan());
        else if (auto a = dynamic_cast<const matrix::Csr<float, int32>*>(op))
            v = b200_csr_plan_parts(a->get_plan());
    });
    return v;
}

// gko::read_generic<Csr<double, int32>>(file) / gko::write(file, csr) / write_binary
void* gkob_csr_read_f64_i32(void* exec, const char* path)
{
    auto e = static_cast<Handle*>(exec)->exec;
    Handle* h = new Handle{e, nullptr};
    if (guarded([&] {
            std::ifstream is(path, std::ios::binary);
            if (!is) throw StreamError(std::string("cannot open ") + path);
            h->op = read_generic<matrix::Csr<double, int32>>(is, e);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}
// layout: 0 coordinate, 1 array, 2 binary
int gkob_csr_write_f64_i32(void* csr, const char* path, int layout)
{
    return guarded([&] {
        auto a = dynamic_cast<const matrix::Csr<double, int32>*>(static_cast<Handle*>(csr)->op.get());
        if (!a) throw NotSupported("gkob_csr_write: not a Csr<double, int32>");
        std::ofstream os(path, std::ios::binary);
        if (!os) throw StreamError(std::string("cannot open ") + path);
        os << std::setprecision(17);
        if (layout == 2)
            write_binary(os, a);
        else
            write(os, a, layout == 1 ? layout_type::array : layout_type::coordinate);
    });
}
// gko::read_generic<Format<double, int32>>(file): fmt "csr" | "ell" | "sellp" | "coo" | "hybrid"
void* gkob_read_f64_i32(void* exec, const char* path, const char* fmt)
{
    auto e = static_cast<Handle*>(exec)->exec;
    Handle* h = new Handle{e, nullptr};
    if (guarded([&] {
            std::ifstream is(path, std::ios::binary);
            if (!is) throw StreamError(std::string("cannot open ") + path);
            const std::string f(fmt);
            if (f == "csr")
                h->op = read_generic<matrix::Csr<double, int32>>(is, e);
            else if (f == "ell")
                h->op = read_generic<matrix::Ell<double, int32>>(is, e);
            else if (f == "sellp")
                h->op = read_generic<matrix::Sellp<double, int32>>(is, e);
            else if (f == "coo")
                h->op = read_generic<matrix::Coo<double, int32>>(is, e);
            else if (f == "hybrid")
                h->op = read_generic<matrix::Hybrid<double, int32>>(is, e);
            else if (f == "dense")
                h->op = read_generic<matrix::Dense<double>>(is, e);
            else
                throw NotSupported("gkob_read: unknown format " + f);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}
// gko::write / write_binary of any of the five formats (layout: 0 coordinate, 1 array, 2 binary)
int gkob_write_f64_i32(void* op, const char* path, int layout)
{
    return guarded([&] {
        auto p = static_cast<Handle*>(op)->op.get();
        std::ofstream os(path, std::ios::binary);
        if (!os) throw StreamError(std::string("cannot open ") + path);
        os << std::setprecision(17);
        auto put = [&](auto* a) {
            if (layout == 2)
                write_binary(os, a);
            else
                write(os, a, layout == 1 ? layout_type::array : layout_type::coordinate);
        };
        if (auto a = dynamic_cast<const matrix::Csr<double, int32>*>(p))
            put(a);
        else if (auto a = dynamic_cast<const matrix::Ell<double, int32>*>(p))
            put(a);
        else if (auto a = dynamic_cast<const matrix::Sellp<double, int32>*>(p))
            put(a);
        else if (auto a = dynamic_cast<const matrix::Coo<double, int32>*>(p))
            put(a);
        else if (auto a = dynamic_cast<const matrix::Hybrid<double, int32>*>(p))
            put(a);
        else if (auto a = dynamic_cast<const matrix::Dense<double>*>(p))
            put(a);
        else
            throw NotSupported("gkob_write: not a <double, int32> matrix format");
    });
}
long long gkob_num_rows(void* op) { return (long long)static_cast<Handle*>(op)->op->get_size().rows; }
long long gkob_num_cols(void* op) { return (long long)static_cast<Handle*>(op)->op->get_size().cols; }

// parameters for the next gkob_solver_create_* of kind 5 (Ir: relaxation_factor) or 6
// (Chebyshev: foci)
void gkob_solver_guess(int mode) { g_ir_guess = mode; }
// the next gkob_solver_create_* takes this generated preconditioner (e.g. a gkob_jacobi_create handle)
// through with_generated_preconditioner instead of precond_max_bs; NULL clears it
void gkob_solver_preconditioner(void* pre) { g_generated_pre = pre ? static_cast<Handle*>(pre)->op : nullptr; }
void gkob_solver_params(double relaxation_factor, double foci_lo, double foci_hi)
{
    g_relaxation = relaxation_factor;
    g_foci_lo = foci_lo;
    g_foci_hi = foci_hi;
}

// locality of the gathers the tuned plan measured (distinct 128-byte lines of b per gathered element)
double gkob_csr_gather_lines(void* csr)
{
    double v = -1.0;
    guarded([&] {
        auto op = static_cast<Handle*>(csr)->op.get();
        if (auto a = dynamic_cast<const matrix::Csr<double, int32>*>(op))
            v = b200_csr_plan_gather_lines(a->get_plan());
        else if (auto a = dynamic_cast<const matrix::Csr<float, int32>*>(op))
            v = b200_csr_plan_gather_lines(a->get_plan());
    });
    return v;
}

// kernel variant the tuned plan of a Csr handle uses (2 = gather_pipe, 4 = warp_pipe, 5 = cta ring); -1 if
// the handle is not a double/int32 or float/int32 Csr
int gkob_csr_kernel_variant(void* csr)
{
    int v = -1;
    guarded([&] {
        auto op = static_cast<Handle*>(csr)->op.get();
        if (auto a = dynamic_cast<const matrix::Csr<double, int32>*>(op))
            v = b200_csr_plan_variant(a->get_plan());
        else if (auto a = dynamic_cast<const matrix::Csr<float, int32>*>(op))
            v = b200_csr_plan_variant(a->get_plan());
    });
    return v;
}

#define GKOB_DEF(V, S)                                                                          \
    void* gkob_csr_view_##S##_i32(void* exec, long long n, long long m, long long nnz,         \
                                  int32* rp, int32* ci, V* va)                                  \
    {                                                                                           \
        auto e = static_cast<Handle*>(exec)->exec;                                              \
        Handle* h = new Handle{e, nullptr};                                                     \
        if (guarded([&] {                                                                       \
                h->op = matrix::Csr<V, int32>::create(                                          \
                    e, dim2{(size_type)n, (size_type)m}, array<V>::view(e, nnz, va),            \
                    array<int32>::view(e, nnz, ci), array<int32>::view(e, n + 1, rp));          \
            })) {                                                                               \
            delete h;                                                                           \
            return nullptr;                                                                     \
        }                                                                                       \
        return h;                                                                               \
    }                                                                                           \
    void* gkob_csr_view_##S##_i64(void* exec, long long n, long long m, long long nnz,         \
                                  int64* rp, int64* ci, V* va)                                  \
    {                                                                                           \
        auto e = static_cast<Handle*>(exec)->exec;                                              \
        Handle* h = new Handle{e, nullptr};                                                     \
        if (guarded([&] {                                                                       \
                h->op = matrix::Csr<V, int64>::create(                                          \
                    e, dim2{(size_type)n, (size_type)m}, array<V>::view(e, nnz, va),            \
                    array<int64>::view(e, nnz, ci), array<int64>::view(e, n + 1, rp));          \
            })) {                                                                               \
            delete h;                                                                           \
            return nullptr;                                                                     \
        }                                                                                       \
        return h;                                                                               \
    }                                                                                           \
    void* gkob_dense_view_##S(void* exec, long long rows, long long cols, long long stride,     \
                              V* ptr)                                                           \
    {                                                                                           \
        auto e = static_cast<Handle*>(exec)->exec;                                              \
        Handle* h = new Handle{e, nullptr};                                                     \
        if (guarded([&] {                                                                       \
                h->op = matrix::Dense<V>::create_view(                                          \
                    e, dim2{(size_type)rows, (size_type)cols}, ptr, (size_type)stride);         \
            })) {                                                                               \
            delete h;                                                                           \
            return nullptr;                                                                     \
        }                                                                                       \
        return h;                                                                               \
    }                                                                                           \
    void* gkob_solver_create_##S(void* exec, int kind, void* matrix, int precond_max_bs,        \
                                 const int32* block_ptrs, long long nblocks,                    \
                                 long long max_iters, int res_kind, int baseline,               \
                                 double reduction, int iter_first, int krylov_dim, int ortho,   \
                                 int fused, int check_every)                                    \
    {                                                                                           \
        auto e = static_cast<Handle*>(exec)->exec;                                              \
        Handle* h = new Handle{e, nullptr};                                                     \
        auto gen_pre = std::move(g_generated_pre); /* for this solver only */                   \
        g_generated_pre = nullptr;                                                              \
        if (guarded([&] {                                                                       \
                h->op = make_solver<V>(e, kind, static_cast<Handle*>(matrix)->op,               \
                                       precond_max_bs, block_ptrs, nblocks, max_iters,          \
                                       res_kind, baseline, reduction, iter_first, krylov_dim,   \
                                       ortho, fused, check_every, gen_pre);                     \
            })) {                                                                               \
            delete h;                                                                           \
            return nullptr;                                                                     \
        }                                                                                       \
        return h;                                                                               \
    }                                                                                           \
    int gkob_solver_info_##S(void* solver, long long* iters, unsigned char* status,             \
                             int* used_fused)                                                   \
    {                                                                                           \
        return guarded([&] {                                                                    \
            auto op = static_cast<Handle*>(solver)->op.get();                                   \
            auto sb = dynamic_cast<solver::SolverBase<V>*>(op);                                 \
            if (!sb) throw NotSupported("not a solver");                                        \
            *iters = (long long)sb->get_num_iterations();                                       \
            *status = sb->get_stop_status(0);                                                   \
            auto cg = dynamic_cast<solver::Cg<V>*>(op);                                         \
            auto bicgstab = dynamic_cast<solver::Bicgstab<V>*>(op);                             \
            auto gmres = dynamic_cast<solver::Gmres<V>*>(op);                                   \
            auto minres = dynamic_cast<solver::Minres<V>*>(op);                                 \
            *used_fused = cg         ? (int)cg->used_fused_path()                               \
                          : bicgstab ? (int)bicgstab->used_fused_path()                         \
                          : gmres    ? (int)gmres->used_fused_path()                            \
                          : minres   ? (int)minres->used_fused_path()                           \
                                     : 0;                                                       \
        });                                                                                     \
    }                                                                                           \
    /* the stopping status of columns 0..cols-1 after the last apply (0 beyond the solved ones) */ \
    int gkob_solver_statuses_##S(void* solver, unsigned char* out, long long cols)              \
    {                                                                                           \
        return guarded([&] {                                                                    \
            auto sb = dynamic_cast<solver::SolverBase<V>*>(static_cast<Handle*>(solver)->op.get()); \
            if (!sb) throw NotSupported("not a solver");                                        \
            for (long long c = 0; c < cols; ++c) out[c] = sb->get_stop_status((size_type)c);    \
        });                                                                                     \
    }
GKOB_DEF(double, f64)
GKOB_DEF(float, f32)

// ---- multi-GPU ------------------------------------------------------------------------------
struct DistHandle {
    std::shared_ptr<Executor> exec;
    std::shared_ptr<distributed::communicator> comm;
    std::shared_ptr<distributed::Matrix<double, int32>> A;
    std::unique_ptr<distributed::Cg<double, int32>> cg;
};

int gkob_dist_unique_id(unsigned char* id128)
{
    return guarded([&] {
        uint8 id[128];
        distributed::communicator::get_unique_id(id);
        std::memcpy(id128, id, 128);
    });
}

// local rows (rp, ci_local, va device views), halo description from distributed.build_partition
void* gkob_dist_matrix_create_f64_i32(void* exec, const unsigned char* id128, int rank, int nranks,
                                      long long n_local, long long n_ghost, long long nnz,
                                      int32* rp, int32* ci_local, double* va,
                                      const long long* send_counts, const long long* recv_counts,
                                      const int32* send_idx_dev)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new DistHandle();
    h->exec = e;
    if (guarded([&] {
            h->comm = distributed::communicator::create(e, id128, rank, nranks);
            auto local = matrix::Csr<double, int32>::create(
                e, dim2{(size_type)n_local, (size_type)(n_local + n_ghost)},
                array<double>::view(e, nnz, va), array<int32>::view(e, nnz, ci_local),
                array<int32>::view(e, n_local + 1, rp));
            std::vector<int64> sc(send_counts, send_counts + nranks), rc(recv_counts,
                                                                         recv_counts + nranks);
            h->A = std::make_shared<distributed::Matrix<double, int32>>(
                e, h->comm, std::move(local), (size_type)n_ghost, sc, rc, send_idx_dev);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

int gkob_dist_spmv_f64(void* dist, double* x_ext, double* y_local)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        auto n = h->A->n_local(), ng = h->A->n_ghost();
        auto xe = matrix::Dense<double>::create_view(h->exec, dim2{n + ng, 1}, x_ext, 1);
        auto y = matrix::Dense<double>::create_view(h->exec, dim2{n, 1}, y_local, 1);
        h->A->apply_extended(xe.get(), y.get());
    });
}

// pipelined (owner-block, arrival-order) exchange on / off; returns through *active whether the next
// gkob_dist_spmv_f64 will use it (collective decisions are local: every rank qualifies alike)
int gkob_dist_set_overlap(void* dist, int on)
{
    return guarded([&] { static_cast<DistHandle*>(dist)->A->set_overlap(on != 0); });
}
int gkob_dist_pipelined(void* dist) { return static_cast<DistHandle*>(dist)->A->pipelined() ? 1 : 0; }

// ghosts_out[0 .. n_ghost) = the ghost entries the last gkob_dist_spmv_f64 gathered from (the peer-memory
// path reads them in place from the landing slot instead of copying them into the caller's x_ext)
int gkob_dist_last_ghosts_f64(void* dist, double* ghosts_out)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        auto n = h->A->n_local(), ng = h->A->n_ghost();
        const double* src = h->A->last_extended();
        if (!src) throw NotSupported("no distributed apply yet");
        if (ng) h->exec->copy(ghosts_out, src + n, ng);
    });
}

int gkob_dist_cg_create_f64(void* dist, int scalar_jacobi, long long max_iters, int res_kind,
                            int baseline, double reduction, int iter_first, int check_every)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        h->cg.reset(new distributed::Cg<double, int32>(h->exec, h->A, scalar_jacobi != 0, max_iters,
                                                       res_kind, baseline, reduction,
                                                       iter_first != 0, check_every));
    });
}

int gkob_dist_cg_apply_f64(void* dist, const double* b_local, double* x_local, long long* iters,
                           unsigned char* status)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        auto n = h->A->n_local();
        auto b = matrix::Dense<double>::create_view(h->exec, dim2{n, 1},
                                                    const_cast<double*>(b_local), 1);
        auto x = matrix::Dense<double>::create_view(h->exec, dim2{n, 1}, x_local, 1);
        h->cg->apply(b.get(), x.get());
        *iters = h->cg->get_num_iterations();
        *status = h->cg->get_stop_status();
    });
}

// any solver of make_solver on the distributed matrix: b_local / x_local are this rank's rows
// (device pointers), wrapped as distributed::Vector so that dots and norms sum over the ranks;
// the preconditioner is generated from the local block.  Collective.
// schwarz_sweeps: 0 = Jacobi(precond_max_bs) generated from the local block; -1 = Schwarz whose
// local solver is that Jacobi on the square local block; k > 0 = Schwarz whose local solver is k
// Richardson sweeps (Ir, relaxation from gkob_solver_params) preconditioned by that Jacobi
// b_local / x_local: n_local x nrhs, row-major
int gkob_dist_solve_f64(void* dist, int kind, int precond_max_bs, int schwarz_sweeps, const double* b_local,
                        double* x_local, long long global_rows, long long max_iters, int res_kind,
                        int baseline, double reduction, int iter_first, int krylov_dim, int ortho, int nrhs,
                        long long* iters, unsigned char* status)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        const size_type n = h->A->n_local();
        const size_type k = (size_type)nrhs;
        auto b = distributed::Vector<double>::create_view(h->exec, h->comm, dim2{(size_type)global_rows, k},
                                                          dim2{n, k}, const_cast<double*>(b_local), k);
        auto x = distributed::Vector<double>::create_view(h->exec, h->comm, dim2{(size_type)global_rows, k},
                                                          dim2{n, k}, x_local, k);
        std::unique_ptr<LinOp> solver;
        if (schwarz_sweeps == 0) {
            solver = make_solver<double>(h->exec, kind, h->A, precond_max_bs, nullptr, 0, max_iters, res_kind,
                                         baseline, reduction, iter_first, krylov_dim, ortho, 0, 1);
        } else {
            using jac = preconditioner::Jacobi<double, int32>;
            std::shared_ptr<const LinOpFactory> local =
                jac::build().with_max_block_size((uint32)std::max(precond_max_bs, 1)).on(h->exec);
            if (schwarz_sweeps > 0)
                local = solver::Ir<double>::build()
                            .with_criteria(stop::Iteration::build().with_max_iters((size_type)schwarz_sweeps))
                            .with_solver(local)
                            .with_relaxation_factor(g_relaxation)
                            .with_default_initial_guess(solver::initial_guess_mode::zero)
                            .on(h->exec);
            std::shared_ptr<const LinOp> schwarz = distributed::preconditioner::Schwarz<double, int32>::build()
                                                       .with_local_solver(local)
                                                       .on(h->exec)
                                                       ->generate(h->A);
            solver = make_solver<double>(h->exec, kind, h->A, 0, nullptr, 0, max_iters, res_kind, baseline,
                                         reduction, iter_first, krylov_dim, ortho, 0, 1, schwarz);
        }
        solver->apply(b.get(), x.get());
        auto base = dynamic_cast<solver::SolverBase<double>*>(solver.get());
        *iters = base ? (long long)base->get_num_iterations() : -1;
        *status = base ? base->get_stop_status() : 0;
    });
}

// LinOp::apply of the distributed matrix on the local rows of distributed vectors
// (n_local_cols x nrhs -> n_local x nrhs, row-major)
int gkob_dist_apply_f64(void* dist, const double* b_local, double* x_local, int nrhs)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        const size_type k = (size_type)nrhs;
        auto b = matrix::Dense<double>::create_view(h->exec, dim2{h->A->n_local_cols(), k},
                                                    const_cast<double*>(b_local), k);
        auto x = matrix::Dense<double>::create_view(h->exec, dim2{h->A->n_local(), k}, x_local, k);
        static_cast<const LinOp*>(h->A.get())->apply(b.get(), x.get());
    });
}

void gkob_dist_destroy(void* dist) { delete static_cast<DistHandle*>(dist); }

// ---- distributed set-up: Partition<int32, int64>, assemble_local, read_distributed ---------
using part_t = distributed::Partition<int32, int64>;
struct PartHandle {
    std::shared_ptr<Executor> exec;
    std::shared_ptr<const part_t> part;
};
struct AssemblyHandle {
    std::shared_ptr<Executor> exec;
    distributed::local_assembly<double, int32, int64> a;
};

void* gkob_partition_from_mapping(void* exec, const int* mapping_host, long long n, int num_parts)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new PartHandle{e, nullptr};
    if (guarded([&] {
            array<int32> m(e, std::vector<int32>(mapping_host, mapping_host + n));
            h->part = part_t::build_from_mapping(e, m, num_parts);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

void* gkob_partition_from_contiguous(void* exec, const long long* ranges_host, long long num_ranges,
                                     const int* part_ids_host)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new PartHandle{e, nullptr};
    if (guarded([&] {
            array<int64> r(e, std::vector<int64>(ranges_host, ranges_host + num_ranges + 1));
            if (part_ids_host) {
                array<int32> ids(e, std::vector<int32>(part_ids_host, part_ids_host + num_ranges));
                h->part = part_t::build_from_contiguous(e, r, ids);
            } else {
                h->part = part_t::build_from_contiguous(e, r);
            }
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

void* gkob_partition_uniform(void* exec, int num_parts, long long global_size)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new PartHandle{e, nullptr};
    if (guarded([&] { h->part = part_t::build_from_global_size_uniform(e, num_parts, global_size); })) {
        delete h;
        return nullptr;
    }
    return h;
}

// meta = {size, num_ranges, num_parts, num_empty_parts, has_connected_parts, has_ordered_parts};
// the arrays (may be NULL) are copied to the host
int gkob_partition_info(void* part, long long* meta, long long* bounds, int* part_ids, int* starting,
                        int* sizes)
{
    return guarded([&] {
        auto h = static_cast<PartHandle*>(part);
        auto& p = *h->part;
        const size_type nr = p.get_num_ranges();
        meta[0] = (long long)p.get_size();
        meta[1] = (long long)nr;
        meta[2] = p.get_num_parts();
        meta[3] = p.get_num_empty_parts();
        meta[4] = p.has_connected_parts();
        meta[5] = p.has_ordered_parts();
        if (bounds) {
            std::vector<int64> b(nr + 1);
            h->exec->copy_to_host(b.data(), p.get_range_bounds(), nr + 1);
            std::copy(b.begin(), b.end(), bounds);
        }
        if (part_ids && nr) h->exec->copy_to_host(part_ids, p.get_part_ids(), nr);
        if (starting && nr) h->exec->copy_to_host(starting, p.get_range_starting_indices(), nr);
        if (sizes && p.get_num_parts())
            h->exec->copy_to_host(sizes, p.get_part_sizes(), (size_type)p.get_num_parts());
    });
}

void gkob_partition_destroy(void* part) { delete static_cast<PartHandle*>(part); }

static matrix_data<double, int64> triplets(long long nrows, long long ncols, long long nnz, const long long* rows,
                                           const long long* cols, const double* vals)
{
    matrix_data<double, int64> d(dim2{(size_type)nrows, (size_type)ncols});
    d.nonzeros.reserve((size_t)nnz);
    for (long long i = 0; i < nnz; ++i) d.nonzeros.push_back({(int64)rows[i], (int64)cols[i], vals[i]});
    return d;
}

// the communication-free part of read_distributed for part `rank` (col_part may be NULL)
void* gkob_dist_assemble_f64_i32(void* exec, void* row_part, void* col_part, int rank, long long nrows,
                                 long long ncols, long long nnz, const long long* rows, const long long* cols,
                                 const double* vals)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new AssemblyHandle{e, {}};
    if (guarded([&] {
            auto rp = static_cast<PartHandle*>(row_part)->part;
            auto cp = col_part ? static_cast<PartHandle*>(col_part)->part : rp;
            h->a = distributed::assemble_local<double, int32, int64>(
                e, triplets(nrows, ncols, nnz, rows, cols, vals), rp, cp, rank);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

// out = {n_local_rows, n_local_cols, n_ghost, nnz of the local block, num_parts}
int gkob_dist_assembly_sizes(void* assembly, long long* out)
{
    return guarded([&] {
        auto& a = static_cast<AssemblyHandle*>(assembly)->a;
        out[0] = (long long)a.n_local_rows;
        out[1] = (long long)a.n_local_cols;
        out[2] = (long long)a.n_ghost;
        out[3] = (long long)a.local->get_num_stored_elements();
        out[4] = (long long)a.imap->get_remote_sizes().size();
    });
}

int gkob_dist_assembly_get(void* assembly, int* row_ptrs, int* col_idxs, double* values,
                           long long* recv_counts, long long* remote_global, int* remote_local)
{
    return guarded([&] {
        auto h = static_cast<AssemblyHandle*>(assembly);
        auto& a = h->a;
        const size_type nnz = a.local->get_num_stored_elements();
        h->exec->copy_to_host(row_ptrs, a.local->get_const_row_ptrs(), a.n_local_rows + 1);
        if (nnz) {
            h->exec->copy_to_host(col_idxs, a.local->get_const_col_idxs(), nnz);
            h->exec->copy_to_host(values, a.local->get_const_values(), nnz);
        }
        const auto& rs = a.imap->get_remote_sizes();
        std::copy(rs.begin(), rs.end(), recv_counts);
        if (a.n_ghost) {
            const auto rg = a.imap->get_remote_global_idxs().to_host();
            std::copy(rg.begin(), rg.end(), remote_global);
            h->exec->copy_to_host(remote_local, a.imap->get_remote_local_idxs().get_const_data(), a.n_ghost);
        }
    });
}

int gkob_dist_assembly_map_to_local(void* assembly, int index_space, long long m, const long long* gids_host,
                                    int* out_host)
{
    return guarded([&] {
        auto h = static_cast<AssemblyHandle*>(assembly);
        array<int64> g(h->exec, std::vector<int64>(gids_host, gids_host + m));
        auto res = h->a.imap->map_to_local(g, (distributed::index_space)index_space).to_host();
        std::copy(res.begin(), res.end(), out_host);
    });
}

void gkob_dist_assembly_destroy(void* assembly) { delete static_cast<AssemblyHandle*>(assembly); }

// S[q * P + p] = entries rank q receives from p  ->  what `rank` sends to every q and where
// those entries start in q's remote list
int gkob_dist_send_layout(int P, int rank, const long long* S, long long* send_counts,
                          long long* source_offsets)
{
    return guarded([&] {
        const auto l = distributed::compute_send_layout(std::vector<int64>(S, S + (size_t)P * P), P, rank);
        std::copy(l.send_counts.begin(), l.send_counts.end(), send_counts);
        std::copy(l.source_offsets.begin(), l.source_offsets.end(), source_offsets);
    });
}

// collective: distributed::Matrix::read_distributed of the global triplets (row-major sorted)
void* gkob_dist_matrix_read_f64_i32(void* exec, const unsigned char* id128, int rank, int nranks,
                                    void* row_part, long long nrows, long long ncols, long long nnz,
                                    const long long* rows, const long long* cols, const double* vals,
                                    int keep_local_block)
{
    auto e = static_cast<Handle*>(exec)->exec;
    auto h = new DistHandle();
    h->exec = e;
    if (guarded([&] {
            h->comm = distributed::communicator::create(e, id128, rank, nranks);
            h->A = distributed::Matrix<double, int32>::read_distributed<int64>(
                e, h->comm, triplets(nrows, ncols, nnz, rows, cols, vals),
                static_cast<PartHandle*>(row_part)->part, nullptr, keep_local_block != 0);
        })) {
        delete h;
        return nullptr;
    }
    return h;
}

// out = {n_local rows, n_local columns, n_ghost}; ghost_globals (may be NULL): n_ghost entries
int gkob_dist_matrix_sizes(void* dist, long long* out, long long* ghost_globals)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        out[0] = (long long)h->A->n_local();
        out[1] = (long long)h->A->n_local_cols();
        out[2] = (long long)h->A->n_ghost();
        if (ghost_globals) {
            const auto& g = h->A->get_non_local_to_global();
            std::copy(g.begin(), g.end(), ghost_globals);
        }
    });
}

// distributed::read_distributed_vector on the communicator of `dist`: the local rows (row-major,
// n_local x ncols) are copied to out_host
int gkob_dist_vector_read_f64(void* dist, void* row_part, long long nrows, long long ncols, long long nnz,
                              const long long* rows, const long long* cols, const double* vals, double* out_host)
{
    return guarded([&] {
        auto h = static_cast<DistHandle*>(dist);
        auto v = distributed::read_distributed_vector<double, int32, int64>(
            h->exec, h->comm, triplets(nrows, ncols, nnz, rows, cols, vals),
            static_cast<PartHandle*>(row_part)->part);
        const auto host = v->to_host();
        std::copy(host.begin(), host.end(), out_host);
    });
}



// bit 0: all-reduces run on peer memory, bit 1: the halo exchange does
int gkob_dist_p2p(void* dist)
{
    auto h = static_cast<DistHandle*>(dist);
    return (b200_comm_p2p_enabled(h->comm->get()) ? 1 : 0) |
           (b200_halo_p2p_enabled(h->A->get_halo()) ? 2 : 0);
}

// x = op(b)   /   x = alpha op(b) + beta x  (alpha, beta: 1x1 Dense handles)
int gkob_apply(void* op, void* b, void* x)
{
    return guarded([&] {
        static_cast<Handle*>(op)->op->apply(static_cast<Handle*>(b)->op.get(),
                                            static_cast<Handle*>(x)->op.get());
    });
}
int gkob_apply4(void* op, void* alpha, void* b, void* beta, void* x)
{
    return guarded([&] {
        static_cast<Handle*>(op)->op->apply(
            static_cast<Handle*>(alpha)->op.get(), static_cast<Handle*>(b)->op.get(),
            static_cast<Handle*>(beta)->op.get(), static_cast<Handle*>(x)->op.get());
    });
}
int gkob_synchronize(void* exec)
{
    return guarded([&] { static_cast<Handle*>(exec)->exec->synchronize(); });
}

}  // extern "C"
