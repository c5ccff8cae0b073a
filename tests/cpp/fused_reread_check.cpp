// TEST INFRASTRUCTURE: a fused Cg whose shared Csr is re-read between two applies (compiled against
// the host-memory mock by tests/test_fused_recapture_cpu.py).  Csr::read replaces the arrays the
// captured graph baked in; the second apply, into the same x, must run on the new matrix and give the
// loop's iterations, status and bits of x there.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../ginkgo_b200/host/gko_b200.hpp"

namespace gko = gko_b200;

int main()
{
    using Mtx = gko::matrix::Dense<double>;
    using Csr = gko::matrix::Csr<double, gko::int32>;
    using Cg = gko::solver::Cg<double>;
    auto exec = gko::B200Executor::create(0);
    const gko::int32 n = 40;
    auto tridiagonal = [&](double diag) {
        gko::matrix_data<double, gko::int32> d{gko::dim2(n)};
        for (gko::int32 i = 0; i < n; ++i) {
            if (i > 0) d.nonzeros.push_back({i, i - 1, -1.0});
            d.nonzeros.push_back({i, i, diag});
            if (i + 1 < n) d.nonzeros.push_back({i, i + 1, -1.0});
        }
        return d;
    };
    auto generate = [&](std::shared_ptr<const gko::LinOp> A, bool fused) {
        return Cg::build()
            .with_criteria(gko::stop::Iteration::build().with_max_iters(200u),
                           gko::stop::ResidualNorm<double>::build().with_reduction_factor(1e-12))
            .with_fused(fused)
            .on(exec)
            ->generate(A);
    };
    std::vector<double> bh(n), zeros(n, 0.0);
    for (gko::int32 i = 0; i < n; ++i) bh[i] = std::sin(0.7 * i + 1.0);
    const gko::dim2 col{(gko::size_type)n, 1};
    auto b = Mtx::create_from_host(exec, col, bh.data());
    auto A = gko::share(Csr::create(exec));
    A->read(tridiagonal(2.5));
    auto fused = generate(A, true);
    auto x = Mtx::create_from_host(exec, col, zeros.data());
    fused->apply(b, x);
    A->read(tridiagonal(3.0));
    x->fill(0.0);
    fused->apply(b, x);
    auto loop = generate(A, false);
    auto xl = Mtx::create_from_host(exec, col, zeros.data());
    loop->apply(b, xl);
    auto f = dynamic_cast<Cg*>(fused.get());
    auto l = dynamic_cast<Cg*>(loop.get());
    const auto hf = x->to_host(), hl = xl->to_host();
    const bool same = f->used_fused_path() && !l->used_fused_path() &&
                      f->get_num_iterations() == l->get_num_iterations() &&
                      f->get_stop_status() == l->get_stop_status() &&
                      std::memcmp(hf.data(), hl.data(), n * sizeof(double)) == 0;
    std::printf("fused cg after read: iterations %zu / %zu status %#x / %#x\n", (size_t)f->get_num_iterations(),
                (size_t)l->get_num_iterations(), (unsigned)f->get_stop_status(), (unsigned)l->get_stop_status());
    std::printf("%s\n", same ? "ALL OK" : "FAILED");
    return same ? 0 : 1;
}
