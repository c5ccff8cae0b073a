"""solver::Minres::try_fused on the host-memory mock: the set-up through the loop's own calls, graph
capture and replay, the p / p_prev roles taken from the iteration counter's parity, and polling of
the control block every check_every iterations run on the CPU.  The mock's restatements of the
fused kernels and the kernel-by-kernel loop both add their dot products sequentially in row order,
so the two paths take the same iterations and give the same bits of x."""
import numpy as np
import pytest
import torch

import workloads as W
from tests.helpers import VT


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec
    from tests.mock_minres_build import build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_minres")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def indefinite_laplacian(g, dims, vt, shift, seed=4):
    """the g^dims Laplacian plus diag(uniform(0, 0.5)) - shift I: symmetric indefinite for a shift
    above the smallest Laplacian eigenvalue, with a positive diagonal"""
    rp, ci, va = W.laplace(g, dims, vdtype=np.float64)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    va = va.copy()
    va[ci == rows] += np.random.default_rng(seed).uniform(0, 0.5, n) - shift
    return rp, ci, va.astype(VT[vt])


def solve(host, vt, rp, ci, va, b, precond, block_ptrs=None, **kw):
    from ginkgo_b200 import api
    n = len(rp) - 1
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(b))
    tx = torch.zeros_like(tb)
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "minres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(host, tb), api.host_dense(host, tx))
    return tx.numpy(), s.num_iterations, s.stop_status, s.used_fused


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("baseline,iter_first", [(0, True), (1, False), (2, True), (0, False), (1, True), (2, False)])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_minres_takes_the_loops_iterations(host, vt, precond, baseline, iter_first, check_every):
    rp, ci, va = indefinite_laplacian(12, 2, vt, 0.6)
    n = len(rp) - 1
    b = np.random.default_rng(3).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-9 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10  # absolute threshold
    kw = dict(max_iters=400, reduction=red, res_kind=2, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, usedl = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, vt, rp, ci, va, b, precond, fused_minres=True, check_every=check_every, **kw)
    assert usedf and not usedl
    assert stl & 0x80 and itl > 1  # converged; whatever check_every, the last batch runs past the stop
    assert (itf, stf) == (itl, stl)
    assert np.array_equal(xf, xl)


@pytest.mark.parametrize("max_iters", [0, 1, 5])
@pytest.mark.parametrize("iter_first", [True, False])
@pytest.mark.parametrize("precond", [0, 1])
def test_fused_minres_iteration_limit(host, max_iters, iter_first, precond):
    rp, ci, va = indefinite_laplacian(12, 2, "f64", 0.6)
    n = len(rp) - 1
    b = np.random.default_rng(5).uniform(-1, 1, (n, 1))
    kw = dict(max_iters=max_iters, reduction=1e-12, res_kind=2, iter_first=iter_first)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, precond, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, precond, fused_minres=True, check_every=3, **kw)
    assert used and (itf, stf) == (itl, stl) == (max_iters, 0x40 | (1 if iter_first else 2))
    assert np.array_equal(xf, xl)


def test_fused_minres_iteration_criterion_alone(host):
    rp, ci, va = indefinite_laplacian(10, 2, "f32", 0.6)
    n = len(rp) - 1
    b = np.random.default_rng(8).uniform(-1, 1, (n, 1)).astype(np.float32)
    kw = dict(max_iters=37, res_kind=0)
    xl, itl, stl, _ = solve(host, "f32", rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, "f32", rp, ci, va, b, 1, fused_minres=True, check_every=16, **kw)
    assert used and (itf, stf) == (itl, stl) == (37, 0x40 | 1)
    assert np.array_equal(xf, xl)


def test_fused_minres_graph_is_recaptured_when_x_changes(host):
    from ginkgo_b200 import api
    rp, ci, va = indefinite_laplacian(10, 2, "f64", 0.6)
    n = len(rp) - 1
    rng = np.random.default_rng(9)
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    kw = dict(max_iters=300, reduction=1e-9, res_kind=2)
    s = api.HostSolver(host, "minres", A, precond_max_bs=1, fused_minres=True, check_every=5, **kw)
    xs = [torch.zeros(n, 1, dtype=torch.float64) for _ in range(2)]
    for k in range(4):
        b = rng.uniform(-1, 1, (n, 1))
        tx = xs[k % 2]  # a new x every apply: the graph baked in the previous one
        tx.zero_()
        s.apply(api.host_dense(host, torch.from_numpy(b)), api.host_dense(host, tx))
        assert s.used_fused and s.stop_status == 0x80 | 0x40 | 2
        xl, itl, _, _ = solve(host, "f64", rp, ci, va, b, 1, **kw)
        assert s.num_iterations == itl and np.array_equal(tx.numpy(), xl)


def test_fused_minres_falls_back_to_the_loop(host):
    rp, ci, va = indefinite_laplacian(8, 2, "f64", 0.6)
    n = len(rp) - 1
    rng = np.random.default_rng(2)
    b1, b2 = rng.uniform(-1, 1, (n, 1)), rng.uniform(-1, 1, (n, 2))
    kw = dict(max_iters=200, reduction=1e-8, res_kind=2)
    # block Jacobi, ResidualNorm and several right-hand sides are the loop's
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not solve(host, "f64", rp, ci, va, b1, 4, bp, fused_minres=True, **kw)[3]
    assert not solve(host, "f64", rp, ci, va, b1, 1, fused_minres=True, **dict(kw, res_kind=1))[3]
    x, it, st, used = solve(host, "f64", rp, ci, va, b2, 1, fused_minres=True, **kw)
    assert not used and st == 0x80 | 0x40 | 2
    # off by default, and `fused` alone keeps meaning CG's switch
    assert not solve(host, "f64", rp, ci, va, b1, 1, **kw)[3]
    assert not solve(host, "f64", rp, ci, va, b1, 1, fused=True, **kw)[3]
    assert solve(host, "f64", rp, ci, va, b1, 1, fused_minres=True, **kw)[3]
