"""solver::Bicgstab::try_fused on the host-memory mock: graph capture and replay, polling of the
control block every check_every iterations and the pending-finalize hand-over between step_s and
step_xr run on the CPU.  The mock's restatements of the fused kernels and the kernel-by-kernel
loop both add their dot products sequentially, so the two paths take the same iterations."""
import numpy as np
import pytest
import torch

import workloads as W
from tests.helpers import VT


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_bicgstab")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def convection_diffusion(g, dims, vt, wind=0.8):
    """upwind convection-diffusion on a g^dims grid: the Laplacian stencil with `wind` added to the
    diagonal and subtracted from the upstream neighbour of every axis: nonsymmetric, row sums >= 0"""
    rp, ci, va = W.laplace(g, dims, vdtype=np.float64)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    va = va.copy()
    for d in range(dims):
        up = (ci == rows - g ** d)
        va[up] -= wind
    va[ci == rows] += dims * wind
    return rp, ci, va.astype(VT[vt])


def solve(host, vt, rp, ci, va, b, precond, block_ptrs=None, **kw):
    from ginkgo_b200 import api
    n = len(rp) - 1
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(b))
    tx = torch.zeros_like(tb)
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(host, tb), api.host_dense(host, tx))
    return tx.numpy(), s.num_iterations, s.stop_status, s.used_fused


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("res_kind,baseline,iter_first", [(1, 0, True), (2, 1, False), (1, 2, True), (1, 1, False)])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_bicgstab_takes_the_loops_iterations(host, vt, precond, res_kind, baseline, iter_first, check_every):
    rp, ci, va = convection_diffusion(12, 2, vt)
    n = len(rp) - 1
    b = np.random.default_rng(3).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-9 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10  # absolute threshold
    kw = dict(max_iters=300, reduction=red, res_kind=res_kind, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, usedl = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, vt, rp, ci, va, b, precond, fused_bicgstab=True, check_every=check_every, **kw)
    assert usedf and not usedl
    assert stl & 0x80 and itl > 1  # converged; whatever check_every, the last batch runs past the stop
    assert (itf, stf) == (itl, stl)
    assert np.array_equal(xf, xl)


@pytest.mark.parametrize("max_iters", [0, 1, 5])
@pytest.mark.parametrize("iter_first", [True, False])
def test_fused_bicgstab_iteration_limit(host, max_iters, iter_first):
    rp, ci, va = convection_diffusion(12, 2, "f64")
    n = len(rp) - 1
    b = np.random.default_rng(5).uniform(-1, 1, (n, 1))
    kw = dict(max_iters=max_iters, reduction=1e-12, iter_first=iter_first)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, 1, fused_bicgstab=True, check_every=3, **kw)
    assert used and (itf, stf) == (itl, stl) == (max_iters, 0x40 | (1 if iter_first else 2))
    assert np.array_equal(xf, xl)


def test_fused_bicgstab_stops_at_the_mid_check_and_finalizes(host):
    """A = 4 I: the first half step solves the system, so s = 0 at the mid
    check of iteration 0 and x is completed by bicgstab::finalize (x += alpha y)"""
    n = 50
    rp = np.arange(n + 1, dtype=np.int32)
    ci = np.arange(n, dtype=np.int32)
    va = np.full(n, 4.0)
    b = np.random.default_rng(1).uniform(-1, 1, (n, 1))
    kw = dict(max_iters=20, reduction=1e-10)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 0, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, 0, fused_bicgstab=True, check_every=4, **kw)
    assert used and (itf, stf) == (itl, stl) == (0, 0x80 | 0x40 | 2)
    assert np.array_equal(xf, xl) and np.allclose(xf, b / 4.0, rtol=1e-14)


def test_fused_bicgstab_workspace_and_graph_are_reused(host):
    from ginkgo_b200 import api
    rp, ci, va = convection_diffusion(10, 2, "f64")
    n = len(rp) - 1
    rng = np.random.default_rng(9)
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=1, max_iters=200, reduction=1e-9, fused_bicgstab=True,
                       check_every=5)
    tx = torch.zeros(n, 1, dtype=torch.float64)
    xd = api.host_dense(host, tx)
    for _ in range(3):
        b = rng.uniform(-1, 1, (n, 1))
        tx.zero_()
        s.apply(api.host_dense(host, torch.from_numpy(b)), xd)
        assert s.used_fused and s.stop_status == 0x80 | 0x40 | 2
        xl, itl, _, _ = solve(host, "f64", rp, ci, va, b, 1, max_iters=200, reduction=1e-9)
        assert s.num_iterations == itl and np.array_equal(tx.numpy(), xl)


def test_fused_bicgstab_falls_back_to_the_loop(host):
    rp, ci, va = convection_diffusion(8, 2, "f64")
    n = len(rp) - 1
    rng = np.random.default_rng(2)
    b1, b2 = rng.uniform(-1, 1, (n, 1)), rng.uniform(-1, 1, (n, 2))
    kw = dict(max_iters=100, reduction=1e-8, fused_bicgstab=True)
    # block Jacobi and several right-hand sides are the loop's
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not solve(host, "f64", rp, ci, va, b1, 4, bp, **kw)[3]
    x, it, st, used = solve(host, "f64", rp, ci, va, b2, 1, **kw)
    assert not used and st == 0x80 | 0x40 | 2
    # off by default, and `fused` alone keeps meaning CG's switch
    assert not solve(host, "f64", rp, ci, va, b1, 1, max_iters=100, reduction=1e-8, fused=True)[3]
    assert solve(host, "f64", rp, ci, va, b1, 1, **kw)[3]
