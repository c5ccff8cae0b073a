"""solver::Cg::try_fused_multi_rhs on the host-memory mock: graph capture and replay, polling of the
control block every check_every iterations and the per-column statuses run on the CPU.  The mock's
restatements of the fused kernels and the kernel-by-kernel loop both add every column's dot products
over the rows in order, so the two paths take the same iterations and give the same bits."""
import numpy as np
import pytest
import torch

import workloads as W
from tests.helpers import VT


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_cg_mrhs_build import build_mock_host
    from tests.mock_build import CpuExec
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_cg_mrhs")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def laplacian(g, dims, vt, it="i32"):
    rp, ci, va = W.laplace(g, dims, vdtype=np.float64)
    idx = np.int32 if it == "i32" else np.int64
    return rp.astype(idx), ci.astype(idx), va.astype(VT[vt])


def rhs(n, k, vt, seed=3):
    """k columns; column 1 scaled by 1e-3, so that it converges at another iteration under
    initial_resnorm and absolute baselines than its neighbours"""
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
    b[:, 1] *= 1e-3
    return b.astype(VT[vt])


def solve(host, vt, rp, ci, va, b, precond, x0=None, **kw):
    from ginkgo_b200 import api
    n = len(rp) - 1
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(b))
    tx = torch.zeros_like(tb) if x0 is None else torch.from_numpy(np.ascontiguousarray(x0).copy())
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "cg", A, precond_max_bs=precond, **kw)
    s.apply(api.host_dense(host, tb), api.host_dense(host, tx))
    return tx.numpy(), s.num_iterations, s.stop_statuses, s.used_fused


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("res_kind,baseline,iter_first", [(1, 0, True), (2, 1, False), (1, 2, True), (1, 1, False)])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_multi_rhs_takes_the_loops_iterations(host, vt, precond, res_kind, baseline, iter_first, check_every):
    rp, ci, va = laplacian(12, 2, vt)
    n = len(rp) - 1
    b = rhs(n, 4, vt)
    red = 1e-9 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10  # absolute threshold
    kw = dict(max_iters=300, reduction=red, res_kind=res_kind, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, usedl = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, vt, rp, ci, va, b, precond, fused_multi_rhs=True, check_every=check_every,
                                **kw)
    assert usedf and not usedl
    assert all(s & 0x80 for s in stl) and itl > 1
    assert (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_multi_rhs_columns_stop_on_their_own(host, check_every):
    """a zero column of b stops at iteration 0 under rhs_norm (converged, id 2); the Iteration limit
    then marks only the columns still running (id 1)"""
    rp, ci, va = laplacian(10, 2, "f64", "i64")
    n = len(rp) - 1
    b = rhs(n, 5, "f64", seed=7)
    b[:, 2] = 0
    x0 = np.zeros_like(b)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 0, x0, max_iters=12, reduction=1e-10)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, 0, x0, max_iters=12, reduction=1e-10,
                               fused_multi_rhs=True, check_every=check_every)
    assert used and itf == itl == 12
    assert stf == stl
    assert stf[2] == 0x80 | 0x40 | 2 and all(s == 0x40 | 1 for j, s in enumerate(stf) if j != 2)
    assert xf.tobytes() == xl.tobytes()


def test_fused_multi_rhs_workspace_and_graph_are_reused(host):
    from ginkgo_b200 import api
    rp, ci, va = laplacian(9, 2, "f64")
    n = len(rp) - 1
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    s = api.HostSolver(host, "cg", A, precond_max_bs=1, max_iters=200, reduction=1e-9, fused_multi_rhs=True,
                       check_every=5)
    for k, seed in ((3, 1), (3, 2), (6, 3), (3, 4)):
        b = rhs(n, k, "f64", seed)
        tx = torch.zeros(n, k, dtype=torch.float64)
        s.apply(api.host_dense(host, torch.from_numpy(b)), api.host_dense(host, tx))
        assert s.used_fused and s.stop_statuses == [0x80 | 0x40 | 2] * k
        xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 1, max_iters=200, reduction=1e-9)
        assert s.num_iterations == itl and tx.numpy().tobytes() == xl.tobytes()


def test_fused_multi_rhs_falls_back_to_the_loop(host):
    rp, ci, va = laplacian(8, 2, "f64")
    n = len(rp) - 1
    kw = dict(max_iters=100, reduction=1e-8)
    b33 = rhs(n, 33, "f64")
    assert not solve(host, "f64", rp, ci, va, b33, 1, fused_multi_rhs=True, **kw)[3]
    b4 = rhs(n, 4, "f64")
    # off by default
    x, it, st, used = solve(host, "f64", rp, ci, va, b4, 1, **kw)
    assert not used and st == [0x80 | 0x40 | 2] * 4
    # block Jacobi is the loop's
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    from ginkgo_b200 import api
    t = [torch.from_numpy(a) for a in (va, ci, rp)]
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "cg", A, precond_max_bs=4, block_ptrs=bp, fused_multi_rhs=True, **kw)
    tx = torch.zeros(n, 4, dtype=torch.float64)
    s.apply(api.host_dense(host, torch.from_numpy(b4)), api.host_dense(host, tx))
    assert not s.used_fused
    # one column keeps the one-column path, whatever the switch
    b1 = b4[:, :1].copy()
    x1, it1, st1, used1 = solve(host, "f64", rp, ci, va, b1, 1, fused_multi_rhs=True, **kw)
    x0, it0, st0, used0 = solve(host, "f64", rp, ci, va, b1, 1, **kw)
    assert used1 and used0 and (it1, st1) == (it0, st0) and x1.tobytes() == x0.tobytes()
