"""solver::Bicgstab::try_fused_multi_rhs on the host-memory mock: graph capture and replay, polling of the
control block every check_every iterations, the per-column statuses and the finalize owed after a stop at
the mid-iteration check run on the CPU.  The mock's restatements of the fused kernels and the
kernel-by-kernel loop both add every column's dot products over the rows in order, so the two paths
take the same iterations and give the same bits."""
import numpy as np
import pytest
import torch

from tests.helpers import VT
from tests.test_fused_bicgstab_gpu import upwind

FIN_CONV_2 = 0x80 | 0x40 | 2  # converged by the residual criterion, second of Iteration first


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_bicgstab_mrhs")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def system(vt, it="i32", g=12):
    rp, ci, va = upwind(g, 2, vt)
    idx = np.int32 if it == "i32" else np.int64
    return rp.astype(idx), ci.astype(idx), va


def periodic_upwind(n, vt):
    """periodic 1-D upwind: 2.75 on the diagonal, -1.5 below, -1 above (n even).  Every row sums to 0.25
    and (-1)^i is an eigenvector with eigenvalue 5.25"""
    rows = np.repeat(np.arange(n), 3)
    cols = np.stack([(np.arange(n) - 1) % n, np.arange(n), (np.arange(n) + 1) % n], axis=1).reshape(-1)
    vals = np.tile([-1.5, 2.75, -1.0], n)
    order = np.lexsort((cols, rows))
    rp = np.arange(0, 3 * n + 1, 3, dtype=np.int32)
    return rp, cols[order].astype(np.int32), vals[order].astype(VT[vt])


def rhs(n, k, vt, seed=3):
    """k columns; column 1 scaled by 1e-3, so that it stops at another iteration under initial_resnorm
    and absolute baselines than its neighbours"""
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
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=precond, **kw)
    s.apply(api.host_dense(host, tb), api.host_dense(host, tx))
    return tx.numpy(), s.num_iterations, s.stop_statuses, s.used_fused


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("it,precond", [("i32", 0), ("i32", 1), ("i64", 0)])  # the C handle's Jacobi is int32's
@pytest.mark.parametrize("res_kind,baseline,iter_first", [(1, 0, True), (2, 1, False), (1, 2, True), (1, 1, False)])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_multi_rhs_takes_the_loops_iterations(host, vt, it, precond, res_kind, baseline, iter_first,
                                                    check_every):
    rp, ci, va = system(vt, it)
    n = len(rp) - 1
    b = rhs(n, 4, vt)
    red = 1e-9 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10  # absolute threshold
    kw = dict(max_iters=300, reduction=red, res_kind=res_kind, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, usedl = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, vt, rp, ci, va, b, precond, fused_bicgstab_multi_rhs=True,
                                check_every=check_every, **kw)
    assert usedf and not usedl
    assert all(s & 0x80 for s in stl) and itl > 1
    assert (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_multi_rhs_columns_stop_on_their_own(host, check_every):
    """a zero column of b stops at iteration 0 under rhs_norm (converged, id 2); the Iteration limit
    then marks only the columns still running (id 1)"""
    rp, ci, va = system("f64", "i64", 10)
    n = len(rp) - 1
    b = rhs(n, 5, "f64", seed=7)
    b[:, 2] = 0
    kw = dict(max_iters=6, reduction=1e-14)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 0, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, 0, fused_bicgstab_multi_rhs=True,
                               check_every=check_every, **kw)
    assert used and itf == itl == 6
    assert stf == stl
    assert stf[2] == FIN_CONV_2 and all(s == 0x40 | 1 for j, s in enumerate(stf) if j != 2)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("check_every", [1, 16])
def test_mid_check_stops_among_running_columns(host, precond, check_every):
    """eigenvector columns of the periodic upwind matrix stop at the mid check of iteration 0 and owe
    x_j += alpha_j y_j; a random and a zero column run on beside them"""
    n, vt = 64, "f64"
    rp, ci, va = periodic_upwind(n, vt)
    alt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    b = np.stack([np.ones(n), alt, np.random.default_rng(1).uniform(-1, 1, n), np.zeros(n), 3 * alt], axis=1)
    kw = dict(max_iters=200, reduction=1e-10)
    xl, itl, stl, _ = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, used = solve(host, vt, rp, ci, va, b, precond, fused_bicgstab_multi_rhs=True,
                               check_every=check_every, **kw)
    assert used and (itf, stf) == (itl, stl) and itf > 0
    assert xf.tobytes() == xl.tobytes()
    assert all(s == FIN_CONV_2 for s in stf)
    for j, lam in ((0, 0.25), (1, 5.25), (4, 5.25)):
        assert np.allclose(xf[:, j], b[:, j] / lam, rtol=1e-13, atol=0)
    assert np.all(xf[:, 3] == 0)


@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("check_every", [1, 16])
def test_every_column_stops_at_the_mid_check(host, precond, check_every):
    """only eigenvector columns: the whole solve stops at the mid check of iteration 0, reports 0
    iterations, and x = b / lambda is applied once (not once per replayed iteration)"""
    n, vt = 64, "f64"
    rp, ci, va = periodic_upwind(n, vt)
    alt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    b = np.stack([np.ones(n), alt, 2 * np.ones(n)], axis=1)
    kw = dict(max_iters=200, reduction=1e-10)
    xl, itl, stl, _ = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, used = solve(host, vt, rp, ci, va, b, precond, fused_bicgstab_multi_rhs=True,
                               check_every=check_every, **kw)
    assert used and itf == itl == 0 and stf == stl == [FIN_CONV_2] * 3
    assert xf.tobytes() == xl.tobytes()
    for j, lam in ((0, 0.25), (1, 5.25), (2, 0.25)):
        assert np.allclose(xf[:, j], b[:, j] / lam, rtol=1e-13, atol=0)


def test_fused_multi_rhs_workspace_and_graph_are_reused(host):
    from ginkgo_b200 import api
    rp, ci, va = system("f64", "i32", 9)
    n = len(rp) - 1
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=1, max_iters=200, reduction=1e-9,
                       fused_bicgstab_multi_rhs=True, check_every=5)
    for k, seed in ((3, 1), (3, 2), (6, 3), (3, 4)):
        b = rhs(n, k, "f64", seed)
        tx = torch.zeros(n, k, dtype=torch.float64)
        s.apply(api.host_dense(host, torch.from_numpy(b)), api.host_dense(host, tx))
        assert s.used_fused and s.stop_statuses == [FIN_CONV_2] * k
        xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 1, max_iters=200, reduction=1e-9)
        assert s.num_iterations == itl and tx.numpy().tobytes() == xl.tobytes()


def test_fused_multi_rhs_falls_back_to_the_loop(host):
    rp, ci, va = system("f64", "i32", 8)
    n = len(rp) - 1
    kw = dict(max_iters=100, reduction=1e-8)
    b33 = rhs(n, 33, "f64")
    assert not solve(host, "f64", rp, ci, va, b33, 1, fused_bicgstab_multi_rhs=True, **kw)[3]
    b4 = rhs(n, 4, "f64")
    # off by default
    x, it, st, used = solve(host, "f64", rp, ci, va, b4, 1, **kw)
    assert not used and st == [FIN_CONV_2] * 4
    # block Jacobi is the loop's
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    from ginkgo_b200 import api
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=4, block_ptrs=bp, fused_bicgstab_multi_rhs=True, **kw)
    tx = torch.zeros(n, 4, dtype=torch.float64)
    s.apply(api.host_dense(host, torch.from_numpy(b4)), api.host_dense(host, tx))
    assert not s.used_fused
    # b and x with a stride > k are the loop's
    tb = torch.from_numpy(np.pad(b4, ((0, 0), (0, 2))))
    tx = torch.zeros(n, 6, dtype=torch.float64)
    s = api.HostSolver(host, "bicgstab", A, precond_max_bs=1, fused_bicgstab_multi_rhs=True, **kw)
    s.apply(api.host_dense(host, tb, cols=4), api.host_dense(host, tx, cols=4))
    assert not s.used_fused and s.stop_statuses == [FIN_CONV_2] * 4
    # one column keeps today's behaviour, whatever the switch
    b1 = b4[:, :1].copy()
    x1, it1, st1, used1 = solve(host, "f64", rp, ci, va, b1, 1, fused_bicgstab_multi_rhs=True, **kw)
    x0, it0, st0, used0 = solve(host, "f64", rp, ci, va, b1, 1, **kw)
    assert not used1 and not used0 and (it1, st1) == (it0, st0) and x1.tobytes() == x0.tobytes()
