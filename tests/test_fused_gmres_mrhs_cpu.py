"""solver::Gmres::try_fused_multi_rhs on the host-memory mock (tests/mock): one graph per
batch of check_every iterations, polling of the control block, the per-column statuses and the restart
issued on all k columns run on the CPU.  The mock's restatements and the kernel-by-kernel loop both sum
every column's dots and norms over the rows in order, so the fused path must give the loop's iterations,
per-column statuses and bits of x."""
import numpy as np
import pytest
import torch

from tests.helpers import VT
from tests.test_fused_bicgstab_cpu import convection_diffusion

CONV_2 = 0x80 | 0x40 | 2   # converged (second criterion, Iteration first), finalized by the final update
ITER_1 = 0x40 | 1          # the Iteration limit, finalized


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_gmres_mrhs")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def solve(host, rp, ci, va, b, precond, block_ptrs=None, cols=None, **kw):
    from ginkgo_b200 import api
    n = len(rp) - 1
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(b))
    tx = torch.zeros_like(tb)
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "gmres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(host, tb, cols=cols), api.host_dense(host, tx, cols=cols))
    return tx.numpy(), s.num_iterations, s.stop_statuses, s.used_fused


def case(vt="f64", g=12, k=4, seed=3):
    rp, ci, va = convection_diffusion(g, 2, vt)
    n = len(rp) - 1
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k)).astype(VT[vt])
    return rp, ci, va, b


def staggered(vt="f64", g=12):
    """columns that stop at different cycles (kd = 4): a zero column (iteration 0), a column that is
    almost an eigen-solve of the first cycle (A times a smooth vector, converged inside cycle 1 and
    finalized at the first restart), and random columns that run through several restarts"""
    rp, ci, va, b = case(vt, g, 5, seed=9)
    n = len(rp) - 1
    b[:, 1] = 0
    e = np.zeros(n)
    e[:3] = (1.0, -0.5, 0.25)
    Ae = np.zeros(n)
    for r in range(n):
        Ae[r] = sum(va[q] * e[ci[q]] for q in range(rp[r], rp[r + 1]))
    b[:, 3] = Ae.astype(VT[vt])
    return rp, ci, va, b


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("kd", [4, 20])
@pytest.mark.parametrize("ce", ["1", "3", "kd", "kd+5"])
def test_fused_gmres_multi_rhs_takes_the_loops_bits(host, ortho, precond, vt, kd, ce):
    rp, ci, va, b = case(vt)
    check_every = {"1": 1, "3": 3, "kd": kd, "kd+5": kd + 5}[ce]
    kw = dict(max_iters=400, reduction=1e-10 if vt == "f64" else 1e-5, krylov_dim=kd, ortho=ortho)
    xl, itl, stl, usedl = solve(host, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, rp, ci, va, b, precond, fused_gmres_multi_rhs=True,
                                check_every=check_every, **kw)
    assert usedf and not usedl
    assert all(s & 0x80 for s in stl) and itl > kd  # converged after at least one restart
    assert (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("baseline", [0, 1, 2])
@pytest.mark.parametrize("iter_first", [True, False])
def test_fused_gmres_multi_rhs_baselines_and_orders(host, ortho, baseline, iter_first):
    rp, ci, va, b = case()
    b[:, 1] *= 1e-3  # stops at another iteration than its neighbours under the absolute baseline
    red = 1e-9 * (10 if baseline == 2 else 1)
    kw = dict(max_iters=400, reduction=red, krylov_dim=6, ortho=ortho, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, _ = solve(host, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, rp, ci, va, b, 1, fused_gmres_multi_rhs=True, check_every=4, **kw)
    assert used and all(s & 0x80 for s in stl) and (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("check_every", [1, 3, 4, 9])
def test_columns_stop_at_different_cycles(host, ortho, precond, check_every):
    rp, ci, va, b = staggered()
    kw = dict(max_iters=400, reduction=1e-10, krylov_dim=4, ortho=ortho)
    xl, itl, stl, _ = solve(host, rp, ci, va, b, precond, **kw)
    xf, itf, stf, used = solve(host, rp, ci, va, b, precond, fused_gmres_multi_rhs=True,
                               check_every=check_every, **kw)
    assert used and (itf, stf) == (itl, stl) and itl > 8  # at least two restarts
    assert all(s == CONV_2 for s in stf)
    assert xf.tobytes() == xl.tobytes()
    assert np.all(xf[:, 1] == 0)


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("check_every", [1, 3, 5, 9])
@pytest.mark.parametrize("max_iters", [0, 1, 2, 3, 4, 5, 6, 10])
def test_stop_positions(host, ortho, check_every, max_iters):
    """Iteration stops at iteration 0, mid-batch, at a batch end and at a cycle end (kd = 5: no restart
    may run after a stop at 5 or 10); a zero column has stopped at iteration 0"""
    rp, ci, va, b = case(k=3)
    b[:, 2] = 0
    kw = dict(max_iters=max_iters, reduction=1e-14, krylov_dim=5, ortho=ortho)
    xl, itl, stl, _ = solve(host, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, rp, ci, va, b, 1, fused_gmres_multi_rhs=True, check_every=check_every, **kw)
    assert used and (itf, stf) == (itl, stl)
    # at iteration 0 the Iteration criterion, first in order, also names the zero column
    assert itf == max_iters and stf[:2] == [ITER_1] * 2 and stf[2] == (ITER_1 if max_iters == 0 else CONV_2)
    assert xf.tobytes() == xl.tobytes()


def test_workspace_and_graphs_are_reused(host):
    from ginkgo_b200 import api
    rp, ci, va, _ = case(g=9)
    n = len(rp) - 1
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    kw = dict(max_iters=300, reduction=1e-9, krylov_dim=7, ortho=1)
    s = api.HostSolver(host, "gmres", A, precond_max_bs=1, fused_gmres_multi_rhs=True, check_every=3, **kw)
    for k, seed in ((3, 1), (3, 2), (6, 3), (3, 4)):
        b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
        tx = torch.zeros(n, k, dtype=torch.float64)
        s.apply(api.host_dense(host, torch.from_numpy(b)), api.host_dense(host, tx))
        assert s.used_fused and s.stop_statuses == [CONV_2] * k
        xl, itl, stl, _ = solve(host, rp, ci, va, b, 1, **kw)
        assert s.num_iterations == itl and tx.numpy().tobytes() == xl.tobytes()


def test_fallbacks(host):
    rp, ci, va, b = case(g=8)
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8, krylov_dim=10)
    on = dict(fused_gmres_multi_rhs=True, **kw)
    b33 = np.random.default_rng(5).uniform(-1, 1, (n, 33))
    assert not solve(host, rp, ci, va, b33, 1, **on)[3]
    # off by default, and the one-column switch does not turn it on
    assert not solve(host, rp, ci, va, b, 1, **kw)[3]
    assert not solve(host, rp, ci, va, b, 1, fused_gmres=True, fused_multi_rhs=True, **kw)[3]
    # block Jacobi is the loop's
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not solve(host, rp, ci, va, b, 4, block_ptrs=bp, **on)[3]
    # b and x with a stride > k are the loop's
    x, it, st, used = solve(host, rp, ci, va, np.pad(b, ((0, 0), (0, 2))), 1, cols=4, **on)
    assert not used and st == [CONV_2] * 4
    # ImplicitResidualNorm: NotSupported, as from the loop
    with pytest.raises(Exception):
        solve(host, rp, ci, va, b, 1, res_kind=2, **on)
    # one column keeps today's behaviour, whatever the switch
    b1 = b[:, :1].copy()
    x1, it1, st1, used1 = solve(host, rp, ci, va, b1, 1, **on)
    x0, it0, st0, used0 = solve(host, rp, ci, va, b1, 1, **kw)
    assert not used1 and not used0 and (it1, st1) == (it0, st0) and x1.tobytes() == x0.tobytes()
