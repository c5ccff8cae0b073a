"""solver::Minres::try_fused_multi_rhs on the host-memory mock: the set-up through the loop's own calls on
n x k views, graph capture and replay, the p / p_prev roles taken from the shared iteration counter's
parity, polling of the control block every check_every iterations and the per-column statuses run on the
CPU.  The mock's restatements of the fused kernels and the kernel-by-kernel loop both add every column's
dot products over the rows in order, so the two paths take the same iterations and give the same bits."""
import numpy as np
import pytest
import torch

from tests.helpers import VT
from tests.test_fused_minres_cpu import indefinite_laplacian


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_minres_mrhs")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def rhs(n, k, vt, seed=3):
    """k columns; column 1 scaled by 1e-3, so that it converges at another iteration than its
    neighbours under the absolute baseline"""
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
    b[:, 1] *= 1e-3
    return b.astype(VT[vt])


def solve(host, vt, rp, ci, va, b, precond, block_ptrs=None, strided=0, **kw):
    from ginkgo_b200 import api
    n, k = len(rp) - 1, b.shape[1]
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(np.pad(b, ((0, 0), (0, strided)))))
    tx = torch.zeros_like(tb)
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "minres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(host, tb, cols=k), api.host_dense(host, tx, cols=k))
    return tx.numpy()[:, :k], s.num_iterations, s.stop_statuses, s.used_fused


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("baseline,iter_first", [(0, True), (1, False), (2, True), (0, False), (1, True), (2, False)])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_fused_minres_multi_rhs_takes_the_loops_iterations(host, vt, precond, baseline, iter_first, check_every):
    rp, ci, va = indefinite_laplacian(12, 2, vt, 0.6)
    n = len(rp) - 1
    b = rhs(n, 4, vt)
    red = 1e-9 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10  # absolute threshold
    kw = dict(max_iters=400, reduction=red, res_kind=2, baseline=baseline, iter_first=iter_first)
    xl, itl, stl, usedl = solve(host, vt, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = solve(host, vt, rp, ci, va, b, precond, fused_minres_multi_rhs=True,
                                check_every=check_every, **kw)
    assert usedf and not usedl
    assert all(s & 0x80 for s in stl) and itl > 1  # converged; the last batch runs past the stop
    assert (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("max_iters", [0, 1, 5])
@pytest.mark.parametrize("iter_first", [True, False])
@pytest.mark.parametrize("precond", [0, 1])
def test_fused_minres_multi_rhs_iteration_limit(host, max_iters, iter_first, precond):
    rp, ci, va = indefinite_laplacian(12, 2, "f64", 0.6)
    n = len(rp) - 1
    b = rhs(n, 3, "f64", seed=5)
    kw = dict(max_iters=max_iters, reduction=1e-12, res_kind=2, iter_first=iter_first)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, precond, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, precond, fused_minres_multi_rhs=True, check_every=3,
                               **kw)
    assert used and (itf, stf) == (itl, stl) and itf == max_iters
    assert stf == [0x40 | (1 if iter_first else 2)] * 3
    assert xf.tobytes() == xl.tobytes()


def test_fused_minres_multi_rhs_iteration_criterion_alone(host):
    rp, ci, va = indefinite_laplacian(10, 2, "f32", 0.6)
    n = len(rp) - 1
    b = rhs(n, 5, "f32", seed=8)
    kw = dict(max_iters=37, res_kind=0)
    xl, itl, stl, _ = solve(host, "f32", rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, "f32", rp, ci, va, b, 1, fused_minres_multi_rhs=True, check_every=16, **kw)
    assert used and (itf, stf) == (itl, stl) and (itf, stf) == (37, [0x40 | 1] * 5)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("check_every", [1, 7, 16])
@pytest.mark.parametrize("baseline", [0, 2])
def test_fused_minres_multi_rhs_columns_stop_on_their_own(host, check_every, baseline):
    """a zero column of b stops at iteration 0 (converged, id 2) and keeps x = 0; the Iteration limit
    then marks only the columns still running (id 1); under the absolute baseline the scaled column 1
    converges before the others"""
    rp, ci, va = indefinite_laplacian(10, 2, "f64", 0.6)
    n = len(rp) - 1
    b = rhs(n, 5, "f64", seed=7)
    b[:, 2] = 0
    kw = dict(max_iters=12, reduction=1e-10 if baseline == 0 else 1e-3, res_kind=2, baseline=baseline)
    xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b, 1, fused_minres_multi_rhs=True, check_every=check_every,
                               **kw)
    assert used and itf == itl == 12 and stf == stl
    assert stf[2] == 0x80 | 0x40 | 2 and not np.any(xf[:, 2])
    others = [0, 3, 4] if baseline == 2 else [0, 1, 3, 4]
    assert all(stf[j] == 0x40 | 1 for j in others)
    if baseline == 2:
        assert stf[1] == 0x80 | 0x40 | 2
    assert xf.tobytes() == xl.tobytes()


def test_fused_minres_multi_rhs_workspace_and_graph_are_reused(host):
    """one solver, applies with k = 3, 3, 6, 3, 3 and a new x each time: the workspace is reshaped and the
    graph recaptured whenever k or x changes, and every apply gives the loop's bits"""
    from ginkgo_b200 import api
    rp, ci, va = indefinite_laplacian(9, 2, "f64", 0.6)
    n = len(rp) - 1
    A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
    kw = dict(max_iters=300, reduction=1e-9, res_kind=2)
    s = api.HostSolver(host, "minres", A, precond_max_bs=1, fused_minres_multi_rhs=True, check_every=5, **kw)
    xs = {}
    for i, (k, seed) in enumerate(((3, 1), (3, 2), (6, 3), (3, 4), (3, 5))):
        b = rhs(n, k, "f64", seed)
        tx = xs.setdefault((k, i % 2), torch.zeros(n, k, dtype=torch.float64))
        tx.zero_()
        s.apply(api.host_dense(host, torch.from_numpy(b)), api.host_dense(host, tx))
        assert s.used_fused and s.stop_statuses == [0x80 | 0x40 | 2] * k
        xl, itl, stl, _ = solve(host, "f64", rp, ci, va, b, 1, **kw)
        assert s.num_iterations == itl and tx.numpy().tobytes() == xl.tobytes()


def test_fused_minres_multi_rhs_falls_back_to_the_loop(host):
    rp, ci, va = indefinite_laplacian(8, 2, "f64", 0.6)
    n = len(rp) - 1
    kw = dict(max_iters=200, reduction=1e-8, res_kind=2)
    on = dict(kw, fused_minres_multi_rhs=True)
    b33, b4 = rhs(n, 33, "f64"), rhs(n, 4, "f64")
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not solve(host, "f64", rp, ci, va, b33, 1, **on)[3]                    # more than 32 columns
    assert not solve(host, "f64", rp, ci, va, b4, 1, strided=2, **on)[3]          # stride != k
    assert not solve(host, "f64", rp, ci, va, b4, 4, bp, **on)[3]                 # block Jacobi
    assert not solve(host, "f64", rp, ci, va, b4, 1, **dict(on, res_kind=1))[3]   # ResidualNorm
    x, it, st, used = solve(host, "f64", rp, ci, va, b4, 1, **kw)                 # off by default
    assert not used and st == [0x80 | 0x40 | 2] * 4
    # the one-column switch alone keeps k columns on the loop
    assert not solve(host, "f64", rp, ci, va, b4, 1, fused_minres=True, **kw)[3]
    xf, itf, stf, used = solve(host, "f64", rp, ci, va, b4, 1, **on)
    assert used and (itf, stf) == (it, st) and xf.tobytes() == x.tobytes()


def test_fused_minres_multi_rhs_one_column_keeps_the_one_column_path(host):
    rp, ci, va = indefinite_laplacian(10, 2, "f64", 0.6)
    n = len(rp) - 1
    b1 = rhs(n, 2, "f64", seed=11)[:, :1].copy()
    kw = dict(max_iters=300, reduction=1e-9, res_kind=2, fused_minres=True)
    xa, ita, sta, usa = solve(host, "f64", rp, ci, va, b1, 1, fused_minres_multi_rhs=True, **kw)
    xb, itb, stb, usb = solve(host, "f64", rp, ci, va, b1, 1, **kw)
    assert usa and usb and (ita, sta) == (itb, stb) and xa.tobytes() == xb.tobytes()
    # the new switch alone leaves one column on the loop
    xc, itc, stc, usc = solve(host, "f64", rp, ci, va, b1, 1, **dict(kw, fused_minres=False,
                                                                     fused_minres_multi_rhs=True))
    assert not usc and (itc, stc) == (itb, stb)
