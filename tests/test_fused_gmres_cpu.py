"""solver::Gmres::try_fused on the host-memory mock (tests/mock): one graph per batch of
check_every iterations, polling of the control block, the host-issued restart and the final update
run on the CPU.  The mock's restatements and the kernel-by-kernel loop both sum their dots and norms
sequentially from row 0, so the fused path must give the loop's iterations, status and bits of x."""
import numpy as np
import pytest
import torch

from tests.helpers import VT
from tests.test_fused_bicgstab_cpu import convection_diffusion


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock_gmres")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def solve(host, rp, ci, va, b, precond, block_ptrs=None, **kw):
    from ginkgo_b200 import api
    n = len(rp) - 1
    t = [torch.from_numpy(np.ascontiguousarray(a)) for a in (va, ci, rp)]
    tb = torch.from_numpy(np.ascontiguousarray(b))
    tx = torch.zeros_like(tb)
    A = api.host_csr(host, (n, n), *t)
    s = api.HostSolver(host, "gmres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(host, tb), api.host_dense(host, tx))
    return tx.numpy(), s.num_iterations, s.stop_status, s.used_fused


PRECONDS = {"identity": 0, "scalar": 1, "block": 4}


def case(vt="f64", g=12):
    rp, ci, va = convection_diffusion(g, 2, vt)
    n = len(rp) - 1
    b = np.random.default_rng(3).uniform(-1, 1, (n, 1)).astype(VT[vt])
    return rp, ci, va, b, np.arange(0, n + 1, 4, dtype=np.int32)


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("precond", list(PRECONDS))
@pytest.mark.parametrize("kd", [4, 20])
@pytest.mark.parametrize("ce", ["1", "3", "kd", "kd+5"])
def test_fused_gmres_takes_the_loops_bits(host, ortho, precond, kd, ce):
    rp, ci, va, b, bp = case()
    check_every = {"1": 1, "3": 3, "kd": kd, "kd+5": kd + 5}[ce]
    kw = dict(max_iters=400, reduction=1e-10, krylov_dim=kd, ortho=ortho)
    pc = PRECONDS[precond]
    xl, itl, stl, usedl = solve(host, rp, ci, va, b, pc, bp if pc > 1 else None, **kw)
    xf, itf, stf, usedf = solve(host, rp, ci, va, b, pc, bp if pc > 1 else None, fused_gmres=True,
                                check_every=check_every, **kw)
    assert usedf and not usedl
    assert stl == 0x80 | 0x40 | 2 and itl > kd  # converged after at least one restart
    assert (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("baseline", [0, 1, 2])
def test_fused_gmres_types_and_baselines(host, vt, ortho, baseline):
    rp, ci, va, b, bp = case(vt)
    red = (1e-9 if vt == "f64" else 1e-4) * (10 if baseline == 2 else 1)
    kw = dict(max_iters=400, reduction=red, krylov_dim=6, ortho=ortho, baseline=baseline, iter_first=False)
    xl, itl, stl, _ = solve(host, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, rp, ci, va, b, 1, fused_gmres=True, check_every=4, **kw)
    assert used and stl & 0x80 and (itf, stf) == (itl, stl)
    assert xf.tobytes() == xl.tobytes()


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("check_every", [1, 3, 5, 9])
@pytest.mark.parametrize("max_iters", [0, 1, 2, 3, 4, 5, 6, 10])
def test_fused_gmres_stop_positions(host, ortho, check_every, max_iters):
    """Iteration stops at iteration 0, mid-batch, at a batch end and at a cycle end (kd = 5: no restart
    may run after a stop at 5 or 10): iterations, status and x equal to the loop's"""
    rp, ci, va, b, bp = case()
    kw = dict(max_iters=max_iters, reduction=1e-14, krylov_dim=5, ortho=ortho)
    xl, itl, stl, _ = solve(host, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = solve(host, rp, ci, va, b, 1, fused_gmres=True, check_every=check_every, **kw)
    assert used and (itf, stf) == (itl, stl) == (max_iters, 0x40 | 1)
    assert xf.tobytes() == xl.tobytes()


def test_fused_gmres_zero_rhs(host):
    rp, ci, va, b, bp = case()
    x, it, st, used = solve(host, rp, ci, va, np.zeros_like(b), 1, max_iters=50, reduction=1e-8, baseline=2,
                            fused_gmres=True)
    assert used and it == 0 and st == 0x80 | 0x40 | 2 and np.all(x == 0)


def test_fused_gmres_fallbacks(host):
    rp, ci, va, b, bp = case()
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8, fused_gmres=True)
    b2 = np.random.default_rng(2).uniform(-1, 1, (n, 2))
    assert not solve(host, rp, ci, va, b2, 1, **kw)[3]  # two right-hand sides
    with pytest.raises(Exception):  # ImplicitResidualNorm: NotSupported, as from the loop
        solve(host, rp, ci, va, b, 1, res_kind=2, **kw)
    assert not solve(host, rp, ci, va, b, 1, max_iters=300, reduction=1e-8, fused=True, fused_bicgstab=True)[3]
