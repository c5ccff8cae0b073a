"""When the fused solver paths re-capture their graphs, on the host-memory mock.  A captured graph bakes in
x and the matrix arrays; a new x, or a Csr re-read under a live solver, must give the loop's result and
never replay a graph over the old pointers.  The mock's restatements of the fused kernels sum in the
loop's order, so results are compared bit for bit."""
import os
import subprocess

import numpy as np
import pytest
import torch

import workloads as W
from tests.test_fused_bicgstab_cpu import convection_diffusion

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    from ginkgo_b200 import api
    from tests.mock_build import CpuExec, build_mock_host
    lib = build_mock_host(str(tmp_path_factory.mktemp("mock")))
    saved = api._HOST_LIB
    api._HOST_LIB = lib
    yield CpuExec(lib)
    api._HOST_LIB = saved


def laplacian(g, dims, vt):
    assert vt == "f64"
    return W.laplace(g, dims, vdtype=np.float64)


# path: (solver, switch, columns, matrix, Jacobi block size, further keywords)
PATHS = {
    "cg": ("cg", "fused", 1, laplacian, 1, {}),
    "cg_mrhs": ("cg", "fused_multi_rhs", 3, laplacian, 1, {}),
    "bicgstab": ("bicgstab", "fused_bicgstab", 1, convection_diffusion, 1, {}),
    "bicgstab_mrhs": ("bicgstab", "fused_bicgstab_multi_rhs", 3, convection_diffusion, 1, {}),
    "gmres_identity": ("gmres", "fused_gmres", 1, convection_diffusion, 0, {"krylov_dim": 7}),
    "gmres_scalar": ("gmres", "fused_gmres", 1, convection_diffusion, 1, {"krylov_dim": 7}),
    "gmres_block": ("gmres", "fused_gmres", 1, convection_diffusion, 4, {"krylov_dim": 7}),
    "gmres_mrhs": ("gmres", "fused_gmres_multi_rhs", 3, convection_diffusion, 1, {"krylov_dim": 7, "ortho": 1}),
}


@pytest.mark.parametrize("path", list(PATHS))
def test_a_new_x_every_apply_gives_the_loops_result(host, path):
    """two x tensors used in turn across four applies: the paths that bake x into their graphs re-capture,
    the GMRES paths (whose graphs do not hold x) keep theirs, and each apply gives the loop's iterations,
    statuses and bits of x"""
    from ginkgo_b200 import api
    kind, switch, k, matrix, precond, extra = PATHS[path]
    rp, ci, va = (np.ascontiguousarray(a) for a in matrix(10, 2, "f64"))
    n = len(rp) - 1
    bp = np.arange(0, n + 1, 4, dtype=np.int32) if precond > 1 else None
    kw = dict(max_iters=300, reduction=1e-9, **extra)

    def solver(**switches):
        A = api.host_csr(host, (n, n), *[torch.from_numpy(a) for a in (va, ci, rp)])
        return api.HostSolver(host, kind, A, precond_max_bs=precond, block_ptrs=bp, check_every=3, **switches, **kw)

    def statuses(s):
        return s.stop_statuses if k > 1 else s.stop_status

    s = solver(**{"fused": False, switch: True})
    loop = solver(fused=False)
    rng = np.random.default_rng(12)
    xs = [torch.zeros(n, k, dtype=torch.float64) for _ in range(2)]
    for apply in range(4):
        b = torch.from_numpy(rng.uniform(-1, 1, (n, k)))
        tx, xl = xs[apply % 2], torch.zeros(n, k, dtype=torch.float64)
        tx.zero_()
        s.apply(api.host_dense(host, b), api.host_dense(host, tx))
        loop.apply(api.host_dense(host, b), api.host_dense(host, xl))
        assert s.used_fused and not loop.used_fused
        assert (s.num_iterations, statuses(s)) == (loop.num_iterations, statuses(loop))
        assert tx.numpy().tobytes() == xl.numpy().tobytes()


def test_fused_cg_after_the_matrix_is_re_read(tmp_path):
    """tests/cpp/fused_reread_check.cpp: Csr::read between two applies of a fused Cg into the same x; the
    second apply gives the loop's iterations, status and bits of x on the new matrix"""
    from tests.mock_build import build_mock_executable
    exe = build_mock_executable(str(tmp_path), os.path.join(ROOT, "tests", "cpp", "fused_reread_check.cpp"),
                                "fused_reread_check")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
