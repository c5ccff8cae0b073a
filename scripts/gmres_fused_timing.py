"""GMRES (modified Gram-Schmidt) on one GPU: the kernel-by-kernel loop against the fused device-resident
iteration (solver::Gmres::with_fused), alternated in one process after a warm-up solve each.

Problems: cfg4 as bench.py runs it (GMRES(30) + block-Jacobi(16), fp32, reduction 1e-6) and a 3-D upwind
convection-diffusion stencil (fp64, scalar Jacobi, GMRES(30)) at a launch-bound size and at --grid^3.
Per problem and path: iterations, stopping status, true relative residual, wall time per iteration (median
of --reps solves, host clock around an apply that ends in a synchronise), launches issued per iteration,
the byte model of DESIGN.md section 4.5 over the time, and the first apply (graph capture included).
Then a sweep of check_every on the small stencil and on cfg4, fused path only.  Needs a GPU.

  python scripts/gmres_fused_timing.py [--grid 200] [--small 40] [--cfg4-rows 4000000] [--reps 3]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bicgstab_fused_timing import card, upwind3d  # noqa: E402


def model_bytes(it, kd, n, V, b_matrix, b_pre, fused):
    """vector + matrix traffic of `it` MGS iterations at Krylov indices 0, 1, .., kd-1, 0, ..
    loop: B_matrix + (5j + 13) n V, fused: B_matrix + (4j + 10) n V (+ the preconditioner's blocks)"""
    js = np.arange(it) % kd
    per = (4 * js + 10) if fused else (5 * js + 13)
    return float(it * (b_matrix + b_pre) + per.sum() * n * V)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--small", type=int, default=40)
    ap.add_argument("--cfg4-rows", type=int, default=4_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("gmres_fused_timing.py measures on a GPU and none is visible")
    import workloads as W
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())

    def setup(rp, ci, va):
        n = rp.numel() - 1
        with torch.cuda.stream(ex.stream):
            b = torch.ones(n, dtype=va.dtype, device=dev)
        return n, api.host_csr(ex, (n, n), va, ci, rp), b

    def solve(s, bd, x, xd):
        with torch.cuda.stream(ex.stream):
            x.zero_()
        ex.synchronize()
        l0 = ex.launch_count()
        t0 = time.perf_counter()
        s.apply(bd, xd)
        ex.synchronize()
        return time.perf_counter() - t0, ex.launch_count() - l0

    def true_res(A, b, xd):
        one = api.host_dense(ex, torch.ones(1, dtype=b.dtype, device=dev))
        neg = api.host_dense(ex, -torch.ones(1, dtype=b.dtype, device=dev))
        with torch.cuda.stream(ex.stream):
            r = b.clone()
        rd = api.host_dense(ex, r)
        api._hcheck(api._host().gkob_apply4(A.h, neg.h, xd.h, one.h, rd.h))
        ex.synchronize()
        return (r.double().norm() / b.double().norm()).item()

    def problem(label, rp, ci, va, red, pre, note=""):
        n, A, b = setup(rp, ci, va)
        nnz, V, I = va.numel(), va.element_size(), ci.element_size()
        bp = np.arange(0, n + 1, pre, dtype=np.int32) if pre > 1 else None
        kw = dict(precond_max_bs=pre, block_ptrs=bp, max_iters=1000, reduction=red, krylov_dim=30, ortho=0)
        solvers = [api.HostSolver(ex, "gmres", A, **kw), api.HostSolver(ex, "gmres", A, fused_gmres=True, **kw)]
        with torch.cuda.stream(ex.stream):
            xs = [torch.zeros(n, dtype=va.dtype, device=dev) for _ in range(2)]
        bd, xds = api.host_dense(ex, b), [api.host_dense(ex, x) for x in xs]
        first = [solve(solvers[k], bd, xs[k], xds[k])[0] for k in (0, 1)]  # warm-up; fused captures here
        times, launches = [[], []], [0, 0]
        for _ in range(args.reps):
            for k in (0, 1):
                t, nl = solve(solvers[k], bd, xs[k], xds[k])
                times[k].append(t)
                launches[k] = nl
        assert not solvers[0].used_fused and solvers[1].used_fused
        b_matrix = nnz * (V + I) + (n + 1) * I
        b_pre = n * pre * V if pre > 1 else 0  # the inverted blocks (scalar Jacobi: in the vector model)
        per_it = []
        for k, name in ((0, "loop "), (1, "fused")):
            it = max(solvers[k].num_iterations, 1)
            t = sorted(times[k])[len(times[k]) // 2]
            model = model_bytes(it, 30, n, V, b_matrix, b_pre, k == 1)
            per_it.append(t / it)
            print("%-24s %s n=%-9d it=%-4d status=0x%02x  %.3f ms/it (median of %d, min %.3f max %.3f)  "
                  "%.1f launches/it  true rel res %.2e  model %.1f MB/it -> %.0f GB/s  first apply %.1f ms%s" %
                  (label, name, n, solvers[k].num_iterations, solvers[k].stop_status, 1e3 * t / it, len(times[k]),
                   1e3 * min(times[k]) / it, 1e3 * max(times[k]) / it, launches[k] / it,
                   true_res(A, b, xds[k]), model / it / 1e6, model / t / 1e9, 1e3 * first[k], note))
        print("%-24s time per iteration, loop / fused = %.2f (%s)" %
              (label, per_it[0] / per_it[1], "fused faster" if per_it[1] < per_it[0] else "fused SLOWER"))

    def sweep(label, rp, ci, va, red, pre):
        n, A, b = setup(rp, ci, va)
        bp = np.arange(0, n + 1, pre, dtype=np.int32) if pre > 1 else None
        with torch.cuda.stream(ex.stream):
            x = torch.zeros(n, dtype=va.dtype, device=dev)
        bd, xd = api.host_dense(ex, b), api.host_dense(ex, x)
        for ce in (1, 4, 8, 16, 30):
            s = api.HostSolver(ex, "gmres", A, precond_max_bs=pre, block_ptrs=bp, max_iters=1000, reduction=red,
                               krylov_dim=30, ortho=0, check_every=ce, fused_gmres=True)
            solve(s, bd, x, xd)
            ts = sorted(solve(s, bd, x, xd)[0] for _ in range(args.reps))
            it = max(s.num_iterations, 1)
            print("%-24s check_every=%-3d it=%-4d %.3f ms/it" % (label, ce, s.num_iterations, 1e3 * ts[len(ts) // 2] / it))

    with torch.cuda.stream(ex.stream):
        rp, ci, va = W.build("cfg4", xp="torch", device=dev, n=args.cfg4_rows)
    problem("cfg4 f32 bj16", rp, ci, va, 1e-6, 16)
    sweep("cfg4 f32 bj16", rp, ci, va, 1e-6, 16)
    del rp, ci, va
    with torch.cuda.stream(ex.stream):
        small = upwind3d(torch, args.small, dev)
    problem("upwind3d %d^3 f64 jac" % args.small, *small, 1e-8, 1, "  [launch / host-sync bound size]")
    sweep("upwind3d %d^3 f64 jac" % args.small, *small, 1e-8, 1)
    del small
    with torch.cuda.stream(ex.stream):
        big = upwind3d(torch, args.grid, dev)
    problem("upwind3d %d^3 f64 jac" % args.grid, *big, 1e-8, 1)


if __name__ == "__main__":
    main()
