"""BiCGStab on one GPU: the kernel-by-kernel loop against the fused device-resident iteration
(solver::Bicgstab::with_fused), alternated in one process after warming both.

Problems: a 3-D upwind convection-diffusion stencil (fp64, scalar Jacobi) at --grid^3 and at a small
size where launches and host synchronisation dominate, and cfg4's random diagonally dominant matrix
(fp32, scalar Jacobi).  Per problem and path: iterations, stopping status, wall time per iteration
(host clock around an apply that ends in a synchronise), the true relative residual, and the byte
model of DESIGN.md section 4 (2 B_matrix + 36 n V for the loop, 2 B_matrix + 25 n V fused) over the
time, i.e. the HBM rate each path would need to be bandwidth-bound.  Needs a GPU; there is no fallback.

  python scripts/bicgstab_fused_timing.py [--grid 200] [--small 40] [--cfg4-rows 4000000] [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown (nvidia-smi unavailable)"


def upwind3d(torch, g, dev, wind=0.8):
    """7-point Laplacian on a g^3 grid with `wind` added to the diagonal and subtracted from the
    upstream neighbour along every axis (first-order upwind convection): nonsymmetric"""
    import workloads as W
    rp, ci, va = W.laplace(g, 3, xp="torch", device=dev)
    n = g ** 3
    rows = torch.repeat_interleave(torch.arange(n, device=dev), (rp[1:] - rp[:-1]).long())
    col = ci.long()
    for d in range(3):
        va[col == rows - g ** d] -= wind
    va[col == rows] += 3 * wind
    return rp, ci, va


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--small", type=int, default=40)
    ap.add_argument("--cfg4-rows", type=int, default=4_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bicgstab_fused_timing.py measures on a GPU and none is visible")
    import workloads as W
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())

    def problem(label, rp, ci, va, red, note=""):
        n, nnz = rp.numel() - 1, va.numel()
        V, I = va.element_size(), ci.element_size()
        with torch.cuda.stream(ex.stream):
            b = torch.ones(n, dtype=va.dtype, device=dev)
            xs = [torch.zeros(n, dtype=va.dtype, device=dev) for _ in range(2)]
        A = api.host_csr(ex, (n, n), va, ci, rp)
        bd = api.host_dense(ex, b)
        kw = dict(precond_max_bs=1, max_iters=2000, reduction=red)
        solvers = [api.HostSolver(ex, "bicgstab", A, **kw), api.HostSolver(ex, "bicgstab", A, fused_bicgstab=True, **kw)]
        xds = [api.host_dense(ex, x) for x in xs]
        times = [[], []]
        for rep in range(args.reps + 1):  # the first round warms both paths (plan, graph, modules)
            for k in (0, 1):
                with torch.cuda.stream(ex.stream):
                    xs[k].zero_()
                ex.synchronize()
                t0 = time.perf_counter()
                solvers[k].apply(bd, xds[k])
                ex.synchronize()
                if rep:
                    times[k].append(time.perf_counter() - t0)
        assert not solvers[0].used_fused and solvers[1].used_fused
        one = api.host_dense(ex, torch.ones(1, dtype=va.dtype, device=dev))
        neg = api.host_dense(ex, -torch.ones(1, dtype=va.dtype, device=dev))
        b_matrix = nnz * (V + I) + (n + 1) * I
        for k, name in ((0, "loop "), (1, "fused")):
            with torch.cuda.stream(ex.stream):
                r = b.clone()
            rd = api.host_dense(ex, r)
            api._hcheck(api._host().gkob_apply4(A.h, neg.h, xds[k].h, one.h, rd.h))
            ex.synchronize()
            res = (r.double().norm() / b.double().norm()).item()
            it = solvers[k].num_iterations
            t = sorted(times[k])[len(times[k]) // 2]
            model = 2 * b_matrix + (36 if k == 0 else 25) * n * V
            print("%-22s %s n=%-9d nnz=%-10d it=%-4d status=0x%02x  %.3f ms/it (median of %d, min %.3f max %.3f)  "
                  "true rel res %.2e  model %.1f MB/it -> %.0f GB/s%s" %
                  (label, name, n, nnz, it, solvers[k].stop_status, 1e3 * t / max(it, 1), len(times[k]),
                   1e3 * min(times[k]) / max(it, 1), 1e3 * max(times[k]) / max(it, 1), res, model / 1e6,
                   model * max(it, 1) / t / 1e9, note))
        t_loop = sorted(times[0])[len(times[0]) // 2] / max(solvers[0].num_iterations, 1)
        t_fused = sorted(times[1])[len(times[1]) // 2] / max(solvers[1].num_iterations, 1)
        print("%-22s time per iteration, loop / fused = %.2f" % (label, t_loop / t_fused))

    with torch.cuda.stream(ex.stream):
        small = upwind3d(torch, args.small, dev)
        big = upwind3d(torch, args.grid, dev)
    problem("upwind3d %d^3 f64" % args.small, *small, 1e-8, "  [launch / host-sync bound size]")
    del small
    problem("upwind3d %d^3 f64" % args.grid, *big, 1e-8)
    del big
    with torch.cuda.stream(ex.stream):
        rp, ci, va = W.build("cfg4", xp="torch", device=dev, n=args.cfg4_rows)
    problem("cfg4 random f32", rp, ci, va, 1e-5)


if __name__ == "__main__":
    main()
