"""MINRES on one GPU: the kernel-by-kernel loop against the fused device-resident iteration
(solver::Minres::with_fused), alternated in one process after one warm-up solve each.

Problem: the 3-D 7-point Laplacian plus diag(uniform(0, 0.5)) - sigma I, symmetric indefinite with a
positive diagonal (so scalar Jacobi is SPD), fp64, scalar Jacobi.
  1. --grid^3: 200 iterations with the Iteration criterion only, so both paths do the same work;
  2. --small^3: ImplicitResidualNorm to 1e-8 (and at most 2000 iterations).
Per problem and path: iterations, stopping status, wall time per iteration (host clock around an
apply that ends in a synchronise, median of --reps), host launches per iteration, the true relative
residual, and the byte model of DESIGN.md section 4.9 (B_matrix + 26 n V for the loop, B_matrix + 19 n V
fused) over the time.  Then each of the three fused launches at --grid^3, timed with CUDA events over
back-to-back launches.  Needs a GPU; there is no fallback.

  python scripts/minres_fused_timing.py [--grid 200] [--small 40] [--sigma 0.3] [--reps 3]
"""
import argparse
import ctypes
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


def indefinite3d(torch, g, sigma, dev, seed=4):
    import workloads as W
    rp, ci, va = W.laplace(g, 3, xp="torch", device=dev)
    n = g ** 3
    rows = torch.repeat_interleave(torch.arange(n, device=dev), (rp[1:] - rp[:-1]).long())
    gen = torch.Generator(device=dev).manual_seed(seed)
    shift = torch.rand(n, generator=gen, dtype=va.dtype, device=dev) * 0.5 - sigma
    diag = ci.long() == rows
    va[diag] += shift
    return rp, ci, va


def kernel_times(torch, ex, rp, ci, va, reps):
    """ms per launch of spmv_sub_dot, lanczos and update, each launched `reps` times back to back
    between two CUDA events; no criterion is configured, so no launch turns into a no-op"""
    from ginkgo_b200 import _lib
    lib = _lib.lib()
    n, nnz = rp.numel() - 1, va.numel()
    it = "i32" if ci.element_size() == 4 else "i64"
    ctx = ctypes.c_void_p()
    assert lib.b200_ctx_create(0, ex.stream.cuda_stream, ctypes.byref(ctx)) == 0
    plan = ctypes.c_void_p()
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    assert getattr(lib, "b200_csr_plan_create_f64_" + it)(ctx, n, nnz, P(rp), ctypes.byref(plan)) == 0
    assert getattr(lib, "b200_csr_plan_tune_f64_" + it)(ctx, plan, n, n, nnz, P(rp), P(ci), P(va)) == 0
    dev = ex.device
    with torch.cuda.stream(ex.stream):
        vecs = [torch.empty(n, dtype=torch.float64, device=dev).uniform_(-1, 1) for _ in range(7)]
        x, p0, p1, z, q, v, d = vecs
        d.abs_().add_(0.1)
        sc = torch.zeros(16, dtype=torch.float64, device=dev)
        sc[0:4] = torch.tensor([0.5, 0.7, 0.3, 0.2])  # alpha, beta, gamma, delta: no zero divisor
        sc[9:13] = torch.tensor([0.6, 0.8, 0.8, 0.6])
        sc[6] = 1
        ctl = torch.tensor([0, 0, -1, 0, 1, 0, 0, 0], dtype=torch.int32, device=dev)
        work = torch.zeros(lib.b200_minres_fused_work_size_f64(ctx), dtype=torch.float64, device=dev)
    sub_dot = getattr(lib, "b200_csr_spmv_sub_dot_f64_" + it)
    b_matrix = nnz * (8 + ci.element_size()) + (n + 1) * rp.element_size()
    calls = [
        ("spmv_sub_dot", lambda: sub_dot(ctx, plan, n, n, nnz, P(rp), P(ci), P(va), P(z), P(v), P(sc), P(work),
                                         P(ctl)), b_matrix + 3 * n * 8),
        ("lanczos", lambda: lib.b200_minres_fused_lanczos_f64(ctx, n, P(v), P(q), P(d), P(sc), P(ctl), P(work)),
         4 * n * 8),
        ("update", lambda: lib.b200_minres_fused_update_f64(ctx, n, P(x), P(p0), P(p1), P(z), P(q), P(v), P(d),
                                                            P(sc), P(ctl)), 12 * n * 8),
    ]
    total = 0.0
    for name, fn, model in calls:
        with torch.cuda.stream(ex.stream):
            sc[0:4] = torch.tensor([0.5, 0.7, 0.3, 0.2])
            sc[6] = 1
            for t in (x, p0, p1, z, q, v):
                t.uniform_(-1, 1)
        assert fn() == 0  # warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ex.stream)
        for _ in range(reps):
            fn()
        e1.record(ex.stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / reps
        total += ms
        print("kernel %-13s n=%-9d %.3f ms/launch  model %.1f MB -> %.0f GB/s" %
              (name, n, ms, model / 1e6, model / ms / 1e6))
    assert ctl[0].item() == 0, "a kernel turned into a no-op"
    print("kernel sum of one fused iteration: %.3f ms (3 launches)" % total)
    lib.b200_csr_plan_destroy(plan)
    lib.b200_ctx_destroy(ctx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--small", type=int, default=40)
    ap.add_argument("--sigma", type=float, default=0.3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("minres_fused_timing.py measures on a GPU and none is visible")
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())

    def problem(label, rp, ci, va, kw, note=""):
        n, nnz = rp.numel() - 1, va.numel()
        V, I = va.element_size(), ci.element_size()
        with torch.cuda.stream(ex.stream):
            b = torch.ones(n, dtype=va.dtype, device=dev)
            xs = [torch.zeros(n, dtype=va.dtype, device=dev) for _ in range(2)]
        A = api.host_csr(ex, (n, n), va, ci, rp)
        bd = api.host_dense(ex, b)
        solvers = [api.HostSolver(ex, "minres", A, precond_max_bs=1, **kw),
                   api.HostSolver(ex, "minres", A, precond_max_bs=1, fused_minres=True, **kw)]
        xds = [api.host_dense(ex, x) for x in xs]
        times, launches = [[], []], [0, 0]
        for rep in range(args.reps + 1):  # the first round warms both paths (plan, graph, modules)
            for k in (0, 1):
                with torch.cuda.stream(ex.stream):
                    xs[k].zero_()
                ex.synchronize()
                l0 = ex.launch_count()
                t0 = time.perf_counter()
                solvers[k].apply(bd, xds[k])
                ex.synchronize()
                if rep:
                    times[k].append(time.perf_counter() - t0)
                    launches[k] = ex.launch_count() - l0
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
            model = b_matrix + (26 if k == 0 else 19) * n * V
            print("%-20s %s n=%-9d nnz=%-10d it=%-4d status=0x%02x  %.3f ms/it (median of %d, min %.3f max %.3f)  "
                  "%.1f launches/it  true rel res %.2e  model %.1f MB/it -> %.0f GB/s%s" %
                  (label, name, n, nnz, it, solvers[k].stop_status, 1e3 * t / max(it, 1), len(times[k]),
                   1e3 * min(times[k]) / max(it, 1), 1e3 * max(times[k]) / max(it, 1), launches[k] / max(it, 1),
                   res, model / 1e6, model * max(it, 1) / t / 1e9, note))
        t_loop = sorted(times[0])[len(times[0]) // 2] / max(solvers[0].num_iterations, 1)
        t_fused = sorted(times[1])[len(times[1]) // 2] / max(solvers[1].num_iterations, 1)
        print("%-20s time per iteration, loop / fused = %.2f" % (label, t_loop / t_fused))

    with torch.cuda.stream(ex.stream):
        big = indefinite3d(torch, args.grid, args.sigma, dev)
    problem("indef3d %d^3 f64" % args.grid, *big, dict(max_iters=200, res_kind=0), "  [Iteration only]")
    kernel_times(torch, ex, *big, args.kernel_reps)
    del big
    with torch.cuda.stream(ex.stream):
        small = indefinite3d(torch, args.small, args.sigma, dev)
    problem("indef3d %d^3 f64" % args.small, *small, dict(max_iters=2000, res_kind=2, reduction=1e-8),
            "  [ImplicitResidualNorm 1e-8]")


if __name__ == "__main__":
    main()
