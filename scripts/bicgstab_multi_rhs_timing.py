"""BiCGStab for k right-hand sides of one system on one GPU, three ways, alternated in one process after
one warm-up solve each:
  (a) k one-column fused solves (solver::Bicgstab with_fused, once per column),
  (b) the kernel-by-kernel loop on the n x k Dense,
  (c) the fused path for several right-hand sides (with_fused_multi_rhs: one matrix pass per SpMV).

Problems: upwind convection-diffusion 200^3 in fp64 with scalar Jacobi (bicgstab_fused_timing.upwind3d;
columns of b from workloads.vector on distinct streams), k in --ks, once with a fixed --iters iterations
(Iteration only) and once to 1e-8 (rhs_norm); then cfg4's scattered non-symmetric dominant random matrix
of --rand-rows rows, k in --rand-ks, to 1e-8.  Per run and path: ms per iteration and per iteration and
right-hand side (median of --reps solves, host clock around work that ends in a synchronise), the byte
model over that time, host-issued launches per iteration, the true relative residual of every column
and the stop statuses.  Byte models per iteration of the n x k system (B = matrix bytes, V = value
bytes, scalar Jacobi): (a) k (2 B + 25 n V), (b) 2 B + 36 n k V, (c) 2 B + 23 n k V + 2 n V.
Then the time of each of the five launches of (c) at k = --kernel-k on upwind --grid^3, from CUDA events
around --kernel-reps back-to-back launches of that kernel.  Needs a GPU.

  python scripts/bicgstab_multi_rhs_timing.py [--grid 200] [--ks 2,4,8,16] [--iters 200] [--rand-rows 2000000]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bicgstab_fused_timing import card, upwind3d  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--ks", default="2,4,8,16")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rand-rows", type=int, default=2_000_000)
    ap.add_argument("--rand-ks", default="4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-k", type=int, default=8)
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bicgstab_multi_rhs_timing.py measures on a GPU and none is visible")
    import workloads as W
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())

    def timed(fn):
        ex.synchronize()
        l0 = ex.launch_count()
        t0 = time.perf_counter()
        fn()
        ex.synchronize()
        return time.perf_counter() - t0, ex.launch_count() - l0

    def true_res(A, b, x):
        """|| b_j - A x_j || / || b_j || per column"""
        k = b.shape[1]
        one = api.host_dense(ex, torch.ones(1, dtype=b.dtype, device=dev))
        neg = api.host_dense(ex, -torch.ones(1, dtype=b.dtype, device=dev))
        with torch.cuda.stream(ex.stream):
            r = b.clone()
        xd, rd = api.host_dense(ex, x), api.host_dense(ex, r)  # the views must outlive the call
        api._hcheck(api._host().gkob_apply4(A.h, neg.h, xd.h, one.h, rd.h))
        ex.synchronize()
        rn = r.double().norm(dim=0) / b.double().norm(dim=0)
        del r
        return [float(v) for v in rn.cpu()]

    def run(label, A, n, nnz, V, I, k, b, crit, pre=1):
        b_matrix = nnz * (V + I) + (n + 1) * I
        kw = dict(precond_max_bs=pre, **crit)
        with torch.cuda.stream(ex.stream):
            cols = [b[:, j].contiguous().reshape(n, 1) for j in range(k)]
            xs1 = [torch.zeros(n, 1, dtype=b.dtype, device=dev) for _ in range(k)]
            xl = torch.zeros(n, k, dtype=b.dtype, device=dev)
            xf = torch.zeros(n, k, dtype=b.dtype, device=dev)
        s1 = api.HostSolver(ex, "bicgstab", A, fused_bicgstab=True, **kw)
        sl = api.HostSolver(ex, "bicgstab", A, **kw)
        sf = api.HostSolver(ex, "bicgstab", A, fused_bicgstab_multi_rhs=True, **kw)
        bd, bcols = api.host_dense(ex, b), [api.host_dense(ex, c) for c in cols]
        x1d, xld, xfd = [api.host_dense(ex, x) for x in xs1], api.host_dense(ex, xl), api.host_dense(ex, xf)
        iters1, st1 = [0] * k, [0] * k

        def one_column():
            for j in range(k):
                xs1[j].zero_()
                s1.apply(bcols[j], x1d[j])
                iters1[j], st1[j] = s1.num_iterations, s1.stop_status

        def loop():
            xl.zero_()
            sl.apply(bd, xld)

        def fused():
            xf.zero_()
            sf.apply(bd, xfd)

        paths = [("(a) k x one-column", one_column), ("(b) loop n x k", loop), ("(c) fused n x k", fused)]
        for _, fn in paths:  # warm-up; the fused paths capture their graphs here
            with torch.cuda.stream(ex.stream):
                timed(fn)
        times, launches = [[] for _ in paths], [0] * len(paths)
        for _ in range(args.reps):
            for p, (_, fn) in enumerate(paths):
                with torch.cuda.stream(ex.stream):
                    t, nl = timed(fn)
                times[p].append(t)
                launches[p] = nl
        assert s1.used_fused and not sl.used_fused and sf.used_fused
        with torch.cuda.stream(ex.stream):
            x1 = torch.cat(xs1, dim=1)
        res = [true_res(A, b, x) for x in (x1, xl, xf)]
        its = [sum(iters1), sl.num_iterations, sf.num_iterations]  # (a): iterations summed over its k solves
        stats = [st1, sl.stop_statuses, sf.stop_statuses]
        models = [(2 * b_matrix + 25 * n * V) * its[0], 2 * b_matrix + 36 * n * k * V,
                  2 * b_matrix + 23 * n * k * V + 2 * n * V]
        per_rhs = []
        for p, (name, _) in enumerate(paths):
            t = sorted(times[p])[len(times[p]) // 2]
            it = max(its[p], 1)
            # ms per iteration of the n x k system: (a) counts k one-column iterations as one
            it_sys = it / k if p == 0 else it
            model = models[p] * (1 if p == 0 else it)
            per_rhs.append(t / it_sys / k)
            print("%-28s k=%-2d %-20s it=%-5s %.3f ms/it  %.4f ms/(it*rhs)  (median of %d, min %.3f max %.3f ms/it)  "
                  "model %.0f MB/it -> %.0f GB/s  %.1f launches/it  status %s  true rel res %s" %
                  (label, k, name, ("%d" % its[p]) if p else "%d/%d" % (its[p], k), 1e3 * t / it_sys,
                   1e3 * t / it_sys / k, len(times[p]), 1e3 * min(times[p]) / it_sys, 1e3 * max(times[p]) / it_sys,
                   model / it_sys / 1e6, model / t / 1e9, launches[p] / it_sys,
                   ",".join("%02x" % s for s in stats[p]), ",".join("%.2e" % v for v in res[p])))
        print("%-28s k=%-2d per right-hand side and iteration: one-column / fused = %.2f, loop / fused = %.2f" %
              (label, k, per_rhs[0] / per_rhs[2], per_rhs[1] / per_rhs[2]))
        del xs1, xl, xf, cols, x1

    with torch.cuda.stream(ex.stream):
        rp, ci, va = upwind3d(torch, args.grid, dev)
    n, nnz = rp.numel() - 1, va.numel()
    A = api.host_csr(ex, (n, n), va, ci, rp)
    label = "upwind %d^3 f64 jac" % args.grid
    for k in [int(s) for s in args.ks.split(",")]:
        with torch.cuda.stream(ex.stream):
            b = torch.stack([W.vector(n, stream=11 + j, xp="torch", device=dev) for j in range(k)], dim=1)
            b = b.to(torch.float64).contiguous()
        run(label + " fixed", A, n, nnz, 8, 4, k, b, dict(max_iters=args.iters, res_kind=0))
        run(label + " 1e-8", A, n, nnz, 8, 4, k, b, dict(max_iters=5000, reduction=1e-8))
        del b
    kernel_times(torch, ex, rp, ci, va, args.kernel_k, args.kernel_reps, label)
    del A, rp, ci, va

    with torch.cuda.stream(ex.stream):
        rp, ci, va = W.build("cfg4", xp="torch", device=dev, n=args.rand_rows)
        va = va.to(torch.float64)
    m = rp.numel() - 1
    A = api.host_csr(ex, (m, m), va, ci, rp)
    label = "cfg4 %.1fM f64 jac" % (m / 1e6)
    for k in [int(s) for s in args.rand_ks.split(",")]:
        with torch.cuda.stream(ex.stream):
            b = torch.stack([W.vector(m, stream=11 + j, xp="torch", device=dev) for j in range(k)], dim=1)
            b = b.to(torch.float64).contiguous()
        run(label + " 1e-8", A, m, va.numel(), 8, ci.element_size(), k, b, dict(max_iters=5000, reduction=1e-8))
        del b


def kernel_times(torch, ex, rp, ci, va, k, reps, label):
    """ms per launch of each of the five kernels of one iteration of (c), each launched `reps` times
    back to back between two CUDA events on the solver's stream; Iteration only with no limit, so no
    launch turns into a no-op"""
    import ctypes
    from ginkgo_b200 import _lib
    lib = _lib.lib()
    n = rp.numel() - 1
    ctx = ctypes.c_void_p()
    assert lib.b200_ctx_create(0, ex.stream.cuda_stream, ctypes.byref(ctx)) == 0
    dev = ex.device
    with torch.cuda.stream(ex.stream):
        vec = {nm: torch.zeros(n, k, dtype=torch.float64, device=dev) for nm in ("x", "r", "rr", "p", "v", "y", "s", "t", "z")}
        vec["r"].uniform_(-1, 1)
        diag = torch.ones(n, dtype=torch.float64, device=dev)
        sc = torch.zeros(10 * k, dtype=torch.float64, device=dev)
        sc[4 * k:5 * k] = 1
        status = torch.zeros(k, dtype=torch.uint8, device=dev)
        ctl = torch.zeros(8, dtype=torch.int32, device=dev)
        work = torch.zeros(lib.b200_bicgstab_mrhs_work_size_f64(ctx, k), dtype=torch.float64, device=dev)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    V = {nm: P(t) for nm, t in vec.items()}
    d, s_, st, c, w = P(diag), P(sc), P(status), P(ctl), P(work)
    A = (P(rp), P(ci), P(va))
    assert lib.b200_bicgstab_mrhs_init_f64(ctx, n, k, V["r"], V["rr"], V["p"], V["v"], V["y"], V["s"], V["t"], V["z"],
                                           s_, st, c, w, 1 << 40, 0, 1, 2, ctypes.c_double(0.0)) == 0
    mdot2 = getattr(lib, "b200_csr_spmv_mdot2_f64_" + ("i32" if ci.element_size() == 4 else "i64"))
    sc_at = lambda j: ctypes.c_void_p(sc.data_ptr() + 8 * j * k)  # noqa: E731
    calls = [
        ("step_p", lambda: lib.b200_bicgstab_mrhs_step_p_f64(ctx, n, k, V["p"], V["r"], V["v"], V["y"], d, s_, st, c)),
        ("spmv_mdot2 (v = A y)", lambda: mdot2(ctx, n, n, va.numel(), *A, V["y"], k, V["v"],
                                                                          V["rr"], sc_at(2), None, w, c)),
        ("step_s", lambda: lib.b200_bicgstab_mrhs_step_s_f64(ctx, n, k, V["r"], V["v"], V["s"], V["z"], d, s_, st, c, w)),
        ("spmv_mdot2 (t = A z)", lambda: mdot2(ctx, n, n, va.numel(), *A, V["z"], k, V["t"],
                                                                          V["s"], sc_at(8), sc_at(2), w, c)),
        ("step_xr", lambda: lib.b200_bicgstab_mrhs_step_xr_f64(ctx, n, k, V["x"], V["r"], V["s"], V["t"], V["y"], V["z"],
                                                                V["rr"], s_, st, c, w)),
    ]
    b_matrix = va.numel() * (8 + ci.element_size()) + (n + 1) * rp.element_size()
    bytes_of = {"step_p": (5 * k + 1) * n * 8, "step_s": (4 * k + 1) * n * 8, "step_xr": 8 * k * n * 8}
    total = 0.0
    for name, fn in calls:
        assert fn() == 0  # warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ex.stream)
        for _ in range(reps):
            fn()
        e1.record(ex.stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / reps
        total += ms
        model = bytes_of.get(name, b_matrix + 3 * k * n * 8)
        print("%-28s k=%-2d kernel %-22s %.3f ms/launch  model %.0f MB -> %.0f GB/s" %
              (label, k, name, ms, model / 1e6, model / ms / 1e6))
    assert ctl[0].item() == 0, "a kernel turned into a no-op"
    print("%-28s k=%-2d five launches: %.3f ms" % (label, k, total))
    lib.b200_ctx_destroy(ctx)


if __name__ == "__main__":
    main()
