"""MINRES on one GPU for k right-hand sides of one system: (a) k one-column fused solves
(solver::Minres::with_fused), (b) the kernel-by-kernel loop on the n x k Dense, (c) the fused iteration
for several right-hand sides (with_fused_multi_rhs), alternated in one process after one warm-up round.

Problem: the --grid^3 indefinite Laplacian of DESIGN.md section 4.9 (7-point Laplacian plus
diag(uniform(0, 0.5)) - sigma I, symmetric indefinite with a positive diagonal), fp64, int32 indices,
scalar Jacobi, the Iteration criterion only (--iters), so that all three paths do the same work.  Per k
and path: wall time per iteration and right-hand side (host clock around the solve, which ends in a
synchronise; median of --reps), launches per iteration, the largest relative difference of x from path
(b), and the byte model of DESIGN.md section 4.10 over the time:
  (a) k (B_matrix + 19 n V)   (b) B_matrix + 25 n k V + n V   (c) B_matrix + 17 n k V + 2 n V
Then the three launches of (c) at --kernel-k, timed with CUDA events over back-to-back launches.  Needs
a GPU; there is no fallback.

  python scripts/minres_multi_rhs_timing.py [--grid 200] [--ks 2,4,8,16] [--iters 200] [--reps 3]
"""
import argparse
import ctypes
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

from minres_fused_timing import card, indefinite3d  # noqa: E402


def kernel_times(torch, ex, rp, ci, va, k, reps):
    """ms per launch of spmv_sub_mdot, lanczos and update at k columns, each launched `reps` times back
    to back between two CUDA events; no criterion is configured, so no launch turns into a no-op"""
    from ginkgo_b200 import _lib
    lib = _lib.lib()
    n, nnz = rp.numel() - 1, va.numel()
    it = "i32" if ci.element_size() == 4 else "i64"
    ctx = ctypes.c_void_p()
    assert lib.b200_ctx_create(0, ex.stream.cuda_stream, ctypes.byref(ctx)) == 0
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    dev = ex.device
    with torch.cuda.stream(ex.stream):
        x, p0, p1, z, q, v = (torch.empty(n * k, dtype=torch.float64, device=dev).uniform_(-1, 1) for _ in range(6))
        d = torch.empty(n, dtype=torch.float64, device=dev).uniform_(0.1, 1)
        sc = torch.zeros(16, k, dtype=torch.float64, device=dev)
        status = torch.zeros(k, dtype=torch.uint8, device=dev)
        ctl = torch.tensor([0, 0, -1, 0, 1, 0, 0, 0], dtype=torch.int32, device=dev)
        work = torch.zeros(lib.b200_minres_mrhs_work_size_f64(ctx, k), dtype=torch.float64, device=dev)

    def reset():
        with torch.cuda.stream(ex.stream):
            sc[0:4] = torch.tensor([0.5, 0.7, 0.3, 0.2], dtype=torch.float64, device=dev)[:, None]
            sc[9:13] = torch.tensor([0.6, 0.8, 0.8, 0.6], dtype=torch.float64, device=dev)[:, None]
            sc[6] = 1
            for t in (x, p0, p1, z, q, v):
                t.uniform_(-1, 1)

    sub = getattr(lib, "b200_csr_spmv_sub_mdot_f64_" + it)
    b_matrix = nnz * (8 + ci.element_size()) + (n + 1) * rp.element_size()
    calls = [
        ("spmv_sub_mdot", lambda: sub(ctx, n, n, nnz, P(rp), P(ci), P(va), P(z), k, P(v), P(sc), P(work), P(ctl)),
         b_matrix + 3 * n * k * 8),
        ("lanczos", lambda: lib.b200_minres_mrhs_lanczos_f64(ctx, n, k, P(v), P(q), P(d), P(sc), P(status), P(ctl),
                                                             P(work)), (3 * n * k + n) * 8),
        ("update", lambda: lib.b200_minres_mrhs_update_f64(ctx, n, k, P(x), P(p0), P(p1), P(z), P(q), P(v), P(d),
                                                           P(sc), P(status), P(ctl)), (11 * n * k + n) * 8),
    ]
    total = 0.0
    print("CUDA events, k = %d, n = %d, %d launches each:" % (k, n, reps))
    print("| launch | ms/launch | model MB | GB/s |")
    print("|---|---|---|---|")
    for name, fn, model in calls:
        reset()
        assert fn() == 0  # warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ex.stream)
        for _ in range(reps):
            fn()
        e1.record(ex.stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / reps
        total += ms
        print("| %s | %.3f | %.1f | %.0f |" % (name, ms, model / 1e6, model / ms / 1e6))
    assert ctl[0].item() == 0, "a kernel turned into a no-op"
    print("kernel sum of one iteration at k = %d: %.3f ms (%.3f ms per right-hand side)" % (k, total, total / k))
    lib.b200_ctx_destroy(ctx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--sigma", type=float, default=0.3)
    ap.add_argument("--ks", default="2,4,8,16")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-k", type=int, default=8)
    ap.add_argument("--kernel-reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("minres_multi_rhs_timing.py measures on a GPU and none is visible")
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())
    with torch.cuda.stream(ex.stream):
        rp, ci, va = indefinite3d(torch, args.grid, args.sigma, dev)
    n, nnz = rp.numel() - 1, va.numel()
    V, I = va.element_size(), ci.element_size()
    b_matrix = nnz * (V + I) + (n + 1) * I
    A = api.host_csr(ex, (n, n), va, ci, rp)
    kw = dict(precond_max_bs=1, max_iters=args.iters, res_kind=0)
    loop = api.HostSolver(ex, "minres", A, **kw)
    multi = api.HostSolver(ex, "minres", A, fused_minres_multi_rhs=True, **kw)
    print("indef3d %d^3 f64 i32, n=%d nnz=%d, scalar Jacobi, Iteration(%d) only" % (args.grid, n, nnz, args.iters))
    print("| k | path | ms/it/rhs (median of %d) | min | max | launches/it | model GB/it | GB/s | max rel diff to (b) |"
          % args.reps)
    print("|---|---|---|---|---|---|---|---|---|")
    for k in [int(s) for s in args.ks.split(",")]:
        with torch.cuda.stream(ex.stream):
            gen = torch.Generator(device=dev).manual_seed(k)
            b = torch.empty(n, k, dtype=torch.float64, device=dev).uniform_(-1, 1, generator=gen)
            cols = [b[:, j:j + 1].contiguous() for j in range(k)]
            xa = [torch.zeros(n, 1, dtype=torch.float64, device=dev) for _ in range(k)]
            xb, xc = torch.zeros(n, k, dtype=torch.float64, device=dev), torch.zeros(n, k, dtype=torch.float64,
                                                                                      device=dev)
        bd, bcols = api.host_dense(ex, b), [api.host_dense(ex, c) for c in cols]
        # one solver per column: a fused graph bakes in x, so one solver for all k would recapture
        one_cols = [api.HostSolver(ex, "minres", A, fused_minres=True, **kw) for _ in range(k)]
        xad, xbd, xcd = [api.host_dense(ex, t) for t in xa], api.host_dense(ex, xb), api.host_dense(ex, xc)

        def run_a():
            for j in range(k):
                one_cols[j].apply(bcols[j], xad[j])

        paths = [("(a) k one-column fused", run_a, xa),
                 ("(b) loop on n x k", lambda: loop.apply(bd, xbd), [xb]),
                 ("(c) fused n x k", lambda: multi.apply(bd, xcd), [xc])]
        times, launches = [[] for _ in paths], [0] * len(paths)
        for rep in range(args.reps + 1):  # the first round warms every path (graphs, modules)
            for i, (_, fn, xs) in enumerate(paths):
                with torch.cuda.stream(ex.stream):
                    for t in xs:
                        t.zero_()
                ex.synchronize()
                l0 = ex.launch_count()
                t0 = time.perf_counter()
                fn()
                ex.synchronize()
                if rep:
                    times[i].append(time.perf_counter() - t0)
                    launches[i] = ex.launch_count() - l0
        assert all(s.used_fused and s.num_iterations == args.iters for s in one_cols)
        assert not loop.used_fused and multi.used_fused
        assert loop.num_iterations == multi.num_iterations == args.iters
        ref = xb.double()
        xa_all = torch.cat(xa, dim=1)
        models = [k * (b_matrix + 19 * n * V), b_matrix + 25 * n * k * V + n * V, b_matrix + 17 * n * k * V + 2 * n * V]
        meds = []
        for i, (name, _, _) in enumerate(paths):
            x = xa_all if i == 0 else (xb if i == 1 else xc)
            diff = ((x.double() - ref).norm(dim=0) / ref.norm(dim=0)).max().item()
            ts = sorted(times[i])
            per = 1e3 / (args.iters * k)
            med = ts[len(ts) // 2]
            meds.append(med)
            print("| %d | %s | %.4f | %.4f | %.4f | %.1f | %.2f | %.0f | %.1e |" %
                  (k, name, med * per, ts[0] * per, ts[-1] * per, launches[i] / args.iters, models[i] / 1e9,
                   models[i] * args.iters / med / 1e9, diff))
        print("k = %d: (c) is %.2fx faster than (a) and %.2fx faster than (b) per right-hand side" %
              (k, meds[0] / meds[2], meds[1] / meds[2]))
        del b, cols, xa, xb, xc, bd, bcols, xad, xbd, xcd, paths, one_cols
        torch.cuda.empty_cache()
    kernel_times(torch, ex, rp, ci, va, args.kernel_k, args.kernel_reps)


if __name__ == "__main__":
    main()
