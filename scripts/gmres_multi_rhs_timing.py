"""GMRES for k right-hand sides of one system on one GPU, three ways, alternated in one process after one
warm-up solve each:
  (a) k one-column fused solves (solver::Gmres with_fused, once per column),
  (b) the kernel-by-kernel loop on the n x k Dense,
  (c) the fused path for several right-hand sides (with_fused_multi_rhs: one matrix pass per SpMV).

GMRES(--kd) in fp64 with scalar Jacobi, MGS and CGS, a fixed --iters iterations (Iteration only, so the
three paths do the same work; 2 x kd iterations give a mean Krylov index of (kd - 1) / 2):
upwind convection-diffusion --grid^3 (bicgstab_fused_timing.upwind3d) for k in --ks, the same at
--grid16^3 for k = 16 (where the bases of (b) and (c) both fit), and cfg4's scattered non-symmetric
dominant random matrix of --rand-rows rows for k in --rand-ks.  Per run and path: ms per iteration and per
iteration and right-hand side (median of --reps solves, host clock around work that ends in a
synchronise), the byte model over that time, and host-issued launches per iteration.  Byte models per
iteration at Krylov index j (B = matrix bytes, V = value bytes, scalar Jacobi), MGS:
(a) k (B + (4j + 10) n V), (b) B + (5j + 12) n k V + n V, (c) B + (4j + 9) n k V + n V; CGS:
(a) k (B + (2j + 11) n V), (b) B + (4j + 12) n k V + n V, (c) B + (2j + 10) n k V + n V.
Then the time of each launch of (c) at k = --kernel-k and Krylov index --kernel-j on upwind --grid^3,
from CUDA events around --kernel-reps back-to-back launches of that kernel.  Needs a GPU.

  python scripts/gmres_multi_rhs_timing.py [--grid 200] [--ks 2,4,8] [--grid16 150] [--rand-rows 2000000]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bicgstab_fused_timing import card, upwind3d  # noqa: E402

ORTHOS = {"mgs": 0, "cgs": 1}


def model_bytes(ortho, path, j, n, k, b_matrix, V=8):
    """bytes of one iteration at Krylov index j (see the module docstring)"""
    if ortho == "mgs":
        per = {"a": k * (b_matrix + (4 * j + 10) * n * V), "b": b_matrix + (5 * j + 12) * n * k * V + n * V,
               "c": b_matrix + (4 * j + 9) * n * k * V + n * V}
    else:
        per = {"a": k * (b_matrix + (2 * j + 11) * n * V), "b": b_matrix + (4 * j + 12) * n * k * V + n * V,
               "c": b_matrix + (2 * j + 10) * n * k * V + n * V}
    return per[path]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--ks", default="2,4,8")
    ap.add_argument("--grid16", type=int, default=150)
    ap.add_argument("--rand-rows", type=int, default=2_000_000)
    ap.add_argument("--rand-ks", default="2,4,8")
    ap.add_argument("--kd", type=int, default=30)
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-k", type=int, default=8)
    ap.add_argument("--kernel-j", type=int, default=14)
    ap.add_argument("--kernel-reps", type=int, default=30)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("gmres_multi_rhs_timing.py measures on a GPU and none is visible")
    import workloads as W
    from ginkgo_b200 import api
    ex = api.HostExecutor(0)
    dev = ex.device
    print("card (name, power limit, max SM clock):", card())
    kd, iters = args.kd, args.iters

    def timed(fn):
        ex.synchronize()
        l0 = ex.launch_count()
        t0 = time.perf_counter()
        fn()
        ex.synchronize()
        return time.perf_counter() - t0, ex.launch_count() - l0

    def run(label, A, n, nnz, I, k, b, ortho):
        b_matrix = nnz * (8 + I) + (n + 1) * I
        kw = dict(precond_max_bs=1, max_iters=iters, res_kind=0, krylov_dim=kd, ortho=ORTHOS[ortho])
        with torch.cuda.stream(ex.stream):
            cols = [b[:, j].contiguous().reshape(n, 1) for j in range(k)]
            xs1 = [torch.zeros(n, 1, dtype=b.dtype, device=dev) for _ in range(k)]
            xl = torch.zeros(n, k, dtype=b.dtype, device=dev)
            xf = torch.zeros(n, k, dtype=b.dtype, device=dev)
        s1 = api.HostSolver(ex, "gmres", A, fused_gmres=True, **kw)
        sl = api.HostSolver(ex, "gmres", A, **kw)
        sf = api.HostSolver(ex, "gmres", A, fused_gmres_multi_rhs=True, **kw)
        bd, bcols = api.host_dense(ex, b), [api.host_dense(ex, c) for c in cols]
        x1d, xld, xfd = [api.host_dense(ex, x) for x in xs1], api.host_dense(ex, xl), api.host_dense(ex, xf)

        def one_column():
            for j in range(k):
                xs1[j].zero_()
                s1.apply(bcols[j], x1d[j])

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
        assert s1.num_iterations == sl.num_iterations == sf.num_iterations == iters
        js = [it % kd for it in range(iters)]
        per_rhs = []
        for p, (name, _) in enumerate(paths):
            t = sorted(times[p])[len(times[p]) // 2]
            model = sum(model_bytes(ortho, "abc"[p], j, n, k, b_matrix) for j in js)
            per_rhs.append(t / iters / k)
            print("%-26s %-4s k=%-2d %-20s %.3f ms/it  %.4f ms/(it*rhs)  (median of %d, min %.3f max %.3f)  "
                  "model %.0f MB/it -> %.0f GB/s  %.1f launches/it" %
                  (label, ortho, k, name, 1e3 * t / iters, 1e3 * t / iters / k, len(times[p]),
                   1e3 * min(times[p]) / iters, 1e3 * max(times[p]) / iters, model / iters / 1e6, model / t / 1e9,
                   launches[p] / iters))
        print("%-26s %-4s k=%-2d per right-hand side and iteration: one-column / fused = %.2f, loop / fused = %.2f" %
              (label, ortho, k, per_rhs[0] / per_rhs[2], per_rhs[1] / per_rhs[2]))
        sys.stdout.flush()
        del xs1, xl, xf, cols, s1, sl, sf

    def cases(label, A, n, nnz, I, ks):
        for k in ks:
            with torch.cuda.stream(ex.stream):
                b = torch.stack([W.vector(n, stream=11 + j, xp="torch", device=dev) for j in range(k)], dim=1)
                b = b.to(torch.float64).contiguous()
            for ortho in ORTHOS:
                run(label, A, n, nnz, I, k, b, ortho)
            del b
            torch.cuda.empty_cache()

    with torch.cuda.stream(ex.stream):
        rp, ci, va = upwind3d(torch, args.grid, dev)
    n, nnz = rp.numel() - 1, va.numel()
    A = api.host_csr(ex, (n, n), va, ci, rp)
    label = "upwind %d^3 f64 jac" % args.grid
    cases(label, A, n, nnz, 4, [int(s) for s in args.ks.split(",")])
    kernel_times(torch, ex, rp, ci, va, args.kernel_k, args.kernel_j, kd, args.kernel_reps, label)
    del A, rp, ci, va
    torch.cuda.empty_cache()

    with torch.cuda.stream(ex.stream):
        rp, ci, va = upwind3d(torch, args.grid16, dev)
    n, nnz = rp.numel() - 1, va.numel()
    A = api.host_csr(ex, (n, n), va, ci, rp)
    cases("upwind %d^3 f64 jac" % args.grid16, A, n, nnz, 4, [16])
    del A, rp, ci, va
    torch.cuda.empty_cache()

    with torch.cuda.stream(ex.stream):
        rp, ci, va = W.build("cfg4", xp="torch", device=dev, n=args.rand_rows)
        va = va.to(torch.float64)
    m = rp.numel() - 1
    A = api.host_csr(ex, (m, m), va, ci, rp)
    cases("cfg4 %.1fM f64 jac" % (m / 1e6), A, m, va.numel(), ci.element_size(),
          [int(s) for s in args.rand_ks.split(",")])


def kernel_times(torch, ex, rp, ci, va, k, j, kd, reps, label):
    """ms per launch of each kernel of one iteration of (c) at Krylov index j, each launched `reps` times
    back to back between two CUDA events on the solver's stream; no column ever stops, so no launch turns
    into a no-op"""
    import ctypes
    from ginkgo_b200 import _lib
    lib = _lib.lib()
    n = rp.numel() - 1
    ctx = ctypes.c_void_p()
    assert lib.b200_ctx_create(0, ex.stream.cuda_stream, ctypes.byref(ctx)) == 0
    dev = ex.device
    nk = n * k
    with torch.cuda.stream(ex.stream):
        K = torch.empty((j + 2) * nk, dtype=torch.float64, device=dev).uniform_(-1, 1)
        z = torch.zeros(nk, dtype=torch.float64, device=dev)
        diag = torch.ones(n, dtype=torch.float64, device=dev)
        hess = torch.full(((j + 2) * k,), 0.5, dtype=torch.float64, device=dev)  # no coefficient skips its basis
        haux = torch.zeros((kd + 1) * k, dtype=torch.float64, device=dev)
        sc = torch.ones(3 * k, dtype=torch.float64, device=dev)
        sc[2 * k:] = 0  # threshold 0: never converged
        gsin = torch.zeros((j + 1) * k, dtype=torch.float64, device=dev)
        gcos = torch.ones((j + 1) * k, dtype=torch.float64, device=dev)  # identity rotations keep hess nonzero
        rnc = torch.ones((j + 2) * k, dtype=torch.float64, device=dev)
        rnorm = torch.zeros(k, dtype=torch.float64, device=dev)
        fin = torch.zeros(k, dtype=torch.int64, device=dev)
        status = torch.zeros(k, dtype=torch.uint8, device=dev)
        ctl = torch.tensor([0, 0, -1, 0, 1, 0, 0, 0], dtype=torch.int32, device=dev)  # no criterion can stop
        work = torch.zeros(lib.b200_gmres_mrhs_work_size_f64(ctx, k, kd), dtype=torch.float64, device=dev)
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + 8 * off)  # noqa: E731
    vj, w = P(K, j * nk), P(K, (j + 1) * nk)
    hcol = P(hess)
    st, c, wk, s_ = P(status), P(ctl), P(work), P(sc)
    mdot2 = getattr(lib, "b200_csr_spmv_mdot2_f64_" + ("i32" if ci.element_size() == 4 else "i64"))
    final_j = j

    def final_pass(first):
        # the final pass's Givens update at a fixed index: fin and the iteration count grow, nothing stops
        return lib.b200_gmres_mrhs_final_pass_f64(ctx, n, k, w, P(K), first, hcol, None, hcol, final_j, P(gsin),
                                                  P(gcos), P(rnorm), P(rnc), P(fin), st, s_, c, wk)
    calls = [
        ("scale", lambda: lib.b200_gmres_mrhs_scale_f64(ctx, n, k, vj, P(z), P(diag), s_, st, c, 1), (3 * k + 1) * n * 8),
        ("spmv_mdot2", lambda: mdot2(ctx, n, n, va.numel(), P(rp), P(ci), P(va), P(z), k, w, P(K), hcol, None, wk, c),
         None),
        ("mgs_pass", lambda: lib.b200_gmres_mrhs_mgs_pass_f64(ctx, n, k, w, P(K), P(K, nk), hcol, 1, st, c, wk),
         4 * nk * 8),
        ("final_pass (MGS)", lambda: final_pass(j), 3 * nk * 8),
        ("multi_dot (CGS, j bases)", lambda: lib.b200_gmres_mrhs_multi_dot_f64(ctx, n, k, j, kd, P(K, nk), w,
                                                                              P(haux), st, c, wk), (j + 1) * nk * 8),
        ("final_pass (CGS)", lambda: final_pass(0), (j + 3) * nk * 8),
    ]
    b_matrix = va.numel() * (8 + ci.element_size()) + (n + 1) * rp.element_size()
    mgs_total = 0.0
    cgs_total = 0.0
    for name, fn, model in calls:
        assert fn() == 0  # warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ex.stream)
        for _ in range(reps):
            fn()
        e1.record(ex.stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / reps
        model = model if model is not None else b_matrix + 3 * nk * 8
        if name in ("scale", "spmv_mdot2"):
            mgs_total += ms
            cgs_total += ms
        elif name == "mgs_pass":
            mgs_total += j * ms
        elif name == "final_pass (MGS)":
            mgs_total += ms
        else:
            cgs_total += ms
        print("%-26s k=%-2d j=%-2d kernel %-26s %.3f ms/launch  model %.0f MB -> %.0f GB/s" %
              (label, k, j, name, ms, model / 1e6, model / ms / 1e6))
    assert ctl[0].item() == 0, "a kernel turned into a no-op"
    print("%-26s k=%-2d j=%-2d one iteration: MGS %.3f ms (%d launches), CGS %.3f ms (4 launches)" %
          (label, k, j, mgs_total, j + 3, cgs_total))
    lib.b200_ctx_destroy(ctx)


if __name__ == "__main__":
    main()
