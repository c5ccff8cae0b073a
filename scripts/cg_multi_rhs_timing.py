"""CG for k right-hand sides of one system on one GPU, three ways, alternated in one process after one
warm-up solve each:
  (a) k one-column fused solves (solver::Cg's default fused path, once per column),
  (b) the kernel-by-kernel loop on the n x k Dense,
  (c) the fused path for several right-hand sides (with_fused_multi_rhs: one matrix pass per iteration).

Problems: the 7-pt Laplacian 200^3 in fp64 with scalar Jacobi (cfg3's matrix; columns of b from
workloads.vector on distinct streams), k in --ks, once with a fixed --iters iterations (Iteration only)
and once to 1e-8 (rhs_norm); then an SPD matrix with scattered columns (workloads.random_csr of
--rand-rows rows and 8 per row, symmetrised, diagonal = row sum of |a| + 1), k in --rand-ks, to 1e-8.
Per run and path: ms per iteration and per iteration and right-hand side (median of --reps solves, host
clock around work that ends in a synchronise), the byte model over that time, host-issued launches per
iteration, the true relative residual of every column and the stop statuses.  Byte models per iteration
of the n x k system (B = matrix bytes, V = value bytes; with scalar Jacobi, Identity one n V less per
column): (a) k (B + 13 n V), (b) B + 19 n k V, (c) B + 13 n k V.  Needs a GPU.

  python scripts/cg_multi_rhs_timing.py [--grid 200] [--ks 2,4,8,16] [--iters 200] [--rand-rows 2000000]
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bicgstab_fused_timing import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=200)
    ap.add_argument("--ks", default="2,4,8,16")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rand-rows", type=int, default=2_000_000)
    ap.add_argument("--rand-ks", default="4,8")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("cg_multi_rhs_timing.py measures on a GPU and none is visible")
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
        d = 1 if pre else 0  # the diagonal, counted once per column as in the one-column model
        kw = dict(precond_max_bs=pre, **crit)
        with torch.cuda.stream(ex.stream):
            cols = [b[:, j].contiguous().reshape(n, 1) for j in range(k)]
            xs1 = [torch.zeros(n, 1, dtype=b.dtype, device=dev) for _ in range(k)]
            xl = torch.zeros(n, k, dtype=b.dtype, device=dev)
            xf = torch.zeros(n, k, dtype=b.dtype, device=dev)
        s1 = api.HostSolver(ex, "cg", A, **kw)
        sl = api.HostSolver(ex, "cg", A, fused=False, **kw)
        sf = api.HostSolver(ex, "cg", A, fused_multi_rhs=True, **kw)
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
        models = [(b_matrix + (12 + d) * n * V) * its[0], b_matrix + (18 + d) * n * k * V,
                  b_matrix + (12 + d) * n * k * V]
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
        rp, ci, va = W.laplace(args.grid, 3, xp="torch", device=dev)
    n, nnz = rp.numel() - 1, va.numel()
    A = api.host_csr(ex, (n, n), va, ci, rp)
    label = "laplace7 %d^3 f64 jac" % args.grid
    for k in [int(s) for s in args.ks.split(",")]:
        with torch.cuda.stream(ex.stream):
            b = torch.stack([W.vector(n, stream=11 + j, xp="torch", device=dev) for j in range(k)], dim=1)
            b = b.to(torch.float64).contiguous()
        run(label + " fixed", A, n, nnz, 8, 4, k, b, dict(max_iters=args.iters, res_kind=0))
        run(label + " 1e-8", A, n, nnz, 8, 4, k, b, dict(max_iters=5000, reduction=1e-8))
        del b
    del A, rp, ci, va

    import scipy.sparse as sp
    m = args.rand_rows
    rp, ci, va = W.random_csr(m, 8)
    S = sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(m, m))
    S = (S + S.T).tocsr()
    S.setdiag(0)
    S.eliminate_zeros()
    d = np.asarray(abs(S).sum(axis=1)).ravel() + 1.0
    S = (S + sp.diags(d)).tocsr()
    S.sort_indices()
    with torch.cuda.stream(ex.stream):
        t = [torch.from_numpy(a).to(dev) for a in (S.data.astype(np.float64), S.indices.astype(np.int32),
                                                    S.indptr.astype(np.int32))]
    A = api.host_csr(ex, (m, m), *t)
    label = "random sym %dM f64 jac" % (m // 1_000_000)
    for k in [int(s) for s in args.rand_ks.split(",")]:
        with torch.cuda.stream(ex.stream):
            b = torch.stack([W.vector(m, stream=11 + j, xp="torch", device=dev) for j in range(k)], dim=1)
            b = b.to(torch.float64).contiguous()
        run(label + " 1e-8", A, m, S.nnz, 8, 4, k, b, dict(max_iters=5000, reduction=1e-8))
        del b


if __name__ == "__main__":
    main()
