"""Times every column part of the cfg2 plan on its own (b200_csr_spmv_part_f64_i32), CUDA events over
--reps launches each, plus the whole 5-part apply.  Part 0 writes c = A_0 b; parts 1.. read c and write
c = A_p b + c.  Prints the card name and power limit first, then one line per part with its time, its
HBM bytes (values + column indices + row pointers + c) and the gather rate.

  python scripts/cfg2_parts_timing.py [--reps 50]
"""
import argparse
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    import workloads as W
    from ginkgo_b200 import _lib, api

    print("card: %s" % card())
    ex = api.B200Executor.create(0)
    dev = ex.device
    n = W.CONFIGS["cfg2"]["n"]
    with torch.cuda.stream(ex.stream):
        rp, ci, va = W.build("cfg2", xp="torch", device=dev)
        x = W.vector(n, xp="torch", device=dev)
        y = torch.empty(n, dtype=torch.float64, device=dev)
    A = api.Csr(ex, (n, n), va, ci, rp)
    plan = A.plan()
    l = _lib.lib()
    parts = l.b200_csr_plan_parts(plan)
    print("cfg2: n=%d nnz=%d, %d column parts, kernel variant %d" % (n, va.numel(), parts,
                                                                     l.b200_csr_plan_variant(plan)))
    if parts < 2:
        raise SystemExit("the cfg2 plan has no column-blocked copy on this device")
    col_block = -(-n // parts)
    with torch.cuda.stream(ex.stream):
        part_nnz = [int(((ci >= p * col_block) & (ci < min(n, (p + 1) * col_block))).sum().item())
                    for p in range(parts)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        for _ in range(3):
            fn()
        ex.synchronize()
        e0.record(ex.stream)
        for _ in range(args.reps):
            fn()
        e1.record(ex.stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.reps

    total = 0.0
    for p in range(parts):
        ms = timed(lambda: ex.run("b200_csr_spmv_part_f64_i32", plan, p, int(p > 0), x, 1, y, 1, None, 0))
        nbytes = part_nnz[p] * 12 + (n + 1) * 4 + n * 8 * (2 if p > 0 else 1)
        total += ms
        print("part %d (%s): nnz %d, %.4f ms, %.1f GB/s HBM, %.1f G gathers/s" %
              (p, "reads c" if p else "no c read", part_nnz[p], ms, nbytes / ms / 1e6, part_nnz[p] / ms / 1e6))
    whole = timed(lambda: A.apply(api.Dense(ex, x), api.Dense(ex, y)))
    print("sum of parts %.4f ms; whole apply %.4f ms (%.1f GFLOP/s)" % (total, whole, 2 * va.numel() / whole / 1e6))


if __name__ == "__main__":
    main()
