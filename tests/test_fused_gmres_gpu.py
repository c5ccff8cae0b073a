"""The fused GMRES iteration (csrc/fused_gmres.cu, the ctl-aware block-Jacobi instance of stop_jacobi.cu
and solver::Gmres::try_fused): each kernel through the C ABI against a numpy restatement, then the host
solver against the device loop and the oracle.

Assertions as in tests/test_fused_bicgstab_gpu.py: element-wise updates and the scalars derived from
given sums BIT FOR BIT, reductions on small-integer data for EQUALITY with the exact sum, reductions on
random data against math.fsum within gamma_h * sum |t|."""
import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import VT
from tests.test_fused_bicgstab_gpu import SYSTEMS, convective_arrow, true_rel_res, upwind
from tests.test_fused_cg_gpu import (STOPPED, VTS, arrow_inv_diag, assert_sum_within, backend,  # noqa: F401
                                     dev, hexec, nans)

pytestmark = pytest.mark.gpu

SC, CTL = 8, 8  # sc: 0 ||w|| of the last final pass, 1 tau0, 2 threshold


def vec(vt, n, data, seed):
    rng = np.random.default_rng(seed)
    if data == "int":
        return rng.integers(-3, 4, size=n).astype(VT[vt])
    return rng.uniform(-1, 1, size=n).astype(VT[vt])


def assert_norm_within(nrm, w, vt):
    """nrm = sqrt of the sum of w^2 in some order: |nrm^2 - S| <= (gamma_(n-1) + 3u) sum w^2 (the sum's
    any-order bound, plus the rounding of the square root and of squaring it back)"""
    import math
    u = float(np.finfo(VT[vt]).eps) / 2
    t = (w.astype(np.float64) ** 2)
    S = math.fsum(t)
    h = max(len(t) - 1, 0)
    gamma = h * u / (1 - h * u)
    assert abs(float(nrm) ** 2 - S) <= (gamma + 3 * u) * S * (1 + 2.0 ** -40) + 1e-300, (float(nrm) ** 2, S)


SIZES = [0, 1, 7, 1000, 300_001]  # the last one fills the grid cap of the element-wise kernels


# --------------------------------------------------------------------------- A. scale
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("divide", [0, 1])
def test_scale(dev, n, vt, precond, divide):
    T = VT[vt]
    w, d = vec(vt, n, "rand", 1), vec(vt, n, "rand", 2)
    h = T(0.37)
    sc = dev.put(np.array([h] + [0] * 7, T))
    ctl = dev.put(np.zeros(CTL, np.int32))
    vd, zd, dd = dev.put(w), dev.put(nans(n, vt)), dev.put(d)
    dev.call("gmres_fused_scale_" + vt, n, vd, zd if precond else None, dd if precond else None, sc, ctl, divide)
    v_ref = (w / h).astype(T) if divide else w
    assert vd.get().tobytes() == v_ref.tobytes()
    if precond:
        assert zd.get().tobytes() == (v_ref * d).astype(T).tobytes()
    else:
        assert np.isnan(zd.get()).all()
    # stopped: nothing is written
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    v2, z2 = dev.put(w), dev.put(nans(n, vt))
    dev.call("gmres_fused_scale_" + vt, n, v2, z2, dd, sc, ctl, 1)
    assert v2.get().tobytes() == w.tobytes() and np.isnan(z2.get()).all()


# --------------------------------------------------------------------------- B. MGS passes
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_mgs_passes(dev, n, vt, data):
    """passes i = 1..j on j + 1 bases: w bit-equal to sequential sub_scaled, every h_i checked"""
    T = VT[vt]
    j = 4
    V = np.stack([vec(vt, n, data, 10 + i) for i in range(j + 1)])
    w = vec(vt, n, data, 3)
    h0 = T(2) if data == "int" else T(0.3)
    hcol = np.full(j + 2, np.nan, T)
    hcol[0] = h0
    Vd, wd, hd = dev.put(V), dev.put(w), dev.put(hcol)
    ctl, work = dev.put(np.zeros(CTL, np.int32)), dev.work(vt)
    w_ref = w.copy()
    for i in range(1, j + 1):
        dev.call("gmres_fused_mgs_pass_" + vt, n, wd, Vd.at((i - 1) * n), Vd.at(i * n), hd, i, ctl, work)
        h_prev = hd.get()[i - 1]
        w_ref = (w_ref - (h_prev * V[i - 1]).astype(T)).astype(T) if h_prev != 0 else w_ref
        got_w, got_h = wd.get(), hd.get()[i]
        assert got_w.tobytes() == w_ref.tobytes(), i
        terms = (V[i] * w_ref).astype(T)
        if data == "int":
            prods = V[i].astype(np.int64) * w_ref.astype(np.int64)
            if np.abs(prods).sum() < (2 ** 24 if vt == "f32" else 2 ** 53):  # every partial sum exact
                assert float(got_h) == int(prods.sum()), i
        assert_sum_within(got_h, terms, vt, "h_%d" % i)
        if data == "int" and abs(float(got_h)) > 1e6:
            break  # keep the integer data exact
    # stopped: nothing is written
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    before_w, before_h = wd.get(), hd.get()
    dev.call("gmres_fused_mgs_pass_" + vt, n, wd, Vd.at(0), Vd.at(n), hd, 1, ctl, work)
    assert wd.get().tobytes() == before_w.tobytes() and hd.get().tobytes() == before_h.tobytes()


# --------------------------------------------------------------------------- C. final pass
def givens_ref(T, gsin, gcos, rnc, h, it):
    """hessenberg_qr (reference/solver/common_gmres_kernels.cpp) for one right-hand side, in T"""
    hj = h[0]
    for j in range(it):
        c, s, hj1 = gcos[j], gsin[j], h[j + 1]
        h[j] = T(T(c * hj) + T(s * hj1))
        hj = T(T(-s * hj) + T(c * hj1))
    this, nxt = hj, h[it + 1]
    if this == 0:
        c, s = T(0), T(1)
    else:
        scale = T(abs(this) + abs(nxt))
        a, b = abs(T(this / scale)), abs(T(nxt / scale))
        hyp = T(scale * np.sqrt(T(T(a * a) + T(b * b))))
        c, s = T(this / hyp), T(nxt / hyp)
    gcos[it], gsin[it] = c, s
    h[it] = T(T(c * this) + T(s * nxt))
    h[it + 1] = T(0)
    old = rnc[it]
    rnc[it + 1] = T(-s * old)
    rnc[it] = T(c * old)
    return abs(rnc[it + 1])


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("n", [1, 1000, 300_001])
def test_final_pass_givens(dev, vt, n):
    """iterations j = 0..kd-1 of final passes on made-up Hessenberg columns: w, the norm, the Givens
    values, rnc and the column bit-equal to the restatement, the status byte untouched while running"""
    T = VT[vt]
    kd = 6
    rng = np.random.default_rng(5)
    gsin, gcos = np.zeros(kd, T), np.zeros(kd, T)
    rnc = np.zeros(kd + 1, T)
    rnc[0] = T(3.5)
    gs, gc, rn = dev.put(gsin), dev.put(gcos), dev.put(rnc)
    rnorm, fin, stop = dev.put(np.zeros(1, T)), dev.put(np.zeros(1, np.uint64)), dev.put(np.zeros(1, np.uint8))
    sc = dev.put(np.array([0, 1, 0] + [0] * 5, T))  # threshold 0: never converged
    ctl = dev.put(np.array([0, 0, -1, 1, 1, 0, 0, 0], np.int32))
    work = dev.work(vt)
    for j in range(kd):
        h = np.concatenate([rng.uniform(-1, 1, j + 1), [np.nan]]).astype(T)
        if j == 2:
            h[j] = T(0)  # no subtraction, and ...
        w, v = vec(vt, n, "rand", 20 + j), vec(vt, n, "rand", 40 + j)
        if j == 3:
            w = np.zeros(n, T)  # ... a zero norm, which the Givens update must take
            h[:j + 1] = 0
        K = np.concatenate([np.full(j * n, np.nan, T), v])  # MGS: only basis j is subtracted
        hd, wd, Kd = dev.put(h), dev.put(w), dev.put(K)
        dev.call("gmres_fused_final_pass_" + vt, n, wd, Kd, j, hd, None, hd, j, gs, gc, rnorm, rn, fin, stop, sc,
                 ctl, work)
        w_ref = (w - (h[j] * v).astype(T)).astype(T) if h[j] != 0 else w
        assert wd.get().tobytes() == w_ref.tobytes()
        nrm = sc.get()[0]
        assert_norm_within(nrm, w_ref, vt)
        h_ref = h.copy()
        h_ref[j + 1] = nrm
        tau = givens_ref(T, gsin, gcos, rnc, h_ref, j)
        assert hd.get().tobytes() == h_ref.tobytes(), j
        assert gs.get().tobytes() == gsin.tobytes() and gc.get().tobytes() == gcos.tobytes()
        assert rn.get().tobytes() == rnc.tobytes()
        assert rnorm.get()[0] == tau and fin.get()[0] == j + 1
        assert stop.get()[0] == 0 and ctl.get()[0] == 0 and ctl.get()[1] == j + 1


def run_check(dev, vt, tau, tau0, factor, max_iters, res_kind, iter_first, iters_done, baseline=2):
    """the stopping check of the final pass, fed one Givens update whose |rnc[1]| is exactly tau"""
    T = VT[vt]
    # a column with this == 0 gives c = 0, s = 1: rnc[1] = -rnc[0], |rnc[1]| = rnc[0]
    gs, gc = dev.put(np.zeros(1, T)), dev.put(np.zeros(1, T))
    rn = dev.put(np.array([tau, np.nan], T))
    rnorm, fin, stop = dev.put(np.zeros(1, T)), dev.put(np.zeros(1, np.uint64)), dev.put(np.zeros(1, np.uint8))
    sc = dev.put(np.array([0, tau0, T(factor) * T(tau0)] + [0] * 5, T))
    ctl = dev.put(np.array([0, iters_done, max_iters, res_kind, int(iter_first), 0, 0, 0], np.int32))
    n = 16
    hd, wd, vd = dev.put(np.zeros(2, T)), dev.put(np.zeros(n, T)), dev.put(np.zeros(n, T))
    dev.call("gmres_fused_final_pass_" + vt, n, wd, vd, 0, hd, None, hd, 0, gs, gc, rnorm, rn, fin, stop, sc,
             ctl, dev.work(vt))
    assert rnorm.get()[0] == T(tau)
    c = ctl.get()
    assert c[1] == iters_done + 1 and c[0] == stop.get()[0]
    return int(c[0])


@pytest.mark.parametrize("vt", VTS)
def test_stopping_table(dev, vt):
    """Iteration x ResidualNorm in both orders; tau exactly on the threshold converges; no finalized bit"""
    T = VT[vt]
    thr_tau0, f = T(2.0), 0.25  # threshold 0.5, exact in both types
    conv = 0x80
    for iter_first in (True, False):
        it_id, res_id = (1, 2) if iter_first else (2, 1)
        # neither
        assert run_check(dev, vt, 0.75, thr_tau0, f, 10, 1, iter_first, 3) == 0
        # tau on the threshold: converged
        assert run_check(dev, vt, 0.5, thr_tau0, f, 10, 1, iter_first, 3) == conv | res_id
        # iteration limit reached (iteration 4 >= 4)
        assert run_check(dev, vt, 0.75, thr_tau0, f, 4, 1, iter_first, 3) == it_id
        # both: the first in the user's order wins
        both = run_check(dev, vt, 0.25, thr_tau0, f, 4, 1, iter_first, 3)
        assert both == (it_id if iter_first else conv | res_id)
    # one criterion alone takes id 1
    assert run_check(dev, vt, 0.25, thr_tau0, f, -1, 1, True, 3) == conv | 1
    assert run_check(dev, vt, 0.25, thr_tau0, f, 4, 0, True, 3) == 1


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
@pytest.mark.parametrize("rn0", [0.0, 3.0])
def test_init(dev, vt, baseline, rn0):
    """baseline, threshold and the iteration-0 check; a zero initial residual stops at iteration 0"""
    T = VT[vt]
    rnorm, stop = dev.put(np.array([rn0], T)), dev.put(np.full(1, 0x3f, np.uint8))
    bnorm = T(8.0)
    sc = dev.put(np.array([np.nan, bnorm] + [np.nan] * 6, T))
    ctl = dev.put(np.full(CTL, 77, np.int32))
    dev.call("gmres_fused_init_" + vt, rnorm, sc, ctl, stop, 100, 1, 1, baseline, T(0.125))
    tau0 = {0: bnorm, 1: T(rn0), 2: T(1)}[baseline]
    s, c = sc.get(), ctl.get()
    assert s[1] == tau0 and s[2] == T(0.125) * tau0
    assert list(c[1:5]) == [0, 100, 1, 1]
    expect = 0x80 | 2 if T(rn0) <= T(0.125) * tau0 else 0
    assert c[0] == expect and stop.get()[0] == expect


# --------------------------------------------------------------------------- D. the host solver
def host_gmres(hexec, rp, ci, va, b, precond, block_ptrs=None, **kw):
    import torch
    from ginkgo_b200 import api
    n = len(rp) - 1
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(b)).to(hexec.device)
        tx = torch.zeros_like(tb)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "gmres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
    hexec.synchronize()
    return tx.cpu().numpy(), s.num_iterations, s.stop_status, s.used_fused


PRECONDS = {"identity": (0, None), "scalar": (1, None), "block_given": (8, "given"), "block_detected": (8, None)}


def precond_args(name, n):
    pc, bp = PRECONDS[name]
    if bp == "given":
        bp = np.unique(np.concatenate([np.arange(0, n, 5), [n]])).astype(np.int32)
    return pc, bp


@pytest.mark.parametrize("system", list(SYSTEMS))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", list(PRECONDS))
@pytest.mark.parametrize("kd,check_every", [(5, 1), (5, 3), (20, 20), (30, 8), (30, 40)])
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_fused_gmres_matches_loop(hexec, system, vt, precond, kd, check_every, ortho):
    rp, ci, va = SYSTEMS[system](vt)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-10 if vt == "f64" else 1e-5
    pc, bp = precond_args(precond, n)
    kw = dict(max_iters=600, reduction=red, krylov_dim=kd, ortho=ortho, check_every=check_every)
    xl, itl, stl, usedl = host_gmres(hexec, rp, ci, va, b, pc, bp, **kw)
    xf, itf, stf, usedf = host_gmres(hexec, rp, ci, va, b, pc, bp, fused_gmres=True, **kw)
    assert usedf and not usedl
    assert abs(itf - itl) <= 2, (itf, itl)
    assert stf == stl
    if stl & 0x80:
        assert true_rel_res(rp, ci, va, b, xf) <= 20 * red
    assert H.rel_err(xl, xf) <= (1e-8 if vt == "f64" else 1e-3)


@pytest.mark.parametrize("system", ["upwind2d", "dominant_random"])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("kd", [5, 30])
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_fused_gmres_matches_oracle(hexec, system, vt, precond, kd, ortho):
    rp, ci, va = SYSTEMS[system](vt)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-9 if vt == "f64" else 1e-4
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    xo, ito, stop_o = H.orc_solve("gmres", vt, rp, ci, va, b, np.zeros((n, 1), VT[vt]), precond, jac,
                                  max_iters=600, reduction=red, krylov_dim=kd, ortho=ortho)
    xd, itd, stop_d, used = host_gmres(hexec, rp, ci, va, b, precond, max_iters=600, reduction=red, krylov_dim=kd,
                                       ortho=ortho, fused_gmres=True)
    assert used
    assert abs(itd - ito) <= 2, (itd, ito)
    assert stop_d == stop_o[0]
    assert true_rel_res(rp, ci, va, b, xd) <= 20 * red
    assert H.rel_err(xo, xd) <= (1e-8 if vt == "f64" else 1e-3)


@pytest.mark.parametrize("kd,check_every", [(5, 1), (5, 3), (5, 5), (5, 9)])
@pytest.mark.parametrize("max_iters", [0, 1, 2, 3, 4, 5, 6, 10, 15])
def test_stop_positions(hexec, kd, check_every, max_iters):
    """stops by the Iteration criterion at iteration 0, mid-batch, at a batch end and at a cycle end:
    the fused path reports the loop's iterations and status, and x matches (no restart after a stop)"""
    rp, ci, va = upwind(12, 2, "f64")
    n = len(rp) - 1
    b = np.random.default_rng(3).uniform(-1, 1, (n, 1))
    kw = dict(max_iters=max_iters, reduction=1e-14, krylov_dim=kd, check_every=check_every)
    xl, itl, stl, _ = host_gmres(hexec, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = host_gmres(hexec, rp, ci, va, b, 1, fused_gmres=True, **kw)
    assert used and itf == itl == max_iters and stf == stl == 0x40 | 1
    assert H.rel_err(xl, xf) <= 1e-10


def test_zero_rhs_stops_at_iteration_zero(hexec):
    rp, ci, va = upwind(10, 2, "f64")
    n = len(rp) - 1
    x, it, st, used = host_gmres(hexec, rp, ci, va, np.zeros((n, 1)), 1, max_iters=50, reduction=1e-8,
                                 baseline=2, fused_gmres=True)
    assert used and it == 0 and st == 0x80 | 0x40 | 2
    assert np.all(x == 0)


def test_repeated_applies_reuse_graphs(hexec):
    """the graphs are cached on the solver: a second apply on the same matrix gives the same bits"""
    import torch
    from ginkgo_b200 import api
    rp, ci, va = upwind(30, 2, "f64")
    n = len(rp) - 1
    b = np.random.default_rng(4).uniform(-1, 1, (n, 1))
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(b).to(hexec.device)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "gmres", A, precond_max_bs=8, max_iters=300, reduction=1e-10, krylov_dim=10,
                       check_every=4, fused_gmres=True)
    xs = []
    for _ in range(2):
        with torch.cuda.stream(hexec.stream):
            tx = torch.zeros_like(tb)
        s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
        hexec.synchronize()
        assert s.used_fused
        xs.append((tx.cpu().numpy().tobytes(), s.num_iterations, s.stop_status))
    assert xs[0] == xs[1]


def test_cfg4_full_size_fused(hexec, backend):
    """test_fullsize_gpu.py's cfg4 gate (GMRES(30, MGS) + block-Jacobi(16), fp32, n = 4M) on the fused path"""
    if backend.mock:
        pytest.skip("mock: a full-size solve on the host is out of reach")
    import torch
    import workloads as W
    from ginkgo_b200 import api
    from tests.test_fullsize_gpu import _fullsize_reference
    dev_ = hexec.device
    n = W.CONFIGS["cfg4"]["n"]
    with torch.cuda.stream(hexec.stream):
        rp, ci, va = W.build("cfg4", xp="torch", device=dev_)
        b = torch.ones(n, dtype=torch.float32, device=dev_)
        x = torch.zeros(n, dtype=torch.float32, device=dev_)
    A = api.host_csr(hexec, (n, n), va, ci, rp)
    bp = np.arange(0, n + 1, 16, dtype=np.int32)
    s = api.HostSolver(hexec, "gmres", A, precond_max_bs=16, block_ptrs=bp, max_iters=1000, reduction=1e-6,
                       krylov_dim=30, ortho=0, fused_gmres=True)
    bd, xd = api.host_dense(hexec, b), api.host_dense(hexec, x)  # the handles live as long as these
    s.apply(bd, xd)
    r = b.clone()
    h = api._host()
    one = api.host_dense(hexec, torch.ones(1, dtype=torch.float32, device=dev_))
    neg = api.host_dense(hexec, -torch.ones(1, dtype=torch.float32, device=dev_))
    rd = api.host_dense(hexec, r)
    api._hcheck(h.gkob_apply4(A.h, neg.h, xd.h, one.h, rd.h))
    hexec.synchronize()
    res = (r.double().norm() / b.double().norm()).item()
    exp = _fullsize_reference()["cfg4"]
    assert s.used_fused
    assert s.stop_status == (0x80 | 0x40 | 2)
    assert res <= 1.0e-6
    assert s.num_iterations <= max(exp["reference"]["iterations"], exp["omp"]["iterations"])


def test_fused_gmres_fallbacks_say_so(hexec):
    rp, ci, va = upwind(20, 2, "f64")
    n = len(rp) - 1
    rng = np.random.default_rng(2)
    b1, b2 = rng.uniform(-1, 1, (n, 1)), rng.uniform(-1, 1, (n, 2))
    kw = dict(max_iters=300, reduction=1e-8, fused_gmres=True)
    x, it, st, used = host_gmres(hexec, rp, ci, va, b2, 1, **kw)  # two right-hand sides
    assert not used and st == 0x80 | 0x40 | 2
    with pytest.raises(Exception):  # ImplicitResidualNorm: NotSupported, as from the loop
        host_gmres(hexec, rp, ci, va, b1, 1, res_kind=2, **kw)
    # off by default, and the other solvers' switches do not turn it on
    base = dict(max_iters=300, reduction=1e-8)
    assert not host_gmres(hexec, rp, ci, va, b1, 1, **base)[3]
    assert not host_gmres(hexec, rp, ci, va, b1, 1, fused=True, fused_bicgstab=True, **base)[3]
    assert host_gmres(hexec, rp, ci, va, b1, 1, **kw)[3]


# --------------------------------------------------------------------------- E. CGS / CGS2 kernels
@pytest.mark.parametrize("n", [1, 1000, 300_001])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_multi_dot_and_sub_passes(dev, n, vt, data):
    """CGS2 at j = 3: multi_dot of bases 1..j, the plain subtract pass, the multi-dot of bases 0..j into
    haux, the final pass adding haux; w bit-equal to sequential sub_scaled, the dots exact / bounded"""
    T = VT[vt]
    j = 3
    V = np.stack([vec(vt, n, data, 60 + i) for i in range(j + 1)])
    w0 = vec(vt, n, data, 7)
    Kd, wd = dev.put(V), dev.put(w0)
    hcol = np.full(j + 2, np.nan, T)
    hcol[0] = T(1) if data == "int" else T(0.25)
    hd, haux = dev.put(hcol), dev.put(np.full(j + 1, np.nan, T))
    ctl, work = dev.put(np.zeros(CTL, np.int32)), dev.put(np.full(
        getattr(dev.l, "b200_gmres_fused_work_size_" + vt)(dev.ctx, 30), np.nan, T))

    def check_dots(got, ws, bases):
        for q, i in enumerate(bases):
            terms = (V[i] * ws).astype(T)
            if data == "int":
                prods = V[i].astype(np.int64) * ws.astype(np.int64)
                if np.abs(prods).sum() < (2 ** 24 if vt == "f32" else 2 ** 53):
                    assert float(got[q]) == int(prods.sum()), i
            assert_sum_within(got[q], terms, vt, "v_%d . w" % i)

    dev.call("gmres_fused_multi_dot_" + vt, n, j, Kd.at(n), wd, hd.at(1), ctl, work)
    h = hd.get()
    check_dots(h[1:j + 1], w0, range(1, j + 1))
    w_ref = w0.copy()
    for i in range(j + 1):
        if h[i] != 0:
            w_ref = (w_ref - (h[i] * V[i]).astype(T)).astype(T)
    dev.call("gmres_fused_sub_pass_" + vt, n, wd, Kd, hd, j, ctl)
    assert wd.get().tobytes() == w_ref.tobytes()
    dev.call("gmres_fused_multi_dot_" + vt, n, j + 1, Kd, wd, haux, ctl, work)
    a = haux.get()
    check_dots(a, w_ref, range(j + 1))
    for i in range(j + 1):
        if a[i] != 0:
            w_ref = (w_ref - (a[i] * V[i]).astype(T)).astype(T)
    kd = 6
    gs, gc = dev.put(np.zeros(kd, T)), dev.put(np.zeros(kd, T))
    rnc = np.zeros(kd + 1, T)
    rnc[0] = T(2)
    rn = dev.put(rnc)
    rnorm, fin, stop = dev.put(np.zeros(1, T)), dev.put(np.zeros(1, np.uint64)), dev.put(np.zeros(1, np.uint8))
    sc = dev.put(np.array([0, 1, 0] + [0] * 5, T))
    before_h = hd.get()
    # the Givens update of the earlier columns is not under test here: j = 3 with zero rotations
    dev.call("gmres_fused_final_pass_" + vt, n, wd, Kd, 0, haux, haux, hd, j, gs, gc, rnorm, rn, fin, stop, sc, ctl,
             work)
    assert wd.get().tobytes() == w_ref.tobytes()
    nrm = sc.get()[0]
    h_ref = (before_h[:j + 1] + a).astype(T)  # the loop's add_scaled of haux, before the rotation
    assert_norm_within(nrm, w_ref, vt)
    col = np.concatenate([h_ref, [nrm]]).astype(T)
    givens_ref(T, np.zeros(kd, T), np.zeros(kd, T), rnc, col, j)
    assert hd.get().tobytes() == col.tobytes()
    # stopped: nothing is written by any of the three
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    snap = [b.get().tobytes() for b in (wd, hd, haux)]
    dev.call("gmres_fused_multi_dot_" + vt, n, j + 1, Kd, wd, haux, ctl, work)
    dev.call("gmres_fused_sub_pass_" + vt, n, wd, Kd, hd, j, ctl)
    dev.call("gmres_fused_final_pass_" + vt, n, wd, Kd, 0, haux, haux, hd, j, gs, gc, rnorm, rn, fin, stop, sc, ctl,
             work)
    assert [b.get().tobytes() for b in (wd, hd, haux)] == snap


# --------------------------------------------------------------------------- F. block Jacobi
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("max_bs,storage", [(4, None), (16, None), (32, None), (8, 0xff), (16, 0xff)])
def test_block_apply_ctl(dev, hexec, vt, max_bs, storage):
    """the ctl-aware instance: bit-equal to b200_jacobi_simple_apply_* (plain and adaptive storage)
    while running, nothing written once stopped"""
    import torch
    from ginkgo_b200 import api
    rp, ci, va = upwind(24, 2, vt)
    n = len(rp) - 1
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
    A = api.host_csr(hexec, (n, n), *t)
    J = api.host_jacobi(A, max_bs, storage_optimization=storage)
    g = api.host_jacobi_get(J)
    blocks, bp = dev.put(g["blocks"]), dev.put(g["block_ptrs"])
    prec = dev.put(g["precisions"]) if g["precisions"] is not None else None
    assert (prec is not None) == (storage is not None)
    b = dev.put(vec(vt, n, "rand", 8))
    ref, got = dev.put(nans(n, vt)), dev.put(nans(n, vt))
    args = (g["num_blocks"], max_bs, g["block_offset"], g["group_offset"], g["group_power"])
    if prec is None:
        dev.call("jacobi_simple_apply_%s_i32" % vt, *args, bp, blocks, b, 1, 1, ref, 1)
    else:
        dev.call("jacobi_simple_apply_adaptive_%s_i32" % vt, *args, prec, bp, blocks, b, 1, 1, ref, 1)
    ctl = dev.put(np.zeros(CTL, np.int32))
    dev.call("gmres_fused_block_apply_%s_i32" % vt, *args, prec, bp, blocks, b, got, ctl)
    assert not np.isnan(ref.get()).any()
    assert got.get().tobytes() == ref.get().tobytes()
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    stopped = dev.put(nans(n, vt))
    dev.call("gmres_fused_block_apply_%s_i32" % vt, *args, prec, bp, blocks, b, stopped, ctl)
    assert np.isnan(stopped.get()).all()


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_fused_gmres_adaptive_block_jacobi(hexec, vt, ortho):
    """adaptive-precision block Jacobi (storage_optimization autodetect), generated outside the solver"""
    import torch
    from ginkgo_b200 import api
    rp, ci, va = SYSTEMS["dominant_random"](vt)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1)).astype(VT[vt])
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
    A = api.host_csr(hexec, (n, n), *t)
    J = api.host_jacobi(A, 16, storage_optimization=0xff)  # detected blocks
    assert api.host_jacobi_get(J)["precisions"] is not None
    red = 1e-10 if vt == "f64" else 1e-5
    out = []
    for fused in (False, True):
        with torch.cuda.stream(hexec.stream):
            tb = torch.from_numpy(b).to(hexec.device)
            tx = torch.zeros_like(tb)
        s = api.HostSolver(hexec, "gmres", A, max_iters=600, reduction=red, krylov_dim=10, ortho=ortho,
                           check_every=4, fused_gmres=fused, preconditioner=J)
        s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
        hexec.synchronize()
        out.append((tx.cpu().numpy(), s.num_iterations, s.stop_status, s.used_fused))
    (xl, itl, stl, ul), (xf, itf, stf, uf) = out
    assert uf and not ul
    assert abs(itf - itl) <= 2 and stf == stl == 0x80 | 0x40 | 2
    assert true_rel_res(rp, ci, va, b, xf) <= 20 * red
    assert H.rel_err(xl, xf) <= (1e-8 if vt == "f64" else 1e-3)


# --------------------------------------------------------------------------- G. matrix paths
@pytest.mark.parametrize("system", ["dominant_random", "convective_arrow"])
@pytest.mark.parametrize("it", ["i32", "i64"])
@pytest.mark.parametrize("kernel,reblock", [("warp", None), ("pipe", None), ("ring", None), ("warp", "3")])
@pytest.mark.parametrize("ortho", [0, 2])
def test_fused_gmres_matrix_paths(hexec, backend, monkeypatch, system, it, kernel, reblock, ortho):
    """int32 / int64 matrices, each SpMV kernel, a column-blocked plan, and rows split over CTAs (the
    arrow matrix: its long rows are split, inside the captured graphs)"""
    if backend.mock and system == "convective_arrow":
        pytest.skip("mock: no split rows")
    monkeypatch.setenv("B200_CSR_KERNEL", kernel)
    if reblock is not None:
        monkeypatch.setenv("B200_CSR_REBLOCK", reblock)
    vt = "f64"
    rp, ci, va = convective_arrow(vt) if system == "convective_arrow" else SYSTEMS[system](vt)
    rp, ci = rp.astype(np.int64 if it == "i64" else np.int32), ci.astype(np.int64 if it == "i64" else np.int32)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1))
    kw = dict(max_iters=600, reduction=1e-10, krylov_dim=20, ortho=ortho, check_every=7)
    pc = 1 if it == "i32" else 0  # the C handle generates Jacobi<V, int32>, from int32 matrices
    xl, itl, stl, usedl = host_gmres(hexec, rp, ci, va, b, pc, **kw)
    xf, itf, stf, usedf = host_gmres(hexec, rp, ci, va, b, pc, fused_gmres=True, **kw)
    assert usedf and not usedl
    assert abs(itf - itl) <= 2 and stf == stl
    if stl & 0x80:
        assert true_rel_res(rp, ci, va, b, xf) <= 20 * 1e-10
        assert H.rel_err(xl, xf) <= 1e-8


# --------------------------------------------------------------------------- H. lock-step
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_lockstep_on_convective_arrow(dev, vt, ortho):
    """36 iterations of the fused kernels with krylov_dim = 5 on the nonsymmetric arrow matrix (rows split
    over CTAs), restarted every 5; after every kernel its output is checked against numpy fed with the
    device's own inputs: bit-equal vectors and Givens values, dots and norms within the any-order bound"""
    from tests.test_fused_cg_gpu import Mat
    T = VT[vt]
    rp, ci, va = convective_arrow(vt)
    n = len(rp) - 1
    A = Mat(dev, vt, "i32", n, n, rp, ci, va, None)
    kd = 5
    K = dev.put(np.zeros((kd + 1) * n, T))
    hess = dev.put(np.zeros(kd * (kd + 1), T))
    small = {k: dev.put(np.zeros(m, T)) for k, m in (("gsin", kd), ("gcos", kd), ("rnc", kd + 1), ("rnorm", 1),
                                                      ("haux", kd + 1))}
    fin, stop = dev.put(np.zeros(1, np.uint64)), dev.put(np.zeros(1, np.uint8))
    sc = dev.put(np.array([0, 1, 0] + [0] * 5, T))  # threshold 0
    ctl = dev.put(np.array([0, 0, 1000, 1, 1, 0, 0, 0], np.int32))
    work = dev.put(np.full(getattr(dev.l, "b200_gmres_fused_work_size_" + vt)(dev.ctx, kd), np.nan, T))
    rng = np.random.default_rng(9)
    Kh = lambda i: K.get()[i * n:(i + 1) * n]  # noqa: E731
    for it_ in range(36):
        j = it_ % kd
        if j == 0:  # a restart: a fresh unit v_0, a zero Hessenberg, rnc[0] = 1
            v0 = rng.uniform(-1, 1, n)
            v0 = (v0 / np.linalg.norm(v0)).astype(T)
            Kall = K.get()
            Kall[:n] = v0
            K.set(Kall)
            hess.set(np.zeros(kd * (kd + 1), T))
            rnc = np.zeros(kd + 1, T)
            rnc[0] = T(1)
            small["rnc"].set(rnc)
            fin.set(np.zeros(1, np.uint64))
        hc = hess.at(j * (kd + 1))
        if j > 0:
            w_old, nrm = Kh(j), sc.get()[0]
            dev.call("gmres_fused_scale_" + vt, n, K.at(j * n), None, None, sc, ctl, 1)
            assert Kh(j).tobytes() == (w_old / nrm).astype(T).tobytes()
        vj = Kh(j)
        dev.call("csr_spmv_dot2_%s_i32" % vt, A.plan, n, n, len(va), A.rp, A.ci, A.va, K.at(j * n), K.at((j + 1) * n),
                 K, hc, None, work, ctl)
        w = Kh(j + 1)
        ref = np.asarray(sp_matvec(rp, ci, va, vj.astype(np.float64)))
        assert np.allclose(w, ref, rtol=1e-10 if vt == "f64" else 1e-4, atol=1e-12 if vt == "f64" else 1e-5)
        h = hess.get()[j * (kd + 1):(j + 1) * (kd + 1)]
        assert_sum_within(h[0], (Kh(0) * w).astype(T), vt, "h_0")
        if ortho == 0:
            for i in range(1, j + 1):
                w_in = Kh(j + 1)
                dev.call("gmres_fused_mgs_pass_" + vt, n, K.at((j + 1) * n), K.at((i - 1) * n), K.at(i * n), hc, i,
                         ctl, work)
                h = hess.get()[j * (kd + 1):(j + 1) * (kd + 1)]
                w_ref = (w_in - (h[i - 1] * Kh(i - 1)).astype(T)).astype(T) if h[i - 1] != 0 else w_in
                assert Kh(j + 1).tobytes() == w_ref.tobytes()
                assert_sum_within(h[i], (Kh(i) * w_ref).astype(T), vt, "h_%d" % i)
            first, coef, add = j, hc, None
        else:
            if j > 0:
                dev.call("gmres_fused_multi_dot_" + vt, n, j, K.at(n), K.at((j + 1) * n), hess.at(j * (kd + 1) + 1),
                         ctl, work)
                h = hess.get()[j * (kd + 1):(j + 1) * (kd + 1)]
                for i in range(1, j + 1):
                    assert_sum_within(h[i], (Kh(i) * w).astype(T), vt, "h_%d" % i)
            first, coef, add = 0, hc, None
            if ortho == 2:
                w_in = Kh(j + 1)
                dev.call("gmres_fused_sub_pass_" + vt, n, K.at((j + 1) * n), K, hc, j, ctl)
                w_ref = w_in.copy()
                for i in range(j + 1):
                    if h[i] != 0:
                        w_ref = (w_ref - (h[i] * Kh(i)).astype(T)).astype(T)
                assert Kh(j + 1).tobytes() == w_ref.tobytes()
                dev.call("gmres_fused_multi_dot_" + vt, n, j + 1, K, K.at((j + 1) * n), small["haux"], ctl, work)
                a = small["haux"].get()
                for i in range(j + 1):
                    assert_sum_within(a[i], (Kh(i) * w_ref).astype(T), vt, "haux_%d" % i)
                coef = add = small["haux"]
        # final pass: the device's own coefficients and Givens state in, bit-equal restatement out
        w_in, h_in = Kh(j + 1), hess.get()[j * (kd + 1):(j + 1) * (kd + 1)].copy()
        cf = (h_in if coef is hc else small["haux"].get())
        gsin, gcos, rnc = small["gsin"].get(), small["gcos"].get(), small["rnc"].get()
        dev.call("gmres_fused_final_pass_" + vt, n, K.at((j + 1) * n), K, first, coef, add, hc, j, small["gsin"],
                 small["gcos"], small["rnorm"], small["rnc"], fin, stop, sc, ctl, work)
        w_ref = w_in.copy()
        for i in range(first, j + 1):
            if cf[i] != 0:
                w_ref = (w_ref - (cf[i] * Kh(i)).astype(T)).astype(T)
        assert Kh(j + 1).tobytes() == w_ref.tobytes()
        nrm = sc.get()[0]
        assert_norm_within(nrm, w_ref, vt)
        col = h_in.copy()
        if add is not None:
            col[:j + 1] = (col[:j + 1] + cf[:j + 1]).astype(T)
        col[j + 1] = nrm
        tau = givens_ref(T, gsin, gcos, rnc, col, j)
        assert hess.get()[j * (kd + 1):(j + 1) * (kd + 1)].tobytes() == col.tobytes()
        assert small["gsin"].get().tobytes() == gsin.tobytes() and small["gcos"].get().tobytes() == gcos.tobytes()
        assert small["rnc"].get().tobytes() == rnc.tobytes() and small["rnorm"].get()[0] == tau
        assert fin.get()[0] == j + 1 and list(ctl.get()[:2]) == [0, it_ + 1]


def sp_matvec(rp, ci, va, x):
    import scipy.sparse as sp
    n = len(rp) - 1
    return sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(n, len(x))) @ x
