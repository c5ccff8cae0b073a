"""The fused CG kernels for several right-hand sides (csrc/fused_cg_mrhs.cu) one at a time through the
C ABI against numpy and the oracle, then solver::Cg with with_fused_multi_rhs(true) against the
oracle's multi-column CG.

As in test_fused_cg_gpu.py: element-wise results are compared BIT FOR BIT (the library is built with
-fmad=false, numpy in the value type rounds as the device does); sums on small-integer data must be
exact (every partial sum of any order is); sums on random data must lie within gamma_h * sum |t| of
math.fsum, which bounds any summation order.  Every vector is n x k row-major (stride k)."""

import numpy as np
import pytest

import workloads as W
from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_fused_cg_gpu import Backend, assert_sum_within, expected_status, int_sum, rand_csr, tau_of
from tests.test_parity_gpu import CSR_KINDS, csr_case
from tests.test_solvers_gpu import ref_jacobi, true_rel_res

pytestmark = pytest.mark.gpu

VTS = ["f64", "f32"]
ITS = ["i32", "i64"]
KS = [2, 3, 5, 8, 17, 32]
STOPPED = 0x40 | 1
SPMV_THREADS, SPMV_CTAS_PER_SM = 256, 8  # fused_cg_mrhs.cu: the SpMV's block size and grid cap per SM


@pytest.fixture(scope="module")
def backend():
    from ginkgo_b200 import _lib
    be = Backend(_lib.lib(), mock=False)
    yield be
    be.close()


@pytest.fixture
def dev(backend):
    yield backend
    backend.release()


@pytest.fixture(scope="module")
def hexec():
    from ginkgo_b200 import api
    return api.HostExecutor(0)


def lanes(k):
    p = 2
    while p < k:
        p *= 2
    return p


def work(dev, vt, k):
    size = getattr(dev.l, "b200_cg_mrhs_work_size_" + vt)(dev.ctx, k)
    return dev.put(np.full(size, np.nan, VT[vt]))


def nans(shape, vt):
    return np.full(shape, np.nan, VT[vt])


def oracle_spmv(orc, vt, it, n, m, rp, ci, va, b, k):
    c = np.zeros((n, k), VT[vt])
    orc("csr_spmv_%s_%s" % (vt, it), n, m, len(va), rp, ci, va, np.ascontiguousarray(b), k, k, c, k)
    return c


def big_case(vt, it, num_sms, k):
    """enough rows for the SpMV grid to reach its cap at this k"""
    n = SPMV_CTAS_PER_SM * num_sms * (SPMV_THREADS // lanes(k)) * 4 + 1000
    rng = np.random.default_rng(5)
    rp, ci = rand_csr(rng, n, n, rng.integers(2, 9, size=n))
    return n, n, rp.astype(IT[it]), ci.astype(IT[it]), rng.uniform(-1, 1, len(ci)).astype(VT[vt])


def check_dots(got, p, q, vt, exact):
    k = p.shape[1]
    for j in range(k):
        if exact:
            assert got[j] == int_sum(p[:, j], q[:, j]), j
        else:
            assert_sum_within(got[j], p[:, j].astype(VT[vt]) * q[:, j], vt, "dot %d" % j)


# --------------------------------------------------------------------------- A. spmv_mdot
def run_spmv_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, data, graph=False):
    rng = np.random.default_rng(k)
    if data == "int":
        va = rng.integers(-1, 2, size=len(va)).astype(VT[vt])
        p = rng.integers(-2, 3, size=(m, k)).astype(VT[vt])
    else:
        p = rng.uniform(-1, 1, size=(m, k)).astype(VT[vt])
    ref = oracle_spmv(orc, vt, it, n, m, rp, ci, va, p, k)
    d = [dev.put(a) for a in (rp, ci, va, p)]
    q, dots, w = dev.put(nans((n, k), vt)), dev.put(nans(k, vt)), work(dev, vt, k)
    args = ("csr_spmv_mdot_%s_%s" % (vt, it), n, m, len(va), d[0], d[1], d[2], d[3], k, q, dots, w, None)
    dev.call(*args)
    got_q, got_dots = q.get().reshape(n, k), dots.get()
    assert got_q.tobytes() == ref.tobytes()
    check_dots(got_dots, p[:n], ref, vt, data == "int")
    if graph:  # a replayed graph gives the eager run's bits, twice
        q.set(nans((n, k), vt))
        dots.set(nans(k, vt))
        g = dev.capture(lambda: dev.call(*args))
        for _ in range(2):
            dev.call("graph_launch", g)
            dev.sync()
            assert q.get().tobytes() == got_q.tobytes() and dots.get().tobytes() == got_dots.tobytes()
    return got_q, got_dots


@pytest.mark.parametrize("kind", CSR_KINDS)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_mdot(dev, orc, kind, k, vt, it, data):
    n, m, rp, ci, va = csr_case(np.random.default_rng(17), kind, vt, it)
    m = max(n, m)  # p has a row per column and the dot reads its first n rows
    run_spmv_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, data)


@pytest.mark.parametrize("k", [2, 8, 32])
@pytest.mark.parametrize("vt,it", [("f64", "i32"), ("f32", "i64")])
def test_spmv_mdot_capped_grid_and_graph(dev, orc, k, vt, it):
    n, m, rp, ci, va = big_case(vt, it, dev.num_sms, k)
    assert n / (SPMV_THREADS // lanes(k) * 4) > SPMV_CTAS_PER_SM * dev.num_sms
    run_spmv_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, "rand", graph=True)
    run_spmv_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, "int")


@pytest.mark.parametrize("vt", VTS)
def test_spmv_mdot_empty_matrix_and_stopped(dev, vt):
    k = 5
    rp = np.zeros(1, np.int32)
    dots, w = dev.put(nans(k, vt)), work(dev, vt, k)
    e = dev.put(np.zeros(1, np.int32))
    dev.call("csr_spmv_mdot_%s_i32" % vt, 0, 0, 0, dev.put(rp), e, e, e, k, e, dots, w, None)
    assert np.array_equal(dots.get(), np.zeros(k, VT[vt]))
    # a raised ctl[0] turns the launch into a no-op
    n = 50
    rp = np.arange(n + 1, dtype=np.int32)
    d = [dev.put(a) for a in (rp, np.arange(n, dtype=np.int32), np.ones(n, VT[vt]), np.ones((n, k), VT[vt]))]
    q, dots = dev.put(nans((n, k), vt)), dev.put(nans(k, vt))
    ctl = dev.put(np.array([1, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dev.call("csr_spmv_mdot_%s_i32" % vt, n, n, n, d[0], d[1], d[2], d[3], k, q, dots, w, ctl)
    assert np.isnan(q.get()).all() and np.isnan(dots.get()).all()


# --------------------------------------------------------------------------- B. step kernels
def scalars(k, vt, rho, prev, pq, rr, tau0, thr):
    return np.concatenate([np.asarray(a, VT[vt]).reshape(k) for a in (rho, prev, pq, rr, tau0, thr)])


@pytest.mark.parametrize("k", [2, 5, 17, 32])
@pytest.mark.parametrize("vt", VTS)
def test_step_p(dev, k, vt):
    v = VT[vt]
    rng = np.random.default_rng(k)
    n = 3001
    z, p = rng.uniform(-1, 1, (n, k)).astype(v), rng.uniform(-1, 1, (n, k)).astype(v)
    rho, prev = rng.uniform(0.5, 2, k).astype(v), rng.uniform(0.5, 2, k).astype(v)
    prev[1] = 0  # p = z
    status = np.zeros(k, np.uint8)
    status[k - 1] = STOPPED
    p[:, k - 1] = np.nan
    sc = scalars(k, vt, rho, prev, np.zeros(k), np.zeros(k), np.zeros(k), np.zeros(k))
    pd, zd, scd, std, ctl = dev.put(p), dev.put(z), dev.put(sc), dev.put(status), dev.put(np.zeros(8, np.int32))
    dev.call("cg_mrhs_step_p_" + vt, n, k, pd, zd, scd, std, ctl)
    want = p.copy()
    for j in range(k - 1):
        want[:, j] = z[:, j] if prev[j] == 0 else z[:, j] + v(rho[j] / prev[j]) * p[:, j]
    got = pd.get().reshape(n, k)
    assert got.tobytes() == want.tobytes()
    # once ctl[0] != 0 nothing moves
    ctl.set(np.array([1, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dev.call("cg_mrhs_step_p_" + vt, n, k, pd, zd, scd, std, ctl)
    assert pd.get().tobytes() == got.tobytes()


def numpy_step_xr(x, r, p, q, inv_diag, sc, status, k, vt):
    """the vectors and sums step_xr produces for every running column"""
    v = VT[vt]
    x, r = x.copy(), r.copy()
    z = np.full_like(r, np.nan)
    for j in range(k):
        if status[j] & 0x3f:
            continue
        pq = sc[2 * k + j]
        if pq != 0:
            alpha = v(sc[j] / pq)
            x[:, j] = x[:, j] + alpha * p[:, j]
            r[:, j] = r[:, j] - alpha * q[:, j]
        z[:, j] = r[:, j] * inv_diag if inv_diag is not None else r[:, j]
    return x, r, z


@pytest.mark.parametrize("k", [2, 5, 17, 32])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("diag", [False, True])
@pytest.mark.parametrize("data", ["int", "rand"])
def test_step_xr(dev, k, vt, diag, data):
    v = VT[vt]
    rng = np.random.default_rng(3 * k)
    n = 4099
    if data == "int":
        mk = lambda: rng.integers(-3, 4, (n, k)).astype(v)  # noqa: E731
        inv_diag = rng.integers(1, 3, n).astype(v) if diag else None
        sc_rho, sc_pq = np.ones(k, v), np.ones(k, v)  # alpha = 1: integer vectors stay integers
    else:
        mk = lambda: rng.uniform(-1, 1, (n, k)).astype(v)  # noqa: E731
        inv_diag = rng.uniform(0.5, 2, n).astype(v) if diag else None
        sc_rho, sc_pq = rng.uniform(0.5, 2, k).astype(v), rng.uniform(0.5, 2, k).astype(v)
    x, r, p, q = mk(), mk(), mk(), mk()
    sc_pq[0] = 0  # no update in column 0
    status = np.zeros(k, np.uint8)
    status[1] = STOPPED  # untouched, NaN sentinels survive
    for a in (x, r, p):
        a[:, 1] = np.nan
    sc = scalars(k, vt, sc_rho, np.ones(k), sc_pq, np.zeros(k), np.ones(k), np.full(k, 1e-30))
    ctl = np.array([0, 4, 100, 1, 1, 0, 0, 0], np.int32)  # iteration 5 next, max 100, ResidualNorm
    d = {nm: dev.put(a) for nm, a in dict(x=x, r=r, p=p, q=q, z=nans((n, k), vt), sc=sc, st=status,
                                          ctl=ctl).items()}
    dd = dev.put(inv_diag) if diag else None
    dev.call("cg_mrhs_step_xr_" + vt, n, k, d["x"], d["r"], d["p"], d["q"], d["z"], dd, d["sc"], d["st"],
             d["ctl"], work(dev, vt, k))
    wx, wr, wz = numpy_step_xr(x, r, p, q, inv_diag, sc, status, k, vt)
    gx, gr, gz = (d[nm].get().reshape(n, k) for nm in ("x", "r", "z"))
    assert gx.tobytes() == wx.tobytes() and gr.tobytes() == wr.tobytes()
    assert np.isnan(gz[:, 1]).all() and np.isnan(d["p"].get().reshape(n, k)[:, 1]).all()
    run = [j for j in range(k) if j != 1]
    assert gz[:, run].tobytes() == wz[:, run].tobytes()
    gsc, gst, gctl = d["sc"].get(), d["st"].get(), d["ctl"].get()
    assert gctl[1] == 5 and gctl[0] == 0 and gst[1] == STOPPED
    for j in run:
        assert gsc[k + j] == sc_rho[j]  # prev_rho = rho
        if data == "int":
            assert gsc[j] == int_sum(wr[:, j], wz[:, j]) and gsc[3 * k + j] == int_sum(wr[:, j], wr[:, j])
        else:
            assert_sum_within(gsc[j], wr[:, j] * wz[:, j], vt, "rho %d" % j)
            assert_sum_within(gsc[3 * k + j], wr[:, j] * wr[:, j], vt, "rr %d" % j)
        assert gst[j] == 0
    # a stopped solver: nothing moves
    d["ctl"].set(np.array([1, 5, 100, 1, 1, 0, 0, 0], np.int32))
    before = [d[nm].get().tobytes() for nm in ("x", "r", "z", "sc", "st")]
    dev.call("cg_mrhs_step_xr_" + vt, n, k, d["x"], d["r"], d["p"], d["q"], d["z"], dd, d["sc"], d["st"],
             d["ctl"], work(dev, vt, k))
    assert [d[nm].get().tobytes() for nm in ("x", "r", "z", "sc", "st")] == before


# --------------------------------------------------------------------------- C. lock-step + stopping table
def arrow(n, vt, it):
    """SPD arrow matrix: a dense first row / column (a row long enough to be split over CTAs by the
    one-column plan) and a dominant diagonal"""
    rows, cols, vals = [], [], []
    for i in range(n):
        if i == 0:
            cs = list(range(n))
        else:
            cs = [0, i]
        for c in cs:
            rows.append(i)
            cols.append(c)
            vals.append(float(n + 2) if c == i else -1.0 / (1 + (i + c) % 7))
    rp = np.zeros(n + 1, np.int64)
    np.add.at(rp, np.array(rows) + 1, 1)
    rp = np.cumsum(rp)
    return rp.astype(IT[it]), np.array(cols).astype(IT[it]), np.array(vals).astype(VT[vt])


@pytest.mark.parametrize("vt,it,k", [("f64", "i32", 5), ("f32", "i64", 3), ("f64", "i64", 17)])
@pytest.mark.parametrize("res_kind,baseline,iter_first", [(1, 0, True), (2, 1, False), (1, 2, True)])
def test_lock_step(dev, orc, vt, it, k, res_kind, baseline, iter_first):
    """30+ iterations one launch at a time against numpy fed the device's scalars: vectors bit-equal,
    every column's status as the criteria say from its own rho / rr, ctl[0] only with the last column"""
    v = VT[vt]
    n = 5000
    rp, ci, va = arrow(n, vt, it)
    rng = np.random.default_rng(k)
    b = rng.uniform(-1, 1, (n, k)).astype(v)
    b[:, 0] = 0  # converges at iteration 0 under rhs_norm / absolute
    b[:, 1] *= 1e-3
    inv_diag = (v(1) / va[np.asarray(rp[:-1], np.int64) + 0]).astype(v)  # diagonal of row 0 is entry 0
    inv_diag[1:] = v(1) / va[np.asarray(rp[1:-1], np.int64) + 1]
    max_iters = 34
    red = 1e-12 if vt == "f64" else 1e-5
    x = np.zeros((n, k), v)
    r = b.copy()  # x = 0
    d = {nm: dev.put(a) for nm, a in dict(x=x, r=r, z=nans((n, k), vt), p=nans((n, k), vt), q=nans((n, k), vt),
                                          sc=np.zeros(6 * k, v), st=np.full(k, 0xff, np.uint8),
                                          ctl=np.zeros(8, np.int32)).items()}
    A = [dev.put(a) for a in (rp, ci, va)]
    dd, w = dev.put(inv_diag), work(dev, vt, k)
    if baseline == 0:
        sc0 = np.zeros(6 * k, v)
        sc0[4 * k:5 * k] = np.sqrt(np.sum(b.astype(np.float64) ** 2, axis=0)).astype(v)
        d["sc"].set(sc0)
    dev.call("cg_mrhs_init_" + vt, n, k, d["r"], d["z"], d["p"], d["q"], dd, d["sc"], d["st"], d["ctl"], w,
             max_iters, res_kind, int(iter_first), baseline, v(red))
    p = np.zeros((n, k), v)
    z = r * inv_diag[:, None]
    sc = d["sc"].get()
    tau0 = sc[4 * k:5 * k]
    if baseline == 1:
        assert tau0.tobytes() == np.sqrt(sc[3 * k:4 * k]).tobytes()
    if baseline == 2:
        assert np.all(tau0 == 1)
    assert sc[5 * k:].tobytes() == (v(red) * tau0).astype(v).tobytes()
    status = np.zeros(k, np.uint8)
    stop_iter = {}
    for iteration in range(0, max_iters + 2):
        sc, st, ctl = d["sc"].get(), d["st"].get(), d["ctl"].get()
        assert ctl[1] == iteration
        if len(stop_iter) < k:
            for j in range(k):
                if status[j] & 0x3f:
                    assert st[j] == status[j]
                    continue
                want = expected_status(iteration, max_iters, res_kind, iter_first,
                                       tau_of(vt, res_kind, sc[j], sc[3 * k + j]), sc[5 * k + j])
                assert st[j] == want, (iteration, j)
                if want:
                    status[j] = want
                    stop_iter[j] = iteration
            assert (ctl[0] != 0) == (len(stop_iter) == k)
        assert np.array_equal(d["z"].get().reshape(n, k)[:, status & 0x3f == 0], z[:, status & 0x3f == 0])
        if ctl[0]:
            frozen = [d[nm].get().tobytes() for nm in ("x", "r", "p", "sc", "st", "ctl")]
        # one iteration, checked kernel by kernel
        dev.call("cg_mrhs_step_p_" + vt, n, k, d["p"], d["z"], d["sc"], d["st"], d["ctl"])
        for j in range(k):
            if not status[j] & 0x3f:
                prev, rho = sc[k + j], sc[j]
                p[:, j] = z[:, j] if prev == 0 else z[:, j] + v(rho / prev) * p[:, j]
        gp = d["p"].get().reshape(n, k)
        if not ctl[0]:
            assert gp.tobytes() == p.tobytes()
        dev.call("csr_spmv_mdot_%s_%s" % (vt, it), n, n, len(va), A[0], A[1], A[2], d["p"], k, d["q"],
                 d["sc"].at(2 * k), w, d["ctl"])
        q = oracle_spmv(orc, vt, it, n, n, rp, ci, va, gp, k)
        if not ctl[0]:
            assert d["q"].get().reshape(n, k).tobytes() == q.tobytes()
        sc_now = d["sc"].get()
        dev.call("cg_mrhs_step_xr_" + vt, n, k, d["x"], d["r"], d["p"], d["q"], d["z"], dd, d["sc"], d["st"],
                 d["ctl"], w)
        if ctl[0]:
            assert [d[nm].get().tobytes() for nm in ("x", "r", "p", "sc", "st", "ctl")] == frozen
            break
        x, r, z = numpy_step_xr(x, r, p, q, inv_diag, sc_now, status, k, vt)
        assert d["x"].get().reshape(n, k).tobytes() == x.tobytes()
        assert d["r"].get().reshape(n, k).tobytes() == r.tobytes()
    assert len(stop_iter) == k and stop_iter[0] == 0 and len(set(stop_iter.values())) >= 2
    st = d["st"].get()
    assert all(s & 0x40 for s in st)  # finalized


# --------------------------------------------------------------------------- D. host solver
def mrhs_rhs(n, k, vt, seed=6):
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
    b[:, 1] *= 1e-3
    return b.astype(VT[vt])


def device_solve(hexec, vt, rp, ci, va, b, x0, precond=0, strided=0, **kw):
    import torch
    from ginkgo_b200 import api
    dev = hexec.device
    k = b.shape[1]
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(dev) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(np.pad(b, ((0, 0), (0, strided))))).to(dev)
        tx = torch.from_numpy(np.ascontiguousarray(np.pad(x0, ((0, 0), (0, strided))))).to(dev).clone()
    n = len(rp) - 1
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "cg", A, precond_max_bs=precond, **kw)
    s.apply(api.host_dense(hexec, tb, cols=k), api.host_dense(hexec, tx, cols=k))
    hexec.synchronize()
    return tx.cpu().numpy()[:, :k], s.num_iterations, s.stop_statuses, s.used_fused


@pytest.mark.parametrize("vt,it,precond", [("f64", "i32", 0), ("f64", "i32", 1), ("f32", "i32", 1),
                                           ("f64", "i64", 0), ("f32", "i64", 0)])
@pytest.mark.parametrize("res_kind", [1, 2])
@pytest.mark.parametrize("baseline", [0, 1, 2])
@pytest.mark.parametrize("iter_first", [True, False])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_solver_matches_oracle(hexec, vt, it, precond, res_kind, baseline, iter_first, check_every):
    rp, ci, va = W.laplace(24, 2, vdtype=VT[vt])
    rp, ci = rp.astype(IT[it]), ci.astype(IT[it])
    n, k = len(rp) - 1, 4
    b = mrhs_rhs(n, k, vt)
    x0 = np.zeros((n, k), VT[vt])
    red = 1e-8 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10
    kw = dict(max_iters=1000, res_kind=res_kind, baseline=baseline, reduction=red)
    jac = ref_jacobi(vt, rp.astype(np.int32), ci.astype(np.int32), va, 1, None) if precond else None
    rp32, ci32 = rp.astype(np.int32), ci.astype(np.int32)  # the oracle's solvers take int32 indices
    xo, ito, stop_o = H.orc_solve("cg", vt, rp32, ci32, va, b, x0, precond, jac, iter_first=int(iter_first), **kw)
    xd, itd, stop_d, used = device_solve(hexec, vt, rp, ci, va, b, x0, precond, iter_first=iter_first,
                                         fused_multi_rhs=True, check_every=check_every, **kw)
    assert used
    assert stop_d == list(stop_o)
    assert abs(itd - ito) <= 2
    tol = 1e-7 if vt == "f64" else 1e-2
    for j in range(k):
        assert H.rel_err(xo[:, j], xd[:, j]) <= tol, j


def test_solver_columns_stop_at_their_own_iterations(hexec):
    """the columns converge at different iterations (column 1 is b scaled by 1e-3, column 3 is zero
    and stops at iteration 0); the statuses are the oracle's and every column is solved"""
    rp, ci, va = W.laplace(40, 2)
    n, k = len(rp) - 1, 5
    b = mrhs_rhs(n, k, "f64", seed=9)
    b[:, 3] = 0
    x0 = np.zeros((n, k))
    kw = dict(max_iters=2000, reduction=1e-9, baseline=0)
    xo, ito, stop_o = H.orc_solve("cg", "f64", rp, ci, va, b, x0, **kw)
    xd, itd, stop_d, used = device_solve(hexec, "f64", rp, ci, va, b, x0, fused_multi_rhs=True, **kw)
    assert used and stop_d == list(stop_o) and abs(itd - ito) <= 2
    assert stop_d[3] == 0x80 | 0x40 | 2 and np.all(xd[:, 3] == 0)
    assert np.all(true_rel_res(rp, ci, va, b[:, [0, 1, 2, 4]], xd[:, [0, 1, 2, 4]]) <= 1.2e-9)


def test_fallbacks(hexec):
    rp, ci, va = W.laplace(12, 2)
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8)
    b33 = mrhs_rhs(n, 33, "f64")
    assert not device_solve(hexec, "f64", rp, ci, va, b33, np.zeros_like(b33), 1, fused_multi_rhs=True, **kw)[3]
    b4 = mrhs_rhs(n, 4, "f64")
    x0 = np.zeros_like(b4)
    # stride != k
    xs, its, sts, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, strided=2, fused_multi_rhs=True, **kw)
    assert not used
    # the switch is off by default: the loop, as before
    xl, itl, stl, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, **kw)
    assert not used and sts == stl == [0x80 | 0x40 | 2] * 4
    # block Jacobi takes the loop
    import torch
    from ginkgo_b200 import api
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(b4).to(hexec.device)
        tx = torch.zeros_like(tb)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "cg", A, precond_max_bs=4, block_ptrs=np.arange(0, n + 1, 4, dtype=np.int32),
                       fused_multi_rhs=True, **kw)
    s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
    assert not s.used_fused
    # the new path agrees with the loop within rounding and in its statuses
    xf, itf, stf, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, fused_multi_rhs=True, **kw)
    assert used and stf == stl and abs(itf - itl) <= 2
    # one column: the one-column path, the same bits with the switch on or off
    b1, x1 = b4[:, :1].copy(), x0[:, :1].copy()
    xa, ita, sta, usa = device_solve(hexec, "f64", rp, ci, va, b1, x1, 1, fused_multi_rhs=True, **kw)
    xb, itb, stb, usb = device_solve(hexec, "f64", rp, ci, va, b1, x1, 1, **kw)
    assert usa and usb and (ita, sta) == (itb, stb) and xa.tobytes() == xb.tobytes()


def test_two_applies_give_the_same_bits(hexec):
    """deterministic sums: the same solve gives the same bits and iterations, with another k between"""
    rp, ci, va = W.laplace(30, 2)
    n = len(rp) - 1
    outs = []
    for k in (6, 3, 6):
        b = mrhs_rhs(n, k, "f64", seed=1)
        outs.append(device_solve(hexec, "f64", rp, ci, va, b, np.zeros_like(b), 1, fused_multi_rhs=True,
                                 max_iters=500, reduction=1e-10))
    assert outs[0][0].tobytes() == outs[2][0].tobytes() and outs[0][1:] == outs[2][1:]
    assert outs[1][2] == [0x80 | 0x40 | 2] * 3
