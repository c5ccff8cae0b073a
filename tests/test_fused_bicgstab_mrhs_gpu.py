"""The fused BiCGStab kernels for several right-hand sides (csrc/fused_bicgstab_mrhs.cu) one at a time
through the C ABI against numpy and the oracle, then solver::Bicgstab with with_fused_multi_rhs(true)
against the oracle's multi-column BiCGStab.

As in test_fused_cg_mrhs_gpu.py: element-wise results are compared BIT FOR BIT (the library is built
with -fmad=false, numpy in the value type rounds as the device does); sums on small-integer data must
be exact; sums on random data must lie within gamma_h * sum |t| of math.fsum, which bounds any
summation order.  Every vector is n x k row-major (stride k).

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock."""
import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_fused_bicgstab_gpu import convective_arrow, true_rel_res, upwind
from tests.test_fused_cg_gpu import (arrow_inv_diag, assert_sum_within, backend, dev,  # noqa: F401
                                     expected_status, hexec, int_sum, tau_of)
from tests.test_fused_cg_mrhs_gpu import big_case, lanes, nans, oracle_spmv
from tests.test_parity_gpu import CSR_KINDS, csr_case

pytestmark = pytest.mark.gpu

VTS = ["f64", "f32"]
ITS = ["i32", "i64"]
KS = [2, 3, 5, 8, 17, 32]
STOPPED = 0x40 | 1
MID_STOPPED = 0x80 | 2     # converged at the mid check, not yet finalized
FIN_CONV_2 = 0x80 | 0x40 | 2
SPMV_THREADS, SPMV_CTAS_PER_SM = 256, 8  # fused_mrhs.cuh: the SpMV's block size and grid cap per SM


def work(dev, vt, k):
    size = getattr(dev.l, "b200_bicgstab_mrhs_work_size_" + vt)(dev.ctx, k)
    return dev.put(np.full(size, np.nan, VT[vt]))


def check_sums(got, a, b, vt, exact, what):
    for j in range(a.shape[1]):
        if exact:
            assert got[j] == int_sum(a[:, j], b[:, j]), (what, j)
        else:
            assert_sum_within(got[j], a[:, j].astype(VT[vt]) * b[:, j], vt, "%s %d" % (what, j))


# --------------------------------------------------------------------------- A. spmv_mdot2
def run_mdot2(dev, orc, vt, it, n, m, rp, ci, va, k, data, graph=False, with_dots2=True):
    rng = np.random.default_rng(k + 100)
    if data == "int":
        va = rng.integers(-1, 2, size=len(va)).astype(VT[vt])
        b = rng.integers(-2, 3, size=(m, k)).astype(VT[vt])
        w = rng.integers(-2, 3, size=(n, k)).astype(VT[vt])
    else:
        b = rng.uniform(-1, 1, size=(m, k)).astype(VT[vt])
        w = rng.uniform(-1, 1, size=(n, k)).astype(VT[vt])
    ref = oracle_spmv(orc, vt, it, n, m, rp, ci, va, b, k)
    d = [dev.put(a) for a in (rp, ci, va, b, w)]
    c, dots, dots2, wk = dev.put(nans((n, k), vt)), dev.put(nans(k, vt)), dev.put(nans(k, vt)), work(dev, vt, k)
    args = ("csr_spmv_mdot2_%s_%s" % (vt, it), n, m, len(va), d[0], d[1], d[2], d[3], k, c, d[4], dots,
            dots2 if with_dots2 else None, wk, None)
    dev.call(*args)
    got_c, got_d, got_d2 = c.get().reshape(n, k), dots.get(), dots2.get()
    assert got_c.tobytes() == ref.tobytes()
    check_sums(got_d, w, ref, vt, data == "int", "w.c")
    if with_dots2:
        check_sums(got_d2, ref, ref, vt, data == "int", "c.c")
    else:
        assert np.isnan(got_d2).all()
    if graph:  # a replayed graph gives the eager run's bits, twice
        c.set(nans((n, k), vt))
        dots.set(nans(k, vt))
        dots2.set(nans(k, vt))
        g = dev.capture(lambda: dev.call(*args))
        for _ in range(2):
            dev.call("graph_launch", g)
            dev.sync()
            assert c.get().tobytes() == got_c.tobytes()
            assert dots.get().tobytes() == got_d.tobytes() and dots2.get().tobytes() == got_d2.tobytes()


@pytest.mark.parametrize("kind", CSR_KINDS)
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_mdot2(dev, orc, kind, k, vt, it, data):
    n, m, rp, ci, va = csr_case(np.random.default_rng(17), kind, vt, it)
    m = max(n, m)
    run_mdot2(dev, orc, vt, it, n, m, rp, ci, va, k, data)


@pytest.mark.parametrize("k", [2, 5, 32])
@pytest.mark.parametrize("vt,it", [("f64", "i32"), ("f32", "i64")])
def test_spmv_mdot2_split_long_rows(dev, orc, k, vt, it):
    """the arrow matrix: a dense first row that the one-column plan splits over CTAs"""
    rp, ci, va = convective_arrow(vt)
    n = len(rp) - 1
    run_mdot2(dev, orc, vt, it, n, n, rp.astype(IT[it]), ci.astype(IT[it]), va, k, "rand")
    run_mdot2(dev, orc, vt, it, n, n, rp.astype(IT[it]), ci.astype(IT[it]), va, k, "int", with_dots2=False)


@pytest.mark.parametrize("k", [2, 8, 32])
@pytest.mark.parametrize("vt,it", [("f64", "i32"), ("f32", "i64")])
def test_spmv_mdot2_capped_grid_and_graph(dev, orc, k, vt, it):
    n, m, rp, ci, va = big_case(vt, it, dev.num_sms, k)
    assert n / (SPMV_THREADS // lanes(k) * 4) > SPMV_CTAS_PER_SM * dev.num_sms
    run_mdot2(dev, orc, vt, it, n, m, rp, ci, va, k, "rand", graph=True)
    run_mdot2(dev, orc, vt, it, n, m, rp, ci, va, k, "int", with_dots2=False)


@pytest.mark.parametrize("vt", VTS)
def test_spmv_mdot2_empty_matrix_and_stopped(dev, vt):
    k = 5
    dots, dots2, w = dev.put(nans(k, vt)), dev.put(nans(k, vt)), work(dev, vt, k)
    e = dev.put(np.zeros(1, np.int32))
    dev.call("csr_spmv_mdot2_%s_i32" % vt, 0, 0, 0, e, e, e, e, k, e, e, dots, dots2, w, None)
    assert np.array_equal(dots.get(), np.zeros(k, VT[vt])) and np.array_equal(dots2.get(), np.zeros(k, VT[vt]))
    # a raised ctl[0] turns the launch into a no-op
    n = 50
    rp = np.arange(n + 1, dtype=np.int32)
    d = [dev.put(a) for a in (rp, np.arange(n, dtype=np.int32), np.ones(n, VT[vt]), np.ones((n, k), VT[vt]))]
    c, dots, dots2 = dev.put(nans((n, k), vt)), dev.put(nans(k, vt)), dev.put(nans(k, vt))
    ctl = dev.put(np.array([1, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dev.call("csr_spmv_mdot2_%s_i32" % vt, n, n, n, d[0], d[1], d[2], d[3], k, c, d[3], dots, dots2, w, ctl)
    assert np.isnan(c.get()).all() and np.isnan(dots.get()).all() and np.isnan(dots2.get()).all()


# --------------------------------------------------------------------------- B. step kernels
def stopped(s):
    return (s & 0x3f) != 0


def np_step_p(p, r, v, d, sc, status, k, vt):
    t = VT[vt]
    p, y = p.copy(), np.full_like(p, np.nan)
    for j in range(k):
        if stopped(status[j]):
            continue
        rho, prev, alpha, omega = sc[j], sc[k + j], sc[6 * k + j], sc[7 * k + j]
        if t(prev * omega) != 0:
            tmp = t(t(t(rho / prev) * alpha) / omega)
            p[:, j] = r[:, j] + tmp * (p[:, j] - omega * v[:, j])
        else:
            p[:, j] = r[:, j]
        y[:, j] = p[:, j] * d if d is not None else p[:, j]
    return p, y


def np_step_s(r, v, d, sc, status, k, vt):
    t = VT[vt]
    s, z = np.full_like(r, np.nan), np.full_like(r, np.nan)
    alpha = {}
    for j in range(k):
        if stopped(status[j]):
            continue
        beta = sc[2 * k + j]
        if beta != 0:
            alpha[j] = t(sc[j] / beta)
            s[:, j] = r[:, j] - alpha[j] * v[:, j]
        else:
            alpha[j] = t(0)
            s[:, j] = r[:, j]
        z[:, j] = s[:, j] * d if d is not None else s[:, j]
    return s, z, alpha


def np_step_xr(x, r, s, t_, y, z, sc, status, k, vt):
    """x, r after step_xr: running columns get bicgstab::step_3, a column stopped at the mid check
    (stopped, not finalized) bicgstab::finalize"""
    t = VT[vt]
    x, r = x.copy(), r.copy()
    for j in range(k):
        alpha = sc[6 * k + j]
        if stopped(status[j]):
            if not status[j] & 0x40:
                x[:, j] = x[:, j] + alpha * y[:, j]
            continue
        beta = sc[2 * k + j]
        omega = t(sc[8 * k + j] / beta) if beta != 0 else t(0)
        x[:, j] = x[:, j] + (alpha * y[:, j] + omega * z[:, j])
        r[:, j] = s[:, j] - omega * t_[:, j]
    return x, r


def scalars(k, vt, **kw):
    names = ["rho", "prev", "beta", "rr", "tau0", "thr", "alpha", "omega", "gamma", "ss"]
    return np.concatenate([np.broadcast_to(np.asarray(kw.get(nm, 0), VT[vt]), (k,)) for nm in names]).copy()


@pytest.mark.parametrize("k", [2, 5, 17, 32])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("diag", [False, True])
def test_step_p(dev, k, vt, diag):
    v = VT[vt]
    rng = np.random.default_rng(k)
    n = 3001
    p, r, vv = (rng.uniform(-1, 1, (n, k)).astype(v) for _ in range(3))
    d = rng.uniform(0.5, 2, n).astype(v) if diag else None
    sc = scalars(k, vt, rho=rng.uniform(0.5, 2, k), prev=rng.uniform(0.5, 2, k), alpha=rng.uniform(0.5, 2, k),
                 omega=rng.uniform(0.5, 2, k))
    sc[k + 0] = 0       # prev_rho = 0: p = r
    sc[7 * k + 1] = 0   # omega = 0: p = r
    status = np.zeros(k, np.uint8)
    status[k - 1] = STOPPED
    p[:, k - 1] = np.nan
    y0 = nans((n, k), vt)
    pd, rd, vd, yd, scd, std = (dev.put(a) for a in (p, r, vv, y0, sc, status))
    ctl = dev.put(np.zeros(8, np.int32))
    dev.call("bicgstab_mrhs_step_p_" + vt, n, k, pd, rd, vd, yd, dev.put(d) if diag else None, scd, std, ctl)
    wp, wy = np_step_p(p, r, vv, d, sc, status, k, vt)
    gp, gy = pd.get().reshape(n, k), yd.get().reshape(n, k)
    assert gp.tobytes() == wp.tobytes() and gy.tobytes() == wy.tobytes()
    assert np.array_equal(gp[:, 0], r[:, 0]) and (k == 2 or np.array_equal(gp[:, 1], r[:, 1]))
    # once ctl[0] != 0 nothing moves
    ctl.set(np.array([1, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dev.call("bicgstab_mrhs_step_p_" + vt, n, k, pd, rd, vd, yd, None, scd, std, ctl)
    assert pd.get().tobytes() == gp.tobytes() and yd.get().tobytes() == gy.tobytes()


@pytest.mark.parametrize("k", [3, 5, 17, 32])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("diag", [False, True])
@pytest.mark.parametrize("data", ["int", "rand"])
def test_step_s_and_mid_check(dev, k, vt, diag, data):
    """s, z bit for bit; ||s||^2 per column; the mid check stops column 2 (its s is zero) without the
    finalized bit and raises ctl[5]; beta = 0 in column 0 gives alpha = 0 and s = r"""
    v = VT[vt]
    rng = np.random.default_rng(5 * k)
    n = 4099
    if data == "int":
        r, vv = rng.integers(-3, 4, (n, k)).astype(v), rng.integers(-3, 4, (n, k)).astype(v)
        d = rng.integers(1, 3, n).astype(v) if diag else None
        rho, beta = np.ones(k, v), np.ones(k, v)
    else:
        r, vv = rng.uniform(-1, 1, (n, k)).astype(v), rng.uniform(-1, 1, (n, k)).astype(v)
        d = rng.uniform(0.5, 2, n).astype(v) if diag else None
        rho, beta = rng.uniform(0.5, 2, k).astype(v), rng.uniform(0.5, 2, k).astype(v)
    beta[0] = 0
    rho[2], beta[2] = 1, 1
    vv[:, 2] = r[:, 2]  # s_2 = r_2 - 1 * r_2 = 0
    status = np.zeros(k, np.uint8)
    status[1] = STOPPED
    sc = scalars(k, vt, rho=rho, beta=beta, thr=np.full(k, 1e-30), alpha=7, ss=7)
    ctl = np.array([0, 4, 100, 1, 1, 0, 0, 0], np.int32)  # iteration 4, max 100, ResidualNorm
    dd = {nm: dev.put(a) for nm, a in dict(r=r, v=vv, s=nans((n, k), vt), z=nans((n, k), vt), sc=sc, st=status,
                                           ctl=ctl).items()}
    dev.call("bicgstab_mrhs_step_s_" + vt, n, k, dd["r"], dd["v"], dd["s"], dd["z"], dev.put(d) if diag else None,
             dd["sc"], dd["st"], dd["ctl"], work(dev, vt, k))
    ws, wz, alpha = np_step_s(r, vv, d, sc, status, k, vt)
    gs, gz = dd["s"].get().reshape(n, k), dd["z"].get().reshape(n, k)
    assert gs.tobytes() == ws.tobytes() and gz.tobytes() == wz.tobytes()  # NaN in the stopped column too
    gsc, gst, gctl = dd["sc"].get(), dd["st"].get(), dd["ctl"].get()
    for j in range(k):
        if j == 1:
            assert gsc[6 * k + j] == 7 and gsc[9 * k + j] == 7 and gst[j] == STOPPED
            continue
        assert gsc[6 * k + j] == alpha[j]
        if data == "int" or j == 2:
            assert gsc[9 * k + j] == int_sum(ws[:, j], ws[:, j])
        else:
            assert_sum_within(gsc[9 * k + j], ws[:, j] * ws[:, j], vt, "ss %d" % j)
        assert gst[j] == (MID_STOPPED if j == 2 else 0), j
    assert gsc[6 * k] == 0 and np.array_equal(gs[:, 0], r[:, 0])
    assert list(gctl[:6]) == [0, 4, 100, 1, 1, 1]
    # every column stopped at the mid check: ctl[0] is raised as well
    st_all = np.full(k, STOPPED, np.uint8)
    st_all[2] = 0
    dd["st"].set(st_all)
    dd["ctl"].set(ctl)
    dev.call("bicgstab_mrhs_step_s_" + vt, n, k, dd["r"], dd["v"], dd["s"], dd["z"], None, dd["sc"], dd["st"],
             dd["ctl"], work(dev, vt, k))
    assert dd["st"].get()[2] == MID_STOPPED and dd["ctl"].get()[0] == 1 and dd["ctl"].get()[5] == 1


@pytest.mark.parametrize("k", [3, 5, 17, 32])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_step_xr_pays_the_finalize_once(dev, k, vt, data):
    """x, r bit for bit; rho = rr.r and ||r||^2 per running column; beta = 0 gives omega = 0; a column
    stopped at the mid check gets only x += alpha y and its finalized bit, a stopped one nothing"""
    v = VT[vt]
    rng = np.random.default_rng(7 * k)
    n = 4099
    if data == "int":
        mk = lambda: rng.integers(-3, 4, (n, k)).astype(v)  # noqa: E731
        alpha, gamma, beta = np.ones(k, v), np.ones(k, v), np.ones(k, v)
    else:
        mk = lambda: rng.uniform(-1, 1, (n, k)).astype(v)  # noqa: E731
        alpha, gamma, beta = (rng.uniform(0.5, 2, k).astype(v) for _ in range(3))
    x, r, s, t, y, z, rr = (mk() for _ in range(7))
    beta[0] = 0
    status = np.zeros(k, np.uint8)
    status[1] = STOPPED          # untouched: NaN sentinels survive
    status[k - 1] = MID_STOPPED  # owes its finalize
    for a in (x, r):
        a[:, 1] = np.nan
    sc = scalars(k, vt, rho=1, prev=1, beta=beta, alpha=alpha, gamma=gamma, thr=np.full(k, 1e-30))
    ctl = np.array([0, 4, 100, 1, 1, 1, 0, 0], np.int32)
    dd = {nm: dev.put(a) for nm, a in dict(x=x, r=r, s=s, t=t, y=y, z=z, rr=rr, sc=sc, st=status,
                                           ctl=ctl).items()}
    wk = work(dev, vt, k)

    def launch():
        dev.call("bicgstab_mrhs_step_xr_" + vt, n, k, dd["x"], dd["r"], dd["s"], dd["t"], dd["y"], dd["z"],
                 dd["rr"], dd["sc"], dd["st"], dd["ctl"], wk)
    launch()
    wx, wr = np_step_xr(x, r, s, t, y, z, sc, status, k, vt)
    gx, gr = dd["x"].get().reshape(n, k), dd["r"].get().reshape(n, k)
    assert gx.tobytes() == wx.tobytes() and gr.tobytes() == wr.tobytes()
    gsc, gst, gctl = dd["sc"].get(), dd["st"].get(), dd["ctl"].get()
    assert gctl[1] == 5 and gctl[0] == 0 and gctl[5] == 0
    assert gst[1] == STOPPED and gst[k - 1] == MID_STOPPED | 0x40
    for j in range(k):
        if stopped(status[j]):
            continue
        assert gsc[k + j] == 1 and gst[j] == 0
        assert gsc[7 * k + j] == (v(gamma[j] / beta[j]) if beta[j] != 0 else 0)
        if data == "int":
            assert gsc[j] == int_sum(rr[:, j], wr[:, j]) and gsc[3 * k + j] == int_sum(wr[:, j], wr[:, j])
        else:
            assert_sum_within(gsc[j], rr[:, j] * wr[:, j], vt, "rho %d" % j)
            assert_sum_within(gsc[3 * k + j], wr[:, j] * wr[:, j], vt, "rr %d" % j)
    # the finalize is paid once: a second launch with every other column stopped moves nothing
    st2 = dd["st"].get()
    st2[[j for j in range(k) if not stopped(st2[j])]] = STOPPED
    dd["st"].set(st2)
    dd["ctl"].set(np.array([1, 5, 100, 1, 1, 0, 0, 0], np.int32))
    before = [dd[nm].get().tobytes() for nm in ("x", "r", "sc", "st", "ctl")]
    launch()
    assert [dd[nm].get().tobytes() for nm in ("x", "r", "sc", "st", "ctl")] == before


@pytest.mark.parametrize("vt", VTS)
def test_step_xr_pays_when_every_column_stopped_at_the_mid_check(dev, vt):
    """ctl[0] raised by the mid check and ctl[5] set: step_xr only pays x += alpha y, sets the
    finalized bits, clears ctl[5], and does not count an iteration"""
    v = VT[vt]
    k, n = 4, 777
    rng = np.random.default_rng(3)
    x, y = rng.uniform(-1, 1, (n, k)).astype(v), rng.uniform(-1, 1, (n, k)).astype(v)
    status = np.array([MID_STOPPED, STOPPED, MID_STOPPED, 0x40 | 0x80 | 1], np.uint8)
    alpha = rng.uniform(0.5, 2, k).astype(v)
    sc = scalars(k, vt, alpha=alpha)
    ctl = np.array([1, 9, 100, 1, 1, 1, 0, 0], np.int32)
    dd = {nm: dev.put(a) for nm, a in dict(x=x, y=y, sc=sc, st=status, ctl=ctl).items()}
    nn = dev.put(nans((n, k), vt))
    dev.call("bicgstab_mrhs_step_xr_" + vt, n, k, dd["x"], nn, nn, nn, dd["y"], nn, nn, dd["sc"], dd["st"],
             dd["ctl"], work(dev, vt, k))
    want = x.copy()
    for j in (0, 2):
        want[:, j] = x[:, j] + alpha[j] * y[:, j]
    assert dd["x"].get().reshape(n, k).tobytes() == want.tobytes()
    assert list(dd["st"].get()) == [MID_STOPPED | 0x40, STOPPED, MID_STOPPED | 0x40, 0x40 | 0x80 | 1]
    assert list(dd["ctl"].get()[:6]) == [1, 9, 100, 1, 1, 0]
    assert np.isnan(nn.get()).all()


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
def test_init(dev, vt, baseline):
    v = VT[vt]
    k, n = 5, 2049
    r = np.random.default_rng(1).integers(-3, 4, (n, k)).astype(v)
    sc0 = np.full(10 * k, np.nan, v)
    sc0[4 * k:5 * k] = 2
    bufs = {nm: dev.put(nans((n, k), vt)) for nm in ("rr", "p", "v", "y", "s", "t", "z")}
    dsc, dst, dctl = dev.put(sc0), dev.put(np.full(k, 0xff, np.uint8)), dev.put(np.full(8, 7, np.int32))
    dev.call("bicgstab_mrhs_init_" + vt, n, k, dev.put(r), *[bufs[nm] for nm in ("rr", "p", "v", "y", "s", "t", "z")],
             dsc, dst, dctl, work(dev, vt, k), 1 << 40, 1, 0, baseline, v(0.5))
    assert bufs["rr"].get().reshape(n, k).tobytes() == r.tobytes()
    for nm in ("p", "v", "y", "s", "t", "z"):
        assert not bufs[nm].get().any()
    sc, st, ctl = dsc.get(), dst.get(), dctl.get()
    rn = np.array([int_sum(r[:, j], r[:, j]) for j in range(k)], v)
    assert np.array_equal(sc[:k], rn) and np.array_equal(sc[3 * k:4 * k], rn)
    assert np.all(sc[k:2 * k] == 1) and np.all(sc[6 * k:9 * k] == 1) and np.all(sc[9 * k:] == 0)
    tau0 = {0: np.full(k, 2, v), 1: np.sqrt(rn), 2: np.ones(k, v)}[baseline]
    assert sc[4 * k:5 * k].tobytes() == tau0.tobytes()
    assert sc[5 * k:6 * k].tobytes() == (v(0.5) * tau0).astype(v).tobytes()
    assert list(ctl[:6]) == [0, 0, 0x7fffffff, 1, 0, 0] and not st.any()


# --------------------------------------------------------------------------- C. lock-step
@pytest.mark.parametrize("vt,it,k", [("f64", "i32", 5), ("f32", "i64", 3), ("f64", "i64", 17), ("f32", "i32", 8)])
@pytest.mark.parametrize("res_kind,baseline,iter_first,diag", [(1, 0, True, True), (2, 1, False, False),
                                                                (1, 2, True, False)])
def test_lock_step(dev, orc, vt, it, k, res_kind, baseline, iter_first, diag):
    """30+ iterations one launch at a time on the convective arrow matrix against numpy fed the
    device's scalars: vectors bit-equal, every column's status at both checks as the criteria say from
    its own scalars, ctl[0] only with the last column"""
    v = VT[vt]
    rp, ci, va = convective_arrow(vt)
    rp, ci = rp.astype(IT[it]), ci.astype(IT[it])
    n = len(rp) - 1
    rng = np.random.default_rng(k)
    b = rng.uniform(-1, 1, (n, k)).astype(v)
    b[:, 0] = 0  # converges at iteration 0 under rhs_norm / absolute
    b[:, 1] *= 1e-3
    d = arrow_inv_diag(rp.astype(np.int64), ci.astype(np.int64), va).astype(v) if diag else None
    max_iters = 34
    red = 1e-13 if vt == "f64" else 1e-6
    nm = ("x", "r", "rr", "p", "v", "y", "s", "t", "z")
    dd = {a: dev.put(np.zeros((n, k), v) if a == "x" else b.copy() if a == "r" else nans((n, k), vt)) for a in nm}
    sc0 = np.zeros(10 * k, v)
    sc0[4 * k:5 * k] = np.sqrt(np.sum(b.astype(np.float64) ** 2, axis=0)).astype(v)
    dd["sc"], dd["st"], dd["ctl"] = dev.put(sc0), dev.put(np.full(k, 0xff, np.uint8)), dev.put(np.zeros(8, np.int32))
    A = [dev.put(a) for a in (rp, ci, va)]
    dp, wk = dev.put(d) if diag else None, work(dev, vt, k)
    dev.call("bicgstab_mrhs_init_" + vt, n, k, dd["r"], dd["rr"], dd["p"], dd["v"], dd["y"], dd["s"], dd["t"], dd["z"],
             dd["sc"], dd["st"], dd["ctl"], wk, max_iters, res_kind, int(iter_first), baseline, v(red))
    x, r, rr, p, vv = np.zeros((n, k), v), b.copy(), b.copy(), np.zeros((n, k), v), np.zeros((n, k), v)
    status = np.zeros(k, np.uint8)
    stop_iter, mid_stops = {}, 0

    def spmv(src, dst, w, dots, dots2):
        dev.call("csr_spmv_mdot2_%s_%s" % (vt, it), n, n, len(va), A[0], A[1], A[2], dd[src], k, dd[dst], dd[w],
                 dd["sc"].at(dots * k), None if dots2 is None else dd["sc"].at(dots2 * k), wk, dd["ctl"])

    def check_top(iteration):
        sc, st = dd["sc"].get(), dd["st"].get()
        for j in range(k):
            if stopped(status[j]):
                assert st[j] & 0x40, (iteration, j)  # finalized
                status[j] = st[j]
                continue
            want = expected_status(iteration, max_iters, res_kind, iter_first,
                                   tau_of(vt, res_kind, sc[j], sc[3 * k + j]), sc[5 * k + j])
            assert st[j] == want, (iteration, j)
            if want:
                status[j] = want
                stop_iter[j] = iteration
    check_top(0)
    counted = 0  # a stop of every column at the mid check counts no further iteration
    for iteration in range(0, max_iters + 2):
        ctl = dd["ctl"].get()
        assert ctl[1] == counted and (ctl[0] != 0) == (len(stop_iter) == k)
        if ctl[0]:
            frozen = [dd[a].get().tobytes() for a in ("x", "r", "p", "sc", "st", "ctl")]
        sc = dd["sc"].get()
        dev.call("bicgstab_mrhs_step_p_" + vt, n, k, dd["p"], dd["r"], dd["v"], dd["y"], dp, dd["sc"], dd["st"],
                 dd["ctl"])
        spmv("y", "v", "rr", 2, None)
        sc_s = dd["sc"].get()
        dev.call("bicgstab_mrhs_step_s_" + vt, n, k, dd["r"], dd["v"], dd["s"], dd["z"], dp, dd["sc"], dd["st"],
                 dd["ctl"], wk)
        mid_ctl, sc_mid = dd["ctl"].get(), dd["sc"].get()
        spmv("z", "t", "s", 8, 2)
        sc_xr = dd["sc"].get()
        dev.call("bicgstab_mrhs_step_xr_" + vt, n, k, dd["x"], dd["r"], dd["s"], dd["t"], dd["y"], dd["z"], dd["rr"],
                 dd["sc"], dd["st"], dd["ctl"], wk)
        if ctl[0]:
            assert [dd[a].get().tobytes() for a in ("x", "r", "p", "sc", "st", "ctl")] == frozen
            break
        # numpy, kernel by kernel, on the device's scalars
        p, y = np_step_p(p, r, vv, d, sc, status, k, vt)
        run = ~np.array([stopped(s_) for s_ in status])
        gy = dd["y"].get().reshape(n, k)
        assert dd["p"].get().reshape(n, k)[:, run].tobytes() == p[:, run].tobytes()
        assert gy[:, run].tobytes() == y[:, run].tobytes()
        vv = oracle_spmv(orc, vt, it, n, n, rp, ci, va, gy, k)
        assert dd["v"].get().reshape(n, k)[:, run].tobytes() == vv[:, run].tobytes()
        s, z, _ = np_step_s(r, vv, d, sc_s, status, k, vt)
        gs, gz = dd["s"].get().reshape(n, k), dd["z"].get().reshape(n, k)
        assert gs[:, run].tobytes() == s[:, run].tobytes() and gz[:, run].tobytes() == z[:, run].tobytes()
        # mid check: each running column's status from its own ||s||^2 and rho
        st_mid = status.copy()
        for j in np.nonzero(run)[0]:
            want = expected_status(iteration, max_iters, res_kind, iter_first,
                                   tau_of(vt, res_kind, sc_mid[j], sc_mid[9 * k + j]), sc_mid[5 * k + j])
            want &= ~0x40
            if want:
                st_mid[j] = want
                stop_iter[j] = iteration
                mid_stops += 1
        assert (mid_ctl[5] != 0) == any(st_mid[j] != status[j] for j in range(k))
        t_ = oracle_spmv(orc, vt, it, n, n, rp, ci, va, gz, k)
        if not mid_ctl[0]:
            assert dd["t"].get().reshape(n, k)[:, run].tobytes() == t_[:, run].tobytes()
        x, r = np_step_xr(x, r, gs, t_, gy, gz, sc_xr, st_mid, k, vt)
        assert dd["x"].get().reshape(n, k).tobytes() == x.tobytes()
        assert dd["r"].get().reshape(n, k)[:, run].tobytes() == r[:, run].tobytes()
        for j in range(k):
            if st_mid[j] != status[j]:
                status[j] = st_mid[j] | 0x40
        if not mid_ctl[0]:
            counted += 1
            check_top(iteration + 1)
    assert len(stop_iter) == k and stop_iter[0] == 0 and len(set(stop_iter.values())) >= 2
    assert all(s_ & 0x40 for s_ in dd["st"].get())


# --------------------------------------------------------------------------- D. host solver
def rhs(n, k, vt, seed=6):
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
    b[:, 1] *= 1e-3
    return b.astype(VT[vt])


def device_solve(hexec, vt, rp, ci, va, b, x0, precond=0, strided=0, block_ptrs=None, **kw):
    import torch
    from ginkgo_b200 import api
    k = b.shape[1]
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(np.pad(b, ((0, 0), (0, strided))))).to(hexec.device)
        tx = torch.from_numpy(np.ascontiguousarray(np.pad(x0, ((0, 0), (0, strided))))).to(hexec.device).clone()
    n = len(rp) - 1
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "bicgstab", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb, cols=k), api.host_dense(hexec, tx, cols=k))
    hexec.synchronize()
    return tx.cpu().numpy()[:, :k], s.num_iterations, s.stop_statuses, s.used_fused


def orc_solve(vt, rp, ci, va, b, precond, **kw):
    rp32, ci32 = rp.astype(np.int32), ci.astype(np.int32)  # the oracle's solvers take int32 indices
    jac = {"blocks": arrow_inv_diag(rp32, ci32, va)} if precond else None
    return H.orc_solve("bicgstab", vt, rp32, ci32, va, b, np.zeros_like(b), precond, jac, **kw)


def assert_matches_oracle(xo, ito, stop_o, xd, itd, stop_d, vt):
    assert stop_d == list(stop_o)
    assert abs(itd - ito) <= max(3, 0.35 * ito), (itd, ito)
    for j in range(xo.shape[1]):
        assert H.rel_err(xo[:, j], xd[:, j]) <= (1e-7 if vt == "f64" else 2e-3), j


@pytest.mark.parametrize("vt,it,precond", [("f64", "i32", 0), ("f64", "i32", 1), ("f32", "i32", 1),
                                           ("f64", "i64", 0), ("f32", "i64", 0)])
@pytest.mark.parametrize("res_kind", [1, 2])
@pytest.mark.parametrize("baseline", [0, 1, 2])
@pytest.mark.parametrize("iter_first", [True, False])
@pytest.mark.parametrize("check_every", [1, 7, 16])
def test_solver_matches_oracle(hexec, vt, it, precond, res_kind, baseline, iter_first, check_every):
    rp, ci, va = upwind(16, 2, vt)
    rp, ci = rp.astype(IT[it]), ci.astype(IT[it])
    n, k = len(rp) - 1, 4
    b = rhs(n, k, vt)
    red = 1e-8 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10
    kw = dict(max_iters=1000, res_kind=res_kind, baseline=baseline, reduction=red)
    xo, ito, stop_o = orc_solve(vt, rp, ci, va, b, precond, iter_first=int(iter_first), **kw)
    xd, itd, stop_d, used = device_solve(hexec, vt, rp, ci, va, b, np.zeros_like(b), precond,
                                         iter_first=iter_first, fused_bicgstab_multi_rhs=True,
                                         check_every=check_every, **kw)
    assert used
    assert_matches_oracle(xo, ito, stop_o, xd, itd, stop_d, vt)


def periodic_upwind(n, vt):
    """periodic 1-D upwind: 2.75 on the diagonal, -1.5 below, -1 above (n even).  Every row sums to 0.25
    and (-1)^i is an eigenvector with eigenvalue 5.25; the Jacobi diagonal is constant, so both are
    eigenvectors of the preconditioned operator too"""
    rows = np.repeat(np.arange(n), 3)
    cols = np.stack([(np.arange(n) - 1) % n, np.arange(n), (np.arange(n) + 1) % n], axis=1).reshape(-1)
    vals = np.tile([-1.5, 2.75, -1.0], n)
    order = np.lexsort((cols, rows))
    return np.arange(0, 3 * n + 1, 3, dtype=np.int32), cols[order].astype(np.int32), vals[order].astype(VT[vt])


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("check_every", [1, 16])
def test_mid_check_stops_beside_running_columns(hexec, vt, precond, check_every):
    """eigenvector columns stop at the mid check of iteration 0 and end with x_j = b_j / lambda (a
    top-check stop would leave x_j = 0); a random and a zero column run on; all against the oracle"""
    n = 1000
    rp, ci, va = periodic_upwind(n, vt)
    alt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    b = np.stack([np.ones(n), alt, np.random.default_rng(1).uniform(-1, 1, n), np.zeros(n), 3 * alt],
                 axis=1).astype(VT[vt])
    kw = dict(max_iters=300, reduction=1e-10 if vt == "f64" else 1e-5)
    xo, ito, stop_o = orc_solve(vt, rp, ci, va, b, precond, **kw)
    xd, itd, stop_d, used = device_solve(hexec, vt, rp, ci, va, b, np.zeros_like(b), precond,
                                         fused_bicgstab_multi_rhs=True, check_every=check_every, **kw)
    assert used and stop_d == [FIN_CONV_2] * 5
    assert_matches_oracle(xo, ito, stop_o, xd, itd, stop_d, vt)
    rt = 1e-12 if vt == "f64" else 1e-5
    for j, lam in ((0, 0.25), (1, 5.25), (4, 5.25)):
        assert np.allclose(xd[:, j], b[:, j] / VT[vt](lam), rtol=rt, atol=0), j
    assert np.all(xd[:, 3] == 0)


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
def test_every_column_stops_at_the_mid_check(hexec, vt, precond):
    """eigenvector columns only: the solve stops at the mid check of iteration 0, reports 0 iterations,
    and with 16 iterations per graph x = b / lambda is applied once, not once per replay"""
    n = 1000
    rp, ci, va = periodic_upwind(n, vt)
    alt = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    b = np.stack([np.ones(n), alt, 2 * np.ones(n)], axis=1).astype(VT[vt])
    kw = dict(max_iters=300, reduction=1e-10 if vt == "f64" else 1e-5)
    xo, ito, stop_o = orc_solve(vt, rp, ci, va, b, precond, **kw)
    xd, itd, stop_d, used = device_solve(hexec, vt, rp, ci, va, b, np.zeros_like(b), precond,
                                         fused_bicgstab_multi_rhs=True, check_every=16, **kw)
    assert used and itd == ito == 0 and stop_d == list(stop_o) == [FIN_CONV_2] * 3
    rt = 1e-12 if vt == "f64" else 1e-5
    for j, lam in ((0, 0.25), (1, 5.25), (2, 0.25)):
        assert np.allclose(xd[:, j], b[:, j] / VT[vt](lam), rtol=rt, atol=0), j
    if precond == 0 and vt == "f64":
        assert np.array_equal(xd[:, 0], np.full(n, 4.0)) and np.array_equal(xd[:, 2], np.full(n, 8.0))


def test_columns_stop_at_their_own_iterations(hexec):
    rp, ci, va = upwind(40, 2, "f64")
    n, k = len(rp) - 1, 5
    b = rhs(n, k, "f64", seed=9)
    b[:, 3] = 0
    kw = dict(max_iters=2000, reduction=1e-9, baseline=0)
    xo, ito, stop_o = orc_solve("f64", rp, ci, va, b, 0, **kw)
    xd, itd, stop_d, used = device_solve(hexec, "f64", rp, ci, va, b, np.zeros_like(b),
                                         fused_bicgstab_multi_rhs=True, **kw)
    assert used
    assert_matches_oracle(xo, ito, stop_o, xd, itd, stop_d, "f64")
    assert stop_d[3] == FIN_CONV_2 and np.all(xd[:, 3] == 0)
    for j in (0, 1, 2, 4):
        assert true_rel_res(rp, ci, va, b[:, j], xd[:, j]) <= 20 * 1e-9


def test_fallbacks(hexec):
    rp, ci, va = upwind(12, 2, "f64")
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8)
    b33 = rhs(n, 33, "f64")
    assert not device_solve(hexec, "f64", rp, ci, va, b33, np.zeros_like(b33), 1, fused_bicgstab_multi_rhs=True,
                            **kw)[3]
    b4 = rhs(n, 4, "f64")
    x0 = np.zeros_like(b4)
    xs, its, sts, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, strided=2, fused_bicgstab_multi_rhs=True,
                                      **kw)
    assert not used
    # the switch is off by default: the loop, as before
    xl, itl, stl, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, **kw)
    assert not used and sts == stl == [FIN_CONV_2] * 4 and its == itl and xs.tobytes() == xl.tobytes()
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not device_solve(hexec, "f64", rp, ci, va, b4, x0, 4, block_ptrs=bp, fused_bicgstab_multi_rhs=True,
                            **kw)[3]
    # the new path agrees with the loop within rounding and in its statuses
    xf, itf, stf, used = device_solve(hexec, "f64", rp, ci, va, b4, x0, 1, fused_bicgstab_multi_rhs=True, **kw)
    assert used and stf == stl and abs(itf - itl) <= max(3, 0.35 * itl)
    # one column: today's paths, the same bits with the switch on or off
    b1, x1 = b4[:, :1].copy(), x0[:, :1].copy()
    for one_col in ((False,) if hexec.stream is None else (False, True)):  # mock: no one-column kernels
        xa, ita, sta, usa = device_solve(hexec, "f64", rp, ci, va, b1, x1, 1, fused_bicgstab_multi_rhs=True,
                                         fused_bicgstab=one_col, **kw)
        xb, itb, stb, usb = device_solve(hexec, "f64", rp, ci, va, b1, x1, 1, fused_bicgstab=one_col, **kw)
        assert usa == usb == one_col and (ita, sta) == (itb, stb) and xa.tobytes() == xb.tobytes()


def test_two_applies_give_the_same_bits(hexec):
    """deterministic sums: the same solve gives the same bits and iterations, with another k between"""
    rp, ci, va = upwind(30, 2, "f64")
    n = len(rp) - 1
    outs = []
    for k in (6, 3, 6):
        b = rhs(n, k, "f64", seed=1)
        outs.append(device_solve(hexec, "f64", rp, ci, va, b, np.zeros_like(b), 1, fused_bicgstab_multi_rhs=True,
                                 max_iters=500, reduction=1e-10))
    assert outs[0][0].tobytes() == outs[2][0].tobytes() and outs[0][1:] == outs[2][1:]
    assert outs[1][2] == [FIN_CONV_2] * 3
