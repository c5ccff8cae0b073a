"""The fused BiCGStab kernels (csrc/fused_bicgstab.cu and the two-sum dot mode of csr_kernels.cuh /
csr_ring.cuh / csr_launch.cuh) one at a time, through the C ABI, against plain numpy restatements.

The three kinds of assertion are those of tests/test_fused_cg_gpu.py, whose backend, buffers and
references this file imports: element-wise updates and the scalars derived from given sums are
compared BIT FOR BIT, reductions on small-integer data for EQUALITY with the exact sum, reductions
on random data against math.fsum within gamma_h * sum |t|.

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock; the asserts about
the device's launch shapes are skipped there, each marked "mock:"."""
import os

import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_fused_cg_gpu import (ITS, STOPPED, VARIANTS, VTS, Backend, Mat, arrow, arrow_inv_diag,  # noqa: F401
                                     assert_sum_within, dev, exact_limit, exact_spmv, expected_status, hexec,
                                     int_sum, nans, spmv_case, step_sizes)
from tests.test_parity_gpu import CSR_KINDS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend(tmp_path_factory):
    """as in test_fused_cg_gpu.py (its `dev` and `hexec` fixtures build on this one); the self-check
    uses the mock that restates the fused BiCGStab entry points"""
    from ginkgo_b200 import _cdecl, _lib
    if os.environ.get("B200_TEST_SELFCHECK") == "1":
        from tests.mock_bicgstab_build import build_mock_host
        lib = build_mock_host(str(tmp_path_factory.mktemp("fused_bicgstab_mock")))
        _cdecl.bind(lib, _lib.declarations())
        be = Backend(lib, mock=True)
    else:
        be = Backend(_lib.lib(), mock=False)
    yield be
    be.close()

SC, CTL = 16, 8  # sc: 0 rho 1 prev_rho 2 beta 3 rr 4 tau0 5 threshold 6 alpha 7 omega 8 gamma 9 ss; ctl[5]: pending


def spmv_dot2(dev, A, b, c, w, dot_ptr, dot2_ptr, work, ctl=None):
    dev.call("csr_spmv_dot2_%s_%s" % (A.vt, A.it), A.plan, A.n, A.ncols, A.nnz, A.rp, A.ci, A.va, b, c, w,
             dot_ptr, dot2_ptr, work, ctl)


def row_vector(vt, n, data, seed=23):
    rng = np.random.default_rng(seed)
    if data == "int":
        return rng.integers(-1, 2, size=n).astype(VT[vt])
    return rng.uniform(-1, 1, size=n).astype(VT[vt])


# --------------------------------------------------------------------------- A. spmv_dot2
@pytest.mark.parametrize("kind", CSR_KINDS + ["rect", "grid_cap"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_dot2(dev, kind, variant, vt, it, data):
    n, ncols, rp, ci, va, b = spmv_case(kind, vt, it, data, dev.num_sms)
    A = Mat(dev, vt, it, n, ncols, rp, ci, va, variant)
    if not dev.mock:  # mock: plans carry no variant and no long-row list
        assert dev.l.b200_csr_plan_variant(A.plan) == variant
        if kind == "split_rows":
            assert dev.l.b200_csr_plan_num_long_rows(A.plan) > 0
    w = row_vector(vt, n, data)  # one entry per ROW (the rectangular case has more columns), not b
    assert n < 8 or not np.array_equal(w, b[:n])
    bd, wd, work = dev.put(b), dev.put(w), dev.work(vt)
    cref = dev.put(nans(n, vt))
    A.spmv(dev, bd, cref)
    c_plain = cref.get()

    # two sums, then one: the second output is optional
    c, dots = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    spmv_dot2(dev, A, bd, c, wd, dots.at(0), dots.at(1), work)
    got_c, (wc, cc) = c.get(), dots.get()
    c1, dots1 = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    spmv_dot2(dev, A, bd, c1, wd, dots1.at(0), None, work)
    assert got_c.tobytes() == c_plain.tobytes() == c1.get().tobytes()
    assert dots1.get()[0].tobytes() == wc.tobytes() and np.isnan(dots1.get()[1])
    if data == "int":
        c_exact, cabs = exact_spmv(n, rp, ci, va, b)
        assert cabs.max(initial=0) < exact_limit(vt)
        assert max(int_sum(np.abs(w), np.abs(c_exact)), int_sum(c_exact, c_exact)) < exact_limit(vt)
        assert np.array_equal(got_c, c_exact)
        assert float(wc) == int_sum(w, c_exact)
        assert float(cc) == int_sum(c_exact, c_exact)
    else:
        assert_sum_within(wc, w * got_c, vt, "w.c")
        assert_sum_within(cc, got_c * got_c, vt, "c.c")

    # deterministic, and the tickets reset themselves
    c2, dots2 = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    spmv_dot2(dev, A, bd, c2, wd, dots2.at(0), dots2.at(1), work)
    assert c2.get().tobytes() == got_c.tobytes() and dots2.get().tobytes() == dots.get().tobytes()

    # a stopped solver: nothing is written (incl. the long-row kernel and its dot fix)
    ctl = dev.put(np.array([STOPPED, 3, 0, 0, 0, 0, 0, 0], np.int32))
    c3, dots3 = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    spmv_dot2(dev, A, bd, c3, wd, dots3.at(0), dots3.at(1), work, ctl)
    assert np.isnan(c3.get()).all() and np.isnan(dots3.get()).all()


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
def test_spmv_dot2_empty_matrix_writes_zeros(dev, vt, it):
    A = Mat(dev, vt, it, 0, 5, np.zeros(1, IT[it]), np.zeros(0, IT[it]), np.zeros(0, VT[vt]))
    b, c, w = dev.put(np.ones(5, VT[vt])), dev.put(nans(0, vt)), dev.put(nans(0, vt))
    dots = dev.put(nans(2, vt))
    spmv_dot2(dev, A, b, c, w, dots.at(0), dots.at(1), dev.work(vt))
    assert dots.get().tolist() == [0.0, 0.0]
    dots = dev.put(nans(2, vt))
    spmv_dot2(dev, A, b, c, w, dots.at(0), None, dev.work(vt))
    assert dots.get()[0] == 0 and np.isnan(dots.get()[1])
    ctl = dev.put(np.array([STOPPED, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dots = dev.put(nans(2, vt))
    spmv_dot2(dev, A, b, c, w, dots.at(0), dots.at(1), dev.work(vt), ctl)
    assert np.isnan(dots.get()).all()


@pytest.mark.parametrize("vt", VTS)
def test_spmv_dot2_refuses_slab_variant(dev, vt):
    if dev.mock:
        pytest.skip("mock: plans carry no variant")
    n, ncols, rp, ci, va, b = spmv_case("laplace_like", vt, "i32", "rand", dev.num_sms)
    A = Mat(dev, vt, "i32", n, ncols, rp, ci, va, 0)
    c, dots, w = dev.put(nans(n, vt)), dev.put(nans(2, vt)), dev.put(row_vector(vt, n, "rand"))
    st = dev.status("csr_spmv_dot2_%s_i32" % vt, A.plan, n, ncols, len(va), A.rp, A.ci, A.va, dev.put(b), c, w,
                    dots.at(0), dots.at(1), dev.work(vt).ptr, None)
    assert st != 0
    assert np.isnan(c.get()).all() and np.isnan(dots.get()).all()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_spmv_dot2_alternating_with_other_reductions(dev, variant, vt):
    """spmv_dot2 shares its ticket with spmv_dot, the step kernels theirs with the fused CG, and
    dense_compute_dot uses the same counter array: each must leave its ticket at 0"""
    rng = np.random.default_rng(6)
    mats = []
    for kind in ("grid_cap", "split_rows"):
        n, ncols, rp, ci, va, b = spmv_case(kind, vt, "i32", "int", dev.num_sms)
        A = Mat(dev, vt, "i32", n, ncols, rp, ci, va, variant)
        c_exact, _ = exact_spmv(n, rp, ci, va, b)
        w = row_vector(vt, n, "int")
        mats.append((A, dev.put(b), dev.put(w), c_exact,
                     (int_sum(w, c_exact), int_sum(c_exact, c_exact), int_sum(b[:n], c_exact))))
    nx = 2048 * 4 * dev.num_sms + 777  # the step kernels at their grid cap
    r = rng.integers(-1, 2, size=nx).astype(VT[vt])
    inv = rng.integers(1, 4, size=nx).astype(VT[vt])
    rd, invd, sd, zd = dev.put(r), dev.put(inv), dev.put(nans(nx, vt)), dev.put(nans(nx, vt))
    sc = dev.put(np.array([1, 1, 0] + [0] * 13, VT[vt]))  # beta = 0: s = r, the sum is exact
    ctl = dev.put(np.array([0, 0, -1, 0, 1, 0, 0, 0], np.int32))
    res, work = dev.put(nans(1, vt)), dev.work(vt)
    for rnd in range(2):
        for A, bd, wd, c_exact, (d_wc, d_cc, d_bc) in mats:
            c, dots = dev.put(nans(A.n, vt)), dev.put(nans(3, vt))
            spmv_dot2(dev, A, bd, c, wd, dots.at(0), dots.at(1), work, ctl)
            A.spmv_dot(dev, bd, c, dots.at(2), work, ctl)
            assert np.array_equal(c.get(), c_exact), rnd
            assert [float(d) for d in dots.get()] == [d_wc, d_cc, d_bc], rnd
            dev.call("bicgstab_fused_step_s_" + vt, nx, rd, rd, sd, zd, invd, sc, ctl, work)
            assert float(sc.get()[9]) == int_sum(r, r) and ctl.get()[0] == 0
            dev.call("dense_compute_dot_" + vt, nx, 1, rd, 1, invd, 1, res)
            assert float(res.get()[0]) == int_sum(r, inv)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_dot2_graph_replay_matches_eager(dev, variant, vt, data):
    """captured with its fork / join on the auxiliary stream (long-row kernel) and the dot fix: the
    rows split over CTAs enter both sums exactly once per replay"""
    n, ncols, rp, ci, va, b = spmv_case("split_rows", vt, "i64", data, dev.num_sms)
    A = Mat(dev, vt, "i64", n, ncols, rp, ci, va, variant)
    bd, wd, work = dev.put(b), dev.put(row_vector(vt, n, data)), dev.work(vt)
    c, dots = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    spmv_dot2(dev, A, bd, c, wd, dots.at(0), dots.at(1), work)
    eager_c, eager_dots = c.get(), dots.get()
    if data == "int":
        c_exact, _ = exact_spmv(n, rp, ci, va, b)
        assert float(eager_dots[1]) == int_sum(c_exact, c_exact)
    c2, dots2 = dev.put(nans(n, vt)), dev.put(nans(2, vt))
    g = dev.capture(lambda: spmv_dot2(dev, A, bd, c2, wd, dots2.at(0), dots2.at(1), work))
    for _ in range(2):
        dev.call("graph_launch", g)
        dev.sync()
        assert c2.get().tobytes() == eager_c.tobytes() and dots2.get().tobytes() == eager_dots.tobytes()
        c2.set(nans(n, vt))
        dots2.set(nans(2, vt))


# --------------------------------------------------------------------------- B. step kernels
def np_step_p(p, r, v, inv, sc):
    """bicgstab::step_1 (reference/solver/bicgstab_kernels.cpp:63-88) + scalar Jacobi apply"""
    rho, prev, alpha, omega = sc[0], sc[1], sc[6], sc[7]
    if prev * omega != 0:
        tmp = rho / prev * alpha / omega
        p1 = r + tmp * (p - omega * v)
    else:
        p1 = r.copy()
    return p1, (p1 * inv if inv is not None else p1)


def np_step_s(r, v, inv, sc):
    """bicgstab::step_2 (:93-116) + scalar Jacobi apply; returns alpha, s, z"""
    beta = sc[2]
    if beta != 0:
        alpha = sc[0] / beta
        s = r - alpha * v
    else:
        alpha, s = r.dtype.type(0), r.copy()
    return alpha, s, (s * inv if inv is not None else s)


def np_step_xr(x, s, t, y, z, sc):
    """bicgstab::step_3 (:121-150); returns omega, x, r"""
    beta = sc[2]
    omega = sc[8] / beta if beta != 0 else x.dtype.type(0)
    return omega, x + (sc[6] * y + omega * z), s - omega * t


def bytes_eq(buf, want):
    return buf.get().tobytes() == np.asarray(want).tobytes()


def rand_vecs(rng, vt, n, k):
    return [rng.uniform(-1, 1, n).astype(VT[vt]) for _ in range(k)]


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
def test_init(dev, size, vt, baseline):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(300 + size)
    r = rng.uniform(-1, 1, n).astype(v)
    rd = dev.put(r)
    others = [dev.put(nans(n, vt)) for _ in range(7)]  # rr p v y s t z
    sc = dev.put(np.array([7] * 4 + [2.5] + [7] * 11, v))  # sc[4]: ||b|| for baseline 0
    ctl = dev.put(np.full(CTL, 7, np.int32))
    factor, max_iters = v(2.0 ** -20), 5
    dev.call("bicgstab_fused_init_" + vt, n, rd, *others, sc, ctl, dev.work(vt), max_iters, 1, 1, baseline,
             float(factor))
    assert bytes_eq(rd, r) and bytes_eq(others[0], r)
    assert all(not o.get().any() for o in others[1:])
    s, c = sc.get(), ctl.get()
    assert c[1:6].tolist() == [0, max_iters, 1, 1, 0]
    # rho = rr.r, moved from the reference's initial 1; the others stay 1 (bicgstab::initialize)
    assert [s[k] for k in (1, 2, 6, 7, 8)] == [1] * 5 and s[9] == 0
    assert_sum_within(s[0], r * r, vt, "rho")
    assert_sum_within(s[3], r * r, vt, "rr")
    tau0 = {0: v(2.5), 1: np.sqrt(s[3]), 2: v(1)}[baseline]
    assert s[4] == tau0 and s[5] == factor * tau0
    assert c[0] == expected_status(0, max_iters, 1, 1, np.sqrt(s[3]), s[5])


@pytest.mark.parametrize("vt", VTS)
def test_init_sums_exact_and_max_iters_clamped(dev, vt):
    n = step_sizes(dev.num_sms)[4]
    r = np.random.default_rng(1).integers(-1, 2, size=n).astype(VT[vt])
    assert n < exact_limit(vt)
    others = [dev.put(nans(n, vt)) for _ in range(7)]
    sc, ctl = dev.put(nans(SC, vt)), dev.put(np.zeros(CTL, np.int32))
    dev.call("bicgstab_fused_init_" + vt, n, dev.put(r), *others, sc, ctl, dev.work(vt), 2 ** 33, 0, 1, 2, 1.0)
    assert (float(sc.get()[0]), float(sc.get()[3])) == (int_sum(r, r), int_sum(r, r))
    assert ctl.get()[:3].tolist() == [0, 0, 2 ** 31 - 1]


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("guard", [None, "prev_rho", "omega"])
def test_step_p(dev, size, vt, precond, guard):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(400 + size)
    p, r, vv = rand_vecs(rng, vt, n, 3)
    inv = rng.uniform(0.5, 2, n).astype(v) if precond else None
    s = rng.uniform(0.5, 2, SC).astype(v)
    if guard:
        s[{"prev_rho": 1, "omega": 7}[guard]] = 0
    pd, rd, vd, yd = dev.put(p), dev.put(r), dev.put(vv), dev.put(nans(n, vt))
    invd = dev.put(inv) if precond else None
    sc, ctl = dev.put(s), dev.put(np.zeros(CTL, np.int32))
    dev.call("bicgstab_fused_step_p_" + vt, n, pd, rd, vd, yd, invd, sc, ctl)
    p1, y1 = np_step_p(p, r, vv, inv, s)
    if guard:
        assert p1.tobytes() == r.tobytes()
    assert bytes_eq(pd, p1) and bytes_eq(yd, y1) and bytes_eq(sc, s)
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    dev.call("bicgstab_fused_step_p_" + vt, n, pd, rd, vd, yd, invd, sc, ctl)
    assert bytes_eq(pd, p1) and bytes_eq(yd, y1)


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("beta_zero", [False, True])
def test_step_s(dev, size, vt, precond, beta_zero):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(500 + size)
    r, vv = rand_vecs(rng, vt, n, 2)
    inv = rng.uniform(0.5, 2, n).astype(v) if precond else None
    s0 = rng.uniform(0.5, 2, SC).astype(v)
    s0[5] = 0  # threshold 0: the mid check does not fire on random data
    if beta_zero:
        s0[2] = 0
    rd, vd, sd, zd = dev.put(r), dev.put(vv), dev.put(nans(n, vt)), dev.put(nans(n, vt))
    invd = dev.put(inv) if precond else None
    sc, ctl = dev.put(s0), dev.put(np.array([0, 3, 10, 1, 1, 0, 0, 0], np.int32))
    dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, invd, sc, ctl, dev.work(vt))
    alpha, s1, z1 = np_step_s(r, vv, inv, s0)
    assert bytes_eq(sd, s1) and bytes_eq(zd, z1) and bytes_eq(rd, r)
    s = sc.get()
    assert s[6].tobytes() == v(alpha).tobytes() and (not beta_zero or s[6] == 0)
    assert_sum_within(s[9], s1 * s1, vt, "ss")
    assert np.delete(s, [6, 9]).tobytes() == np.delete(s0, [6, 9]).tobytes()
    want_ctl = [0, 3, 10, 1, 1, 0, 0, 0]
    if n == 0:  # ||s|| = 0 <= 0: converged at the mid check, finalize pending
        want_ctl[0], want_ctl[5] = 0x80 | 0x40 | 2, 1
    assert ctl.get().tolist() == want_ctl
    state = [b.get().tobytes() for b in (sd, zd, sc)]
    ctl.set(np.array([STOPPED] + [0] * 7, np.int32))
    sd.set(nans(n, vt))
    dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, invd, sc, ctl, dev.work(vt))
    assert np.isnan(sd.get()).all() and [zd.get().tobytes(), sc.get().tobytes()] == state[1:]


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("beta_zero", [False, True])
def test_step_xr(dev, size, vt, beta_zero):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(600 + size)
    x, s_, t, y, z, rr = rand_vecs(rng, vt, n, 6)
    s0 = rng.uniform(0.5, 2, SC).astype(v)
    s0[5] = 0
    if beta_zero:
        s0[2] = 0
    xd, rd = dev.put(x), dev.put(nans(n, vt))
    sd, td, yd, zd, rrd = (dev.put(a) for a in (s_, t, y, z, rr))
    sc, ctl = dev.put(s0), dev.put(np.array([0, 3, 10, 1, 1, 0, 0, 0], np.int32))
    args = (n, xd, rd, sd, td, yd, zd, rrd, sc, ctl, dev.work(vt))
    dev.call("bicgstab_fused_step_xr_" + vt, *args)
    omega, x1, r1 = np_step_xr(x, s_, t, y, z, s0)
    assert bytes_eq(xd, x1) and bytes_eq(rd, r1)
    assert all(bytes_eq(d, a) for d, a in ((sd, s_), (td, t), (yd, y), (zd, z), (rrd, rr)))
    s = sc.get()
    assert s[7].tobytes() == v(omega).tobytes() and (not beta_zero or s[7] == 0)
    assert s[1] == s0[0]  # rho -> prev_rho
    assert_sum_within(s[0], rr * r1, vt, "rho")
    assert_sum_within(s[3], r1 * r1, vt, "rr")
    assert np.delete(s, [0, 1, 3, 7]).tobytes() == np.delete(s0, [0, 1, 3, 7]).tobytes()
    c = ctl.get()
    assert c[1:].tolist() == [4, 10, 1, 1, 0, 0, 0]
    assert c[0] == expected_status(4, 10, 1, 1, np.sqrt(s[3]), s[5])
    # stopped and finalized: a no-op
    ctl.set(np.array([STOPPED, 4, 10, 1, 1, 0, 0, 0], np.int32))
    state = [b.get().tobytes() for b in (xd, rd, sc, ctl)]
    dev.call("bicgstab_fused_step_xr_" + vt, *args)
    assert [b.get().tobytes() for b in (xd, rd, sc, ctl)] == state
    # stopped at the mid check, finalize pending: only x += alpha y, and the word is cleared
    ctl.set(np.array([STOPPED, 4, 10, 1, 1, 1, 0, 0], np.int32))
    dev.call("bicgstab_fused_step_xr_" + vt, *args)
    assert bytes_eq(xd, x1 + s[6] * y) and rd.get().tobytes() == state[1] and sc.get().tobytes() == state[2]
    assert ctl.get().tolist() == [STOPPED, 4, 10, 1, 1, 0, 0, 0]


@pytest.mark.parametrize("vt", VTS)
def test_step_sums_exact_on_integers(dev, vt):
    """s = r (beta = 0) and r = s (beta = 0 => omega = 0) keep integer data: every CTA partial counts"""
    n = step_sizes(dev.num_sms)[4]
    rng = np.random.default_rng(7)
    r, rr = (rng.integers(-1, 2, size=n).astype(VT[vt]) for _ in range(2))
    zeros = np.zeros(n, VT[vt])
    rd, rrd, vd, sd, zd, xd = (dev.put(a) for a in (r, rr, zeros, nans(n, vt), nans(n, vt), zeros))
    s0 = np.zeros(SC, VT[vt])
    s0[0] = 3
    sc, ctl, work = dev.put(s0), dev.put(np.array([0, 0, -1, 0, 1, 0, 0, 0], np.int32)), dev.work(vt)
    dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, None, sc, ctl, work)
    assert float(sc.get()[9]) == int_sum(r, r)
    out = dev.put(nans(n, vt))
    dev.call("bicgstab_fused_step_xr_" + vt, n, xd, out, sd, vd, vd, vd, rrd, sc, ctl, work)
    s = sc.get()
    assert bytes_eq(out, r) and (float(s[0]), float(s[1]), float(s[3])) == (int_sum(rr, r), 3, int_sum(r, r))


# --------------------------------------------------------------------------- C. stopping
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
def test_stopping_table(dev, vt, baseline):
    """both check sites with tau exactly on, above and below the threshold T.  r = (4,4,4,4,0,..):
    rho = ||r||^2 = 64, tau = 8 at the top check of iteration 0.  v = r, beta = 128: alpha = 1/2 and
    s = r/2, ||s|| = 4 at the mid check (ImplicitResidualNorm looks at sqrt|rho| = 8 again).  t = s,
    gamma = beta/2: omega = 1/2, r = s/2 = (1,..), ||r|| = 2 and rho = rr.r = 16, sqrt = 4, at the top
    check of iteration 1.  Every number is a power of two, so nothing is rounded."""
    v = VT[vt]
    n = 8
    r = np.array([4, 4, 4, 4, 0, 0, 0, 0], v)
    y = np.random.default_rng(3).uniform(-1, 1, n).astype(v)
    x = np.random.default_rng(4).uniform(-1, 1, n).astype(v)
    tau0 = {0: 2.0, 1: 8.0, 2: 1.0}[baseline]
    work = dev.work(vt)
    n3, rp, ci, va = 8, np.arange(9, dtype=np.int32), np.arange(8, dtype=np.int32), np.ones(8, v)
    I8 = Mat(dev, vt, "i32", n3, n3, rp, ci, va)
    checked = 0
    for max_iters in (-1, 0, 1, 2):
        for res_kind in (0, 1, 2):
            for iter_first in (0, 1):
                for T in (8.0, 4.0, 2.0, 1.0):
                    what = (max_iters, res_kind, iter_first, T)
                    rd, xd, yd = dev.put(r), dev.put(x), dev.put(nans(n, vt))
                    rrd, pd, vd, sd, td, zd = (dev.put(nans(n, vt)) for _ in range(6))
                    sc = dev.put(np.array([9] * 4 + [2.0] + [9] * 11, v))
                    ctl = dev.put(np.zeros(CTL, np.int32))
                    dev.call("bicgstab_fused_init_" + vt, n, rd, rrd, pd, vd, yd, sd, td, zd, sc, ctl, work,
                             max_iters, res_kind, iter_first, baseline, T / tau0)
                    s, c = sc.get(), ctl.get()
                    assert (s[0], s[3], s[4], s[5]) == (64, 64, tau0, T), what
                    st0 = expected_status(0, max_iters, res_kind, iter_first, 8.0, T)
                    assert c.tolist() == [st0, 0, max_iters, res_kind, iter_first, 0, 0, 0], what

                    def iteration():
                        # the SpMVs are replaced by their results unless stopped: v = r with rr.v = 128;
                        # the second one is really run (identity matrix, z -> t) to see it skipped
                        dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, None, sc, ctl, work)
                        spmv_dot2(dev, I8, zd, td, sd, sc.at(8), sc.at(2), work, ctl)
                        if ctl.get()[0] == 0:
                            s_ = sc.get()
                            s_[8] = s_[2] / 2  # gamma = beta / 2
                            sc.set(s_)
                        dev.call("bicgstab_fused_step_xr_" + vt, n, xd, rd, sd, td, yd, zd, rrd, sc, ctl, work)

                    vd.set(r)
                    yd.set(y)
                    s[2] = 128
                    sc.set(s)
                    tau_mid = 4.0 if res_kind == 1 else 8.0
                    st_mid = st0 or expected_status(0, max_iters, res_kind, iter_first, tau_mid, T)
                    if st0 == 0:
                        dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, None, sc, ctl, work)
                        assert bytes_eq(sd, r / 2) and sc.get()[6] == 0.5 and sc.get()[9] == 16, what
                        assert ctl.get().tolist() == [st_mid, 0, max_iters, res_kind, iter_first, int(st_mid != 0),
                                                      0, 0], what
                        td.set(nans(n, vt))
                        spmv_dot2(dev, I8, zd, td, sd, sc.at(8), sc.at(2), work, ctl)
                        if st_mid:  # the second SpMV did not run
                            assert np.isnan(td.get()).all() and sc.get()[2] == 128, what
                        else:
                            assert bytes_eq(td, r / 2) and (sc.get()[8], sc.get()[2]) == (16, 16), what
                            s_ = sc.get()
                            s_[8] = 8
                            sc.set(s_)
                        dev.call("bicgstab_fused_step_xr_" + vt, n, xd, rd, sd, td, yd, zd, rrd, sc, ctl, work)
                        c = ctl.get()
                        if st_mid:  # bicgstab::finalize only: x += alpha y, r and the iteration count stay
                            assert bytes_eq(xd, x + v(0.5) * y) and bytes_eq(rd, r), what
                            assert c.tolist() == [st_mid, 0, max_iters, res_kind, iter_first, 0, 0, 0], what
                        else:
                            assert bytes_eq(xd, x + (v(0.5) * y + v(0.5) * (r / 2))) and bytes_eq(rd, r / 4), what
                            s = sc.get()
                            assert (s[0], s[1], s[3], s[7]) == (16, 64, 4, 0.5), what
                            tau1 = 2.0 if res_kind == 1 else 4.0
                            st1 = expected_status(1, max_iters, res_kind, iter_first, tau1, T)
                            assert c.tolist() == [st1, 1, max_iters, res_kind, iter_first, 0, 0, 0], what
                    if ctl.get()[0] != 0:
                        # stopped and finalized: a whole iteration leaves every buffer untouched
                        bufs = (xd, rd, rrd, pd, vd, yd, sd, td, zd, sc, ctl)
                        state = [b.get().tobytes() for b in bufs]
                        dev.call("bicgstab_fused_step_p_" + vt, n, pd, rd, vd, yd, None, sc, ctl)
                        iteration()
                        assert [b.get().tobytes() for b in bufs] == state, what
                    checked += 1
    assert checked == 96


# --------------------------------------------------------------------------- D. lock step
def convective_arrow(vt):
    """the arrow matrix of the fused-CG tests (rows of >= 1024 entries, split over CTAs) plus a
    convection term: +-1/2 on the first off-diagonals, which keeps every row's off-diagonal
    absolute sum where the 5-point stencil has both neighbours; nonsymmetric"""
    import scipy.sparse as sp
    rp, ci, va = arrow("f64")
    n = len(rp) - 1
    A = sp.csr_matrix((va, ci, rp), shape=(n, n))
    A = (A + sp.diags([np.full(n - 1, 0.5), np.full(n - 1, -0.5)], [1, -1])).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(VT[vt])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_lockstep_iterations_on_convective_arrow(dev, variant, vt):
    v = VT[vt]
    rp, ci, va = convective_arrow(vt)
    n = len(rp) - 1
    assert (np.diff(rp) >= 1024).sum() == 3
    A = Mat(dev, vt, "i32", n, n, rp, ci, va, variant)
    if not dev.mock:  # mock: plans carry no long-row list
        assert dev.l.b200_csr_plan_num_long_rows(A.plan) == 3
    inv = arrow_inv_diag(rp, ci, va)
    b = np.random.default_rng(4).uniform(-1, 1, n).astype(v)
    xd, rd = dev.put(np.zeros(n, v)), dev.put(b)
    rrd, pd, vd, yd, sd, td, zd = (dev.put(nans(n, vt)) for _ in range(7))
    invd, ref = dev.put(inv), dev.put(nans(n, vt))
    sc, ctl, work = dev.put(nans(SC, vt)), dev.put(np.zeros(CTL, np.int32)), dev.work(vt)
    factor = 1e-12 if vt == "f64" else 1e-6
    dev.call("bicgstab_fused_init_" + vt, n, rd, rrd, pd, vd, yd, sd, td, zd, sc, ctl, work, -1, 1, 1, 1, factor)
    rr = rrd.get()
    assert rr.tobytes() == b.tobytes()

    def step_p():
        dev.call("bicgstab_fused_step_p_" + vt, n, pd, rd, vd, yd, invd, sc, ctl)

    def spmv1():
        spmv_dot2(dev, A, yd, vd, rrd, sc.at(2), None, work, ctl)

    def step_s():
        dev.call("bicgstab_fused_step_s_" + vt, n, rd, vd, sd, zd, invd, sc, ctl, work)

    def spmv2():
        spmv_dot2(dev, A, zd, td, sd, sc.at(8), sc.at(2), work, ctl)

    def step_xr():
        dev.call("bicgstab_fused_step_xr_" + vt, n, xd, rd, sd, td, yd, zd, rrd, sc, ctl, work)

    for it in range(8):
        assert ctl.get()[:2].tolist() == [0, it]
        s0, p0, r0, v0, x0 = sc.get(), pd.get(), rd.get(), vd.get(), xd.get()
        step_p()
        p1, y1 = np_step_p(p0, r0, v0, inv, s0)
        assert bytes_eq(pd, p1) and bytes_eq(yd, y1), it

        spmv1()
        A.spmv(dev, yd, ref)
        v1, s1 = vd.get(), sc.get()
        assert v1.tobytes() == ref.get().tobytes(), it
        assert_sum_within(s1[2], rr * v1, vt, "rr.v")
        assert np.delete(s1, 2).tobytes() == np.delete(s0, 2).tobytes(), it

        step_s()
        alpha, s_1, z1 = np_step_s(r0, v1, inv, s1)
        s2 = sc.get()
        assert bytes_eq(sd, s_1) and bytes_eq(zd, z1) and s2[6].tobytes() == v(alpha).tobytes(), it
        assert_sum_within(s2[9], s_1 * s_1, vt, "s.s")
        assert ctl.get()[0] == 0 and ctl.get()[5] == 0, it

        spmv2()
        A.spmv(dev, zd, ref)
        t1, s3 = td.get(), sc.get()
        assert t1.tobytes() == ref.get().tobytes(), it
        assert_sum_within(s3[8], s_1 * t1, vt, "s.t")
        assert_sum_within(s3[2], t1 * t1, vt, "t.t")

        step_xr()
        omega, x1, r1 = np_step_xr(x0, s_1, t1, y1, z1, s3)
        s4 = sc.get()
        assert bytes_eq(xd, x1) and bytes_eq(rd, r1) and s4[7].tobytes() == v(omega).tobytes(), it
        assert s4[1] == s3[0], it
        assert_sum_within(s4[0], rr * r1, vt, "rho")
        assert_sum_within(s4[3], r1 * r1, vt, "rr")
        assert ctl.get()[0] == expected_status(it + 1, -1, 1, 1, np.sqrt(s4[3]), s4[5]), it

    g = dev.capture(lambda: [f() for _ in range(4) for f in (step_p, spmv1, step_s, spmv2, step_xr)])
    for _ in range(200):
        dev.call("graph_launch", g)
        if ctl.get()[0] != 0:
            break
    c = ctl.get()
    assert c[0] == 0x80 | 0x40 | 1 and c[5] == 0, c
    x = xd.get().astype(np.float64)
    import scipy.sparse as sp
    M = sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(n, n))
    assert np.linalg.norm(b - M @ x) <= 50 * factor * np.linalg.norm(b)
    bufs = (xd, rd, rrd, pd, vd, yd, sd, td, zd, sc, ctl)
    state = [a.get().tobytes() for a in bufs]
    for _ in range(2):
        dev.call("graph_launch", g)
    assert [a.get().tobytes() for a in bufs] == state


# --------------------------------------------------------------------------- E. end to end
def upwind(g, dims, vt, wind=0.8):
    """upwind convection-diffusion on a g^dims grid: the Laplacian stencil with `wind` added to the
    diagonal and subtracted from the upstream neighbour along every axis"""
    import workloads as W
    rp, ci, va = W.laplace(g, dims, vdtype=np.float64)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    va = va.copy()
    for d in range(dims):
        va[ci == rows - g ** d] -= wind
    va[ci == rows] += dims * wind
    return rp, ci, va.astype(VT[vt])


def dominant_random(n, vt):
    """cfg4's kind at a small size: random columns, a dominant diagonal, nonsymmetric"""
    import workloads as W
    rp, ci, va = W.build("cfg4", n=n)
    return rp, ci, va.astype(VT[vt])


def true_rel_res(rp, ci, va, b, x):
    import scipy.sparse as sp
    n = len(rp) - 1
    M = sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(n, n))
    b = b.astype(np.float64).reshape(-1)
    return np.linalg.norm(b - M @ x.astype(np.float64).reshape(-1)) / np.linalg.norm(b)


def host_bicgstab(hexec, rp, ci, va, b, precond, block_ptrs=None, **kw):
    import torch
    from ginkgo_b200 import api
    n = len(rp) - 1
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(b)).to(hexec.device)
        tx = torch.zeros_like(tb)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "bicgstab", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
    hexec.synchronize()
    return tx.cpu().numpy(), s.num_iterations, s.stop_status, s.used_fused


SYSTEMS = {"upwind2d": lambda vt: upwind(40, 2, vt), "upwind3d": lambda vt: upwind(14, 3, vt),
           "dominant_random": lambda vt: dominant_random(3000, vt)}


@pytest.mark.parametrize("system,kernel,reblock",
                         [(s, k, None) for s in SYSTEMS for k in ("warp", "pipe", "ring")] +
                         [("dominant_random", "warp", "3")])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
def test_fused_bicgstab_matches_oracle(hexec, monkeypatch, system, kernel, reblock, vt, precond):
    monkeypatch.setenv("B200_CSR_KERNEL", kernel)
    if reblock is not None:
        monkeypatch.setenv("B200_CSR_REBLOCK", reblock)
    rp, ci, va = SYSTEMS[system](vt)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-9 if vt == "f64" else 1e-4
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    xo, ito, stop_o = H.orc_solve("bicgstab", vt, rp, ci, va, b, np.zeros((n, 1), VT[vt]), precond, jac,
                                  max_iters=400, reduction=red)
    xd, itd, stop_d, used = host_bicgstab(hexec, rp, ci, va, b, precond, max_iters=400, reduction=red,
                                          fused_bicgstab=True)
    assert used
    # the bars of test_solvers_gpu.py::test_solver_matches_oracle for BiCGStab
    assert abs(itd - ito) <= max(3, 0.35 * ito), (itd, ito)
    assert stop_d == stop_o[0] == 0x80 | 0x40 | 2
    assert true_rel_res(rp, ci, va, b, xd) <= 20 * red and true_rel_res(rp, ci, va, b, xo) <= 20 * red
    assert H.rel_err(xo, xd) <= (1e-7 if vt == "f64" else 2e-3)


def test_fused_bicgstab_fallbacks_say_so(hexec):
    rp, ci, va = upwind(20, 2, "f64")
    n = len(rp) - 1
    rng = np.random.default_rng(2)
    b1, b2 = rng.uniform(-1, 1, (n, 1)), rng.uniform(-1, 1, (n, 2))
    kw = dict(max_iters=200, reduction=1e-8, fused_bicgstab=True)
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    x, it, st, used = host_bicgstab(hexec, rp, ci, va, b1, 4, bp, **kw)  # block Jacobi
    assert not used and st == 0x80 | 0x40 | 2
    x, it, st, used = host_bicgstab(hexec, rp, ci, va, b2, 1, **kw)  # two right-hand sides
    assert not used and st == 0x80 | 0x40 | 2
    # `fused` alone is CG's switch; the new one is off by default
    assert not host_bicgstab(hexec, rp, ci, va, b1, 1, max_iters=200, reduction=1e-8, fused=True)[3]
    assert host_bicgstab(hexec, rp, ci, va, b1, 1, **kw)[3]
