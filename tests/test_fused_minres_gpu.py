"""The fused MINRES kernels (csrc/fused_minres.cu) one at a time, through the C ABI, against the loop's
own kernels, and the host solver against the oracle's MINRES.

The kinds of assertion are those of tests/test_fused_cg_gpu.py, whose backend, buffers and references
this file imports: element-wise updates and the scalars derived from given sums are compared BIT FOR
BIT with the kernels the loop runs (b200_csr_advanced_spmv, b200_dense_sub_scaled, the scalar Jacobi
apply, b200_minres_step_1 / step_2), reductions on small-integer data for EQUALITY with the exact sum,
reductions on random data against math.fsum within gamma_h * sum |t|.

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock; the asserts about
the device's launch shapes are skipped there, each marked "mock:"."""
import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_fused_cg_gpu import (ITS, STOPPED, VARIANTS, VTS, Mat, arrow, arrow_inv_diag,  # noqa: F401
                                     assert_sum_within, backend, dev, exact_limit, exact_spmv, expected_status,
                                     hexec, int_sum, nans, spmv_case, step_sizes)
from tests.test_parity_gpu import CSR_KINDS

pytestmark = pytest.mark.gpu

SC, CTL = 16, 8
# sc: 0 alpha 1 beta 2 gamma 3 delta 4 tau0 5 threshold 6 tau 7 eta 8 eta_next 9 cos_prev 10 cos
#     11 sin_prev 12 sin
STEP1_SLOTS = (0, 1, 2, 3, 9, 10, 11, 12, 7, 8, 6)  # b200_minres_step_1's argument order


def sub_dot(dev, A, b, c, dot_ptr, work, ctl=None):
    dev.call("csr_spmv_sub_dot_%s_%s" % (A.vt, A.it), A.plan, A.n, A.ncols, A.nnz, A.rp, A.ci, A.va, b, c,
             dot_ptr, work, ctl)


def advanced(dev, A, b, c):
    """the loop's v = 1 * A z + (-1) * v"""
    ab = dev.put(np.array([1, -1], VT[A.vt]))
    dev.call("csr_advanced_spmv_%s_%s" % (A.vt, A.it), A.plan, A.n, A.ncols, A.nnz, A.rp, A.ci, A.va, ab.at(0),
             b, 1, 1, ab.at(1), c, 1)


def row_vector(vt, n, data, seed=29):
    rng = np.random.default_rng(seed)
    if data == "int":
        return rng.integers(-1, 2, size=n).astype(VT[vt])
    return rng.uniform(-1, 1, size=n).astype(VT[vt])


def mwork(dev, vt):
    size = getattr(dev.l, "b200_minres_fused_work_size_" + vt)(dev.ctx)
    return dev.put(np.full(size, np.nan, VT[vt]))


# --------------------------------------------------------------------------- A. spmv_sub_dot
@pytest.mark.parametrize("kind", CSR_KINDS + ["rect", "grid_cap"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_sub_dot(dev, kind, variant, vt, it, data):
    n, ncols, rp, ci, va, b = spmv_case(kind, vt, it, data, dev.num_sms)
    A = Mat(dev, vt, it, n, ncols, rp, ci, va, variant)
    if not dev.mock:  # mock: plans carry no variant and no long-row list
        assert dev.l.b200_csr_plan_variant(A.plan) == variant
        if kind == "split_rows":
            assert dev.l.b200_csr_plan_num_long_rows(A.plan) > 0
    c0 = row_vector(vt, n, data)
    bd, work = dev.put(b), mwork(dev, vt)
    cref = dev.put(c0)
    advanced(dev, A, bd, cref)
    c_adv = cref.get()

    c, dot = dev.put(c0), dev.put(nans(1, vt))
    sub_dot(dev, A, bd, c, dot.ptr, work)
    got_c, got_dot = c.get(), dot.get()[0]
    # c: the loop's advanced SpMV, with the dot in its epilogue
    assert got_c.tobytes() == c_adv.tobytes()
    if data == "int":
        c_exact, cabs = exact_spmv(n, rp, ci, va, b)
        c_exact = c_exact - c0.astype(np.float64)
        assert cabs.max(initial=0) + 1 < exact_limit(vt)
        assert int_sum(np.abs(b[:n]), np.abs(c_exact)) < exact_limit(vt)
        assert np.array_equal(got_c, c_exact)
        assert float(got_dot) == int_sum(b[:n], c_exact)
    else:
        assert_sum_within(got_dot, b[:n] * got_c, vt, "z.v")

    # deterministic, and the tickets reset themselves
    c2, dot2 = dev.put(c0), dev.put(nans(1, vt))
    sub_dot(dev, A, bd, c2, dot2.ptr, work)
    assert c2.get().tobytes() == got_c.tobytes() and dot2.get().tobytes() == dot.get().tobytes()

    # a stopped solver: nothing is written (incl. the long-row kernel and its dot fix)
    ctl = dev.put(np.array([STOPPED, 3, 0, 0, 0, 0, 0, 0], np.int32))
    c3, dot3 = dev.put(c0), dev.put(nans(1, vt))
    sub_dot(dev, A, bd, c3, dot3.ptr, work, ctl)
    assert c3.get().tobytes() == c0.tobytes() and np.isnan(dot3.get()).all()


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
def test_spmv_sub_dot_empty_matrix_writes_zero(dev, vt, it):
    A = Mat(dev, vt, it, 0, 5, np.zeros(1, IT[it]), np.zeros(0, IT[it]), np.zeros(0, VT[vt]))
    b, c, dot = dev.put(np.ones(5, VT[vt])), dev.put(nans(0, vt)), dev.put(nans(1, vt))
    sub_dot(dev, A, b, c, dot.ptr, mwork(dev, vt))
    assert dot.get().tolist() == [0.0]
    ctl = dev.put(np.array([STOPPED, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dot = dev.put(nans(1, vt))
    sub_dot(dev, A, b, c, dot.ptr, mwork(dev, vt), ctl)
    assert np.isnan(dot.get()).all()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_sub_dot_graph_replay_matches_eager(dev, variant, vt, data):
    """captured with its fork / join on the auxiliary stream (long-row kernel) and the dot fix: the
    rows split over CTAs enter the sum exactly once per replay"""
    n, ncols, rp, ci, va, b = spmv_case("split_rows", vt, "i64", data, dev.num_sms)
    A = Mat(dev, vt, "i64", n, ncols, rp, ci, va, variant)
    c0 = row_vector(vt, n, data)
    bd, work = dev.put(b), mwork(dev, vt)
    c, dot = dev.put(c0), dev.put(nans(1, vt))
    sub_dot(dev, A, bd, c, dot.ptr, work)
    eager_c, eager_dot = c.get(), dot.get()
    c2, dot2 = dev.put(c0), dev.put(nans(1, vt))
    g = dev.capture(lambda: sub_dot(dev, A, bd, c2, dot2.ptr, work))
    for _ in range(2):
        c2.set(c0)
        dot2.set(nans(1, vt))
        dev.call("graph_launch", g)
        dev.sync()
        assert c2.get().tobytes() == eager_c.tobytes() and dot2.get().tobytes() == eager_dot.tobytes()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_spmv_sub_dot_alternating_with_other_reductions(dev, variant, vt):
    """spmv_sub_dot shares its ticket with spmv_dot, lanczos and update theirs with the fused CG's step
    kernels, and dense_compute_dot uses the same counter array: each must leave its ticket at 0"""
    rng = np.random.default_rng(6)
    mats = []
    for kind in ("grid_cap", "split_rows"):
        n, ncols, rp, ci, va, b = spmv_case(kind, vt, "i32", "int", dev.num_sms)
        A = Mat(dev, vt, "i32", n, ncols, rp, ci, va, variant)
        c_exact, _ = exact_spmv(n, rp, ci, va, b)
        mats.append((A, dev.put(b), c_exact, int_sum(b[:n], c_exact)))
    nx = 2048 * 4 * dev.num_sms + 777  # the step kernels at their grid cap
    v = rng.integers(-1, 2, size=nx).astype(VT[vt])
    inv = rng.integers(1, 4, size=nx).astype(VT[vt])
    vd, qd, invd = dev.put(v), dev.put(np.zeros(nx, VT[vt])), dev.put(inv)
    ctl = dev.put(np.array([0, 0, -1, 2, 1, 0, 0, 0], np.int32))
    res, work = dev.put(nans(1, vt)), mwork(dev, vt)
    for rnd in range(2):
        for A, bd, c_exact, d_bc in mats:
            c, dots = dev.put(np.zeros(A.n, VT[vt])), dev.put(nans(2, vt))
            sub_dot(dev, A, bd, c, dots.at(0), work, ctl)
            c1 = dev.put(nans(A.n, vt))
            A.spmv_dot(dev, bd, c1, dots.at(1), work, ctl)
            assert np.array_equal(c.get(), c_exact) and np.array_equal(c1.get(), c_exact), rnd
            assert [float(d) for d in dots.get()] == [d_bc, d_bc], rnd
            # alpha = 0: v stays, beta = v.(d v) exact on integers
            sc = dev.put(np.array([0] * 6 + [1] + [0] * 9, VT[vt]))
            dev.call("minres_fused_lanczos_" + vt, nx, vd, qd, invd, sc, ctl, work)
            assert sc.get()[1] == np.sqrt(VT[vt](int_sum(v * v, inv))), rnd
            dev.call("dense_compute_dot_" + vt, nx, 1, vd, 1, invd, 1, res)
            assert float(res.get()[0]) == int_sum(v, inv), rnd


# --------------------------------------------------------------------------- B. lanczos and update
def loop_lanczos(dev, vt, n, v, q, inv, sc0):
    """the loop's sub_scaled, Jacobi apply, dot and minres::step_1 on copies; returns (v, sc)"""
    vl, ql, L = dev.put(v), dev.put(q), dev.put(sc0)
    dev.call("dense_sub_scaled_" + vt, n, 1, L.at(0), 1, ql, 1, vl, 1)
    zt = dev.put(nans(n, vt))
    if inv is None:
        dev.call("dense_copy_" + vt, n, 1, vl, 1, zt, 1)
    else:
        dev.call("jacobi_simple_scalar_apply_" + vt, n, 1, dev.put(inv), vl, 1, zt, 1)
    dev.call("dense_compute_conj_dot_" + vt, n, 1, vl, 1, zt, 1, L.at(1))
    stop = dev.put(np.zeros(1, np.uint8))
    dev.call("minres_step_1_" + vt, 1, *[L.at(k) for k in STEP1_SLOTS], stop)
    return vl.get(), L.get()


def loop_update(dev, vt, n, x, p_w, p_r, z, q, v, inv, sc):
    """std::swap(p, p_prev) already done: minres::step_2 on copies with z~ = d v; returns x, p, z, q, v"""
    bufs = [dev.put(a) for a in (x, p_w, p_r, z, q, v)]
    xl, pl, ppl, zl, ql, vl = bufs
    zt, qprev = dev.put(nans(n, vt)), dev.put(nans(n, vt))
    if inv is None:
        dev.call("dense_copy_" + vt, n, 1, vl, 1, zt, 1)
    else:
        dev.call("jacobi_simple_scalar_apply_" + vt, n, 1, dev.put(inv), vl, 1, zt, 1)
    L = dev.put(sc)
    stop = dev.put(np.zeros(1, np.uint8))
    dev.call("minres_step_2_" + vt, n, 1, xl, 1, pl, 1, ppl, 1, zl, 1, zt, 1, ql, 1, qprev, 1, vl, 1,
             L.at(0), L.at(1), L.at(2), L.at(3), L.at(10), L.at(7), stop)
    return [b.get() for b in (xl, pl, zl, ql, vl)]


def scalars(rng, vt, **fix):
    sc = rng.uniform(-1, 1, SC).astype(VT[vt])
    sc[4:6] = [1, 1e-3]
    sc[6] = abs(sc[6])
    for k, val in fix.items():
        sc[int(k[1:])] = val
    return sc


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("guard", [None, "alpha", "beta"])
def test_lanczos_matches_the_loop(dev, size, vt, precond, guard):
    """integer data keep both dots exact, so the loop's step_1 sees the fused kernel's beta and every
    scalar must match bit for bit.  guard alpha: alpha = gamma = 0 (no subtraction; the Givens rotation
    takes its zero branch); guard beta: v = alpha q, so v becomes 0 and beta = 0."""
    n = step_sizes(dev.num_sms)[size]
    rng = np.random.default_rng(40 + size)
    v = rng.integers(-2, 3, n).astype(VT[vt])
    q = rng.integers(-2, 3, n).astype(VT[vt])
    inv = rng.integers(1, 4, n).astype(VT[vt]) if precond else None
    sc0 = scalars(rng, vt, s0=VT[vt](2))
    if guard == "alpha":
        sc0[0] = sc0[2] = 0
    if guard == "beta":
        v = (sc0[0] * q).astype(VT[vt])
    work = mwork(dev, vt)
    vd, sc, ctl = dev.put(v), dev.put(sc0), dev.put(np.array([0, 3, -1, 2, 1, 0, 0, 0], np.int32))
    dev.call("minres_fused_lanczos_" + vt, n, vd, dev.put(q), None if inv is None else dev.put(inv), sc, ctl, work)
    vl, L = loop_lanczos(dev, vt, n, v, q, inv, sc0)
    assert vd.get().tobytes() == vl.tobytes()
    assert sc.get().tobytes() == L.tobytes()
    if guard == "beta":
        assert L[1] == 0 and not np.any(vl)
    if guard == "alpha":
        assert vl.tobytes() == v.tobytes() and (L[10], L[12]) == (0, 1)
    assert ctl.get().tolist() == [0, 3, -1, 2, 1, 0, 0, 0]


@pytest.mark.parametrize("vt", VTS)
def test_lanczos_sum_on_random_data(dev, vt):
    n = step_sizes(dev.num_sms)[-1]
    rng = np.random.default_rng(3)
    v, q, inv = (rng.uniform(-1, 1, n).astype(VT[vt]) for _ in range(3))
    sc0 = scalars(rng, vt)
    vd, sc = dev.put(v), dev.put(sc0)
    dev.call("minres_fused_lanczos_" + vt, n, vd, dev.put(q), dev.put(inv), sc,
             dev.put(np.array([0, 0, -1, 0, 1, 0, 0, 0], np.int32)), mwork(dev, vt))
    vl, _ = loop_lanczos(dev, vt, n, v, q, inv, sc0)
    assert vd.get().tobytes() == vl.tobytes()
    # beta = sqrt(sum): square it back in float64 (one rounding of the sqrt, relative 2u, doubled)
    terms = vl * (vl * inv)
    beta_sq = float(sc.get()[1]) ** 2
    ref = float(np.sum(terms.astype(np.float64)))
    tol = 4 * float(np.finfo(VT[vt]).eps) * abs(ref) + n * float(np.finfo(VT[vt]).eps) * float(np.sum(np.abs(terms)))
    assert abs(beta_sq - ref) <= tol


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("parity", [0, 1])
@pytest.mark.parametrize("guard", [None, "alpha", "beta"])
def test_update_matches_step_2(dev, size, vt, precond, parity, guard):
    n = step_sizes(dev.num_sms)[size]
    rng = np.random.default_rng(70 + size)
    x, p0, p1, z, q, v = (rng.uniform(-1, 1, n).astype(VT[vt]) for _ in range(6))
    inv = rng.uniform(0.5, 2, n).astype(VT[vt]) if precond else None
    sc0 = scalars(rng, vt)
    if guard:
        sc0[0 if guard == "alpha" else 1] = 0  # safe_divide's zero divisor
    iters = 4 + parity
    bufs = [dev.put(a) for a in (x, p0, p1, z, q, v)]
    sc = dev.put(sc0)
    ctl = dev.put(np.array([0, iters, -1, 2, 1, 0, 0, 0], np.int32))
    dev.call("minres_fused_update_" + vt, n, *bufs, None if inv is None else dev.put(inv), sc, ctl)
    # iteration k writes p1 when k is even, p0 when odd; the other is p_prev
    p_w, p_r = (p0, p1) if iters % 2 else (p1, p0)
    xl, pl, zl, ql, vl = loop_update(dev, vt, n, x, p_w, p_r, z, q, v, inv, sc0)
    gx, g0, g1, gz, gq, gv = (b.get() for b in bufs)
    gp, gpp = (g0, g1) if iters % 2 else (g1, g0)
    assert gpp.tobytes() == p_r.tobytes()
    for got, want in ((gx, xl), (gp, pl), (gz, zl), (gq, ql), (gv, vl)):
        assert got.tobytes() == want.tobytes()
    want_sc = sc0.copy()
    want_sc[1], want_sc[2] = sc0[2], sc0[1]  # std::swap(gamma, beta)
    assert sc.get().tobytes() == want_sc.tobytes()
    c = ctl.get()
    assert c[1] == iters + 1
    tau = np.sqrt(np.abs(sc0[6]))
    assert c[0] == expected_status(iters + 1, -1, 2, True, tau, sc0[5])


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
def test_stopping_table(dev, vt, baseline):
    """init checks iteration 0, update's last CTA iteration k + 1: ids, converged and finalized bits in
    both criterion orders, the threshold factor * tau0 with tau0 = 1 for the absolute baseline"""
    v = VT[vt]
    factor = v(1e-3)
    tau0 = v(4.0)
    thr = factor * (v(1) if baseline == 2 else tau0)
    n = 100
    cases = 0
    for max_iters in (-1, 0, 1, 2):
        for res_kind in (0, 2):
            if max_iters < 0 and res_kind == 0:
                continue
            for iter_first in (0, 1):
                for tau in (thr * thr * v(0.25), thr * thr, thr * thr * v(4), -thr * thr):
                    sc0 = np.zeros(SC, v)
                    sc0[4], sc0[6] = tau0, tau
                    sc = dev.put(sc0)
                    ctl = dev.put(np.zeros(CTL, np.int32))
                    dev.call("minres_fused_init_" + vt, sc, ctl, max_iters, res_kind, iter_first, baseline, factor)
                    c, s = ctl.get(), sc.get()
                    assert s[5] == thr and s[4] == (1 if baseline == 2 else tau0)
                    assert c[1:5].tolist() == [0, max_iters, res_kind, iter_first]
                    taun = np.sqrt(np.abs(tau))
                    want = expected_status(0, max_iters, res_kind, iter_first, taun, thr)
                    assert c[0] == want, (max_iters, res_kind, iter_first, tau)
                    if want:
                        continue
                    z = [dev.put(np.zeros(n, v)) for _ in range(6)]
                    dev.call("minres_fused_update_" + vt, n, *z, None, sc, ctl)
                    c = ctl.get()
                    assert c[1] == 1 and c[0] == expected_status(1, max_iters, res_kind, iter_first, taun, thr)
                    cases += 1
    assert cases > 8


@pytest.mark.parametrize("vt", VTS)
def test_kernels_are_noops_after_a_stop(dev, vt):
    n = 5000
    rng = np.random.default_rng(1)
    arrs = [rng.uniform(-1, 1, n).astype(VT[vt]) for _ in range(6)]
    bufs = [dev.put(a) for a in arrs]
    sc0 = scalars(rng, vt)
    sc = dev.put(sc0)
    ctl0 = np.array([STOPPED, 7, 9, 2, 1, 0, 0, 0], np.int32)
    ctl = dev.put(ctl0)
    dev.call("minres_fused_lanczos_" + vt, n, bufs[5], bufs[4], None, sc, ctl, mwork(dev, vt))
    dev.call("minres_fused_update_" + vt, n, *bufs, None, sc, ctl)
    assert all(b.get().tobytes() == a.tobytes() for b, a in zip(bufs, arrs))
    assert sc.get().tobytes() == sc0.tobytes() and ctl.get().tobytes() == ctl0.tobytes()


# --------------------------------------------------------------------------- C. lock step
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_lockstep_iterations_on_indefinite_arrow(dev, variant, vt):
    """the arrow matrix (rows split over CTAs) with its diagonal shifted by -3: symmetric indefinite,
    positive diagonal.  Eight iterations launch by launch, each compared with the loop's kernels fed
    the fused path's own scalars; then graphs of five iterations replayed to the stop at 63 iterations,
    and past it without a change."""
    v_ = VT[vt]
    rp, ci, va = arrow(vt, shift=-3)
    n = len(rp) - 1
    inv = arrow_inv_diag(rp, ci, va)
    assert (inv > 0).all()
    A = Mat(dev, vt, "i32", n, n, rp, ci, va, variant)
    if not dev.mock:
        assert dev.l.b200_csr_plan_num_long_rows(A.plan) > 0
    b = np.random.default_rng(5).uniform(-1, 1, n).astype(v_)
    work = mwork(dev, vt)
    invd = dev.put(inv)
    # the loop's set-up with x = 0: r = b, z = M r, beta = r.z, tau = z.z, minres::initialize
    r, z = dev.put(b), dev.put(nans(n, vt))
    dev.call("jacobi_simple_scalar_apply_" + vt, n, 1, invd, r, 1, z, 1)
    sc = dev.put(np.zeros(SC, v_))
    dev.call("dense_compute_conj_dot_" + vt, n, 1, r, 1, z, 1, sc.at(1))
    dev.call("dense_compute_conj_dot_" + vt, n, 1, z, 1, z, 1, sc.at(6))
    x, q, vv, p0, p1 = (dev.put(np.zeros(n, v_)) for _ in range(5))
    stop = dev.put(np.zeros(1, np.uint8))
    dev.call("minres_initialize_" + vt, n, 1, r, 1, z, 1, p0, 1, p1, 1, q, 1, vv, 1, vv, 1, sc.at(1), sc.at(2),
             sc.at(3), sc.at(9), sc.at(10), sc.at(11), sc.at(12), sc.at(8), sc.at(7), stop)
    dev.call("dense_compute_norm2_" + vt, n, 1, dev.put(b), 1, sc.at(4))
    red = 1e-6 if vt == "f64" else 1e-3
    ctl = dev.put(np.zeros(CTL, np.int32))
    dev.call("minres_fused_init_" + vt, sc, ctl, 63, 2, 1, 0, v_(red))
    assert ctl.get()[0] == 0
    for k in range(8):
        # spmv_sub_dot against the loop's advanced SpMV
        zv, vv0 = z.get(), vv.get()
        vl = dev.put(vv0)
        advanced(dev, A, dev.put(zv), vl)
        sub_dot(dev, A, z, vv, sc.at(0), work, ctl)
        assert vv.get().tobytes() == vl.get().tobytes(), k
        s = sc.get()
        assert_sum_within(s[0], zv * vv.get(), vt, "alpha")
        # lanczos: v exactly the loop's; beta within the sum bound; step_1 from that beta
        v_before, q_now = vv.get(), q.get()
        dev.call("minres_fused_lanczos_" + vt, n, vv, q, invd, sc, ctl, work)
        vl, L = loop_lanczos(dev, vt, n, v_before, q_now, inv, s)
        assert vv.get().tobytes() == vl.tobytes(), k
        s1 = sc.get()
        assert abs(float(s1[1]) - float(L[1])) <= 64 * float(np.finfo(v_).eps) * abs(float(L[1])), k
        # update: minres::step_2 fed with the fused scalars
        bufs = [x, p0, p1, z, q, vv]
        before = [a.get() for a in bufs]
        dev.call("minres_fused_update_" + vt, n, *bufs, invd, sc, ctl)
        bx, b0, b1, bz, bq, bv = before
        p_w, p_r = (b0, b1) if k % 2 else (b1, b0)
        want = loop_update(dev, vt, n, bx, p_w, p_r, bz, bq, bv, inv, s1)
        got_p = (p0 if k % 2 else p1).get()
        for got, w in zip((x.get(), got_p, z.get(), q.get(), vv.get()), want):
            assert got.tobytes() == w.tobytes(), k
        c = ctl.get()
        assert c[1] == k + 1 and c[0] == 0, (k, c)
    # the rest of the solve as graphs of 5 iterations, then replays past the stop change nothing
    dev.call("synchronize")

    def batch():
        for _ in range(5):
            sub_dot(dev, A, z, vv, sc.at(0), work, ctl)
            dev.call("minres_fused_lanczos_" + vt, n, vv, q, invd, sc, ctl, work)
            dev.call("minres_fused_update_" + vt, n, x, p0, p1, z, q, vv, invd, sc, ctl)
    g = dev.capture(batch)
    for _ in range(20):
        dev.call("graph_launch", g)
        if ctl.get()[0] != 0:
            break
    c = ctl.get()
    # the Iteration criterion stops the solve in the middle of the twelfth batch
    assert c[0] == 0x40 | 1 and c[1] == 63, c
    assert 0 < sc.get()[6] and np.isfinite(x.get()).all()
    bufs = [x, p0, p1, z, q, vv, sc, ctl]
    state = [a.get().tobytes() for a in bufs]
    for _ in range(2):
        dev.call("graph_launch", g)
    assert [a.get().tobytes() for a in bufs] == state


# --------------------------------------------------------------------------- D. end to end
def indefinite_laplacian(g, dims, shift, vt, seed=12):
    """the g^dims Laplacian plus diag(uniform(0, 0.5)) - shift I"""
    import workloads as W
    rp, ci, va = W.laplace(g, dims, vdtype=np.float64)
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    va = va.copy()
    va[ci == rows] += np.random.default_rng(seed).uniform(0, 0.5, n) - shift
    return rp, ci, va.astype(VT[vt])


def true_rel_res(rp, ci, va, b, x):
    import scipy.sparse as sp
    n = len(rp) - 1
    M = sp.csr_matrix((va.astype(np.float64), ci, rp), shape=(n, n))
    b = b.astype(np.float64).reshape(-1)
    return np.linalg.norm(b - M @ x.astype(np.float64).reshape(-1)) / np.linalg.norm(b)


def host_minres(hexec, rp, ci, va, b, precond, block_ptrs=None, **kw):
    import torch
    from ginkgo_b200 import api
    n = len(rp) - 1
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(b)).to(hexec.device)
        tx = torch.zeros_like(tb)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "minres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
    hexec.synchronize()
    return tx.cpu().numpy(), s.num_iterations, s.stop_status, s.used_fused


SYSTEMS = {"laplace2d": lambda vt: indefinite_laplacian(30, 2, 0.3, vt),
           "laplace3d": lambda vt: indefinite_laplacian(16, 3, 0.5, vt)}


def test_systems_are_indefinite():
    import scipy.sparse as sp
    for name, want in (("laplace2d", 3), ("laplace3d", 4)):
        rp, ci, va = SYSTEMS[name]("f64")
        n = len(rp) - 1
        M = sp.csr_matrix((va, ci, rp), shape=(n, n)).toarray()
        assert np.allclose(M, M.T)
        assert int((np.linalg.eigvalsh(M) < 0).sum()) == want, name


@pytest.mark.parametrize("system", list(SYSTEMS))
@pytest.mark.parametrize("kernel", ["warp", "pipe", "ring"])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
def test_fused_minres_matches_oracle(hexec, monkeypatch, system, kernel, vt, precond):
    monkeypatch.setenv("B200_CSR_KERNEL", kernel)
    rp, ci, va = SYSTEMS[system](vt)
    n = len(rp) - 1
    b = np.random.default_rng(12).uniform(-1, 1, (n, 1)).astype(VT[vt])
    red = 1e-8 if vt == "f64" else 1e-4
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    kw = dict(max_iters=1000, reduction=red, res_kind=2)
    xo, ito, stop_o = H.orc_solve("minres", vt, rp, ci, va, b, np.zeros((n, 1), VT[vt]), precond, jac, **kw)
    xd, itd, stop_d, used = host_minres(hexec, rp, ci, va, b, precond, fused_minres=True, **kw)
    assert used
    # the bars the loop's Minres meets in test_zz_late_gpu.py
    assert abs(itd - ito) <= max(3, 0.2 * ito), (itd, ito)
    assert stop_d == stop_o[0] == 0x80 | 0x40 | 2
    assert true_rel_res(rp, ci, va, b, xd) <= 20 * red and true_rel_res(rp, ci, va, b, xo) <= 20 * red


def test_fused_minres_fallbacks_take_the_loop(hexec):
    rp, ci, va = indefinite_laplacian(20, 2, 0.3, "f64")
    n = len(rp) - 1
    rng = np.random.default_rng(2)
    b1, b2 = rng.uniform(-1, 1, (n, 1)), rng.uniform(-1, 1, (n, 2))
    kw = dict(max_iters=300, reduction=1e-8, res_kind=2)
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    cases = [(b1, 1, None, dict()),                        # the default: off
             (b1, 1, None, dict(fused=True)),              # Cg's switch alone
             (b1, 4, bp, dict(fused_minres=True)),         # block Jacobi
             (b1, 1, None, dict(fused_minres=True, res_kind=1)),  # ResidualNorm
             (b2, 1, None, dict(fused_minres=True))]       # two right-hand sides
    for b, pre, bpp, extra in cases:
        args = dict(kw, **extra)
        x, it, st, used = host_minres(hexec, rp, ci, va, b, pre, bpp, **args)
        assert not used, extra
        args.pop("fused_minres", None)
        args.pop("fused", None)
        xl, itl, stl, usedl = host_minres(hexec, rp, ci, va, b, pre, bpp, fused=False, **args)
        assert (it, st) == (itl, stl) and x.tobytes() == xl.tobytes() and st & 0x80, extra
    assert host_minres(hexec, rp, ci, va, b1, 1, fused_minres=True, **kw)[3]
