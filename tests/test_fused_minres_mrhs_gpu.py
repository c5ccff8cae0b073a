"""The fused MINRES kernels for several right-hand sides (csrc/fused_minres_mrhs.cu) one at a time through
the C ABI against numpy and the oracle, then solver::Minres with with_fused_multi_rhs(true) against the
oracle's multi-column MINRES.

The kinds of assertion are those of test_fused_cg_mrhs_gpu.py and test_fused_minres_gpu.py, whose
backend, buffers and references this file imports: element-wise results and the scalars derived from
given sums are compared BIT FOR BIT with the oracle's advanced SpMV, minres::step_1 and minres::step_2
(the library is built with -fmad=false; numpy in the value type rounds as the device does); sums on
small-integer data must be exact; sums on random data must lie within gamma_h * sum |t| of math.fsum.
Every vector is n x k row-major (stride k), every scalar slot s of column j is sc[s k + j].

Each test item runs every case of its area in a loop (each(): a failure names its case), so the file
adds nine items to the GPU suite rather than one per case.

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock; the asserts about the
device's launch shapes are skipped there, each marked "mock:"."""
import itertools

import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_fused_cg_gpu import (ITS, STOPPED, VTS, arrow, arrow_inv_diag, assert_sum_within,  # noqa: F401
                                     backend, dev, expected_status, hexec, int_sum)
from tests.test_fused_cg_mrhs_gpu import KS, SPMV_CTAS_PER_SM, SPMV_THREADS, big_case, lanes
from tests.test_fused_minres_cpu import indefinite_laplacian
from tests.test_fused_minres_gpu import SC, STEP1_SLOTS, true_rel_res
from tests.test_parity_gpu import CSR_KINDS, csr_case

pytestmark = pytest.mark.gpu

STEP_THREADS, STEP_CTAS_PER_SM = 512, 4  # fused_common.cuh / fused_mrhs.cuh: lanczos and update


def each(cases, check):
    """check(*case) for every case, in one test item; a failure names its case"""
    n = 0
    for case in cases:
        try:
            check(*case)
        except AssertionError as e:
            raise AssertionError("case %r: %s" % (case, e)) from e
        n += 1
    assert n > 0


def nans(shape, vt):
    return np.full(shape, np.nan, VT[vt])


def work(dev, vt, k):
    size = getattr(dev.l, "b200_minres_mrhs_work_size_" + vt)(dev.ctx, k)
    return dev.put(np.full(size, np.nan, VT[vt]))


def step_rows(num_sms, k):
    """row counts for lanczos / update: one row, a few CTAs, and the grid at its cap"""
    return [1, 777, STEP_CTAS_PER_SM * num_sms * (STEP_THREADS // lanes(k)) * 4 + 999]


def slots(sc, k):
    """sc[16k] as 16 contiguous rows of k (slot s of column j at [s, j])"""
    return np.ascontiguousarray(sc.reshape(SC, k))


# --------------------------------------------------------------------------- A. spmv_sub_mdot
def oracle_sub(orc, vt, it, n, m, rp, ci, va, z, c0, k):
    """the loop's v = 1 * A z + (-1) * v with num_rhs = k"""
    c = np.ascontiguousarray(c0).copy()
    one, neg = np.ones(1, VT[vt]), -np.ones(1, VT[vt])
    orc("csr_advanced_spmv_%s_%s" % (vt, it), n, m, len(va), rp, ci, va, one, np.ascontiguousarray(z), k, k,
        neg, c, k)
    return c


def run_sub_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, data, graph=False):
    rng = np.random.default_rng(k + 7)
    if data == "int":
        va = rng.integers(-1, 2, size=len(va)).astype(VT[vt])
        z = rng.integers(-2, 3, size=(m, k)).astype(VT[vt])
        c0 = rng.integers(-1, 2, size=(n, k)).astype(VT[vt])
    else:
        z = rng.uniform(-1, 1, size=(m, k)).astype(VT[vt])
        c0 = rng.uniform(-1, 1, size=(n, k)).astype(VT[vt])
    ref = oracle_sub(orc, vt, it, n, m, rp, ci, va, z, c0, k)
    d = [dev.put(a) for a in (rp, ci, va, z)]
    c, dots, w = dev.put(c0), dev.put(nans(k, vt)), work(dev, vt, k)
    args = ("csr_spmv_sub_mdot_%s_%s" % (vt, it), n, m, len(va), d[0], d[1], d[2], d[3], k, c, dots, w, None)
    dev.call(*args)
    got_c, got_dots = c.get().reshape(n, k), dots.get()
    assert got_c.tobytes() == ref.tobytes()
    for j in range(k):
        if data == "int":
            assert got_dots[j] == int_sum(z[:n, j], ref[:, j]), j
        else:
            assert_sum_within(got_dots[j], z[:n, j] * ref[:, j], vt, "alpha %d" % j)
    if graph:  # a replayed graph gives the eager run's bits, twice
        g = dev.capture(lambda: dev.call(*args))
        for _ in range(2):
            c.set(c0)
            dots.set(nans(k, vt))
            dev.call("graph_launch", g)
            dev.sync()
            assert c.get().tobytes() == got_c.tobytes() and dots.get().tobytes() == got_dots.tobytes()
    # a raised ctl[0]: nothing is written
    c.set(c0)
    dots.set(nans(k, vt))
    dev.call(*(args[:-1] + (dev.put(np.array([1, 0, 0, 0, 0, 0, 0, 0], np.int32)),)))
    assert c.get().tobytes() == c0.tobytes() and np.isnan(dots.get()).all()


def check_spmv_sub_mdot(dev, orc, kind, k, vt, it, data):
    n, m, rp, ci, va = csr_case(np.random.default_rng(17), kind, vt, it)
    m = max(n, m)  # z has a row per column and the dot reads its first n rows
    run_sub_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, data)


def check_spmv_sub_mdot_capped_grid_and_graph(dev, orc, k, vt, it):
    n, m, rp, ci, va = big_case(vt, it, dev.num_sms, k)
    assert n / (SPMV_THREADS // lanes(k) * 4) > SPMV_CTAS_PER_SM * dev.num_sms
    run_sub_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, "rand", graph=True)
    run_sub_mdot(dev, orc, vt, it, n, m, rp, ci, va, k, "int")


def check_spmv_sub_mdot_empty_matrix_writes_zero(dev, vt):
    k = 5
    e = dev.put(np.zeros(1, np.int32))
    dots = dev.put(nans(k, vt))
    dev.call("csr_spmv_sub_mdot_%s_i32" % vt, 0, 0, 0, dev.put(np.zeros(1, np.int32)), e, e, e, k, e, dots,
             work(dev, vt, k), None)
    assert np.array_equal(dots.get(), np.zeros(k, VT[vt]))


def test_spmv_sub_mdot(dev, orc):
    """every CSR_KINDS matrix, k = 2 .. 32, both value and index types, integer and random data"""
    each(itertools.product(CSR_KINDS, KS, VTS, ITS, ["int", "rand"]),
         lambda *case: check_spmv_sub_mdot(dev, orc, *case))


def test_spmv_sub_mdot_capped_grid_graph_and_empty_matrix(dev, orc):
    each(itertools.product([2, 8, 32], [("f64", "i32"), ("f32", "i64")]),
         lambda k, types: check_spmv_sub_mdot_capped_grid_and_graph(dev, orc, k, *types))
    each([(vt,) for vt in VTS], lambda vt: check_spmv_sub_mdot_empty_matrix_writes_zero(dev, vt))


# --------------------------------------------------------------------------- B. lanczos and update
def oracle_step_1(orc, vt, k, S, beta_sq, status):
    """minres::step_1 of the oracle on slot rows S (16 x k) with beta = beta_sq; returns the new rows"""
    S = S.copy()
    S[1] = beta_sq
    orc("minres_step_1_" + vt, k, *[S[s] for s in STEP1_SLOTS], np.ascontiguousarray(status))
    return S


def scalars(rng, vt, k):
    S = rng.uniform(-1, 1, (SC, k)).astype(VT[vt])
    S[4], S[5], S[6] = 1, 1e-3, np.abs(S[6])
    S[13:] = 0
    return S


def check_lanczos_matches_the_loop(dev, orc, k, size, vt, precond):
    """integer data keep the dots exact, so the oracle's step_1 sees the device's beta and every scalar
    must match bit for bit.  Column 0: alpha = gamma = 0 (v -= 0 q still runs; the Givens rotation takes
    its zero branch).  Column 1: v = alpha q, so beta = 0.  Column 2: alpha = 0 with an infinite q entry
    gives the loop's NaN.  The last column has stopped: its NaN sentinels stay."""
    v_ = VT[vt]
    n = step_rows(dev.num_sms, k)[size]
    rng = np.random.default_rng(40 + k + size)
    v = rng.integers(-2, 3, (n, k)).astype(v_)
    q = rng.integers(-2, 3, (n, k)).astype(v_)
    inv = rng.integers(1, 4, n).astype(v_) if precond else None
    S = scalars(rng, vt, k)
    S[0] = 2
    S[0, 0] = S[2, 0] = 0
    v[:, 1] = S[0, 1] * q[:, 1]
    S[0, 2] = 0
    q[0, 2] = np.inf
    status = np.zeros(k, np.uint8)
    status[k - 1] = STOPPED
    S[:, k - 1] = np.nan
    v[:, k - 1] = np.nan
    sc, vd = dev.put(S), dev.put(v)
    ctl = dev.put(np.array([0, 3, -1, 2, 1, 0, 0, 0], np.int32))
    dev.call("minres_mrhs_lanczos_" + vt, n, k, vd, dev.put(q), None if inv is None else dev.put(inv), sc,
             dev.put(status), ctl, work(dev, vt, k))
    # the loop: sub_scaled with a 1 x k alpha (never skipped), the Jacobi apply, the dot, step_1
    want_v = v.copy()
    run = [j for j in range(k) if j != k - 1]
    with np.errstate(invalid="ignore"):  # 0 * inf in column 2
        want_v[:, run] = v[:, run] - S[0, run] * q[:, run]
    got_v = vd.get().reshape(n, k)
    assert np.isnan(got_v[0, 2]) and np.isnan(got_v[:, k - 1]).all()
    finite = np.ones((n, k), bool)
    finite[0, 2] = finite[:, k - 1] = False
    assert got_v[finite].tobytes() == want_v[finite].tobytes()
    zt = want_v * inv[:, None] if precond else want_v
    beta_sq = np.zeros(k, v_)
    for j in run:
        if j != 2:
            beta_sq[j] = int_sum(want_v[:, j], zt[:, j])
    want = oracle_step_1(orc, vt, k, S, beta_sq, status)
    got = slots(sc.get(), k)
    exact = [j for j in run if j != 2]
    assert got[:, exact].tobytes() == want[:, exact].tobytes()
    assert np.isnan(got[:, k - 1]).all()  # the stopped column's scalars: untouched sentinels
    assert np.isnan(got[1, 2])  # the NaN reaches beta
    assert got[1, 1] == 0 and (got[10, 0], got[12, 0]) == (0, 1)
    assert ctl.get().tolist() == [0, 3, -1, 2, 1, 0, 0, 0]


def check_lanczos_sums_on_random_data(dev, vt):
    k = 8
    n = step_rows(dev.num_sms, k)[-1]
    rng = np.random.default_rng(3)
    v, q = (rng.uniform(-1, 1, (n, k)).astype(VT[vt]) for _ in range(2))
    inv = rng.uniform(0.5, 2, n).astype(VT[vt])
    S = scalars(rng, vt, k)
    vd, sc = dev.put(v), dev.put(S)
    dev.call("minres_mrhs_lanczos_" + vt, n, k, vd, dev.put(q), dev.put(inv), sc, dev.put(np.zeros(k, np.uint8)),
             dev.put(np.array([0, 0, -1, 0, 1, 0, 0, 0], np.int32)), work(dev, vt, k))
    want_v = v - S[0] * q
    assert vd.get().reshape(n, k).tobytes() == want_v.tobytes()
    beta = slots(sc.get(), k)[1]
    eps = float(np.finfo(VT[vt]).eps)
    for j in range(k):
        # beta = sqrt(sum): square it back in float64 (one rounding of the sqrt, relative 2u, doubled)
        terms = want_v[:, j] * (want_v[:, j] * inv)
        ref = float(np.sum(terms.astype(np.float64)))
        tol = 4 * eps * abs(ref) + n * eps * float(np.sum(np.abs(terms)))
        assert abs(float(beta[j]) ** 2 - ref) <= tol, j


def test_lanczos_matches_the_loop(dev, orc):
    each(itertools.product([4, 5, 17, 32], range(3), VTS, [False, True]),
         lambda *case: check_lanczos_matches_the_loop(dev, orc, *case))
    each([(vt,) for vt in VTS], lambda vt: check_lanczos_sums_on_random_data(dev, vt))


def oracle_update(orc, vt, k, x, p_w, p_r, z, q, v, inv, S, status):
    """the loop's std::swap(p, p_prev) done: z~ = d v, then the oracle's minres::step_2"""
    x, p_w, z, q, v = (np.ascontiguousarray(a).copy() for a in (x, p_w, z, q, v))
    n = x.shape[0]
    zt = v * inv[:, None] if inv is not None else v.copy()  # step_2 overwrites v before it reads z~
    qprev = nans((n, k), vt)
    orc("minres_step_2_" + vt, n, k, x, k, p_w, k, np.ascontiguousarray(p_r), k, z, k, zt, k, q, k, qprev, k, v, k,
        S[0], S[1], S[2], S[3], S[10], S[7], np.ascontiguousarray(status))
    return x, p_w, z, q, v


def check_update_matches_step_2(dev, orc, k, size, vt, precond, parity):
    """column 0: alpha = 0, column 1: beta = 0 (safe_divide's zero divisors); the last column has
    stopped and keeps its NaN sentinels in every vector and scalar"""
    n = step_rows(dev.num_sms, k)[size]
    rng = np.random.default_rng(70 + k + size)
    x, p0, p1, z, q, v = (rng.uniform(-1, 1, (n, k)).astype(VT[vt]) for _ in range(6))
    inv = rng.uniform(0.5, 2, n).astype(VT[vt]) if precond else None
    S = scalars(rng, vt, k)
    S[0, 0] = 0
    S[1, 1] = 0
    status = np.zeros(k, np.uint8)
    status[k - 1] = STOPPED
    for a in (x, p0, p1, z, q, v):
        a[:, k - 1] = np.nan
    S[:, k - 1] = np.nan
    iters = 4 + parity
    bufs = [dev.put(a) for a in (x, p0, p1, z, q, v)]
    sc, st = dev.put(S), dev.put(status)
    ctl = dev.put(np.array([0, iters, -1, 2, 1, 0, 0, 0], np.int32))
    dev.call("minres_mrhs_update_" + vt, n, k, *bufs, None if inv is None else dev.put(inv), sc, st, ctl)
    # iteration i writes p1 when i is even, p0 when odd; the other is p_prev
    p_w, p_r = (p0, p1) if iters % 2 else (p1, p0)
    want = oracle_update(orc, vt, k, x, p_w, p_r, z, q, v, inv, S, status)
    gx, g0, g1, gz, gq, gv = (b.get().reshape(n, k) for b in bufs)
    gp, gpp = (g0, g1) if iters % 2 else (g1, g0)
    assert gpp.tobytes() == p_r.tobytes()
    for got, w in zip((gx, gp, gz, gq, gv), want):
        assert got.tobytes() == w.tobytes()
    want_S = S.copy()
    want_S[1, :k - 1], want_S[2, :k - 1] = S[2, :k - 1], S[1, :k - 1]  # std::swap(gamma, beta)
    got_S = slots(sc.get(), k)
    assert got_S[:, :k - 1].tobytes() == want_S[:, :k - 1].tobytes() and np.isnan(got_S[:, k - 1]).all()
    c, gst = ctl.get(), st.get()
    assert c[1] == iters + 1 and c[0] == 0 and gst[k - 1] == STOPPED
    for j in range(k - 1):
        assert gst[j] == expected_status(iters + 1, -1, 2, True, np.sqrt(np.abs(S[6, j])), S[5, j]), j


def check_stopping_table(dev, vt, baseline):
    """init checks iteration 0 of every column, update's last CTA iteration 1 of the running ones: ids,
    converged and finalized bits in both criterion orders, the threshold factor * tau0_j (tau0 = 1 for
    the absolute baseline); four columns with four taus around the threshold, ctl[0] raised only once
    all four have stopped"""
    v = VT[vt]
    k, n = 4, 100
    factor = v(1e-3)
    tau0 = np.array([4, 2, 8, 1], v)
    thr = (factor * (np.ones(k, v) if baseline == 2 else tau0)).astype(v)
    taus = (thr * thr * np.array([0.25, 1, 4, -1], v)).astype(v)
    cases = 0
    for max_iters in (-1, 0, 1, 2):
        for res_kind in (0, 2):
            if max_iters < 0 and res_kind == 0:
                continue
            for iter_first in (0, 1):
                S = np.zeros((SC, k), v)
                S[4], S[6] = tau0, taus
                sc, st = dev.put(S), dev.put(np.full(k, 0xff, np.uint8))
                ctl = dev.put(np.zeros(8, np.int32))
                dev.call("minres_mrhs_init_" + vt, k, sc, st, ctl, max_iters, res_kind, iter_first, baseline, factor)
                c, G = ctl.get(), slots(sc.get(), k)
                assert G[5].tobytes() == thr.tobytes() and G[4].tobytes() == (np.ones(k, v) if baseline == 2
                                                                                 else tau0).tobytes()
                assert c[1:8].tolist() == [0, max_iters, res_kind, iter_first, 0, 0, 0]
                taun = np.sqrt(np.abs(taus))
                want = [expected_status(0, max_iters, res_kind, iter_first, taun[j], thr[j]) for j in range(k)]
                assert st.get().tolist() == want
                assert (c[0] != 0) == all(want)
                if all(want):
                    continue
                z = [dev.put(np.zeros((n, k), v)) for _ in range(6)]
                dev.call("minres_mrhs_update_" + vt, n, k, *z, None, sc, st, ctl)
                c = ctl.get()
                want1 = [w or expected_status(1, max_iters, res_kind, iter_first, taun[j], thr[j])
                         for j, w in enumerate(want)]
                assert c[1] == 1 and st.get().tolist() == want1
                assert (c[0] != 0) == all(want1)
                cases += 1
    assert cases > 8


def check_kernels_are_noops_after_a_stop(dev, vt):
    n, k = 5000, 3
    rng = np.random.default_rng(1)
    arrs = [rng.uniform(-1, 1, (n, k)).astype(VT[vt]) for _ in range(6)]
    bufs = [dev.put(a) for a in arrs]
    S = scalars(rng, vt, k)
    sc, st = dev.put(S), dev.put(np.zeros(k, np.uint8))
    ctl0 = np.array([1, 7, 9, 2, 1, 0, 0, 0], np.int32)
    ctl = dev.put(ctl0)
    dev.call("minres_mrhs_lanczos_" + vt, n, k, bufs[5], bufs[4], None, sc, st, ctl, work(dev, vt, k))
    dev.call("minres_mrhs_update_" + vt, n, k, *bufs, None, sc, st, ctl)
    assert all(b.get().tobytes() == a.tobytes() for b, a in zip(bufs, arrs))
    assert sc.get().tobytes() == S.tobytes() and ctl.get().tobytes() == ctl0.tobytes()
    assert not st.get().any()


def test_update_stopping_table_and_noops(dev, orc):
    each(itertools.product([2, 5, 32], range(3), VTS, [False, True], [0, 1]),
         lambda *case: check_update_matches_step_2(dev, orc, *case))
    each(itertools.product(VTS, [0, 1, 2]), lambda vt, baseline: check_stopping_table(dev, vt, baseline))
    each([(vt,) for vt in VTS], lambda vt: check_kernels_are_noops_after_a_stop(dev, vt))


# --------------------------------------------------------------------------- C. lock step
def check_lockstep_iterations_on_indefinite_arrow(dev, orc, vt, it):
    """the arrow matrix with its diagonal shifted by -3 (symmetric indefinite, positive diagonal), k = 5
    columns, column 0 zero (it stops at iteration 0).  Eight iterations launch by launch, each kernel
    compared with the loop's fed the fused path's own scalars; then graphs of five iterations replayed
    until every column has stopped, and past that without a change."""
    v_ = VT[vt]
    k = 5
    rp, ci, va = arrow(vt, shift=-3)
    rp, ci = rp.astype(IT[it]), ci.astype(IT[it])
    n = len(rp) - 1
    inv = arrow_inv_diag(rp, ci, va)
    b = np.random.default_rng(5).uniform(-1, 1, (n, k)).astype(v_)
    b[:, 0] = 0
    A = [dev.put(a) for a in (rp, ci, va)]
    invd, w = dev.put(inv), work(dev, vt, k)
    # the loop's set-up with x = 0: r = b, z = M r, beta = r.z, tau = z.z, minres::initialize, ||b||
    r, z = dev.put(b), dev.put(nans((n, k), vt))
    dev.call("jacobi_simple_scalar_apply_" + vt, n, k, invd, r, k, z, k)
    sc = dev.put(np.zeros(SC * k, v_))
    dev.call("dense_compute_conj_dot_" + vt, n, k, r, k, z, k, sc.at(k))
    dev.call("dense_compute_conj_dot_" + vt, n, k, z, k, z, k, sc.at(6 * k))
    x, q, vv, p0, p1 = (dev.put(np.zeros((n, k), v_)) for _ in range(5))
    st = dev.put(np.full(k, 0xff, np.uint8))
    dev.call("minres_initialize_" + vt, n, k, r, k, z, k, p0, k, p1, k, q, k, vv, k, vv, k,
             *[sc.at(s * k) for s in (1, 2, 3, 9, 10, 11, 12, 8, 7)], st)
    dev.call("dense_compute_norm2_" + vt, n, k, dev.put(b), k, sc.at(4 * k))
    red = 1e-6 if vt == "f64" else 1e-3
    max_iters = 63
    ctl = dev.put(np.zeros(8, np.int32))
    dev.call("minres_mrhs_init_" + vt, k, sc, st, ctl, max_iters, 2, 1, 0, v_(red))
    assert ctl.get()[0] == 0 and st.get().tolist() == [0x80 | 0x40 | 2] + [0] * (k - 1)
    sub = "csr_spmv_sub_mdot_%s_%s" % (vt, it)
    for i in range(8):
        status = st.get()
        # spmv_sub_mdot against the oracle's advanced SpMV
        zv, v0 = z.get().reshape(n, k), vv.get().reshape(n, k)
        dev.call(sub, n, n, len(va), *A, z, k, vv, sc, w, ctl)
        vl = oracle_sub(orc, vt, it, n, n, rp, ci, va, zv, v0, k)
        assert vv.get().reshape(n, k).tobytes() == vl.tobytes(), i
        S = slots(sc.get(), k)
        for j in range(1, k):
            assert_sum_within(S[0, j], zv[:, j] * vl[:, j], vt, "alpha %d" % j)
        # lanczos: v exactly the loop's for every running column; beta within the sum bound
        q_now = q.get().reshape(n, k)
        dev.call("minres_mrhs_lanczos_" + vt, n, k, vv, q, invd, sc, st, ctl, w)
        got_v = vv.get().reshape(n, k)
        want_v = vl - S[0] * q_now
        assert got_v[:, 1:].tobytes() == want_v[:, 1:].tobytes() and got_v[:, 0].tobytes() == vl[:, 0].tobytes()
        S1 = slots(sc.get(), k)
        beta_sq = np.array([np.sum((want_v[:, j] * (want_v[:, j] * inv)).astype(np.float64)) for j in range(k)])
        L = oracle_step_1(orc, vt, k, S, beta_sq.astype(v_), status)
        assert np.all(np.abs(S1[1, 1:].astype(np.float64) - L[1, 1:]) <= 64 * float(np.finfo(v_).eps) *
                      np.abs(L[1, 1:].astype(np.float64))), i
        assert S1[:, 0].tobytes() == S[:, 0].tobytes()  # the stopped column's scalars stay
        # update: the oracle's minres::step_2 fed with the fused scalars
        bufs = [x, p0, p1, z, q, vv]
        bx, b0, b1, bz, bq, bv = (a.get().reshape(n, k) for a in bufs)
        dev.call("minres_mrhs_update_" + vt, n, k, *bufs, invd, sc, st, ctl)
        p_w, p_r = (b0, b1) if i % 2 else (b1, b0)
        want = oracle_update(orc, vt, k, bx, p_w, p_r, bz, bq, bv, inv, S1, status)
        got_p = (p0 if i % 2 else p1).get().reshape(n, k)
        for got, wv in zip((x.get(), got_p, z.get(), q.get(), vv.get()), want):
            assert got.reshape(n, k).tobytes() == wv.tobytes(), i
        c, S2 = ctl.get(), slots(sc.get(), k)
        assert c[1] == i + 1 and c[0] == 0, (i, c)
        for j in range(1, k):
            thr = S2[5, j]
            assert st.get()[j] == expected_status(i + 1, max_iters, 2, True, np.sqrt(np.abs(S2[6, j])), thr), (i, j)
    assert not np.any(x.get().reshape(n, k)[:, 0])

    # the rest of the solve as graphs of 5 iterations; ctl[0] only once every column has stopped
    def batch():
        for _ in range(5):
            dev.call(sub, n, n, len(va), *A, z, k, vv, sc, w, ctl)
            dev.call("minres_mrhs_lanczos_" + vt, n, k, vv, q, invd, sc, st, ctl, w)
            dev.call("minres_mrhs_update_" + vt, n, k, x, p0, p1, z, q, vv, invd, sc, st, ctl)
    g = dev.capture(batch)
    for _ in range(20):
        dev.call("graph_launch", g)
        c, s = ctl.get(), st.get()
        assert (c[0] != 0) == all(s & 0x3f), (c, s)
        if c[0]:
            break
    assert c[0] != 0 and 8 < c[1] <= max_iters and s[0] == 0x80 | 0x40 | 2
    assert all(v_s in (0x80 | 0x40 | 2, 0x40 | 1) for v_s in s)
    assert np.isfinite(x.get()).all() and not np.any(x.get().reshape(n, k)[:, 0])
    state = [a.get().tobytes() for a in (x, p0, p1, z, q, vv, sc, st, ctl)]
    for _ in range(2):
        dev.call("graph_launch", g)
    assert [a.get().tobytes() for a in (x, p0, p1, z, q, vv, sc, st, ctl)] == state


def test_lockstep_iterations_on_indefinite_arrow(dev, orc):
    each([("f64", "i32"), ("f32", "i64")],
         lambda vt, it: check_lockstep_iterations_on_indefinite_arrow(dev, orc, vt, it))


# --------------------------------------------------------------------------- D. host solver
def mrhs_rhs(n, k, vt, seed=6):
    b = np.random.default_rng(seed).uniform(-1, 1, (n, k))
    b[:, 1] *= 1e-3
    return b.astype(VT[vt])


def device_solve(hexec, vt, rp, ci, va, b, precond=0, block_ptrs=None, strided=0, **kw):
    import torch
    from ginkgo_b200 import api
    k = b.shape[1]
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(np.ascontiguousarray(np.pad(b, ((0, 0), (0, strided))))).to(hexec.device)
        tx = torch.zeros_like(tb)
    n = len(rp) - 1
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "minres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb, cols=k), api.host_dense(hexec, tx, cols=k))
    hexec.synchronize()
    return tx.cpu().numpy()[:, :k], s.num_iterations, s.stop_statuses, s.used_fused


def check_solver_matches_oracle(hexec, vt, it, precond, baseline, iter_first, check_every):
    rp, ci, va = indefinite_laplacian(24, 2, vt, 0.6)
    n, k = len(rp) - 1, 4
    b = mrhs_rhs(n, k, vt)
    red = 1e-8 if vt == "f64" else 1e-4
    if baseline == 2:
        red *= 10
    kw = dict(max_iters=1000, res_kind=2, baseline=baseline, reduction=red)
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    xo, ito, stop_o = H.orc_solve("minres", vt, rp, ci, va, b, np.zeros((n, k), VT[vt]), precond, jac,
                                  iter_first=int(iter_first), **kw)
    xd, itd, stop_d, used = device_solve(hexec, vt, rp.astype(IT[it]), ci.astype(IT[it]), va, b, precond,
                                         iter_first=iter_first, fused_minres_multi_rhs=True,
                                         check_every=check_every, **kw)
    assert used
    assert stop_d == list(stop_o) and all(s & 0x80 for s in stop_d)
    # the bar the loop's Minres meets against the oracle (test_fused_minres_gpu.py, test_zz_late_gpu.py):
    # on an indefinite system the implicit residual's recurrence carries the sums' rounding
    assert abs(itd - ito) <= max(3, 0.2 * ito), (itd, ito)
    tol = 1e-7 if vt == "f64" else 1e-2
    for j in range(k):
        # the absolute baseline holds column 1 (b scaled by 1e-3) to the others' absolute threshold, so
        # to a relative accuracy 1e3 coarser
        scale = 1e3 if baseline == 2 and j == 1 else 1
        assert H.rel_err(xo[:, j], xd[:, j]) <= tol * scale, j


def test_solver_matches_oracle(hexec):
    """value / index types with and without scalar Jacobi, every baseline, both criterion orders and
    check_every 1, 7, 16"""
    each(itertools.product([("f64", "i32", 0), ("f64", "i32", 1), ("f32", "i32", 1), ("f64", "i64", 0),
                            ("f32", "i64", 0)], [0, 1, 2], [True, False], [1, 7, 16]),
         lambda types, *rest: check_solver_matches_oracle(hexec, *types, *rest))


def test_solver_columns_stop_at_their_own_iterations(hexec):
    """column 1 is b scaled by 1e-3 and converges first under the absolute baseline, column 3 is zero and
    stops at iteration 0 with x = 0; the statuses are the oracle's and every column is solved"""
    rp, ci, va = indefinite_laplacian(40, 2, "f64", 0.6)
    n, k = len(rp) - 1, 5
    b = mrhs_rhs(n, k, "f64", seed=9)
    b[:, 3] = 0
    kw = dict(max_iters=3000, reduction=1e-9, res_kind=2, baseline=2)
    xo, ito, stop_o = H.orc_solve("minres", "f64", rp, ci, va, b, np.zeros((n, k)), **kw)
    xd, itd, stop_d, used = device_solve(hexec, "f64", rp, ci, va, b, fused_minres_multi_rhs=True, **kw)
    assert used and stop_d == list(stop_o) == [0x80 | 0x40 | 2] * k and abs(itd - ito) <= max(3, 0.2 * ito)
    assert np.all(xd[:, 3] == 0)
    for j in (0, 1, 2, 4):
        assert H.rel_err(xo[:, j], xd[:, j]) <= 1e-6, j
        assert true_rel_res(rp, ci, va, b[:, j], xd[:, j]) <= 1e-6, j


def test_fallbacks(hexec):
    rp, ci, va = indefinite_laplacian(12, 2, "f64", 0.6)
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8, res_kind=2)
    on = dict(kw, fused_minres_multi_rhs=True)
    b33, b4 = mrhs_rhs(n, 33, "f64"), mrhs_rhs(n, 4, "f64")
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    cases = [(b33, 1, None, 0, on),                          # more than 32 columns
             (b4, 1, None, 2, on),                           # stride != k
             (b4, 4, bp, 0, on),                             # block Jacobi
             (b4, 1, None, 0, dict(on, res_kind=1)),         # ResidualNorm
             (b4, 1, None, 0, kw),                           # the switch is off by default
             (b4, 1, None, 0, dict(kw, fused_minres=True))]  # the one-column switch alone
    for b, pre, bpp, strided, args in cases:
        x, it, st, used = device_solve(hexec, "f64", rp, ci, va, b, pre, bpp, strided, **args)
        assert not used, args
        loop = {a: v for a, v in args.items() if not a.startswith("fused")}
        xl, itl, stl, _ = device_solve(hexec, "f64", rp, ci, va, b, pre, bpp, strided, **loop)
        assert (it, st) == (itl, stl) and x.tobytes() == xl.tobytes() and st[0] & 0x80, args
    # one column: the one-column path, the same bits with the new switch on or off
    b1 = b4[:, :1].copy()
    xa, ita, sta, usa = device_solve(hexec, "f64", rp, ci, va, b1, 1, fused_minres=True,
                                     fused_minres_multi_rhs=True, **kw)
    xb, itb, stb, usb = device_solve(hexec, "f64", rp, ci, va, b1, 1, fused_minres=True, **kw)
    assert usa and usb and (ita, sta) == (itb, stb) and xa.tobytes() == xb.tobytes()


def test_two_applies_give_the_same_bits(hexec):
    """deterministic sums: the same solve gives the same bits and iterations, with another k between"""
    rp, ci, va = indefinite_laplacian(30, 2, "f64", 0.6)
    n = len(rp) - 1
    outs = []
    for k in (6, 3, 6):
        b = mrhs_rhs(n, k, "f64", seed=1)
        outs.append(device_solve(hexec, "f64", rp, ci, va, b, 1, fused_minres_multi_rhs=True, max_iters=500,
                                 reduction=1e-10, res_kind=2))
    assert outs[0][0].tobytes() == outs[2][0].tobytes() and outs[0][1:] == outs[2][1:]
    assert outs[1][2] == [0x80 | 0x40 | 2] * 3 and outs[0][3]
