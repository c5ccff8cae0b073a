"""The fused GMRES kernels for several right-hand sides (csrc/fused_gmres_mrhs.cu) one at a time through the
C ABI against numpy, then solver::Gmres with with_fused_multi_rhs(true) against the device loop and the
oracle's multi-column GMRES.

As in test_fused_gmres_gpu.py: element-wise results and the Givens values derived from given sums are
compared BIT FOR BIT (the library is built with -fmad=false, numpy in the value type rounds as the device
does); sums on small-integer data must be exact; sums on random data must lie within gamma_h * sum |t| of
math.fsum.  Every vector is n x k row-major (stride k); column c of basis i is K[i n + r, c].

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock."""
import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import VT
from tests.test_fused_bicgstab_gpu import SYSTEMS, true_rel_res, upwind
from tests.test_fused_cg_gpu import (arrow_inv_diag, assert_sum_within, backend, dev, hexec,  # noqa: F401
                                     int_sum)
from tests.test_fused_cg_mrhs_gpu import nans, oracle_spmv
from tests.test_fused_gmres_gpu import assert_norm_within, givens_ref

pytestmark = pytest.mark.gpu

VTS = ["f64", "f32"]
KS = [2, 3, 5, 8, 17, 32]
CTL = 8
STOPPED = 0x40 | 1        # a stopped column (Iteration, finalized)
CONV_2 = 0x80 | 0x40 | 2  # converged by the residual criterion (second of Iteration first), finalized
THREADS, STEP_CTAS_PER_SM = 512, 4  # fused_common.cuh / fused_mrhs.cuh: the passes' block size and grid cap


def work(dev, vt, k, kd=31):
    size = getattr(dev.l, "b200_gmres_mrhs_work_size_" + vt)(dev.ctx, k, kd)
    return dev.put(np.full(size, np.nan, VT[vt]))


def sizes(dev, k):
    """empty, tiny, and enough rows to fill the capped grid of the passes several times over"""
    num_sms = dev.num_sms
    P = 2
    while P < k:
        P *= 2
    return [0, 3, 1000, (THREADS // P) * 4 * num_sms * STEP_CTAS_PER_SM * 3 + 7]


def mats(vt, n, k, data, seed, count=1):
    rng = np.random.default_rng(seed)
    if data == "int":
        a = rng.integers(-3, 4, size=(count, n, k))
    else:
        a = rng.uniform(-1, 1, size=(count, n, k))
    return a.astype(VT[vt])


def status_of(k, stopped):
    st = np.zeros(k, np.uint8)
    st[list(stopped)] = STOPPED
    return st


def stopped_cols(k):
    return [1] if k < 5 else [1, k - 2]


def check_col_sums(got, a, b, vt, exact, what, cols):
    for c in cols:
        if exact:
            assert got[c] == int_sum(a[:, c], b[:, c]), (what, c)
        else:
            assert_sum_within(got[c], (a[:, c] * b[:, c]).astype(VT[vt]), vt, "%s %d" % (what, c))


# --------------------------------------------------------------------------- A. scale
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("divide", [0, 1])
def test_scale(dev, k, vt, precond, divide):
    T = VT[vt]
    for n in sizes(dev, k):
        (w,) = mats(vt, n, k, "rand", 1)
        d = np.random.default_rng(2).uniform(0.5, 2, n).astype(T)
        h = np.random.default_rng(3).uniform(0.2, 3, k).astype(T)
        stopped = stopped_cols(k)
        sc = dev.put(np.concatenate([h, np.zeros(2 * k, T)]))
        st, ctl = dev.put(status_of(k, stopped)), dev.put(np.zeros(CTL, np.int32))
        vd, zd, dd = dev.put(w), dev.put(nans((n, k), vt)), dev.put(d)
        dev.call("gmres_mrhs_scale_" + vt, n, k, vd, zd if precond else None, dd if precond else None, sc, st, ctl,
                 divide)
        run = [c for c in range(k) if c not in stopped]
        v_ref = w.copy()
        if divide:
            v_ref[:, run] = (w[:, run] / h[run]).astype(T)
        z_ref = nans((n, k), vt)
        if precond:
            z_ref[:, run] = (v_ref[:, run] * d[:, None]).astype(T)
        assert vd.get().reshape(n, k).tobytes() == v_ref.tobytes()
        assert zd.get().reshape(n, k).tobytes() == z_ref.tobytes()  # stopped columns keep their NaNs
        # every column stopped: nothing is written
        ctl.set(np.array([1] + [0] * 7, np.int32))
        v2 = dev.put(w)
        dev.call("gmres_mrhs_scale_" + vt, n, k, v2, zd, dd, sc, st, ctl, 1)
        assert v2.get().reshape(n, k).tobytes() == w.tobytes()


# --------------------------------------------------------------------------- B. MGS passes
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_mgs_passes(dev, k, vt, data):
    """passes i = 1..j: w bit-equal to sequential sub_scaled per column (h = 0 skips), every h_i checked,
    stopped columns untouched in w and h"""
    T = VT[vt]
    j = 4
    stopped = stopped_cols(k)
    run = [c for c in range(k) if c not in stopped]
    for n in sizes(dev, k)[1:]:
        V = mats(vt, n, k, data, 10, j + 1)
        (w,) = mats(vt, n, k, data, 3)
        w[:, stopped] = np.nan
        hcol = nans((j + 2, k), vt)
        hcol[0] = T(2) if data == "int" else T(0.3)
        hcol[0, 0] = 0  # column 0 subtracts nothing in pass 1
        Vd, wd, hd = dev.put(V.reshape(-1)), dev.put(w), dev.put(hcol)
        st, ctl, wk = dev.put(status_of(k, stopped)), dev.put(np.zeros(CTL, np.int32)), work(dev, vt, k)
        w_ref = w.copy()
        for i in range(1, j + 1):
            dev.call("gmres_mrhs_mgs_pass_" + vt, n, k, wd, Vd.at((i - 1) * n * k), Vd.at(i * n * k), hd, i, st, ctl,
                     wk)
            h_all = hd.get().reshape(j + 2, k)
            for c in run:
                hp = h_all[i - 1, c]
                if hp != 0:
                    w_ref[:, c] = (w_ref[:, c] - (hp * V[i - 1][:, c]).astype(T)).astype(T)
            assert wd.get().reshape(n, k).tobytes() == w_ref.tobytes(), i
            exact = data == "int" and np.abs(V[i].astype(np.float64) * w_ref).sum(axis=0)[run].max() < \
                (2 ** 24 if vt == "f32" else 2 ** 53)
            check_col_sums(h_all[i], V[i], w_ref, vt, exact, "h_%d" % i, run)
            assert np.isnan(h_all[i, stopped]).all()
            if data == "int" and np.abs(h_all[i, run]).max() > 1e5:
                break  # keep the integer data exact
        # every column stopped: nothing is written
        ctl.set(np.array([1] + [0] * 7, np.int32))
        bw, bh = wd.get(), hd.get()
        dev.call("gmres_mrhs_mgs_pass_" + vt, n, k, wd, Vd.at(0), Vd.at(n * k), hd, 1, st, ctl, wk)
        assert wd.get().tobytes() == bw.tobytes() and hd.get().tobytes() == bh.tobytes()


# --------------------------------------------------------------------------- C. multi-dot and sub pass
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
@pytest.mark.parametrize("nb", [1, 5, 16, 20, 31])
def test_multi_dot_and_sub_pass(dev, k, vt, data, nb):
    """h_i = v_i . w for nb bases (past one 16-basis sweep), then the plain subtract pass in basis order
    with h = 0 coefficients skipped; stopped columns untouched"""
    T = VT[vt]
    stopped = stopped_cols(k)
    run = [c for c in range(k) if c not in stopped]
    n = sizes(dev, k)[2 if nb > 16 else 3]
    V = mats(vt, n, k, data, 30, nb)
    (w,) = mats(vt, n, k, data, 31)
    w[:, stopped] = np.nan
    Vd, wd = dev.put(V.reshape(-1)), dev.put(w)
    hd = dev.put(nans((nb, k), vt))
    st, ctl, wk = dev.put(status_of(k, stopped)), dev.put(np.zeros(CTL, np.int32)), work(dev, vt, k, 31)
    dev.call("gmres_mrhs_multi_dot_" + vt, n, k, nb, 31, Vd, wd, hd, st, ctl, wk)
    h = hd.get().reshape(nb, k)
    for i in range(nb):
        check_col_sums(h[i], V[i], w, vt, data == "int", "h_%d" % i, run)
        assert np.isnan(h[i, stopped]).all()
    # graph replay gives the eager bits
    hd.set(nans((nb, k), vt))
    g = dev.capture(lambda: dev.call("gmres_mrhs_multi_dot_" + vt, n, k, nb, 31, Vd, wd, hd, st, ctl, wk))
    dev.call("graph_launch", g)
    dev.sync()
    assert hd.get().reshape(nb, k).tobytes() == h.tobytes()
    # subtract pass over bases 0..nb-1 with some zero coefficients
    coef = np.random.default_rng(4).uniform(-1, 1, (nb, k)).astype(T)
    coef[0, 0] = 0
    coef[nb - 1, -1] = 0
    cd = dev.put(coef)
    dev.call("gmres_mrhs_sub_pass_" + vt, n, k, wd, Vd, cd, nb - 1, st, ctl)
    w_ref = w.copy()
    for c in run:
        for i in range(nb):
            if coef[i, c] != 0:
                w_ref[:, c] = (w_ref[:, c] - (coef[i, c] * V[i][:, c]).astype(T)).astype(T)
    assert wd.get().reshape(n, k).tobytes() == w_ref.tobytes()


# --------------------------------------------------------------------------- D. final pass
@pytest.mark.parametrize("k", [2, 3, 5, 8, 17, 32])
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("cgs2", [False, True])
def test_final_pass_givens(dev, k, vt, cgs2):
    """iterations j = 0..kd-1 of final passes on made-up Hessenberg columns, a column stopping on the way:
    w, the norms, the Givens values, rnc, fin and the column bit-equal to the masked hessenberg_qr, the
    stopped columns' NaN sentinels untouched everywhere"""
    T = VT[vt]
    kd, n = 6, sizes(dev, k)[2]
    rng = np.random.default_rng(5)
    gsin, gcos, rnc = nans((kd, k), vt), nans((kd, k), vt), np.zeros((kd + 1, k), T)
    gsin[:, 0] = gcos[:, 0] = 0  # column 0 runs; the rest start with NaN in what they never write
    for c in range(k):
        rnc[0, c] = T(3.5 + c)
    stopped = stopped_cols(k)
    for c in stopped:
        rnc[:, c] = np.nan
    run = [c for c in range(k) if c not in stopped]
    gsin[:, run] = gcos[:, run] = 0
    gs, gc, rn = dev.put(gsin), dev.put(gcos), dev.put(rnc)
    rnorm, fin = dev.put(nans(k, vt)), dev.put(np.zeros(k, np.uint64))
    status = status_of(k, stopped)
    st = dev.put(status)
    sc = dev.put(np.concatenate([nans(k, vt), np.ones(k, T), np.zeros(k, T)]))  # threshold 0: never converged
    ctl = dev.put(np.array([0, 0, -1, 1, 1, 0, 0, 0], np.int32))
    wk = work(dev, vt, k)
    fins = np.zeros(k, np.uint64)
    for j in range(kd):
        h = nans((j + 2, k), vt)
        h[:j + 1] = rng.uniform(-1, 1, (j + 1, k)).astype(T)
        h[:, stopped] = np.nan
        if j == 2:
            h[j, 0] = 0  # no subtraction
        haux = rng.uniform(-1, 1, (j + 1, k)).astype(T) if cgs2 else None
        w = rng.uniform(-1, 1, (n, k)).astype(T)
        if j == 3:
            w[:, 0] = 0  # a zero norm, which the Givens update must take
            h[:j + 1, 0] = 0
            if cgs2:
                haux[:, 0] = 0
        w[:, stopped] = np.nan
        v = rng.uniform(-1, 1, (n, k)).astype(T)
        K = np.concatenate([nans((j * n, k), vt), v])  # MGS: only basis j is subtracted
        coef = haux if cgs2 else h
        hd, wd, Kd = dev.put(h), dev.put(w), dev.put(K)
        ad = dev.put(np.concatenate([haux, nans((1, k), vt)])) if cgs2 else None
        dev.call("gmres_mrhs_final_pass_" + vt, n, k, wd, Kd, j, ad if cgs2 else hd, ad, hd, j, gs, gc, rnorm, rn,
                 fin, st, sc, ctl, wk)
        w_ref = w.copy()
        for c in run:
            if coef[j, c] != 0:
                w_ref[:, c] = (w[:, c] - (coef[j, c] * v[:, c]).astype(T)).astype(T)
        assert wd.get().reshape(n, k).tobytes() == w_ref.tobytes()
        got_sc = sc.get()
        h_ref = h.copy()
        for c in run:
            assert_norm_within(got_sc[c], w_ref[:, c], vt)
            if cgs2:
                h_ref[:j + 1, c] = (h_ref[:j + 1, c] + haux[:, c]).astype(T)
            h_ref[j + 1, c] = got_sc[c]
            col = h_ref[:, c].copy()
            gs_c, gc_c, rnc_c = gsin[:, c].copy(), gcos[:, c].copy(), rnc[:, c].copy()
            tau = givens_ref(T, gs_c, gc_c, rnc_c, col, j)
            h_ref[:, c], gsin[:, c], gcos[:, c], rnc[:, c] = col, gs_c, gc_c, rnc_c
            assert rnorm.get()[c] == tau
            fins[c] += 1
        assert hd.get().reshape(j + 2, k).tobytes() == h_ref.tobytes(), j
        assert gs.get().reshape(kd, k).tobytes() == gsin.tobytes()
        assert gc.get().reshape(kd, k).tobytes() == gcos.tobytes()
        assert rn.get().reshape(kd + 1, k).tobytes() == rnc.tobytes()
        assert np.isnan(rnorm.get()[stopped]).all() and np.isnan(got_sc[stopped]).all()
        assert (fin.get() == fins).all()
        assert st.get().tobytes() == status.tobytes()
        assert list(ctl.get()[:2]) == [0, j + 1]


def run_check(dev, vt, taus, tau0, factor, max_iters, res_kind, iter_first, iters_done, status=None):
    """the per-column stopping check of the final pass, fed one Givens update whose |rnc_c[1]| is
    exactly taus[c] (a zero column: c = 0, s = 1, rnc[1] = -rnc[0])"""
    T = VT[vt]
    k = len(taus)
    status = np.zeros(k, np.uint8) if status is None else status
    gs, gc = dev.put(np.zeros(k, T)), dev.put(np.zeros(k, T))
    rn = dev.put(np.stack([np.array(taus, T), nans(k, vt)]))
    rnorm, fin, st = dev.put(np.zeros(k, T)), dev.put(np.zeros(k, np.uint64)), dev.put(status)
    sc = dev.put(np.concatenate([np.zeros(k, T), np.full(k, tau0, T), np.full(k, T(factor) * T(tau0), T)]))
    ctl = dev.put(np.array([0, iters_done, max_iters, res_kind, int(iter_first), 0, 0, 0], np.int32))
    n = 16
    hd, wd, vd = dev.put(np.zeros((2, k), T)), dev.put(np.zeros((n, k), T)), dev.put(np.zeros((n, k), T))
    dev.call("gmres_mrhs_final_pass_" + vt, n, k, wd, vd, 0, hd, None, hd, 0, gs, gc, rnorm, rn, fin, st, sc, ctl,
             work(dev, vt, k))
    c = ctl.get()
    assert c[1] == iters_done + 1
    out = [int(s) for s in st.get()]
    assert c[0] == (1 if all(s & 0x3f for s in out) else 0)
    return out


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", ["rhs_norm", "initial_resnorm", "absolute"])
def test_stopping_table(dev, vt, baseline):
    """Iteration x ResidualNorm in both orders, per column; tau exactly on the threshold converges; no
    finalized bit; a column stopped before keeps its status; ctl[0] only once every column stopped.
    The baseline only sets tau0 (init), so each is fed here as its tau0."""
    T = VT[vt]
    tau0 = {"rhs_norm": T(2.0), "initial_resnorm": T(4.0), "absolute": T(1.0)}[baseline]
    f = 0.25
    thr = float(T(f) * tau0)
    taus = [1.5 * thr, thr, 0.5 * thr]  # above, on, below the threshold
    conv = 0x80
    for iter_first in (True, False):
        it_id, res_id = (1, 2) if iter_first else (2, 1)
        assert run_check(dev, vt, taus, tau0, f, 10, 1, iter_first, 3) == [0, conv | res_id, conv | res_id]
        assert run_check(dev, vt, taus, tau0, f, 4, 1, iter_first, 3) == \
            [it_id] + [it_id if iter_first else conv | res_id] * 2
    assert run_check(dev, vt, taus, tau0, f, -1, 1, True, 3) == [0, conv | 1, conv | 1]
    assert run_check(dev, vt, taus, tau0, f, 4, 0, True, 3) == [1, 1, 1]
    # a stopped column keeps its byte; the others stop: ctl[0] is raised
    assert run_check(dev, vt, [thr, thr, 9 * thr], tau0, f, 10, 1, True, 3,
                     status=np.array([0, 0, STOPPED], np.uint8)) == [conv | 2, conv | 2, STOPPED]


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2])
@pytest.mark.parametrize("k", [2, 5, 32])
def test_init_and_replay_past_the_stop(dev, vt, baseline, k):
    """baselines, thresholds and the iteration-0 check per column (a zero residual stops at iteration 0);
    then a graph of iterations replayed past the point where every column stopped changes nothing"""
    T = VT[vt]
    rn0 = np.full(k, 3.0, T)
    rn0[1] = 0
    rnorm = dev.put(rn0)
    bnorm = np.arange(1, k + 1).astype(T) * T(8)
    sc = dev.put(np.concatenate([nans(k, vt), bnorm, nans(k, vt)]))
    st, ctl = dev.put(np.full(k, 0x3f, np.uint8)), dev.put(np.full(CTL, 77, np.int32))
    dev.call("gmres_mrhs_init_" + vt, k, rnorm, sc, st, ctl, 100, 1, 1, baseline, T(0.125))
    tau0 = {0: bnorm, 1: rn0, 2: np.ones(k, T)}[baseline]
    s, c, got = sc.get(), ctl.get(), st.get()
    assert s[k:2 * k].tobytes() == tau0.tobytes() and s[2 * k:].tobytes() == (T(0.125) * tau0).astype(T).tobytes()
    assert (s[:k] == 0).all() and list(c[:5]) == [0, 0, 100, 1, 1]
    for j in range(k):
        assert got[j] == (0x80 | 2 if rn0[j] <= T(0.125) * tau0[j] else 0)
    # every column stopped (the Iteration limit 0): ctl[0] raised, and a replayed iteration is a no-op
    dev.call("gmres_mrhs_init_" + vt, k, rnorm, sc, st, ctl, 0, 1, 1, baseline, T(0.125))
    assert ctl.get()[0] == 1 and all(s & 0x3f for s in st.get())
    n = 500
    (w,) = mats(vt, n, k, "rand", 8)
    K = mats(vt, n, k, "rand", 9, 3)
    wd, Kd, hd = dev.put(w), dev.put(K.reshape(-1)), dev.put(nans((3, k), vt))
    gs, gc, rn, fin = dev.put(nans(k, vt)), dev.put(nans(k, vt)), dev.put(nans((2, k), vt)), dev.put(
        np.zeros(k, np.uint64))
    wk = work(dev, vt, k)
    before = [a.get().tobytes() for a in (wd, Kd, hd, sc, st, ctl, gs, gc, rn, fin)]

    def iteration():
        dev.call("gmres_mrhs_scale_" + vt, n, k, Kd, wd, None, sc, st, ctl, 0)
        dev.call("gmres_mrhs_multi_dot_" + vt, n, k, 1, 31, Kd, wd, hd, st, ctl, wk)
        dev.call("gmres_mrhs_mgs_pass_" + vt, n, k, wd, Kd, Kd.at(n * k), hd, 1, st, ctl, wk)
        dev.call("gmres_mrhs_final_pass_" + vt, n, k, wd, Kd, 0, hd, None, hd, 0, gs, gc, rn, rn, fin, st, sc, ctl, wk)
    g = dev.capture(iteration)
    for _ in range(3):
        dev.call("graph_launch", g)
    dev.sync()
    assert [a.get().tobytes() for a in (wd, Kd, hd, sc, st, ctl, gs, gc, rn, fin)] == before


# --------------------------------------------------------------------------- D2. lock step
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("ortho", ["mgs", "cgs", "cgs2"])
def test_lockstep_on_convective_arrow(dev, orc, vt, ortho):
    """13 iterations of GMRES(5) with scalar Jacobi on the nonsymmetric arrow matrix (rows split over
    CTAs), k = 3, across two restarts done here the way gmres_restart does them: every launch checked
    against numpy on the device's own inputs -- element-wise results and Givens values bit for bit,
    sums within the any-order bound -- and column 2 stopped by a raised threshold half-way through"""
    from tests.test_fused_bicgstab_gpu import convective_arrow
    T = VT[vt]
    rp, ci, va = convective_arrow(vt)
    n, k, kd = len(rp) - 1, 3, 5
    d = arrow_inv_diag(rp, ci, va)
    rng = np.random.default_rng(21)
    nk = n * k
    K = dev.put(np.zeros(((kd + 1) * n, k), T))
    z, hess = dev.put(np.zeros((n, k), T)), dev.put(np.zeros((kd, (kd + 1) * k), T))
    gs, gc, rn = dev.put(np.zeros((kd, k), T)), dev.put(np.zeros((kd, k), T)), dev.put(np.zeros((kd + 1, k), T))
    haux, rnorm = dev.put(np.zeros((kd + 1, k), T)), dev.put(np.zeros(k, T))
    fin, st = dev.put(np.zeros(k, np.uint64)), dev.put(np.zeros(k, np.uint8))
    sc, ctl, wk = dev.put(np.zeros(3 * k, T)), dev.put(np.zeros(CTL, np.int32)), work(dev, vt, k, kd)
    dd = dev.put(d)
    d_rp, d_ci, d_va = dev.put(rp), dev.put(ci), dev.put(va)
    hs = (kd + 1) * k

    def restart():
        """basis 0 = r / ||r|| per column, rnc[0] = ||r||, fin = 0 (a made-up residual)"""
        r = rng.uniform(-1, 1, (n, k)).astype(T)
        nrm = np.sqrt((r.astype(np.float64) ** 2).sum(axis=0)).astype(T)
        Kh = K.get().reshape((kd + 1) * n, k)
        Kh[:n] = (r / nrm).astype(T)
        K.set(Kh)
        rnc = rn.get().reshape(kd + 1, k)
        rnc[0] = nrm
        rn.set(rnc)
        rnorm.set(nrm)
        fin.set(np.zeros(k, np.uint64))
        return nrm

    nrm0 = restart()
    dev.call("gmres_mrhs_init_" + vt, k, rnorm, sc, st, ctl, 13, 1, 1, 2, T(1e-30))
    assert list(st.get()) == [0] * k
    for it in range(13):
        j = it % kd
        if j == 0 and it > 0:
            restart()
        if it == 7:  # column 2 stops at the next check
            s_h = sc.get()
            s_h[2 * k + 2] = T(1e30)
            sc.set(s_h)
        status = st.get()
        run = [c for c in range(k) if not status[c] & 0x3f]
        Kh = K.get().reshape(kd + 1, n, k)
        # scale
        s_h = sc.get()
        dev.call("gmres_mrhs_scale_" + vt, n, k, K.at(j * nk), z, dd, sc, st, ctl, int(j > 0))
        vj = Kh[j].copy()
        if j > 0:
            vj[:, run] = (vj[:, run] / s_h[run]).astype(T)
        Kh[j] = vj
        assert K.get().reshape(kd + 1, n, k)[j].tobytes() == vj.tobytes(), it
        zh = z.get().reshape(n, k)
        assert zh[:, run].tobytes() == (vj[:, run] * d[:, None]).astype(T).tobytes(), it
        # SpMV + h_0 (w is basis j + 1)
        dev.call("csr_spmv_mdot2_%s_i32" % vt, n, n, len(va), d_rp, d_ci, d_va, z, k, K.at((j + 1) * nk), K,
                 hess.at(j * hs), None, wk, ctl)
        w = oracle_spmv(orc, vt, "i32", n, n, rp, ci, va, zh, k)
        assert K.get().reshape(kd + 1, n, k)[j + 1].tobytes() == w.tobytes(), it
        h = hess.get().reshape(kd, kd + 1, k)[j].copy()
        check_col_sums(h[0], Kh[0], w, vt, False, "h_0", run)
        coef, add, first = h, None, j
        if ortho == "mgs":
            for i in range(1, j + 1):
                dev.call("gmres_mrhs_mgs_pass_" + vt, n, k, K.at((j + 1) * nk), K.at((i - 1) * nk), K.at(i * nk),
                         hess.at(j * hs), i, st, ctl, wk)
                for c in run:
                    if h[i - 1, c] != 0:
                        w[:, c] = (w[:, c] - (h[i - 1, c] * Kh[i - 1][:, c]).astype(T)).astype(T)
                assert K.get().reshape(kd + 1, n, k)[j + 1].tobytes() == w.tobytes(), (it, i)
                h = hess.get().reshape(kd, kd + 1, k)[j].copy()
                check_col_sums(h[i], Kh[i], w, vt, False, "h_%d" % i, run)
            coef = h
        else:
            if j > 0:
                dev.call("gmres_mrhs_multi_dot_" + vt, n, k, j, kd, K.at(nk), K.at((j + 1) * nk), hess.at(j * hs + k),
                         st, ctl, wk)
                h = hess.get().reshape(kd, kd + 1, k)[j].copy()
                for i in range(1, j + 1):
                    check_col_sums(h[i], Kh[i], w, vt, False, "h_%d" % i, run)
            coef, first = h, 0
            if ortho == "cgs2":
                dev.call("gmres_mrhs_sub_pass_" + vt, n, k, K.at((j + 1) * nk), K, hess.at(j * hs), j, st, ctl)
                for c in run:
                    for i in range(j + 1):
                        if h[i, c] != 0:
                            w[:, c] = (w[:, c] - (h[i, c] * Kh[i][:, c]).astype(T)).astype(T)
                assert K.get().reshape(kd + 1, n, k)[j + 1].tobytes() == w.tobytes(), it
                dev.call("gmres_mrhs_multi_dot_" + vt, n, k, j + 1, kd, K, K.at((j + 1) * nk), haux, st, ctl, wk)
                coef = haux.get().reshape(kd + 1, k)
                for i in range(j + 1):
                    check_col_sums(coef[i], Kh[i], w, vt, False, "haux_%d" % i, run)
                add = haux
        # final pass
        gsin, gcos = gs.get().reshape(kd, k), gc.get().reshape(kd, k)
        rnc, fins = rn.get().reshape(kd + 1, k), fin.get()
        dev.call("gmres_mrhs_final_pass_" + vt, n, k, K.at((j + 1) * nk), K, first,
                 haux if ortho == "cgs2" else hess.at(j * hs), add, hess.at(j * hs), j, gs, gc, rnorm, rn, fin, st, sc,
                 ctl, wk)
        for c in run:
            for i in range(first, j + 1):
                if coef[i, c] != 0:
                    w[:, c] = (w[:, c] - (coef[i, c] * Kh[i][:, c]).astype(T)).astype(T)
        assert K.get().reshape(kd + 1, n, k)[j + 1].tobytes() == w.tobytes(), it
        s_new = sc.get()
        h_ref = h.copy()
        for c in run:
            assert_norm_within(s_new[c], w[:, c], vt)
            if add is not None:
                h_ref[:j + 1, c] = (h_ref[:j + 1, c] + coef[:j + 1, c]).astype(T)
            h_ref[j + 1, c] = s_new[c]
            col, g_s, g_c, r_c = h_ref[:j + 2, c].copy(), gsin[:, c].copy(), gcos[:, c].copy(), rnc[:, c].copy()
            givens_ref(T, g_s, g_c, r_c, col, j)
            h_ref[:j + 2, c], gsin[:, c], gcos[:, c], rnc[:, c] = col, g_s, g_c, r_c
            fins[c] += 1
        got_h = hess.get().reshape(kd, kd + 1, k)[j]
        assert got_h[:j + 2][:, run].tobytes() == h_ref[:j + 2][:, run].tobytes(), it
        assert gs.get().reshape(kd, k)[:, run].tobytes() == gsin[:, run].tobytes(), it
        assert gc.get().reshape(kd, k)[:, run].tobytes() == gcos[:, run].tobytes(), it
        assert rn.get().reshape(kd + 1, k)[:, run].tobytes() == rnc[:, run].tobytes(), it
        assert (fin.get() == fins).all(), it
        stopped_now = [int(x) for x in st.get()]
        assert ctl.get()[1] == it + 1
        if it < 12:
            assert stopped_now == [0, 0, 0x80 | 2 if it >= 7 else 0], it
    # the Iteration limit (13) stops the running columns at the last check; ctl[0] raised
    assert list(st.get()) == [1, 1, 0x80 | 2] and ctl.get()[0] == 1
    assert (nrm0 > 0).all()


# --------------------------------------------------------------------------- E. the host solver
def host_gmres(hexec, rp, ci, va, b, precond, block_ptrs=None, strided=0, **kw):
    import torch
    from ginkgo_b200 import api
    n, k = len(rp) - 1, b.shape[1]
    bb = np.ascontiguousarray(np.pad(b, ((0, 0), (0, strided))))
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(bb).to(hexec.device)
        tx = torch.zeros_like(tb)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "gmres", A, precond_max_bs=precond, block_ptrs=block_ptrs, **kw)
    s.apply(api.host_dense(hexec, tb, cols=k), api.host_dense(hexec, tx, cols=k))
    hexec.synchronize()
    return tx.cpu().numpy()[:, :k], s.num_iterations, s.stop_statuses, s.used_fused


def cfg4_like(vt):
    return SYSTEMS["dominant_random"](vt)


MRHS_SYSTEMS = {"upwind": lambda vt: upwind(40, 2, vt), "cfg4_like": cfg4_like}


def rhs(n, k, vt, seed=12):
    return np.random.default_rng(seed).uniform(-1, 1, (n, k)).astype(VT[vt])


@pytest.mark.parametrize("system", list(MRHS_SYSTEMS))
@pytest.mark.parametrize("vt,it,precond", [("f64", "i32", 0), ("f64", "i32", 1), ("f32", "i32", 0), ("f32", "i32", 1),
                                           ("f64", "i64", 0), ("f32", "i64", 0)])  # the C handle's Jacobi is int32's
@pytest.mark.parametrize("kd,check_every", [(5, 1), (5, 3), (5, 10), (20, 20), (30, 3), (30, 35)])
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_matches_loop(hexec, system, vt, it, precond, kd, check_every, ortho):
    rp, ci, va = MRHS_SYSTEMS[system](vt)
    idx = np.int32 if it == "i32" else np.int64
    rp, ci = rp.astype(idx), ci.astype(idx)
    n, k = len(rp) - 1, 4
    b = rhs(n, k, vt)
    red = 1e-10 if vt == "f64" else 1e-5
    kw = dict(max_iters=600, reduction=red, krylov_dim=kd, ortho=ortho, check_every=check_every)
    xl, itl, stl, usedl = host_gmres(hexec, rp, ci, va, b, precond, **kw)
    xf, itf, stf, usedf = host_gmres(hexec, rp, ci, va, b, precond, fused_gmres_multi_rhs=True, **kw)
    assert usedf and not usedl
    assert abs(itf - itl) <= 2, (itf, itl)
    assert stf == stl
    for c in range(k):
        if stl[c] & 0x80:  # GMRES stops on its residual estimate: as close to b as the loop's x, or closer
            res_l = true_rel_res(rp, ci, va, b[:, c], xl[:, c])
            assert true_rel_res(rp, ci, va, b[:, c], xf[:, c]) <= max(20 * red, 2 * res_l), c
        assert H.rel_err(xl[:, c], xf[:, c]) <= (1e-8 if vt == "f64" else 1e-3), c


@pytest.mark.parametrize("system", list(MRHS_SYSTEMS))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [0, 1])
@pytest.mark.parametrize("kd", [5, 30])
@pytest.mark.parametrize("ortho", [0, 1, 2])
def test_matches_oracle(hexec, system, vt, precond, kd, ortho):
    rp, ci, va = MRHS_SYSTEMS[system](vt)
    n, k = len(rp) - 1, 3
    b = rhs(n, k, vt)
    red = 1e-9 if vt == "f64" else 1e-4
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    xo, ito, stop_o = H.orc_solve("gmres", vt, rp, ci, va, b, np.zeros((n, k), VT[vt]), precond, jac,
                                  max_iters=600, reduction=red, krylov_dim=kd, ortho=ortho)
    xd, itd, stop_d, used = host_gmres(hexec, rp, ci, va, b, precond, max_iters=600, reduction=red, krylov_dim=kd,
                                       ortho=ortho, fused_gmres_multi_rhs=True)
    assert used
    assert abs(itd - ito) <= 2, (itd, ito)
    assert stop_d == list(stop_o)
    for c in range(k):
        res_o = true_rel_res(rp, ci, va, b[:, c], xo[:, c])
        assert true_rel_res(rp, ci, va, b[:, c], xd[:, c]) <= max(20 * red, 2 * res_o), c
        assert H.rel_err(xo[:, c], xd[:, c]) <= (1e-8 if vt == "f64" else 1e-3), c


@pytest.mark.parametrize("ortho", [0, 1, 2])
@pytest.mark.parametrize("check_every", [1, 3, 5])
def test_columns_stop_at_different_cycles(hexec, ortho, check_every):
    """kd = 5: a zero column stops at iteration 0; A e for a vector e with three nonzeros converges inside
    cycle 1 and is finalized at the first restart; random columns run through several restarts"""
    rp, ci, va = upwind(16, 2, "f64")
    n, k = len(rp) - 1, 5
    b = rhs(n, k, "f64", seed=9)
    b[:, 1] = 0
    e = np.zeros(n)
    e[:3] = (1.0, -0.5, 0.25)
    import scipy.sparse as sp
    b[:, 3] = sp.csr_matrix((va, ci, rp), shape=(n, n)) @ e
    kw = dict(max_iters=600, reduction=1e-10, krylov_dim=5, ortho=ortho, check_every=check_every)
    xl, itl, stl, _ = host_gmres(hexec, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = host_gmres(hexec, rp, ci, va, b, 1, fused_gmres_multi_rhs=True, **kw)
    assert used and stf == stl == [CONV_2] * k and abs(itf - itl) <= 2 and itf > 10
    assert np.all(xf[:, 1] == 0)
    for c in range(k):
        assert H.rel_err(xl[:, c], xf[:, c]) <= 1e-8, c


@pytest.mark.parametrize("check_every", [1, 3, 5, 9])
@pytest.mark.parametrize("max_iters", [0, 1, 2, 3, 4, 5, 6, 10, 15])
def test_stop_positions(hexec, check_every, max_iters):
    rp, ci, va = upwind(12, 2, "f64")
    n = len(rp) - 1
    b = rhs(n, 3, "f64", seed=3)
    kw = dict(max_iters=max_iters, reduction=1e-14, krylov_dim=5, check_every=check_every)
    xl, itl, stl, _ = host_gmres(hexec, rp, ci, va, b, 1, **kw)
    xf, itf, stf, used = host_gmres(hexec, rp, ci, va, b, 1, fused_gmres_multi_rhs=True, **kw)
    assert used and itf == itl == max_iters and stf == stl == [STOPPED] * 3
    assert H.rel_err(xl, xf) <= 1e-10


def test_two_applies_give_the_same_bits(hexec):
    rp, ci, va = upwind(30, 2, "f64")
    n = len(rp) - 1
    outs = []
    for k in (6, 3, 6):
        outs.append(host_gmres(hexec, rp, ci, va, rhs(n, k, "f64", seed=1), 1, fused_gmres_multi_rhs=True,
                               max_iters=500, reduction=1e-10, krylov_dim=20, ortho=1))
    assert outs[0][3] and outs[0][0].tobytes() == outs[2][0].tobytes() and outs[0][1:] == outs[2][1:]


def test_fallbacks(hexec):
    rp, ci, va = upwind(12, 2, "f64")
    n = len(rp) - 1
    kw = dict(max_iters=300, reduction=1e-8, krylov_dim=10)
    on = dict(fused_gmres_multi_rhs=True, **kw)
    assert not host_gmres(hexec, rp, ci, va, rhs(n, 33, "f64"), 1, **on)[3]
    b = rhs(n, 4, "f64")
    assert not host_gmres(hexec, rp, ci, va, b, 1, strided=2, **on)[3]
    bp = np.arange(0, n + 1, 4, dtype=np.int32)
    assert not host_gmres(hexec, rp, ci, va, b, 4, block_ptrs=bp, **on)[3]
    with pytest.raises(Exception):  # ImplicitResidualNorm: NotSupported, as from the loop
        host_gmres(hexec, rp, ci, va, b, 1, res_kind=2, **on)
    xl, itl, stl, used = host_gmres(hexec, rp, ci, va, b, 1, fused_gmres=hexec.stream is not None, **kw)  # off
    assert not used and stl == [CONV_2] * 4
    xf, itf, stf, used = host_gmres(hexec, rp, ci, va, b, 1, **on)
    assert used and stf == stl and abs(itf - itl) <= 2
    # one column: the one-column path or the loop, the same bits with the switch on or off
    b1 = b[:, :1].copy()
    for one in ((False,) if hexec.stream is None else (False, True)):  # mock: no one-column kernels
        xa, ita, sta, usa = host_gmres(hexec, rp, ci, va, b1, 1, fused_gmres=one, **on)
        xb, itb, stb, usb = host_gmres(hexec, rp, ci, va, b1, 1, fused_gmres=one, **kw)
        assert usa == usb == one and (ita, sta) == (itb, stb) and xa.tobytes() == xb.tobytes()
