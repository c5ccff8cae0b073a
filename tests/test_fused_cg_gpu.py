"""The fused CG kernels (csrc/fused_cg.cu and the DOT paths of csr_kernels.cuh / csr_ring.cuh /
csr_launch.cuh) one at a time, through the C ABI, against plain numpy restatements.

How every assertion holds for a correct kernel by construction:
 * Element-wise updates (p = z + (rho/prev) p, x += alpha p, r -= alpha q, z = r inv_diag,
   alpha = rho/pq, sc[5] = factor sc[4], sqrt) are compared BIT FOR BIT: the library is built with
   -fmad=false and without fast math, so numpy in the value type rounds exactly as the device does.
 * Reductions on INTEGER data are compared for EQUALITY with the exact sum (Python int): values are
   small integers and sum |t| stays below 2^24 (f32) / 2^53 (f64), so every partial sum of any
   summation order is exact.  A missing or doubled row, tile, CTA partial or long-row chunk changes
   the result.
 * Reductions on RANDOM data are checked against math.fsum of the products rounded in the value
   type, within gamma_h * sum |t| (gamma_h = h u / (1 - h u)) with h = number of terms - 1, which
   bounds the error of any summation order.  A tree sum is not correctly rounded; nothing here
   asserts that it is.

B200_TEST_SELFCHECK=1 runs the same bodies on the host-memory mock of tests/mock (num_sms = 1,
sequential restatements of these entry points, graph capture included); the few asserts about the
device's launch shapes are skipped there, each marked "mock:"."""
import ctypes
import functools
import math
import os

import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import IT, VT
from tests.test_parity_gpu import CSR_KINDS, EXACT_KINDS, csr_case

pytestmark = pytest.mark.gpu

VTS = ["f64", "f32"]
ITS = ["i32", "i64"]
VARIANTS = [2, 4, 5]  # gather_pipe, warp_pipe, cta_ring
STOPPED = 0x40 | 1    # any nonzero stopping status turns the fused kernels into no-ops
WARP_TILE_MAX_ITEMS = 320  # kWMaxItems of csr_kernels.cuh: the largest warp tile a plan may choose


# --------------------------------------------------------------------------- backend
class Buf:
    """an array in the backend's memory (device memory, or host memory on the mock)"""

    def __init__(self, be, a):
        a = np.ascontiguousarray(a).reshape(-1)
        self.be, self.dtype, self.n = be, a.dtype, a.size
        host = a.copy() if a.size else np.zeros(1, a.dtype)  # empty arrays still get a valid pointer
        if be.mock:
            self.t = host
            self.ptr = host.ctypes.data
        else:
            torch = be.torch
            with torch.cuda.stream(be.stream):
                self.t = torch.from_numpy(host).cuda()
            self.ptr = self.t.data_ptr()

    def at(self, k):
        return self.ptr + k * self.dtype.itemsize

    def get(self):
        if self.be.mock:
            return self.t[:self.n].copy()
        self.be.stream.synchronize()
        return self.t.cpu().numpy()[:self.n].copy()

    def set(self, a):
        a = np.ascontiguousarray(a, dtype=self.dtype).reshape(-1)
        assert a.size == self.n
        if self.be.mock:
            self.t[:self.n] = a
        else:
            torch = self.be.torch
            with torch.cuda.stream(self.be.stream):
                self.t[:self.n].copy_(torch.from_numpy(a.copy()))
            self.be.stream.synchronize()


class Backend:
    """b200_* entry points on a context of the CUDA library, or of the host-memory mock"""

    def __init__(self, lib, mock):
        self.l, self.mock = lib, mock
        ctx = ctypes.c_void_p()
        if mock:
            self.stream = None
            self.check(lib.b200_ctx_create(0, None, ctypes.byref(ctx)))
        else:
            import torch
            self.torch = torch
            if not torch.cuda.is_available():
                raise RuntimeError("no CUDA device: the gpu tests need an H100")
            self.stream = torch.cuda.Stream()
            self.check(lib.b200_ctx_create(0, self.stream.cuda_stream, ctypes.byref(ctx)))
        self.ctx = ctx
        self.num_sms = lib.b200_ctx_num_sms(ctx)
        self._plans, self._graphs = [], []

    def check(self, st):
        if st != 0:
            msg = self.l.b200_last_error()
            raise RuntimeError("b200 status %d: %s" % (st, msg.decode() if msg else ""))

    def put(self, a):
        return Buf(self, a)

    def call(self, name, *args):
        self.check(self.status(name, *args))

    def status(self, name, *args):
        conv = [a.ptr if isinstance(a, Buf) else a for a in args]
        return getattr(self.l, "b200_" + name)(self.ctx, *conv)

    def work(self, vt):
        size = getattr(self.l, "b200_cg_fused_work_size_" + vt)(self.ctx)
        return self.put(np.full(size, np.nan, VT[vt]))

    def plan(self, vt, it, n, nnz, rp, variant=None):
        p = ctypes.c_void_p()
        self.call("csr_plan_create_%s_%s" % (vt, it), n, nnz, rp, ctypes.byref(p))
        self._plans.append(p)
        if variant is not None:
            self.l.b200_csr_plan_set_variant(p, variant)
        return p

    def capture(self, body):
        self.call("graph_begin_capture")
        try:
            body()
        finally:
            g = ctypes.c_void_p()
            self.call("graph_end_capture", ctypes.byref(g))
        self._graphs.append(g)
        return g

    def sync(self):
        self.call("synchronize")

    def release(self):
        self.sync()
        for g in self._graphs:
            self.l.b200_graph_destroy(g)
        for p in self._plans:
            self.l.b200_csr_plan_destroy(p)
        self._graphs, self._plans = [], []

    def close(self):
        self.release()
        self.l.b200_ctx_destroy(self.ctx)


@pytest.fixture(scope="module")
def backend(tmp_path_factory):
    from ginkgo_b200 import _cdecl, _lib
    if os.environ.get("B200_TEST_SELFCHECK") == "1":
        # harness self-check (no GPU): the host-memory mock stands in for the device, to debug
        # the TEST BODIES themselves.  Never set on the GPU box.
        from tests.mock_build import build_mock_host
        lib = build_mock_host(str(tmp_path_factory.mktemp("fused_cg_mock")))
        _cdecl.bind(lib, _lib.declarations())
        be = Backend(lib, mock=True)
    else:
        be = Backend(_lib.lib(), mock=False)
    yield be
    be.close()


@pytest.fixture
def dev(backend):
    yield backend
    backend.release()


@pytest.fixture(scope="module")
def hexec(backend):
    """the C++ host layer on the same library"""
    from ginkgo_b200 import api
    if backend.mock:
        from tests.mock_build import CpuExec
        saved = api._HOST_LIB
        api._HOST_LIB = backend.l
        yield CpuExec(backend.l)
        api._HOST_LIB = saved
    else:
        yield api.HostExecutor(0)


# --------------------------------------------------------------------------- references
def unit_roundoff(vt):
    return float(np.finfo(VT[vt]).eps) / 2


def assert_sum_within(dev_value, terms, vt, what):
    """dev_value is a sum of `terms` (already rounded in the value type) in SOME order:
    |dev - S*| <= gamma_h sum|t| with h = len - 1 (any order).  S = fsum is S* rounded to f64
    (|S - S*| <= 2^-53 |S*|), and the bound is evaluated in f64 (relative slack 2^-40)."""
    t = np.asarray(terms, dtype=VT[vt]).astype(np.float64)
    s = math.fsum(t)
    a = math.fsum(np.abs(t))
    h = max(len(t) - 1, 0)
    u = unit_roundoff(vt)
    gamma = h * u / (1 - h * u)
    tol = gamma * a * (1 + 2.0 ** -40) + 2.0 ** -52 * abs(s)
    assert abs(float(dev_value) - s) <= tol, (what, float(dev_value), s, tol)


def exact_limit(vt):
    return 2 ** 24 if vt == "f32" else 2 ** 53


def int_sum(a, b):
    """exact sum of a[i] * b[i] for integer-valued float arrays"""
    return int(np.dot(a.astype(np.int64), b.astype(np.int64)))


def expected_status(iters, max_iters, res_kind, iter_first, tau, threshold):
    """the reference's stop::Combined over Iteration and (Implicit)ResidualNorm
    (core/stop/combined.cpp, iteration.cpp, residual_norm.cpp): the criteria are checked in the
    configured order, the first that holds sets the status: id = its position among the CONFIGURED
    criteria (1-based), 0x40 finalized, 0x80 converged (residual criteria only)."""
    order = ("it", "res") if iter_first else ("res", "it")
    configured = [c for c in order if (c == "it" and max_iters >= 0) or (c == "res" and res_kind != 0)]
    for ident, c in enumerate(configured, start=1):
        if c == "it" and iters >= max_iters:
            return 0x40 | ident
        if c == "res" and tau <= threshold:
            return 0x80 | 0x40 | ident
    return 0


def tau_of(vt, res_kind, rho, rr):
    v = VT[vt]
    return np.sqrt(v(rr)) if res_kind == 1 else np.sqrt(np.abs(v(rho)))


def rand_csr(rng, n, m, lens):
    """random columns, sorted per row (vectorised: sizes of millions of entries)"""
    lens = np.asarray(lens, np.int64)
    rows = np.repeat(np.arange(n), lens)
    cols = rng.integers(0, m, size=len(rows))
    order = np.lexsort((cols, rows))
    rp = np.zeros(n + 1, np.int64)
    rp[1:] = np.cumsum(lens)
    return rp, cols[order]


def grid_cap_rows(num_sms):
    """rows enough for a gather_pipe / warp_pipe grid at its cap of 2 * num_sms CTAs: 5 entries per
    row on average = 7 merge items per row; a warp tile holds at most 320 items and a CTA takes 8
    tiles, so 3000 rows per SM give >= 7 * 3000 / 320 / 8 = 8.2 CTAs per SM wanted"""
    return 3000 * num_sms


@functools.lru_cache(maxsize=None)
def spmv_case(kind, vt, it, data, num_sms):
    """(n, num_cols, rp, ci, va, b): the matrices of test_parity_gpu.py plus a rectangular one and
    one that fills the capped grids.  num_cols >= n always: the dot reads b[0..n) (the distributed
    CG calls spmv_dot with the n + n_ghost columns of its local block)."""
    rng = np.random.default_rng(17)
    if kind in CSR_KINDS:
        n, m, rp, ci, va = csr_case(rng, kind, vt, it)
    elif kind == "rect":
        n, m = 3000, 7000
        rp, ci, va = H.random_csr(rng, n, m, rng.integers(0, 13, size=n), vt, it)
    elif kind == "grid_cap":
        n = m = grid_cap_rows(num_sms)
        rp, ci = rand_csr(rng, n, m, rng.integers(2, 9, size=n))
        va = rng.uniform(-1, 1, size=len(ci)).astype(VT[vt])
    else:
        raise ValueError(kind)
    ncols = max(n, m)
    nnz = len(ci)
    if data == "int":
        va = rng.integers(-1, 2, size=nnz).astype(VT[vt])
        b = rng.integers(-1, 2, size=ncols).astype(VT[vt])
    else:
        b = rng.uniform(-1, 1, size=ncols).astype(VT[vt])
    return n, ncols, rp.astype(IT[it]), ci.astype(IT[it]), va, b


def exact_spmv(n, rp, ci, va, b):
    """integer data: c (exact, float64) and sum |products| per row"""
    lens = np.diff(rp.astype(np.int64))
    rows = np.repeat(np.arange(n), lens)
    prod = va.astype(np.float64) * b.astype(np.float64)[ci.astype(np.int64)]
    c = np.bincount(rows, weights=prod, minlength=n)
    cabs = np.bincount(rows, weights=np.abs(prod), minlength=n)
    return c, cabs


class Mat:
    """a CSR matrix, its plan and b in the backend's memory"""

    def __init__(self, dev, vt, it, n, ncols, rp, ci, va, variant=None):
        self.vt, self.it, self.n, self.ncols, self.nnz = vt, it, n, ncols, len(va)
        self.rp, self.ci, self.va = dev.put(rp), dev.put(ci), dev.put(va)
        self.plan = dev.plan(vt, it, n, self.nnz, self.rp, variant)

    def spmv(self, dev, b, c):
        dev.call("csr_spmv_%s_%s" % (self.vt, self.it), self.plan, self.n, self.ncols, self.nnz, self.rp,
                 self.ci, self.va, b, 1, 1, c, 1)

    def spmv_dot(self, dev, b, c, dot_ptr, work, ctl=None):
        dev.call("csr_spmv_dot_%s_%s" % (self.vt, self.it), self.plan, self.n, self.ncols, self.nnz,
                 self.rp, self.ci, self.va, b, c, dot_ptr, work, ctl)


def nans(n, vt):
    return np.full(n, np.nan, VT[vt])


# --------------------------------------------------------------------------- A. spmv_dot
@pytest.mark.parametrize("kind", CSR_KINDS + ["rect", "grid_cap"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_dot(dev, orc, kind, variant, vt, it, data):
    n, ncols, rp, ci, va, b = spmv_case(kind, vt, it, data, dev.num_sms)
    A = Mat(dev, vt, it, n, ncols, rp, ci, va, variant)
    if not dev.mock:  # mock: plans carry no variant and no long-row list
        assert dev.l.b200_csr_plan_variant(A.plan) == variant
        if kind == "split_rows":
            assert dev.l.b200_csr_plan_num_long_rows(A.plan) > 0
    if kind == "grid_cap":
        # more CTAs wanted than the cap of 2 * num_sms (see grid_cap_rows)
        assert (2 * n + len(va)) / WARP_TILE_MAX_ITEMS > 8 * 2 * dev.num_sms
    bd, work = dev.put(b), dev.work(vt)

    cref = dev.put(nans(n, vt))
    A.spmv(dev, bd, cref)
    c_plain = cref.get()

    c, dot = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    A.spmv_dot(dev, bd, c, dot.ptr, work)
    got_c, got_dot = c.get(), dot.get()[0]
    # c: the same kernel with the dot fused in its epilogue
    assert got_c.tobytes() == c_plain.tobytes()
    if kind in EXACT_KINDS or data == "int":
        c_orc = nans(n, vt)
        orc("csr_spmv_%s_%s" % (vt, it), n, ncols, len(va), rp, ci, va, b, 1, 1, c_orc, 1)
        assert np.array_equal(got_c, c_orc)
    if data == "int":
        c_exact, cabs = exact_spmv(n, rp, ci, va, b)
        assert cabs.max(initial=0) < exact_limit(vt)  # every partial row sum is exact
        assert int_sum(np.abs(b[:n]), np.abs(c_exact)) < exact_limit(vt)  # every partial dot sum is exact
        assert np.array_equal(got_c, c_exact)
        assert float(got_dot) == int_sum(b[:n], c_exact)
    else:
        assert_sum_within(got_dot, b[:n] * got_c, vt, "b.c")

    # deterministic, and the tickets reset themselves
    c2, dot2 = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    A.spmv_dot(dev, bd, c2, dot2.ptr, work)
    assert c2.get().tobytes() == got_c.tobytes() and dot2.get().tobytes() == dot.get().tobytes()

    # a stopped solver: nothing is written (incl. the long-row kernel and its dot fix)
    ctl = dev.put(np.array([STOPPED, 3, 0, 0, 0, 0, 0, 0], np.int32))
    c3, dot3 = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    A.spmv_dot(dev, bd, c3, dot3.ptr, work, ctl)
    assert np.isnan(c3.get()).all() and np.isnan(dot3.get()).all()


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("it", ITS)
def test_spmv_dot_empty_matrix_writes_zero(dev, vt, it):
    A = Mat(dev, vt, it, 0, 5, np.zeros(1, IT[it]), np.zeros(0, IT[it]), np.zeros(0, VT[vt]))
    b, c, dot = dev.put(np.ones(5, VT[vt])), dev.put(nans(0, vt)), dev.put(nans(1, vt))
    A.spmv_dot(dev, b, c, dot.ptr, dev.work(vt))
    assert dot.get().tolist() == [0.0]
    ctl = dev.put(np.array([STOPPED, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dot = dev.put(nans(1, vt))
    A.spmv_dot(dev, b, c, dot.ptr, dev.work(vt), ctl)
    assert np.isnan(dot.get()).all()


@pytest.mark.parametrize("vt", VTS)
def test_spmv_dot_refuses_slab_variant(dev, vt):
    if dev.mock:
        pytest.skip("mock: plans carry no variant")
    n, ncols, rp, ci, va, b = spmv_case("laplace_like", vt, "i32", "rand", dev.num_sms)
    A = Mat(dev, vt, "i32", n, ncols, rp, ci, va, 0)
    c, dot = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    st = dev.status("csr_spmv_dot_%s_i32" % vt, A.plan, n, ncols, len(va), A.rp, A.ci, A.va, dev.put(b), c,
                    dot.ptr, dev.work(vt).ptr, None)
    assert st != 0
    assert np.isnan(c.get()).all() and np.isnan(dot.get()).all()


def step_xr_exact_case(rng, vt, n):
    """r in {-1, 0, 1}, inv_diag in {1, 2, 3}: sum |r z| <= 3 n, exact for every n used here"""
    r = rng.integers(-1, 2, size=n).astype(VT[vt])
    inv = rng.integers(1, 4, size=n).astype(VT[vt])
    assert 3 * n < exact_limit(vt)
    return r, inv


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_spmv_dot_alternating_with_other_reductions(dev, variant, vt):
    """spmv_dot, step_xr and dense_compute_dot share ctx->counters: each must leave its ticket at 0"""
    rng = np.random.default_rng(5)
    mats = []
    for kind in ("grid_cap", "split_rows"):
        n, ncols, rp, ci, va, b = spmv_case(kind, vt, "i32", "int", dev.num_sms)
        A = Mat(dev, vt, "i32", n, ncols, rp, ci, va, variant)
        c_exact, _ = exact_spmv(n, rp, ci, va, b)
        mats.append((A, dev.put(b), c_exact, int_sum(b[:n], c_exact)))
    nx = 2048 * 4 * dev.num_sms + 777  # step_xr at its grid cap
    r, inv = step_xr_exact_case(rng, vt, nx)
    rd, zd, invd = dev.put(r), dev.put(nans(nx, vt)), dev.put(inv)
    zeros = dev.put(np.zeros(nx, VT[vt]))
    sc = dev.put(np.array([1, 1, 0, 0, 0, 0, 0, 0], VT[vt]))  # pq = 0: r stays, sums are exact
    ctl = dev.put(np.array([0, 0, -1, 0, 1, 0, 0, 0], np.int32))
    res = dev.put(nans(1, vt))
    work = dev.work(vt)
    for rnd in range(2):
        for A, bd, c_exact, d_exact in mats:
            c, dot = dev.put(nans(A.n, vt)), dev.put(nans(1, vt))
            A.spmv_dot(dev, bd, c, dot.ptr, work, ctl)
            assert np.array_equal(c.get(), c_exact) and float(dot.get()[0]) == d_exact, rnd
            dev.call("cg_fused_step_xr_" + vt, nx, zeros, rd, zeros, zeros, zd, invd, sc, ctl, work, 1)
            s = sc.get()
            assert float(s[0]) == int_sum(r, r * inv) and float(s[3]) == int_sum(r, r)
            dev.call("dense_compute_dot_" + vt, nx, 1, rd, 1, invd, 1, res)
            assert float(res.get()[0]) == int_sum(r, inv)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("data", ["int", "rand"])
def test_spmv_dot_graph_replay_matches_eager(dev, variant, vt, data):
    """captured with its fork / join on the auxiliary stream (long-row kernel) and the dot fix"""
    n, ncols, rp, ci, va, b = spmv_case("split_rows", vt, "i64", data, dev.num_sms)
    A = Mat(dev, vt, "i64", n, ncols, rp, ci, va, variant)
    bd, work = dev.put(b), dev.work(vt)
    c, dot = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    A.spmv_dot(dev, bd, c, dot.ptr, work)
    eager_c, eager_dot = c.get(), dot.get()
    c2, dot2 = dev.put(nans(n, vt)), dev.put(nans(1, vt))
    g = dev.capture(lambda: A.spmv_dot(dev, bd, c2, dot2.ptr, work))
    for _ in range(2):
        dev.call("graph_launch", g)
        dev.sync()
        assert c2.get().tobytes() == eager_c.tobytes() and dot2.get().tobytes() == eager_dot.tobytes()
        c2.set(nans(n, vt))
        dot2.set(nans(1, vt))


# --------------------------------------------------------------------------- B. step kernels
def step_sizes(num_sms):
    # 0, one element, one CTA -1 / +1, and step_xr's grid at its cap of 4 * num_sms CTAs of 512
    # threads, each looping over 4 * 512 elements: more partials than the last CTA has threads
    return [0, 1, 511, 513, 2048 * 4 * num_sms + 3 * 2048 + 5]


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("prev_zero", [False, True])
def test_step_p(dev, size, vt, prev_zero):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(size)
    z, p = rng.uniform(-1, 1, n).astype(v), rng.uniform(-1, 1, n).astype(v)
    rho, prev = v(rng.uniform(0.5, 2)), v(0 if prev_zero else rng.uniform(0.5, 2))
    pd, zd = dev.put(p), dev.put(z)
    sc = dev.put(np.array([rho, prev, 0, 0, 0, 0, 0, 0], v))
    ctl = dev.put(np.zeros(8, np.int32))
    dev.call("cg_fused_step_p_" + vt, n, pd, zd, sc, ctl)
    want = z if prev_zero else z + (rho / prev) * p
    assert pd.get().tobytes() == want.tobytes()
    ctl.set(np.array([STOPPED, 0, 0, 0, 0, 0, 0, 0], np.int32))
    dev.call("cg_fused_step_p_" + vt, n, pd, zd, sc, ctl)
    assert pd.get().tobytes() == want.tobytes()


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
@pytest.mark.parametrize("finalize", [1, 0])
def test_init_and_step_xr(dev, size, vt, precond, finalize):
    n = step_sizes(dev.num_sms)[size]
    v = VT[vt]
    rng = np.random.default_rng(100 + size)
    x, r = rng.uniform(-1, 1, n).astype(v), rng.uniform(-1, 1, n).astype(v)
    inv = rng.uniform(0.5, 2, n).astype(v) if precond else None
    xd, rd, zd, pd, qd = (dev.put(a) for a in (x, r, nans(n, vt), nans(n, vt), nans(n, vt)))
    invd = dev.put(inv) if precond else None
    sc = dev.put(np.array([7, 7, 7, 7, 2.5, 7, 7, 7], v))  # sc[4]: ||b|| for baseline 0
    ctl = dev.put(np.full(8, 7, np.int32))
    work = dev.work(vt)
    factor, max_iters = v(2.0 ** -20), 5
    dev.call("cg_fused_init_" + vt, n, rd, zd, pd, qd, invd, sc, ctl, work, max_iters, 1, 1, 0,
             float(factor), finalize)
    z = r * inv if precond else r
    assert zd.get().tobytes() == z.tobytes() and rd.get().tobytes() == r.tobytes()
    assert not pd.get().any() and not qd.get().any()
    s, c = sc.get(), ctl.get()
    assert c[1:5].tolist() == [0 if finalize else -1, max_iters, 1, 1]
    assert s[4] == v(2.5)
    if finalize:
        assert s[1] == 1 and s[2] == 0 and s[6] == 0 and s[7] == 0
        assert_sum_within(s[0], r * z, vt, "rho")
        assert_sum_within(s[3], r * r, vt, "rr")
        assert s[5] == factor * v(2.5)
        assert c[0] == expected_status(0, max_iters, 1, 1, tau_of(vt, 1, s[0], s[3]), s[5])
    else:
        assert s[:4].tolist() == [1, 1, 0, 0]
        assert_sum_within(s[6], r * z, vt, "rho")
        assert_sum_within(s[7], r * r, vt, "rr")
        assert c[0] == 0

    for pq_zero in (False, True):
        x0, r0, z0 = xd.get(), rd.get(), zd.get()
        s0, c0 = sc.get(), ctl.get()
        p, q = rng.uniform(-1, 1, n).astype(v), rng.uniform(-1, 1, n).astype(v)
        pd.set(p)
        qd.set(q)
        s0[2] = 0 if pq_zero else v(rng.uniform(0.5, 2))
        sc.set(s0)
        dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, finalize)
        s, c = sc.get(), ctl.get()
        if c0[0] != 0:  # stopped at init (n = 0: ||r|| = 0): a no-op
            assert (xd.get().tobytes(), rd.get().tobytes(), zd.get().tobytes()) == \
                (x0.tobytes(), r0.tobytes(), z0.tobytes())
            assert s.tobytes() == s0.tobytes() and c.tobytes() == c0.tobytes()
            continue
        if pq_zero:
            x1, r1 = x0, r0
        else:
            alpha = s0[0] / s0[2]
            x1, r1 = x0 + alpha * p, r0 - alpha * q
        z1 = r1 * inv if precond else r1
        assert xd.get().tobytes() == x1.tobytes()
        assert rd.get().tobytes() == r1.tobytes()
        assert zd.get().tobytes() == z1.tobytes()
        if finalize:
            assert s[1] == s0[0] and s[2] == s0[2] and s[4:].tobytes() == s0[4:].tobytes()
            assert_sum_within(s[0], r1 * z1, vt, "rho")
            assert_sum_within(s[3], r1 * r1, vt, "rr")
            assert c[1] == c0[1] + 1
            assert c[0] == expected_status(c[1], max_iters, 1, 1, tau_of(vt, 1, s[0], s[3]), s[5])
        else:
            assert s[:6].tobytes() == s0[:6].tobytes() and c.tobytes() == c0.tobytes()
            assert_sum_within(s[6], r1 * z1, vt, "rho")
            assert_sum_within(s[7], r1 * r1, vt, "rr")


@pytest.mark.parametrize("size", range(5))
@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("precond", [False, True])
def test_step_xr_sums_exact_on_integers(dev, size, vt, precond):
    n = step_sizes(dev.num_sms)[size]
    rng = np.random.default_rng(200 + size)
    r, inv = step_xr_exact_case(rng, vt, n)
    if not precond:
        inv = np.ones(n, VT[vt])
    rho, rr = int_sum(r, r * inv), int_sum(r, r)
    rd, zd, pd, qd = (dev.put(a) for a in (r, nans(n, vt), nans(n, vt), nans(n, vt)))
    invd = dev.put(inv) if precond else None
    xd = dev.put(np.zeros(n, VT[vt]))
    sc, ctl, work = dev.put(nans(8, vt)), dev.put(np.zeros(8, np.int32)), dev.work(vt)
    # no criterion: never stops
    dev.call("cg_fused_init_" + vt, n, rd, zd, pd, qd, invd, sc, ctl, work, -1, 0, 1, 2, 1.0, 1)
    s = sc.get()
    assert (float(s[0]), float(s[3])) == (rho, rr)
    for k in range(2):  # pq = 0 after init: r stays integer
        dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 1)
        s, c = sc.get(), ctl.get()
        assert (float(s[0]), float(s[1]), float(s[3])) == (rho, rho, rr)
        assert c[:2].tolist() == [0, k + 1]
    dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 0)
    s = sc.get()
    assert (float(s[6]), float(s[7])) == (rho, rr)


@pytest.mark.parametrize("vt", VTS)
def test_init_clamps_max_iters(dev, vt):
    n = 4
    bufs = [dev.put(np.ones(n, VT[vt])) for _ in range(4)]
    sc, ctl = dev.put(nans(8, vt)), dev.put(np.zeros(8, np.int32))
    dev.call("cg_fused_init_" + vt, n, *bufs, None, sc, ctl, dev.work(vt), 2 ** 33, 1, 1, 2, 0.5, 1)
    assert ctl.get()[2] == 2 ** 31 - 1


def stop_case(vt, baseline, res_kind, rel):
    """r = (4, 4, 4, 4, 0, ...), inv_diag = 1/4: rr = 64, rho = 16, so tau = 8 (ResidualNorm) or 4
    (ImplicitResidualNorm); tau0 by baseline: 0 ||b|| = 2 (preset), 1 sqrt(rr) = 8, 2 absolute 1,
    3 sqrt(||b||^2 = 4) = 2.  factor = tau / tau0 * rel: powers of two, so rel = 1 puts tau exactly
    on the threshold (the criterion is tau <= threshold: it stops)."""
    tau = 8.0 if res_kind != 2 else 4.0
    tau0 = {0: 2.0, 1: 8.0, 2: 1.0, 3: 2.0}[baseline]
    preset = {0: 2.0, 3: 4.0}.get(baseline, 123.0)
    return VT[vt](tau / tau0 * rel), preset


@pytest.mark.parametrize("vt", VTS)
@pytest.mark.parametrize("baseline", [0, 1, 2, 3])
def test_stopping_table(dev, vt, baseline):
    """every criterion set through init + step_xr(finalize=1), and through the multi-GPU split
    finalize=0 + cg_fused_finish (the only path for baseline 3, whose sc[4] is the global ||b||^2)"""
    v = VT[vt]
    n = 8
    r = np.array([4, 4, 4, 4, 0, 0, 0, 0], v)
    inv = np.full(n, 0.25, v)
    rr, rho = v(64), v(16)
    work = dev.work(vt)
    rd, invd = dev.put(r), dev.put(inv)
    xd = dev.put(np.zeros(n, v))

    def run(split, max_iters, res_kind, iter_first, factor, preset):
        bufs = [dev.put(nans(n, vt)) for _ in range(3)]  # z p q
        sc = dev.put(np.array([9, 9, 9, 9, preset, 9, 9, 9], v))
        ctl = dev.put(np.zeros(8, np.int32))
        dev.call("cg_fused_init_" + vt, n, rd, *bufs, invd, sc, ctl, work, max_iters, res_kind, iter_first,
                 baseline, float(factor), 0 if split else 1)
        if split:
            dev.call("cg_fused_finish_" + vt, sc, ctl, 1, baseline, float(factor))
        after_init = (sc.get(), ctl.get())
        z, p, q = bufs
        dev.call("cg_fused_step_xr_" + vt, n, xd, rd, p, q, z, invd, sc, ctl, work, 0 if split else 1)
        if split:
            dev.call("cg_fused_finish_" + vt, sc, ctl, 0, baseline, float(factor))
        return after_init, (sc.get(), ctl.get())

    checked = 0
    for max_iters in (-1, 0, 1):
        for res_kind in (0, 1, 2):
            for iter_first in (0, 1):
                for rel in (0.5, 1.0, 2.0):
                    factor, preset = stop_case(vt, baseline, res_kind, rel)
                    tau0 = {0: v(preset), 1: np.sqrt(rr), 2: v(1), 3: np.sqrt(v(preset))}[baseline]
                    threshold = factor * tau0
                    tau = tau_of(vt, res_kind, rho, rr)
                    st0 = expected_status(0, max_iters, res_kind, iter_first, tau, threshold)
                    st1 = st0 or expected_status(1, max_iters, res_kind, iter_first, tau, threshold)
                    clamp = max_iters
                    runs = [True] if baseline == 3 else [False, True]
                    results = [run(split, max_iters, res_kind, iter_first, factor, preset) for split in runs]
                    for (si, ci), (ss, cs) in results:
                        what = (max_iters, res_kind, iter_first, rel)
                        assert ci[:5].tolist() == [st0, 0, clamp, res_kind, iter_first], what
                        assert si[4] == tau0 and si[5] == threshold, what
                        assert (si[0], si[1], si[3]) == (rho, 1, rr), what
                        assert cs[:2].tolist() == [st1, 1 if st0 == 0 else 0], what
                        if st0 == 0:
                            assert (ss[0], ss[1], ss[3]) == (rho, rho, rr), what
                    if len(results) == 2:
                        # the split leaves sc[0..5] and ctl as finalize = 1 does; sc[6..7] hold the sums
                        # finalize = 1 put into sc[0] / sc[3]
                        (f_si, f_ci), (f_ss, f_cs) = results[0]
                        (s_si, s_ci), (s_ss, s_cs) = results[1]
                        assert s_si[:6].tobytes() == f_si[:6].tobytes() and s_ci.tobytes() == f_ci.tobytes()
                        assert (s_si[6], s_si[7]) == (f_si[0], f_si[3])
                        assert s_ss[:6].tobytes() == f_ss[:6].tobytes() and s_cs.tobytes() == f_cs.tobytes()
                        if f_ci[0] == 0:
                            assert (s_ss[6], s_ss[7]) == (f_ss[0], f_ss[3])
                    checked += 1
    assert checked == 54


@pytest.mark.parametrize("vt", VTS)
def test_kernels_are_noops_after_a_stop(dev, vt):
    rng = np.random.default_rng(8)
    rp, ci, va = arrow(vt)
    n = len(rp) - 1
    A = Mat(dev, vt, "i32", n, n, rp, ci, va)
    v = VT[vt]
    arrays = [rng.uniform(-1, 1, n).astype(v) for _ in range(5)]
    xd, rd, zd, pd, qd = (dev.put(a) for a in arrays)
    invd = dev.put(rng.uniform(0.5, 2, n).astype(v))
    sc, ctl, work = dev.put(nans(8, vt)), dev.put(np.zeros(8, np.int32)), dev.work(vt)
    # max_iters = 0: stopped right at init
    dev.call("cg_fused_init_" + vt, n, rd, zd, pd, qd, invd, sc, ctl, work, 0, 1, 1, 2, 0.5, 1)
    assert ctl.get()[0] == 0x40 | 1
    pd.set(arrays[3])
    qd.set(arrays[4])
    state = [b.get().tobytes() for b in (xd, rd, zd, pd, qd, sc, ctl)]
    dev.call("cg_fused_step_p_" + vt, n, pd, zd, sc, ctl)
    A.spmv_dot(dev, pd, qd, sc.at(2), work, ctl)
    dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 1)
    dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 0)
    dev.call("cg_fused_finish_" + vt, sc, ctl, 0, 2, 0.5)
    assert [b.get().tobytes() for b in (xd, rd, zd, pd, qd, sc, ctl)] == state


# --------------------------------------------------------------------------- C. lock step
def arrow(vt, g=72, links=(1100, 2000, 4500), seed=11, shift=0):
    """SPD 'arrow' matrix: the 5-point Laplacian on a g x g grid plus hub rows / columns with
    `links` off-diagonal -1 entries each (rows of >= 1024 entries: split over CTAs; 4500 > one
    chunk of 4096), every link adding 1 to both diagonals: symmetric, irreducibly diagonally dominant
    with a positive diagonal.  `shift` is added to the whole diagonal.  Integer values."""
    import scipy.sparse as sp
    import workloads as W
    rp, ci, va = W.laplace(g, 2)
    n = g * g
    L = sp.csr_matrix((va, ci, rp), shape=(n, n))
    rng = np.random.default_rng(seed)
    hubs = np.linspace(0, n - 1, len(links) + 2).astype(np.int64)[1:-1]
    rows, cols = [], []
    for h, k in zip(hubs, links):
        others = rng.choice(np.delete(np.arange(n), h), size=k, replace=False)
        rows += [np.full(k, h), others]
        cols += [others, np.full(k, h)]
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    E = sp.csr_matrix((-np.ones(len(rows)), (rows, cols)), shape=(n, n))
    A = (L + E + sp.diags(np.asarray(abs(E).sum(axis=1)).ravel() + shift)).tocsr()
    A.sum_duplicates()
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(VT[vt])


def arrow_inv_diag(rp, ci, va):
    n = len(rp) - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    diag = va[rows == ci]
    assert len(diag) == n
    return (va.dtype.type(1) / diag).astype(va.dtype)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("vt", VTS)
def test_lockstep_iterations_on_arrow(dev, orc, variant, vt):
    v = VT[vt]
    rp, ci, va = arrow(vt)
    n, nnz = len(rp) - 1, len(va)
    lens = np.diff(rp)
    assert lens.max() >= 4096 and (lens >= 1024).sum() == 3
    A = Mat(dev, vt, "i32", n, n, rp, ci, va, variant)
    if not dev.mock:  # mock: plans carry no long-row list
        assert dev.l.b200_csr_plan_num_long_rows(A.plan) == 3
    inv = arrow_inv_diag(rp, ci, va)
    rng = np.random.default_rng(4)
    b = rng.uniform(-1, 1, n).astype(v)
    xd, rd, zd, pd, qd = (dev.put(a) for a in (np.zeros(n, v), b, nans(n, vt), nans(n, vt), nans(n, vt)))
    invd = dev.put(inv)
    qref = dev.put(nans(n, vt))
    sc, ctl, work = dev.put(nans(8, vt)), dev.put(np.zeros(8, np.int32)), dev.work(vt)
    # converges after about 44 (f64) / 29 (f32) iterations: the graph below runs past the stop
    factor = 1e-12 if vt == "f64" else 1e-7
    dev.call("cg_fused_init_" + vt, n, rd, zd, pd, qd, invd, sc, ctl, work, -1, 1, 1, 1, factor, 1)
    s = sc.get()
    assert zd.get().tobytes() == (b * inv).tobytes()
    assert_sum_within(s[0], b * (b * inv), vt, "rho")
    assert_sum_within(s[3], b * b, vt, "rr")
    assert s[4] == np.sqrt(s[3]) and s[5] == v(factor) * s[4]
    short = lens < 64  # summed by one thread, left to right: the oracle's bits
    for it in range(24):
        assert ctl.get()[0] == 0, it
        s, p0, z0 = sc.get(), pd.get(), zd.get()
        dev.call("cg_fused_step_p_" + vt, n, pd, zd, sc, ctl)
        p1 = z0 + (s[0] / s[1]) * p0 if s[1] != 0 else z0
        assert pd.get().tobytes() == p1.tobytes(), it

        A.spmv_dot(dev, pd, qd, sc.at(2), work, ctl)
        A.spmv(dev, pd, qref)
        q1, s1 = qd.get(), sc.get()
        assert q1.tobytes() == qref.get().tobytes(), it
        q_orc = nans(n, vt)
        orc("csr_spmv_%s_i32" % vt, n, n, nnz, rp, ci, va, p1, 1, 1, q_orc, 1)
        assert np.array_equal(q1[short], q_orc[short]), it
        for row in np.flatnonzero(~short):  # tree / chunk order: within the bound of any order
            s_, e_ = rp[row], rp[row + 1]
            assert_sum_within(q1[row], va[s_:e_] * p1[ci[s_:e_]], vt, ("row", row, it))
        assert_sum_within(s1[2], p1 * q1, vt, "p.q")
        assert np.delete(s1, 2).tobytes() == np.delete(s, 2).tobytes(), it

        x0, r0, c0 = xd.get(), rd.get(), ctl.get()
        dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 1)
        alpha = s1[0] / s1[2]
        x1, r1 = x0 + alpha * p1, r0 - alpha * q1
        z1 = r1 * inv
        assert xd.get().tobytes() == x1.tobytes(), it
        assert rd.get().tobytes() == r1.tobytes(), it
        assert zd.get().tobytes() == z1.tobytes(), it
        s2, c2 = sc.get(), ctl.get()
        assert s2[1] == s1[0] and s2[2] == s1[2] and s2[4:].tobytes() == s1[4:].tobytes(), it
        assert_sum_within(s2[0], r1 * z1, vt, "rho")
        assert_sum_within(s2[3], r1 * r1, vt, "rr")
        assert c2[1] == c0[1] + 1 == it + 1
        assert c2[0] == expected_status(c2[1], -1, 1, 1, np.sqrt(s2[3]), s2[5]), it

    def iteration():
        dev.call("cg_fused_step_p_" + vt, n, pd, zd, sc, ctl)
        A.spmv_dot(dev, pd, qd, sc.at(2), work, ctl)
        dev.call("cg_fused_step_xr_" + vt, n, xd, rd, pd, qd, zd, invd, sc, ctl, work, 1)

    k = 8
    g = dev.capture(lambda: [iteration() for _ in range(k)])
    for _ in range(400):
        dev.call("graph_launch", g)
        if ctl.get()[0] != 0:
            break
    c = ctl.get()
    assert c[0] == 0x80 | 0x40 | 1, c
    state = [a.get().tobytes() for a in (xd, rd, zd, pd, qd, sc, ctl)]
    for _ in range(2):
        dev.call("graph_launch", g)
    assert [a.get().tobytes() for a in (xd, rd, zd, pd, qd, sc, ctl)] == state


# --------------------------------------------------------------------------- D. end to end
def host_solve(hexec, vt, rp, ci, va, b, precond, **kw):
    import torch
    from ginkgo_b200 import api
    n = len(rp) - 1
    with torch.cuda.stream(hexec.stream):
        t = [torch.from_numpy(a).to(hexec.device) for a in (va, ci, rp)]
        tb = torch.from_numpy(b.reshape(n, 1).copy()).to(hexec.device)
        tx = torch.zeros(n, 1, dtype=tb.dtype, device=hexec.device)
    A = api.host_csr(hexec, (n, n), *t)
    s = api.HostSolver(hexec, "cg", A, precond_max_bs=precond, fused=True, **kw)
    s.apply(api.host_dense(hexec, tb), api.host_dense(hexec, tx))
    hexec.synchronize()
    parts = api._host().gkob_csr_plan_parts(A.h) if vt == "f64" else None
    return tx.cpu().numpy(), s.num_iterations, s.stop_status, s.used_fused, parts


@pytest.mark.parametrize("kernel,reblock,vt,precond",
                         [(k, None, vt, pre) for k in ("warp", "pipe", "ring") for vt in VTS for pre in (0, 1)] +
                         [("warp", "3", "f64", 1)])
def test_fused_cg_on_arrow_matches_oracle(hexec, monkeypatch, kernel, reblock, vt, precond):
    # read by the plan's kernel choice on every call (B200_CSR_KERNEL) and by the tuning of the plan
    # (B200_CSR_REBLOCK: a column-blocked copy next to the fused loop, which does not use it)
    monkeypatch.setenv("B200_CSR_KERNEL", kernel)
    if reblock is not None:
        monkeypatch.setenv("B200_CSR_REBLOCK", reblock)
    # the unit shift keeps unpreconditioned fp32 CG within the +-2 iterations of the oracle whatever
    # the order of its dot products (without it, 43..47 iterations depending on the order)
    rp, ci, va = arrow(vt, g=60, links=(1100, 1500, 3000), shift=1)
    n = len(rp) - 1
    rng = np.random.default_rng(12)
    b = rng.uniform(-1, 1, n).astype(VT[vt])
    red = 1e-9 if vt == "f64" else 1e-4
    jac = {"blocks": arrow_inv_diag(rp, ci, va)} if precond else None
    xo, ito, stop_o = H.orc_solve("cg", vt, rp, ci, va, b, np.zeros(n, VT[vt]), precond, jac, max_iters=2000,
                                  reduction=red)
    xd, itd, stop_d, used, parts = host_solve(hexec, vt, rp, ci, va, b, precond, max_iters=2000,
                                              reduction=red)
    assert used
    if reblock is not None and not hexec.device.type == "cpu":  # mock: plans carry no column-blocked copy
        assert parts == int(reblock)
    assert abs(itd - ito) <= 2, (itd, ito)
    assert stop_d == stop_o[0] == 0x80 | 0x40 | 2
    assert H.rel_err(xo, xd) <= (1e-8 if vt == "f64" else 1e-3)
