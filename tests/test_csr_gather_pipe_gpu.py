"""The gather-pipe CSR SpMV kernel (csr_kernels.cuh, plan variant 2): the tuned plan picks it for
matrices with scattered gathers, unblocked and column-blocked, and its results equal the oracle's
left-to-right row sums bit for bit (torch.equal).

Two matrices:
 * `short`: about 3 entries per row, uniformly random columns and values -- the shape of one column
   part of cfg2.  Every row is summed by one lane in storage order, so the comparison checks the order
   of the additions as well.
 * `mixed`: stretches of empty rows (tiles of more rows than the row-pointer prefetch covers), rows of
   64..300 entries (summed by the whole warp), rows of 400..1000 entries (the last row of a tile that
   does not fit the products strip) and rows of >= 1024 entries (split over CTAs).  Values and x are
   small integers, so every partial sum is exact and any summation order gives the same bits: the
   comparison checks which products each row receives."""
import numpy as np
import pytest

from tests import helpers as H
from tests.helpers import VT

pytestmark = pytest.mark.gpu


def make(kind, vt, it, seed=3):
    rng = np.random.default_rng(seed)
    if kind == "short":
        n = m = 60_000
        lens = rng.poisson(3.0, size=n)
        rp, ci, va = H.random_csr(rng, n, m, lens, vt, it)
        x = rng.uniform(-1, 1, size=m).astype(VT[vt])
    else:
        n = m = 12_000
        lens = rng.integers(0, 6, size=n)
        lens[rng.integers(0, n, size=n // 3)] = 0
        lens[2000:2600] = 0
        lens[9000:9400] = 0
        lens[[10, 500, 501, 3000, 7000]] = [64, 65, 90, 150, 300]
        lens[[20, 4000, 8000]] = [400, 700, 1000]
        lens[[30, 5000, 11_999]] = [1024, 3000, 5000]
        rp, ci, va = H.random_csr(rng, n, m, lens, vt, it)
        va = rng.integers(-4, 5, size=len(va)).astype(VT[vt])
        x = rng.integers(-4, 5, size=m).astype(VT[vt])
    return n, m, rp, ci, va, x


def oracle_apply(orc, vt, it, n, m, rp, ci, va, x, alpha=None, beta=None, y0=None):
    y = np.zeros((n, 1), VT[vt]) if y0 is None else y0.copy().reshape(n, 1)
    if alpha is None:
        orc("csr_spmv_%s_%s" % (vt, it), n, m, len(va), rp, ci, va, x.reshape(m, 1), 1, 1, y, 1)
    else:
        orc("csr_advanced_spmv_%s_%s" % (vt, it), n, m, len(va), rp, ci, va, np.array([alpha], VT[vt]),
            x.reshape(m, 1), 1, 1, np.array([beta], VT[vt]), y, 1)
    return y.reshape(-1)


def device_apply(ex, A, x, alpha=None, beta=None, y0=None):
    import torch
    from ginkgo_b200 import api
    dt = A.values.dtype
    with torch.cuda.stream(ex.stream):
        xd = torch.from_numpy(x).to(ex.device)
        y = (torch.full((A.size[0],), float("nan"), dtype=dt) if y0 is None else torch.from_numpy(y0.copy()))
        y = y.to(ex.device)
    Y = api.Dense(ex, y)
    if alpha is None:
        A.apply(api.Dense(ex, xd), Y)
    else:
        with torch.cuda.stream(ex.stream):
            a = torch.tensor([alpha], dtype=dt, device=ex.device)
            b = torch.tensor([beta], dtype=dt, device=ex.device)
        A.apply(api.Dense(ex, a), api.Dense(ex, xd), api.Dense(ex, b), Y)
    ex.synchronize()
    return Y.values.reshape(-1).cpu()


def check_all_modes(orc, ex, A, vt, it, n, m, rp, ci, va, x):
    import torch
    rng = np.random.default_rng(9)
    y0 = rng.integers(-4, 5, size=n).astype(VT[vt])
    got = device_apply(ex, A, x)
    assert torch.equal(got, torch.from_numpy(oracle_apply(orc, vt, it, n, m, rp, ci, va, x)))
    for alpha, beta in [(-1.5, 0.0), (0.5, 2.0), (1.0, 1.0)]:
        yin = np.full(n, np.nan, VT[vt]) if beta == 0.0 else y0
        got = device_apply(ex, A, x, alpha, beta, yin)
        want = oracle_apply(orc, vt, it, n, m, rp, ci, va, x, alpha, beta, yin)
        assert torch.equal(got, torch.from_numpy(want)), (alpha, beta)


def csr(ex, n, m, rp, ci, va):
    import torch
    from ginkgo_b200 import api
    with torch.cuda.stream(ex.stream):
        t = [torch.from_numpy(a).to(ex.device) for a in (va, ci, rp)]
    return api.Csr(ex, (n, m), *t)


@pytest.fixture(scope="module")
def ex():
    from ginkgo_b200 import api
    return api.B200Executor.create(0)


def test_plan_picks_gather_pipe_for_scattered_gathers(ex):
    from ginkgo_b200 import _lib
    n, m, rp, ci, va, x = make("short", "f64", "i32")
    A = csr(ex, n, m, rp, ci, va)
    l = _lib.lib()
    assert l.b200_csr_plan_variant(A.plan()) == 2
    assert l.b200_csr_plan_gather_lines(A.plan()) > 0.9
    assert l.b200_csr_plan_parts(A.plan()) == 0


@pytest.mark.parametrize("kind", ["short", "mixed"])
@pytest.mark.parametrize("vt", ["f64", "f32"])
@pytest.mark.parametrize("it", ["i32", "i64"])
def test_gather_pipe_matches_oracle(orc, ex, kind, vt, it):
    from ginkgo_b200 import _lib
    n, m, rp, ci, va, x = make(kind, vt, it)
    A = csr(ex, n, m, rp, ci, va)
    assert _lib.lib().b200_csr_plan_variant(A.plan()) == 2
    if kind == "mixed":
        assert _lib.lib().b200_csr_plan_num_long_rows(A.plan()) == 3
    check_all_modes(orc, ex, A, vt, it, n, m, rp, ci, va, x)


@pytest.mark.parametrize("parts", [2, 3, 4, 5])
@pytest.mark.parametrize("kind", ["short", "mixed"])
@pytest.mark.parametrize("vt,it", [("f64", "i32"), ("f32", "i64")])
def test_gather_pipe_column_parts_match_oracle(orc, ex, monkeypatch, parts, kind, vt, it):
    from ginkgo_b200 import _lib
    monkeypatch.setenv("B200_CSR_REBLOCK", str(parts))
    n, m, rp, ci, va, x = make(kind, vt, it, seed=5)
    A = csr(ex, n, m, rp, ci, va)
    l = _lib.lib()
    assert l.b200_csr_plan_parts(A.plan()) == parts
    assert l.b200_csr_plan_variant(A.plan()) == 2
    check_all_modes(orc, ex, A, vt, it, n, m, rp, ci, va, x)
