"""Scalar float64 routines of csrc/tsfx_math.cuh (the single-lane sections of the kernels), compiled for
the host with g++ and checked against scipy / numpy.  CPU-only."""
import ctypes
import os
import subprocess
import warnings

import numpy as np
import pytest
from scipy import special, stats

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hm(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hm") / "libhostmath.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", "-ffp-contract=off",
                           os.path.join(HERE, "native", "host_math_shim.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    d = ctypes.c_double
    for name, n in (("hm_incbeta", 3), ("hm_student2", 2), ("hm_mackinnon", 1), ("hm_cubic", 4)):
        getattr(lib, name).restype = d
        getattr(lib, name).argtypes = [d] * n
    lib.hm_quantile.restype = d
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def test_incbeta_and_student(hm):
    rng = np.random.default_rng(0)
    for _ in range(300):
        a, b, x = rng.uniform(0.5, 200), rng.uniform(0.5, 5), rng.uniform(0, 1)
        assert hm.hm_incbeta(a, b, x) == pytest.approx(special.betainc(a, b, x), rel=1e-10, abs=1e-300)
    for df in (1, 2, 3, 8, 24, 50, 254, 1022):
        for t in (0.0, 1e-3, 0.5, 1.0, 2.0, 2.5, 7.0, 30.0, -3.0):
            assert hm.hm_student2(t, df) == pytest.approx(2 * special.stdtr(df, -abs(t)), rel=1e-9)
    assert np.isnan(hm.hm_student2(0.0, 0.0))


def test_cubic_max_real_root(hm):
    rng = np.random.default_rng(1)
    for i in range(500):
        c = rng.standard_normal(4) * 10 ** rng.uniform(-3, 3, 4)
        if i % 7 == 0:
            c[0] = 0.0
        if i % 11 == 0:
            c[3] = 0.0
        want = np.max(np.real(np.roots(c)))
        got = hm.hm_cubic(*c)
        assert got == pytest.approx(want, rel=1e-8, abs=1e-10), c
    assert np.isnan(hm.hm_cubic(np.nan, 1, 1, 1))


def test_polyfit3(hm):
    rng = np.random.default_rng(2)
    for k in (1, 2, 3, 4, 5, 12, 30):
        x = np.sort(rng.standard_normal(k) * 2)
        y = rng.standard_normal(k)
        c = np.zeros(5)
        assert hm.hm_polyfit3(_p(x), _p(y), k, _p(c))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = np.polyfit(x, y, 3)
        np.testing.assert_allclose(c[:4], want, rtol=1e-7, atol=1e-9)


def _shifted_fits():
    """(level, r, bin means x, y) of the Friedrich fit (the oracle's bin means) on walks b + 0.3 cumsum(N(0, 1)) of 256
    float32 samples, and on 31-sample N(0, 1) series for k = 1 .. 3 bins"""
    from oracle.calculators import friedrich_points
    rng = np.random.default_rng(11)
    out = []
    for level in (0.0, 30.0, 100.0, 300.0, 1e3, 3e3, 1e4, -1e3):
        for i in range(6):
            walk = (level + 0.3 * rng.standard_normal(256).cumsum()).astype(np.float32).astype(np.float64)
            short = (level + rng.standard_normal(31)).astype(np.float32).astype(np.float64)
            for s, r in ((walk, 4), (walk, 5), (walk, 10), (walk, 30), (short, 1), (short, 2), (short, 3)):
                pts = friedrich_points(s, r)
                out.append((level, r, pts.xm.to_numpy(np.float64), pts.ym.to_numpy(np.float64)))
    return out


def test_polyfit3_shifted_abscissae(hm):
    """Bin means at levels up to 1e4: the coefficients against the exact least-squares (k >= 4) or minimum-norm (k < 4)
    fit within the least-squares perturbation bound (tests/helpers.py:polyfit3_accepts), against np.polyfit at
    rtol 1e-5 where that bound is below 1e-7, and the largest real root against np.roots of the exact fit"""
    from oracle.extract import NOISE_FLOOR
    from tests.helpers import exact_polyfit3, polyfit3_bound, polyfit3_error
    failures = []
    for level, r, x, y in _shifted_fits():
        k = len(x)
        c = np.zeros(5)
        if not hm.hm_polyfit3(_p(x), _p(y), k, _p(c)):
            failures.append((level, r, k, "no fit"))
            continue
        ex, S = exact_polyfit3(x, y)
        err, bound = polyfit3_error(c[:4], ex, S), polyfit3_bound(x, y, ex, S)
        if not err <= max(1e-5, bound):
            failures.append((level, r, k, "coefficients", err, bound))
        if bound < 1e-7:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                want = np.polyfit(x, y, 3)
            if not np.allclose(c[:4], want, rtol=1e-5, atol=0):
                failures.append((level, r, k, "np.polyfit", list(c[:4]), list(want)))
        # the roots live at the scale of the abscissae: one bin gives the cubic c (t^3 + t^2 x + t x^2 + x^3) with the
        # roots -x and +-ix, so a largest real part of exactly 0 that both sides compute as rounding noise of order eps |x|
        root = np.max(np.real(np.roots([float(v) for v in ex])))
        if not np.isclose(c[4], root, rtol=1e-5, atol=NOISE_FLOOR * max(1.0, np.abs(x).max())):
            failures.append((level, r, k, "max_langevin", c[4], root))
    assert not failures, "%d failures, first: %r" % (len(failures), failures[:10])


def test_levinson_quantile_linreg_cholesky(hm):
    rng = np.random.default_rng(3)
    from oracle import thirdparty as tp
    x = rng.standard_normal(200)
    acv = tp.acovf_adjusted(x)[:10].copy()
    out, work = np.zeros(10), np.zeros(20)
    hm.hm_levinson(_p(acv), 9, _p(out), _p(work))
    np.testing.assert_allclose(out, tp.levinson_durbin_pacf(acv, 9), rtol=1e-12)
    s = np.sort(rng.standard_normal(37))
    for q in (0.0, 0.1, 0.25, 0.5, 0.55, 0.9, 1.0, 1 / 3):
        assert hm.hm_quantile(_p(s), 37, ctypes.c_double(q)) == np.quantile(s, q)
    y = rng.standard_normal(50).cumsum()
    t = np.arange(50.0)
    lr = stats.linregress(t, y)
    o = np.zeros(5)
    hm.hm_linreg.argtypes = [ctypes.c_double] * 6 + [ctypes.POINTER(ctypes.c_double)]
    hm.hm_linreg(50.0, t.mean(), y.mean(), np.mean((t - t.mean()) ** 2), np.mean((y - y.mean()) ** 2),
                 np.mean((t - t.mean()) * (y - y.mean())), _p(o))
    np.testing.assert_allclose(o, [lr.pvalue, lr.rvalue, lr.intercept, lr.slope, lr.stderr], rtol=1e-9)
    A = rng.standard_normal((8, 8))
    A = A @ A.T + np.eye(8)
    b = rng.standard_normal(8)
    want = np.linalg.solve(A, b)
    Ac, bc = A.copy(), b.copy()
    assert hm.hm_cholesky_solve(_p(Ac), 8, _p(bc))
    np.testing.assert_allclose(bc, want, rtol=1e-10)


def test_mackinnon(hm):
    from oracle import thirdparty as tp
    for s in (-25.0, -15.3, -3.0, -1.61, -1.0, 0.0, 2.0, 3.0):
        assert hm.hm_mackinnon(s) == pytest.approx(tp.mackinnonp_c(s), rel=1e-12)
