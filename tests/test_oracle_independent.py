"""Second, independent derivations of the two calculators whose reference arithmetic lives in packages that cannot be
installed here (statsmodels adfuller, PyWavelets cwt) -- the 63 columns SURVEY.md section 8c calls "parity unpinned".
They are NOT statsmodels / pywt (those are absent from this image); they bound what the restatements in
oracle/thirdparty.py can be wrong about:

  * augmented_dickey_fuller: a from-scratch OLS route (explicit design matrices, numpy.linalg.lstsq, information
    criteria from the residual variance) must give the same usedlag and test statistic as the restatement, and the
    MacKinnon p-value surface must reproduce the published asymptotic critical values of the constant-only test
    (-3.43 / -2.86 / -2.57 at 1 % / 5 % / 10 %).
  * cwt_coefficients: the continuous wavelet transform with the Mexican-hat wavelet evaluated by EXACT integration
    (closed-form antiderivative, series piecewise constant on [k, k+1)) must agree with the restated pywt algorithm
    (integrated wavelet sampled on a 1024-point grid) to the discretisation error of that algorithm (< 2 % of the
    largest coefficient at every scale tsfresh uses, on signals smooth at the sample scale; correlation > 0.98 on
    white noise, where the floor()-resampled kernel of the pywt algorithm itself is the error)."""
import math

import numpy as np
import pytest

from oracle import thirdparty as tp


def adf_lstsq(x, autolag="AIC"):
    """Dickey-Fuller regression  dx_t = c + g x_{t-1} + sum_j b_j dx_{t-j} + e_t  with lag order chosen by AIC / BIC on
    the common sample, re-fitted on the longest sample of the chosen order; statistic = g / se(g)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    maxlag = min(int(math.ceil(12.0 * (n / 100.0) ** 0.25)), n // 2 - 2)
    dx = x[1:] - x[:-1]

    def design(p, first):
        # rows t = first .. n-2 (index into dx); columns: level x_t, dx_{t-1} .. dx_{t-p}, constant
        rows = range(first, len(dx))
        X = np.array([[x[t]] + [dx[t - j] for j in range(1, p + 1)] + [1.0] for t in rows])
        y = np.array([dx[t] for t in rows])
        return X, y

    def fit(X, y):
        beta, *_ = np.linalg.lstsq(X, y, rcond=None)
        r = y - X @ beta
        return beta, float(r @ r)

    if autolag is None:
        p_best = maxlag
    else:
        best = None
        for p in range(maxlag + 1):
            X, y = design(p, maxlag)
            _, ssr = fit(X, y)
            m, k = len(y), X.shape[1]
            loglik = -0.5 * m * (math.log(2.0 * math.pi) + math.log(ssr / m) + 1.0)
            crit = -2.0 * loglik + (2.0 * k if autolag == "AIC" else math.log(m) * k)
            if best is None or crit < best[0]:
                best = (crit, p)
        p_best = best[1]
    X, y = design(p_best, p_best)
    beta, ssr = fit(X, y)
    cov = np.linalg.inv(X.T @ X) * ssr / (len(y) - X.shape[1])
    return beta[0] / math.sqrt(cov[0, 0]), p_best


@pytest.mark.parametrize("kind", ["walk", "noise", "ar1", "trend"])
@pytest.mark.parametrize("n", [40, 256, 1024])
@pytest.mark.parametrize("autolag", ["AIC", "BIC", None])
def test_adfuller_restatement_against_an_independent_ols_route(kind, n, autolag):
    rng = np.random.default_rng(hash((kind, n)) % 2 ** 31)
    e = rng.standard_normal(n)
    if kind == "walk":
        x = e.cumsum()
    elif kind == "noise":
        x = e
    elif kind == "ar1":
        x = np.zeros(n)
        for t in range(1, n):
            x[t] = 0.7 * x[t - 1] + e[t]
    else:
        x = 0.05 * np.arange(n) + e
    stat, p, lag = tp.adfuller(x, autolag=autolag)
    stat2, lag2 = adf_lstsq(x, autolag)
    assert lag == lag2
    assert stat == pytest.approx(stat2, rel=1e-8, abs=1e-10)
    assert 0.0 <= p <= 1.0


def test_mackinnon_pvalues_reproduce_the_published_critical_values():
    # asymptotic critical values of the constant-only Dickey-Fuller distribution (Fuller 1976 / MacKinnon 1994/2010)
    for stat, level in ((-3.43, 0.01), (-2.86, 0.05), (-2.57, 0.10)):
        assert tp.mackinnonp_c(stat) == pytest.approx(level, rel=0.02)
    # monotone, continuous at the switch point of the two polynomials, saturating at the tabulated limits
    grid = np.linspace(-19.0, 3.0, 2201)
    p = np.array([tp.mackinnonp_c(s) for s in grid])
    assert (np.diff(p) >= -1e-12).all()
    assert abs(tp.mackinnonp_c(-1.61) - tp.mackinnonp_c(-1.61 + 1e-9)) < 1e-3
    assert tp.mackinnonp_c(-18.84) == 0.0 and tp.mackinnonp_c(2.75) == 1.0


@pytest.mark.parametrize("scale", [2, 5, 10, 20])
@pytest.mark.parametrize("kind", ["walk", "noise"])
def test_cwt_restatement_against_exact_integration_of_the_mexican_hat(scale, kind):
    rng = np.random.default_rng(scale)
    x = rng.standard_normal(300)
    if kind == "walk":
        x = x.cumsum()
    got = tp.cwt(x, [scale])[0][0]
    c = 2.0 / (math.sqrt(3.0) * math.pi ** 0.25)

    def antiderivative(u):                      # d/du [c u exp(-u^2/2)] = c (1 - u^2) exp(-u^2/2) = psi(u)
        return c * u * np.exp(-u * u / 2.0)

    n = len(x)
    b = np.arange(n)[:, None]
    k = np.arange(n)[None, :]
    # C(a, b) = 1/sqrt(a) * int x(t) psi((t - b) / a) dt with x(t) = x[k] on [k, k + 1)
    exact = (math.sqrt(scale) * (antiderivative((k + 1 - b) / scale) - antiderivative((k - b) / scale)) * x[None, :]).sum(axis=1)
    if kind == "walk":
        assert np.max(np.abs(exact - got)) < 0.02 * np.max(np.abs(got))
        # what tsfresh reads: coefficients 0..14 of each scale
        assert np.max(np.abs(exact[:15] - got[:15])) < 0.02 * np.max(np.abs(got))
    else:
        # white noise: pywt resamples its 1024-point integrated wavelet with floor() indices, a sub-sample jitter of the
        # kernel that a rough signal does not average out (up to ~18 % of the largest coefficient at scale 20); the two
        # transforms are still the same transform
        assert np.corrcoef(exact, got)[0, 1] > 0.98


# approximate_entropy: the oracle counts template matches over column blocks of the distance matrix, so that series of
# 21 000 samples need 32 MB instead of an N x N x m array of 10 GB.  The counts are integers and the maximum of the
# absolute differences is exact in any order, so the blocked form must equal the whole-array form bit for bit.
def _apen_inputs():
    rng = np.random.default_rng(11)
    out = [rng.standard_normal(n) for n in (1, 2, 3, 4, 5, 8, 33, 100, 257, 600)]
    out += [rng.standard_normal(600).cumsum(), np.round(rng.standard_normal(600) * 2) / 2,      # walk, many ties
            np.zeros(50), np.full(300, 3.25), np.array([-1.0, 1.0] * 150), np.arange(200, dtype=np.float64)]
    return [np.asarray(x, dtype=np.float32).astype(np.float64) for x in out]


@pytest.mark.parametrize("m,r", [(2, 0.1), (2, 0.3), (2, 0.5), (2, 0.7), (2, 0.9), (3, 0.2)])
def test_approximate_entropy_blocked_equals_whole_array(m, r):
    from oracle import calculators
    for x in _apen_inputs():
        whole = calculators.approximate_entropy_blocked(x, m, r, block_cols=None)
        for cols in (0, 1, 7, 64):
            got = calculators.approximate_entropy_blocked(x, m, r, block_cols=cols)
            assert got == whole or (np.isnan(got) and np.isnan(whole)), (len(x), cols, got, whole)
        assert calculators.approximate_entropy(x, m, r) == whole or np.isnan(whole)
