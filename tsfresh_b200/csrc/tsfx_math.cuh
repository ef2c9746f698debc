// tsfx_math.cuh -- scalar float64 routines used by single lanes inside the warp kernels.
// Plain C++ (compiles with g++ for the host-side unit test tests/test_host_math.py and with nvcc for
// the device).  Nothing here touches memory except through the pointers it is given.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define TSFX_HD __host__ __device__ __forceinline__
#define TSFX_HD_NOINLINE static __host__ __device__ __noinline__
#else
#define TSFX_HD inline
#define TSFX_HD_NOINLINE inline
#endif

namespace tsfx {

TSFX_HD double m_nan() {
#ifdef __CUDA_ARCH__
    return __longlong_as_double(0x7ff8000000000000LL);
#else
    return NAN;
#endif
}

// ------------------------------------------------------------------ regularised incomplete beta
// Continued fraction (modified Lentz) for I_x(a,b); relative accuracy ~1e-14.
TSFX_HD double m_betacf(double a, double b, double x) {
    const double TINY = 1e-300, EPS = 1e-16;
    double qab = a + b, qap = a + 1.0, qam = a - 1.0;
    double c = 1.0, d = 1.0 - qab * x / qap;
    if (fabs(d) < TINY) d = TINY;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= 400; ++m) {
        double m2 = 2.0 * m;
        double aa = m * (b - m) * x / ((qam + m2) * (a + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < TINY) d = TINY;
        c = 1.0 + aa / c;
        if (fabs(c) < TINY) c = TINY;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < TINY) d = TINY;
        c = 1.0 + aa / c;
        if (fabs(c) < TINY) c = TINY;
        d = 1.0 / d;
        double del = d * c;
        h *= del;
        if (fabs(del - 1.0) < EPS) break;
    }
    return h;
}

TSFX_HD double m_incbeta(double a, double b, double x) {
    if (!(x >= 0.0) || !(x <= 1.0)) return m_nan();
    if (x == 0.0) return 0.0;
    if (x == 1.0) return 1.0;
    double lbt = lgamma(a + b) - lgamma(a) - lgamma(b) + a * log(x) + b * log1p(-x);
    double bt = exp(lbt);
    if (x < (a + 1.0) / (a + b + 2.0)) return bt * m_betacf(a, b, x) / a;
    return 1.0 - bt * m_betacf(b, a, 1.0 - x) / b;
}

// 2 * stdtr(df, -|t|): the two-sided p-value scipy.stats.linregress reports (_stats_py.py linregress).
TSFX_HD_NOINLINE double m_student_two_sided(double t, double df) {
    if (!(df > 0.0) || t != t) return m_nan();
    double t2 = t * t;
    if (isinf(t2)) return 0.0;
    return m_incbeta(0.5 * df, 0.5, df / (df + t2));
}

TSFX_HD double m_norm_cdf(double z) { return 0.5 * erfc(-z * 0.70710678118654752440); }

// MacKinnon (1994) approximate p-value for the ADF statistic, regression "c", N=1
// (statsmodels.tsa.adfvalues.mackinnonp as called by adfuller; oracle/thirdparty.py mackinnonp_c).
TSFX_HD double m_mackinnon_p_c(double stat) {
    if (stat != stat) return m_nan();
    if (stat > 2.74) return 1.0;
    if (stat < -18.83) return 0.0;
    double z;
    if (stat <= -1.61) z = 2.1659 + stat * (1.4412 + stat * 3.8269e-2);
    else z = 1.7339 + stat * (9.3202e-1 + stat * (-1.2745e-1 + stat * (-1.0368e-2)));
    return m_norm_cdf(z);
}

// ------------------------------------------------------------------ linregress finishing step
struct LinReg { double rvalue, intercept, slope, stderr_, tstat, df; };

// scipy.stats.linregress from the averaged centred sums (ssxm, ssym, ssxym), the means and n.
TSFX_HD LinReg m_linregress(double n, double xmean, double ymean, double ssxm, double ssym, double ssxym) {
    LinReg R;
    if (n < 2.0) { R.rvalue = R.intercept = R.slope = R.stderr_ = R.tstat = m_nan(); R.df = n - 2.0; return R; }
    double r;
    if (ssxm == 0.0 || ssym == 0.0) r = (ssxym == 0.0) ? m_nan() : 0.0;
    else {
        r = ssxym / sqrt(ssxm * ssym);
        if (r > 1.0) r = 1.0;
        if (r < -1.0) r = -1.0;
    }
    R.rvalue = r;
    R.slope = ssxym / ssxm;
    R.intercept = ymean - R.slope * xmean;
    double df = n - 2.0;
    double t = r * sqrt(df / ((1.0 - r + 1e-20) * (1.0 + r + 1e-20)));
    R.tstat = t;          // the p-value (an incomplete-beta evaluation) is formed only when asked for
    R.df = df;
    // df == 0 (two points): r is +-1 up to rounding, so scipy's (1 - r^2) * ssym / ssxm / 0 is 0/0 = NaN
    // or tiny/0 = inf depending on the last bit of r; the mathematically exact value is returned here.
    R.stderr_ = (df == 0.0) ? m_nan() : sqrt((1.0 - r * r) * ssym / ssxm / df);
    return R;
}

TSFX_HD double m_linreg_pick(const LinReg& R, int attr) {
    switch (attr) {
        case 0: return m_student_two_sided(R.tstat, R.df);
        case 1: return R.rvalue;
        case 2: return R.intercept;
        case 3: return R.slope;
        default: return R.stderr_;
    }
}

// intercept_stderr of the same fit (scipy: slope_stderr * sqrt(ssxm + xmean^2)); the callers pick it before
// m_linreg_pick, whose LinReg does not carry the regressor's moments
TSFX_HD double m_intercept_stderr(double slope_stderr, double xmean, double ssxm) {
    return slope_stderr * sqrt(ssxm + xmean * xmean);
}

// ------------------------------------------------------------------ dense SPD solves (row-major, lda)
// In-place lower Cholesky of the leading n x n block.  Returns false on a non-positive pivot.
TSFX_HD bool m_cholesky(double* A, int n, int lda) {
    for (int j = 0; j < n; ++j) {
        double d = A[j * lda + j];
        for (int k = 0; k < j; ++k) d -= A[j * lda + k] * A[j * lda + k];
        if (!(d > 0.0)) return false;
        d = sqrt(d);
        A[j * lda + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[i * lda + j];
            for (int k = 0; k < j; ++k) s -= A[i * lda + k] * A[j * lda + k];
            A[i * lda + j] = s / d;
        }
    }
    return true;
}
// forward substitution L z = b (in place in b)
TSFX_HD void m_forward(const double* L, int n, int lda, double* b) {
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= L[i * lda + k] * b[k];
        b[i] = s / L[i * lda + i];
    }
}
// back substitution L^T x = z (in place)
TSFX_HD void m_backward(const double* L, int n, int lda, double* b) {
    for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int k = i + 1; k < n; ++k) s -= L[k * lda + i] * b[k];
        b[i] = s / L[i * lda + i];
    }
}

// ------------------------------------------------------------------ Levinson-Durbin partial autocorrelation
// acv[0..nlags] autocovariances; out[0..nlags] = pacf (out[0] = 1).  work: 2*(nlags+1) doubles.
// (statsmodels levinson_durbin(..., isacov=True)[2]; oracle/thirdparty.py levinson_durbin_pacf)
TSFX_HD void m_levinson_pacf(const double* acv, int nlags, double* out, double* work) {
    double* prev = work;
    double* cur = work + (nlags + 1);
    out[0] = 1.0;
    if (nlags < 1) return;
    double phi = acv[1] / acv[0];
    double sig = acv[0] - phi * acv[1];
    prev[1] = phi;
    out[1] = phi;
    for (int k = 2; k <= nlags; ++k) {
        double num = acv[k];
        for (int j = 1; j < k; ++j) num -= prev[j] * acv[k - j];
        double pk = num / sig;
        for (int j = 1; j < k; ++j) cur[j] = prev[j] - pk * prev[k - j];
        cur[k] = pk;
        sig = sig * (1.0 - pk * pk);
        out[k] = pk;
        for (int j = 1; j <= k; ++j) prev[j] = cur[j];
    }
}

// ------------------------------------------------------------------ cubic: largest real part of the roots
// np.max(np.real(np.roots([c0,c1,c2,c3]))) (feature_calculators.py:2163): leading zeros are stripped,
// trailing zeros contribute roots at 0.
TSFX_HD double m_quadratic_max_real(double a, double b, double c) {
    double disc = b * b - 4.0 * a * c;
    if (disc < 0.0) return -b / (2.0 * a);
    double q = -0.5 * (b + (b >= 0.0 ? 1.0 : -1.0) * sqrt(disc));
    double r1 = q / a, r2 = (q != 0.0) ? c / q : -b / a - r1;
    return r1 > r2 ? r1 : r2;
}

TSFX_HD double m_poly3_max_real_root(double c0, double c1, double c2, double c3) {
    if (c0 != c0 || c1 != c1 || c2 != c2 || c3 != c3) return m_nan();
    if (isinf(c0) || isinf(c1) || isinf(c2) || isinf(c3)) return m_nan();
    // strip leading zeros
    if (c0 == 0.0) {
        if (c1 == 0.0) {
            if (c2 == 0.0) return m_nan();          // np.roots -> [] -> np.max raises ValueError -> NaN
            return -c3 / c2;
        }
        if (c3 == 0.0) {                             // roots: 0 and -c2/c1
            double r = -c2 / c1;
            return r > 0.0 ? r : 0.0;
        }
        return m_quadratic_max_real(c1, c2, c3);
    }
    double a = c1 / c0, b = c2 / c0, c = c3 / c0;
    // depressed cubic t^3 + p t + q, x = t - a/3
    double a3 = a / 3.0;
    double p = b - a * a3;
    double q = 2.0 * a3 * a3 * a3 - a3 * b + c;
    double disc = 0.25 * q * q + p * p * p / 27.0;
    double best;
    if (disc > 0.0) {               // one real root r, complex pair with real part -(r_t)/2
        double sq = sqrt(disc);
        double u = cbrt(-0.5 * q + sq), v = cbrt(-0.5 * q - sq);
        double t = u + v;
        // polish the real root with Newton on the original cubic
        double x = t - a3;
        for (int it = 0; it < 3; ++it) {
            double f = ((x + a) * x + b) * x + c;
            double fp = (3.0 * x + 2.0 * a) * x + b;
            if (fp != 0.0) x -= f / fp;
        }
        double pair_re = -0.5 * (x + a);            // sum of roots = -a
        best = x > pair_re ? x : pair_re;
    } else {                        // three real roots
        double m = 2.0 * sqrt(-p / 3.0);
        double arg = (p != 0.0) ? (3.0 * q / (p * m)) : 0.0;
        if (arg > 1.0) arg = 1.0;
        if (arg < -1.0) arg = -1.0;
        double th = acos(arg) / 3.0;
        double x = m * cos(th) - a3;                 // k = 0 gives the largest root
        for (int it = 0; it < 3; ++it) {
            double f = ((x + a) * x + b) * x + c;
            double fp = (3.0 * x + 2.0 * a) * x + b;
            if (fp != 0.0) x -= f / fp;
        }
        best = x;
    }
    return best;
}

// ------------------------------------------------------------------ cubic least squares (np.polyfit deg 3)
// np.polyfit(x, y, 3) scales the Vandermonde columns [x^3, x^2, x, 1] to unit 2-norm and solves by least squares,
// minimum-norm when k < 4.  For k >= 4 the answer is unique, so it is computed in the centred variable
// u = (x - mu) / h, mu and h the midpoint and half-width of the points' range: the scaled Vandermonde of u in [-1, 1] is
// well conditioned whatever the level of x, while that of raw x has a condition number growing like (level/spread)^3,
// which normal equations would square (NaN or wrong coefficients for series hovering around 300).  The fit in u is then
// expanded to monomial coefficients of x.  For k < 4 the minimum-norm solution depends on the basis, so it stays in
// numpy's column-scaled monomial basis, solved by a Householder LQ of the k x 4 matrix.

// mu, h of the centred variable for points in [lo, hi]; false when they do not span a positive, finite range
TSFX_HD bool m_cubic_centre(double lo, double hi, double* mu, double* h) {
    *mu = 0.5 * lo + 0.5 * hi;
    *h = 0.5 * hi - 0.5 * lo;
    return *h > 0.0 && *h < INFINITY && *mu == *mu;
}

// column-scaled centred basis [u^3, u^2, u, 1] / sc
TSFX_HD void m_cubic_cols(double u, const double* sc, double* col) {
    const double u2 = u * u;
    col[0] = u2 * u / sc[0]; col[1] = u2 / sc[1]; col[2] = u / sc[2]; col[3] = 1.0 / sc[3];
}

// a[0..3]: coefficients of u^3 .. u^0.  coef[0..3] = monomial coefficients of x (np.polyfit order), coef[4] =
// np.max(np.real(np.roots(coef[0..3]))) taken as mu + h * (largest real part of the u-cubic's roots): x -> u is
// increasing and affine, and leading zeros of the two coefficient vectors coincide.
TSFX_HD void m_cubic_from_centred(const double* a, double mu, double h, double* coef /*5*/) {
    double b[4];
    double hp = 1.0;
    for (int j = 3; j >= 0; --j) { b[j] = a[j] / hp; hp *= h; }   // polynomial in d = x - mu
    for (int i = 0; i < 3; ++i)                                    // Taylor shift: q(x - mu) by synthetic division
        for (int j = 1; j < 4 - i; ++j) b[j] -= mu * b[j - 1];
    for (int j = 0; j < 4; ++j) coef[j] = b[j];
    coef[4] = mu + h * m_poly3_max_real_root(a[0], a[1], a[2], a[3]);
}

TSFX_HD bool m_coef_finite(const double* coef) {
    for (int c = 0; c < 4; ++c)
        if (!(fabs(coef[c]) < INFINITY)) return false;
    return true;
}

// k < 4 points: A = [L 0] H_{k-1} .. H_0 with Householder reflections H_i acting on columns i..3 from the right; the
// minimum-norm solution of A w = y is w = H_0 .. H_{k-1} [L^-1 y; 0].  Outputs as m_polyfit3.
TSFX_HD_NOINLINE bool m_polyfit3_minnorm(const double* x, const double* y, int k, double* coef /*5*/) {
    if (k <= 0 || k >= 4) return false;
    double S[4] = {0, 0, 0, 0};
    for (int i = 0; i < k; ++i) {
        const double v = x[i], v2 = v * v, v3 = v2 * v;
        S[0] += v3 * v3; S[1] += v2 * v2; S[2] += v * v; S[3] += 1.0;
    }
    for (int j = 0; j < 4; ++j) S[j] = sqrt(S[j]);
    double A[12], V[12], tau[3], w[4] = {0, 0, 0, 0};
    for (int i = 0; i < k; ++i) {
        const double v = x[i];
        A[i * 4 + 0] = v * v * v / S[0]; A[i * 4 + 1] = v * v / S[1];
        A[i * 4 + 2] = v / S[2];         A[i * 4 + 3] = 1.0 / S[3];
    }
    for (int i = 0; i < k; ++i) {
        double nrm = 0.0;
        for (int c = i; c < 4; ++c) nrm += A[i * 4 + c] * A[i * 4 + c];
        nrm = sqrt(nrm);
        const double alpha = A[i * 4 + i] >= 0.0 ? -nrm : nrm;
        double vv = 0.0;
        for (int c = i; c < 4; ++c) { V[i * 4 + c] = A[i * 4 + c] - (c == i ? alpha : 0.0); vv += V[i * 4 + c] * V[i * 4 + c]; }
        tau[i] = vv > 0.0 ? 2.0 / vv : 0.0;
        for (int r = i; r < k; ++r) {
            double s = 0.0;
            for (int c = i; c < 4; ++c) s += A[r * 4 + c] * V[i * 4 + c];
            s *= tau[i];
            for (int c = i; c < 4; ++c) A[r * 4 + c] -= s * V[i * 4 + c];
        }
    }
    for (int i = 0; i < k; ++i) {                 // L z = y; L[i][i] = alpha_i
        double s = y[i];
        for (int m = 0; m < i; ++m) s -= A[i * 4 + m] * w[m];
        w[i] = s / A[i * 4 + i];
    }
    for (int i = k - 1; i >= 0; --i) {
        double s = 0.0;
        for (int c = i; c < 4; ++c) s += V[i * 4 + c] * w[c];
        s *= tau[i];
        for (int c = i; c < 4; ++c) w[c] -= s * V[i * 4 + c];
    }
    for (int c = 0; c < 4; ++c) coef[c] = w[c] / S[c];
    coef[4] = m_poly3_max_real_root(coef[0], coef[1], coef[2], coef[3]);
    return m_coef_finite(coef);
}

// Fits the cubic to k points (any order, x, y not modified).  coef[0..3] as np.polyfit(x, y, 3), coef[4] the largest
// real part of its roots (max_langevin_fixed_point).  Returns false when the data are not finite or the fit is singular.
TSFX_HD bool m_polyfit3(const double* x, const double* y, int k, double* coef /*5*/) {
    if (k < 4) return m_polyfit3_minnorm(x, y, k, coef);
    {
        double lo = x[0], hi = x[0];
        for (int i = 1; i < k; ++i) { lo = fmin(lo, x[i]); hi = fmax(hi, x[i]); }
        double mu, h;
        if (!m_cubic_centre(lo, hi, &mu, &h)) return false;
        const double ih = 1.0 / h;
        double sc[4] = {0, 0, 0, 0};
        for (int i = 0; i < k; ++i) {
            const double u = (x[i] - mu) * ih, u2 = u * u, u3 = u2 * u;
            sc[0] += u3 * u3; sc[1] += u2 * u2; sc[2] += u * u; sc[3] += 1.0;
        }
        for (int j = 0; j < 4; ++j) sc[j] = sqrt(sc[j]);
        // normal equations of the scaled centred columns (condition number of G below ~1e4 for k >= 4 distinct points
        // spread over [-1, 1]), Cholesky, two refinement steps with residuals formed from the data
        double L[16], sol[4];
        for (int a = 0; a < 16; ++a) L[a] = 0.0;
        for (int a = 0; a < 4; ++a) sol[a] = 0.0;
        for (int i = 0; i < k; ++i) {
            double col[4];
            m_cubic_cols((x[i] - mu) * ih, sc, col);
            for (int a = 0; a < 4; ++a) {
                sol[a] += col[a] * y[i];
                for (int b = 0; b <= a; ++b) L[a * 4 + b] += col[a] * col[b];
            }
        }
        if (!m_cholesky(L, 4, 4)) return false;
        m_forward(L, 4, 4, sol);
        m_backward(L, 4, 4, sol);
        for (int it = 0; it < 2; ++it) {
            double r[4] = {0, 0, 0, 0};
            for (int i = 0; i < k; ++i) {
                double col[4];
                m_cubic_cols((x[i] - mu) * ih, sc, col);
                const double e = y[i] - (col[0] * sol[0] + col[1] * sol[1] + col[2] * sol[2] + col[3] * sol[3]);
                for (int a = 0; a < 4; ++a) r[a] += col[a] * e;
            }
            m_forward(L, 4, 4, r);
            m_backward(L, 4, 4, r);
            for (int a = 0; a < 4; ++a) sol[a] += r[a];
        }
        for (int a = 0; a < 4; ++a) sol[a] /= sc[a];
        m_cubic_from_centred(sol, mu, h, coef);
    }
    return m_coef_finite(coef);
}

// ------------------------------------------------------------------ numpy linear quantile on a sorted array
// np.quantile(method="linear") incl. numpy's two-sided lerp (a + (b-a)*t for t < 0.5, b - (b-a)*(1-t) else).
template <typename T>
TSFX_HD double m_quantile_sorted(const T* s, int n, double q) {
    double pos = q * (double)(n - 1);
    double fl = floor(pos);
    int lo = (int)fl;
    if (lo < 0) lo = 0;
    if (lo > n - 1) lo = n - 1;
    int hi = lo + 1 > n - 1 ? n - 1 : lo + 1;
    double t = pos - fl;
    double a = (double)s[lo], b = (double)s[hi];
    double d = b - a;
    if (t >= 0.5) return b - d * (1.0 - t);
    return a + d * t;
}

}  // namespace tsfx
