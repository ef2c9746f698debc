// Host-side C shim over tsfresh_b200/csrc/tsfx_math.cuh so pytest (ctypes) can check the scalar
// routines the kernels' single-lane sections use.  Built by tests/test_host_math.py with g++.
#include "../../tsfresh_b200/csrc/tsfx_math.cuh"
using namespace tsfx;
extern "C" {
double hm_incbeta(double a, double b, double x) { return m_incbeta(a, b, x); }
double hm_student2(double t, double df) { return m_student_two_sided(t, df); }
double hm_mackinnon(double s) { return m_mackinnon_p_c(s); }
double hm_cubic(double a, double b, double c, double d) { return m_poly3_max_real_root(a, b, c, d); }
int hm_polyfit3(const double* x, const double* y, int k, double* c /*5*/) { return m_polyfit3(x, y, k, c) ? 1 : 0; }
void hm_levinson(const double* acv, int nlags, double* out, double* work) { m_levinson_pacf(acv, nlags, out, work); }
double hm_quantile(const double* s, int n, double q) { return m_quantile_sorted(s, n, q); }
void hm_linreg(double n, double xm, double ym, double sxx, double syy, double sxy, double* o) {
    LinReg r = m_linregress(n, xm, ym, sxx, syy, sxy);
    o[0] = m_linreg_pick(r, 0); o[1] = r.rvalue; o[2] = r.intercept; o[3] = r.slope; o[4] = r.stderr_;
}
int hm_cholesky_solve(double* A, int n, double* b) {
    if (!m_cholesky(A, n, n)) return 0;
    m_forward(A, n, n, b); m_backward(A, n, n, b); return 1;
}
}
