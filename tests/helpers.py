import multiprocessing as mp
import os
from fractions import Fraction

import numpy as np

from oracle.extract import compare, oracle_rows
from tsfresh_b200.plan import Plan


def cores():
    """CPUs this process may use (affinity, and the cgroup quota where one is set)"""
    n = len(os.sched_getaffinity(0))
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(round(int(quota) / int(period)))))
    except Exception:
        pass
    return max(1, n)


def _single_threaded(fn_args):
    for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS"):
        os.environ[k] = "1"
    fn, args = fn_args
    return fn(args)


def pool_map(fn, tasks):
    """[fn(t) for t in tasks] in a spawned process pool with single-threaded BLAS; fn must be importable"""
    with mp.get_context("spawn").Pool(cores()) as pool:
        return pool.map(_single_threaded, [(fn, t) for t in tasks], chunksize=1)


# ---------------------------------------------------------------------------------------------- exact cubic fit
def _solve_exact(M, b):
    """Gauss-Jordan on Fractions"""
    n = len(b)
    M = [list(row) + [bi] for row, bi in zip(M, b)]
    for c in range(n):
        p = next(r for r in range(c, n) if M[r][c] != 0)
        M[c], M[p] = M[p], M[c]
        for r in range(n):
            if r != c and M[r][c] != 0:
                f = M[r][c] / M[c][c]
                M[r] = [a - f * e for a, e in zip(M[r], M[c])]
    return [M[i][n] / M[i][i] for i in range(n)]


def exact_polyfit3(x, y):
    """np.polyfit(x, y, 3) in exact rational arithmetic on the float64 inputs (every float64 is a rational).  For k >= 4
    points the least-squares solution, which is unique; for k < 4 the minimum-norm solution in numpy's basis, the
    Vandermonde columns divided by their float64 2-norms S (the minimum-norm answer depends on that scaling).
    Returns (coefficients as Fractions, highest power first, S)."""
    x = np.asarray(x, np.float64)
    V = np.vander(x, 4)
    S = np.sqrt((V * V).sum(axis=0))
    X = [Fraction(v) for v in x]
    Y = [Fraction(v) for v in np.asarray(y, np.float64)]
    if len(X) >= 4:
        pw = [sum(xi ** m for xi in X) for m in range(7)]
        G = [[pw[6 - a - b] for b in range(4)] for a in range(4)]
        rhs = [sum(xi ** (3 - a) * yi for xi, yi in zip(X, Y)) for a in range(4)]
        return _solve_exact(G, rhs), S
    W = [1 / Fraction(s) ** 2 for s in S]
    P = [[xi ** (3 - j) for j in range(4)] for xi in X]
    H = [[sum(p[j] * q[j] * W[j] for j in range(4)) for q in P] for p in P]
    z = _solve_exact(H, Y)
    return [W[j] * sum(p[j] * zi for p, zi in zip(P, z)) for j in range(4)], S


POLYFIT_C = 64          # constant of the least-squares perturbation bound below


def polyfit3_bound(x, y, c_exact, S):
    """C * 2^-53 * (2 kappa / cos(theta) + kappa^2 tan(theta)): the relative error, in the column-scaled norm, that a
    backward-stable least-squares solver may make on these data.  kappa is the condition number of the column-scaled
    Vandermonde, theta the angle between y and its range.  0 when the exact fit is 0."""
    x = np.asarray(x, np.float64)
    sv = np.linalg.svd(np.vander(x, 4) / S, compute_uv=False)
    kappa = sv[0] / sv[-1]
    X = [Fraction(v) for v in x]
    fit = [sum(xi ** (3 - j) * c_exact[j] for j in range(4)) for xi in X]
    fn = np.sqrt(float(sum(f * f for f in fit)))
    if fn == 0.0:
        return 0.0
    rn = np.sqrt(float(sum((Fraction(v) - f) ** 2 for v, f in zip(np.asarray(y, np.float64), fit))))
    yn = np.hypot(fn, rn)
    return POLYFIT_C * 2.0 ** -53 * (2 * kappa * yn / fn + kappa ** 2 * rn / fn)


def polyfit3_error(got, c_exact, S):
    """||S (got - exact)|| / ||S exact|| (inf where the exact fit is 0 and got is not)"""
    ex = np.array([float(v) for v in c_exact])
    num = np.linalg.norm(S * (np.asarray(got, np.float64) - ex))
    den = np.linalg.norm(S * ex)
    return num / den if den > 0 else (0.0 if num == 0 else np.inf)


def polyfit3_accepts(got, x, y):
    """(accepted, relative error, bound, exact coefficients): the comparison rule for friedrich_coefficients, error
    within max(1e-5, the perturbation bound) of the exact fit"""
    c, S = exact_polyfit3(x, y)
    err = polyfit3_error(got, c, S)
    bound = polyfit3_bound(x, y, c, S)
    return err <= max(1e-5, bound), err, bound, c


def synthetic_series(seed, n_series, length, kind="normal"):
    rng = np.random.default_rng(seed)
    if kind == "normal":
        v = rng.standard_normal((n_series, length))
    elif kind == "walk":
        v = rng.standard_normal((n_series, length)).cumsum(axis=1)
    elif kind == "rounded":            # many ties / duplicates
        v = np.round(rng.standard_normal((n_series, length)) * 2) / 2
    else:
        raise ValueError(kind)
    return v.astype(np.float32)


def to_csr(series):
    lens = np.array([len(s) for s in series], dtype=np.int32)
    begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    values = np.concatenate([np.asarray(s, dtype=np.float32) for s in series]) if len(series) else np.zeros(0, np.float32)
    return values, begin, lens


def gpu_vs_oracle(ctx, settings, series, rtol=1e-5, atol=0.0):
    """Runs `settings` over the list of float32 series on the GPU (C-ABI, CSR path) and in the oracle;
    returns (mismatches, plan, gpu_matrix, oracle_matrix)."""
    from tsfresh_b200._lib import DevicePlan
    plan = Plan(settings)
    dp = DevicePlan(ctx, plan)
    try:
        values, begin, lens = to_csr(series)
        got = dp.extract_csr(values, begin, lens)
    finally:
        dp.close()
    want = oracle_rows([np.asarray(s, dtype=np.float32).astype(np.float64) for s in series], settings)
    return compare(got, want, plan.suffixes, rtol=rtol, atol=atol), plan, got, want
