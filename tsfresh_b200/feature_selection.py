"""Feature selection on the feature matrix -- the step after the hot path (SURVEY.md section 8f row 4).

Mirrors tsfresh/feature_selection/relevance.py:31-322 (`calculate_relevance_table`, `combine_relevance_tables`,
`infer_ml_task`, `get_feature_type`) and selection.py:17-200 (`select_features`) for CLASSIFICATION targets (binary and
multiclass): same arguments, same relevance table (index / columns / order / dtypes), same decisions.

The reference runs one scipy test per feature column in a Python loop (783 calls per class label, each sorting the column on
the CPU).  Here every column of the matrix is sorted ONCE on the GPU and the sufficient statistics of all tests come out of
one pass over the sorted column (tsfx_select_classification, csrc/tsfx_select.cu):

  real feature,   target binary:  Mann-Whitney U + tie term  (significance_tests.py:84-132, scipy.stats.mannwhitneyu)
                                  or the two-sample Kolmogorov-Smirnov statistic ('smir', scipy.stats.ks_2samp)
  binary feature, target binary:  the 2 x 2 contingency table  (significance_tests.py:43-81, scipy.stats.fisher_exact)

What is left for the host is O(n_features): the p-value of each statistic (the closed forms scipy itself evaluates: normal
tail with continuity and tie correction / exact U distribution for tiny untied samples, hypergeometric tail, Kolmogorov
distributions) and the Benjamini-Hochberg / Benjamini-Yekutieli step-up decision (statsmodels.stats.multitest.multipletests
in the reference, relevance.py:347-351).

REGRESSION targets (relevance.py:282-296) take tsfx_select_regression: real features need Kendall's tau -- the rows are
brought into (x, rank(y)) order by two stable device sorts, the discordant pairs are the strict inversions of the rank
sequence (bottom-up merge, one kernel per level), tie sums come from the runs; binary features need the two-sample KS of
the target between their two groups (one pass over the y-sorted rows).

A feature matrix already on the GPU (extract_features_device) takes calculate_relevance_table_device /
select_features_device: the library reads the CUDA tensor in place (TSFX_FLAG_DEVICE_PTRS) instead of staging a host
copy, and the same host code turns the statistics into the table (_relevance_table).
"""
import contextlib
import math
import warnings
from functools import reduce

import numpy as np
import pandas as pd

from . import _lib
from .extraction import N_PROCESSES, get_context

TEST_FOR_BINARY_TARGET_BINARY_FEATURE = "fisher"        # tsfresh/defaults.py:15-20
TEST_FOR_BINARY_TARGET_REAL_FEATURE = "mann"
TEST_FOR_REAL_TARGET_BINARY_FEATURE = "mann"
TEST_FOR_REAL_TARGET_REAL_FEATURE = "kendall"
FDR_LEVEL = 0.05
HYPOTHESES_INDEPENDENT = False


# ------------------------------------------------------------------------------------------ p-values from statistics
def _norm_sf(z):
    return 0.5 * math.erfc(z / math.sqrt(2.0))


def _mwu_exact_sf(k, n1, n2):
    """P(U >= k) for the Mann-Whitney U of a sample of n1 against n2 without ties: coefficients of the Gaussian binomial
    prod_{i=1..n1} (1 - q^(n2+i)) / (1 - q^i) (what scipy's _MWU tabulates)."""
    n1, n2 = int(n1), int(n2)
    if n1 > n2:
        n1, n2 = n2, n1
    size = n1 * n2 + 1
    c = np.zeros(size, dtype=np.float64)
    c[0] = 1.0
    for i in range(1, n1 + 1):
        num = n2 + i
        if num < size:                               # multiply by (1 - q^num)
            c[num:] -= c[:-num].copy()
        for u in range(i, size):                     # divide by (1 - q^i)
            c[u] += c[u - i]
    total = c.sum()
    k = max(0, int(k))
    return float(c[k:].sum() / total) if k < size else 0.0


def mannwhitneyu_pvalue(U1, n1, n2, tie_term, distinct):
    """scipy.stats.mannwhitneyu(x_y1, x_y0, use_continuity=True, alternative="two-sided") p-value from its statistics
    (method="auto": exact for a sample of <= 8 without ties, else the normal approximation with tie correction)."""
    if n1 == 0 or n2 == 0:
        raise ValueError("`x` and `y` must be of nonzero size.")
    n = n1 + n2
    ties = distinct < n
    if (n1 <= 8 or n2 <= 8) and not ties:
        U = max(U1, n1 * n2 - U1)
        return float(min(1.0, max(0.0, 2.0 * _mwu_exact_sf(int(U), n1, n2))))
    mu = n1 * n2 / 2.0
    with np.errstate(all="ignore"):
        s = math.sqrt(n1 * n2 / 12.0 * ((n + 1) - tie_term / (n * (n - 1.0))))
        num = U1 - mu
        num -= 0.5 * np.sign(num)
        z = num / s if s != 0 else (math.nan if num == 0 else math.copysign(math.inf, num))
    if z != z:
        return math.nan
    return float(min(1.0, max(0.0, 2.0 * _norm_sf(abs(z)))))


def ks_2samp_pvalue(d, n1, n2):
    """scipy.stats.ks_2samp(..., alternative="two-sided", method="auto") p-value from the statistic: exact for samples of
    at most 10 000 rows (scipy's lattice-path count), else the asymptotic Kolmogorov distribution."""
    from scipy import stats
    n1, n2 = int(n1), int(n2)
    g = math.gcd(n1, n2)
    if max(n1, n2) <= 10000:
        try:
            from scipy.stats._stats_py import _attempt_exact_2kssamp
            ok, d2, prob = _attempt_exact_2kssamp(n1, n2, g, d, "two-sided")
            if ok:
                return float(np.clip(prob, 0, 1))
        except Exception:
            pass
    m, n = sorted([float(n1), float(n2)], reverse=True)
    en = m * n / (m + n)
    return float(np.clip(stats.distributions.kstwo.sf(d, np.round(en)), 0, 1))


def kendall_pvalue(n, dis, xtie, x0, x1, ntie, ytie, y0, y1):
    """scipy.stats.kendalltau(x, y, method="asymptotic").pvalue (tau-b) from its sufficient statistics: discordant pairs,
    the tie sums sum t(t-1)/2, sum t(t-1)(t-2), sum t(t-1)(2t+5) of x and y and the joint ties (scipy _stats_py.py)."""
    tot = n * (n - 1) // 2
    if xtie == tot or ytie == tot:
        return math.nan
    con_minus_dis = tot - xtie - ytie + ntie - 2 * dis
    m = n * (n - 1.0)
    var = (m * (2 * n + 5) - x1 - y1) / 18 + (2 * xtie * ytie) / m + x0 * y0 / (9 * m * (n - 2))
    z = con_minus_dis / math.sqrt(var)
    return math.erfc(abs(z) / math.sqrt(2.0))


def fisher_pvalue(n_y1_x1, n_y1_x0, n_y0_x1, n_y0_x0):
    from scipy import stats
    table = np.array([[n_y1_x1, n_y1_x0], [n_y0_x1, n_y0_x0]], dtype=np.int64)
    return float(stats.fisher_exact(table, alternative="two-sided")[1])


def benjamini_reject(pvals, alpha, independent):
    """statsmodels.stats.multitest.multipletests(pvals, alpha, "fdr_bh" | "fdr_by")[0] (relevance.py:347-351): the
    Benjamini-Hochberg step-up procedure; for arbitrary dependence the thresholds are divided by sum(1 / i)."""
    p = np.asarray(pvals, dtype=np.float64)
    m = len(p)
    if m == 0:
        return np.zeros(0, dtype=bool)
    order = np.argsort(p)
    ps = p[order]
    factor = np.arange(1, m + 1) / float(m)
    if not independent:
        factor = factor / np.sum(1.0 / np.arange(1, m + 1))
    reject = ps <= factor * alpha
    if reject.any():
        reject[:np.max(np.nonzero(reject)[0]) + 1] = True
    out = np.empty(m, dtype=bool)
    out[order] = reject
    return out


# ------------------------------------------------------------------------------------------ reference API
def infer_ml_task(y):
    """relevance.py:354-375"""
    if y.dtype.kind in np.typecodes["AllInteger"] or y.dtype == object or isinstance(y.dtype, pd.StringDtype):
        return "classification"
    return "regression"


def get_feature_type(feature_column):
    """relevance.py:398-414 (one column; calculate_relevance_table types all columns on the device)"""
    n_unique_values = len(set(np.asarray(feature_column)))
    return "constant" if n_unique_values == 1 else ("binary" if n_unique_values == 2 else "real")


def combine_relevance_tables(relevance_tables):
    """relevance.py:378-395"""
    def _combine(a, b):
        a.relevant |= b.relevant
        a.p_value = a.p_value.combine(b.p_value, min, 1)
        return a
    return reduce(_combine, relevance_tables)


def _table_for_label(features, types, stats, test_real, fdr_level, hypotheses_independent):
    """relevance.py:325-351 for one implicit binary target, from the device statistics [n_features, 8]"""
    real = [i for i, t in enumerate(types) if t == "real"]
    binary = [i for i, t in enumerate(types) if t == "binary"]
    p = {}
    for i in real:
        s = stats[i]
        if test_real == "mann":
            p[i] = mannwhitneyu_pvalue(s[3], s[1], s[2], s[4], s[6])
        elif test_real == "smir":
            p[i] = ks_2samp_pvalue(s[5], s[1], s[2])
        else:
            raise ValueError("Please use a valid entry for test_for_binary_target_real_feature. "
                             "Valid entries are 'mann' and 'smir'.")
    for i in binary:
        s = stats[i]
        p[i] = fisher_pvalue(int(s[3]), int(s[4]), int(s[5]), int(s[6]))
    idx = real + binary                                   # pd.concat([table_real, table_binary])
    table = pd.DataFrame({"feature": [features[i] for i in idx], "type": [types[i] for i in idx],
                          "p_value": [p[i] for i in idx]}, index=pd.Index([features[i] for i in idx], name="feature"))
    table["relevant"] = benjamini_reject(table.p_value.to_numpy(), fdr_level, hypotheses_independent)
    return table.sort_values("p_value")


def calculate_relevance_table(X, y, ml_task="auto", multiclass=False, n_significant=1, n_jobs=N_PROCESSES, show_warnings=False,
                              chunksize=None, test_for_binary_target_binary_feature=TEST_FOR_BINARY_TARGET_BINARY_FEATURE,
                              test_for_binary_target_real_feature=TEST_FOR_BINARY_TARGET_REAL_FEATURE,
                              test_for_real_target_binary_feature=TEST_FOR_REAL_TARGET_BINARY_FEATURE,
                              test_for_real_target_real_feature=TEST_FOR_REAL_TARGET_REAL_FEATURE, fdr_level=FDR_LEVEL,
                              hypotheses_independent=HYPOTHESES_INDEPENDENT, device=None):
    """GPU implementation of tsfresh.feature_selection.relevance.calculate_relevance_table (relevance.py:31-322)."""
    y = y.sort_index()
    X = X.sort_index()
    assert list(y.index) == list(X.index), "The index of X and y need to be the same"

    def host_matrix():                   # the library copies it to the device (the context's selection scratch)
        return np.ascontiguousarray(X.to_numpy(dtype=np.float64))
    return _relevance_table(
        list(X.columns), y, lambda codes, k: get_context(device).select_classification(host_matrix(), codes, k),
        lambda yv: get_context(device).select_regression(host_matrix(), yv), ml_task, multiclass, n_significant,
        show_warnings, test_for_binary_target_real_feature, fdr_level, hypotheses_independent)


def _relevance_table(features, y, class_stats, regression_stats, ml_task, multiclass, n_significant, show_warnings,
                     test_for_binary_target_real_feature, fdr_level, hypotheses_independent):
    """relevance.py:172-322 from the sufficient statistics of the feature matrix, whose columns are `features` and
    whose rows are the positions of the host Series `y`.  The matrix is only read through the two callables, called
    after every argument check: class_stats(int32 codes, n_labels) -> [n_labels, n_features, 8] and
    regression_stats(float64 y) -> ([n_features, 8], (ytie, y0, y1, n)), raising a ValueError that mentions NaN for a
    NaN in the matrix."""
    if ml_task not in ["auto", "classification", "regression"]:
        raise ValueError("ml_task must be one of: 'auto', 'classification', 'regression'")
    elif ml_task == "auto":
        ml_task = infer_ml_task(y)
    if multiclass:
        assert ml_task == "classification", "ml_task must be classification for multiclass problem"
        assert len(y.unique()) >= n_significant, "n_significant must not exceed the total number of classes"
        if len(y.unique()) <= 2:
            warnings.warn("Two or fewer classes, binary feature selection will be used (multiclass = False)")
            multiclass = False

    with warnings.catch_warnings():
        warnings.simplefilter("default" if show_warnings else "ignore")
        try:
            if ml_task == "classification":
                labels = list(y.unique())                # order of appearance, as the reference's loop (relevance.py:248)
                codes = pd.Categorical(y, categories=labels).codes.astype(np.int32)
                stats = class_stats(codes, len(labels))                   # [n_labels, n_features, 8]
                type_col = stats[0, :, 0]
            else:
                yv = np.ascontiguousarray(y.to_numpy(dtype=np.float64))
                if np.isnan(yv).any():
                    raise ValueError("Target y contains NaN values")
                rstats, ytail = regression_stats(yv)                         # [n_features, 8], (ytie, y0, y1, n)
                type_col = rstats[:, 0]
        except ValueError as e:
            if "NaN" in str(e) and "Target" not in str(e):
                raise ValueError("Feature {} contains NaN values".format("matrix")) from None
            raise
        type_names = {0: "constant", 1: "binary", 2: "real"}
        types = [type_names[int(t)] for t in type_col]
        const = [i for i, t in enumerate(types) if t == "constant"]
        table_const = pd.DataFrame({"feature": [features[i] for i in const], "type": ["constant"] * len(const)},
                                   index=pd.Index([features[i] for i in const], name="feature"))
        table_const["p_value"] = np.nan
        table_const["relevant"] = False
        if not table_const.empty:
            warnings.warn("[test_feature_significance] Constant features: {}".format(", ".join(map(str, table_const.feature))),
                          RuntimeWarning)
        if len(table_const) == len(features):
            return table_const

        if ml_task == "regression":
            # relevance.py:282-296: Kendall's tau for real features, two-sample KS of the target for binary ones
            n = int(ytail[3])
            real = [i for i, t in enumerate(types) if t == "real"]
            binary = [i for i, t in enumerate(types) if t == "binary"]
            p = {}
            for i in real:
                s_ = rstats[i]
                p[i] = kendall_pvalue(n, int(s_[2]), int(s_[3]), s_[4], s_[5], int(s_[6]), int(ytail[0]), ytail[1], ytail[2])
            for i in binary:
                s_ = rstats[i]
                p[i] = ks_2samp_pvalue(s_[2], s_[3], s_[4])
            idx = real + binary
            relevance_table = pd.DataFrame({"feature": [features[i] for i in idx], "type": [types[i] for i in idx],
                                            "p_value": [p[i] for i in idx]}, index=pd.Index([features[i] for i in idx], name="feature"))
            relevance_table["relevant"] = benjamini_reject(relevance_table.p_value.to_numpy(), fdr_level, hypotheses_independent)
            relevance_table = relevance_table.sort_values("p_value")
            labels = []
        tables = []
        for k, label in enumerate(labels):
            tmp = _table_for_label(features, types, stats[k], test_for_binary_target_real_feature, fdr_level,
                                   hypotheses_independent)
            if multiclass:
                tmp = tmp.reset_index(drop=True)
                tmp.columns = tmp.columns.map(lambda x: (x + "_" + str(label) if x != "feature" and x != "type" else x))
            tables.append(tmp)
        if ml_task == "regression":
            pass
        elif multiclass:
            relevance_table = reduce(lambda left, right: pd.merge(left, right, on=["feature", "type"], how="outer"), tables)
            relevance_table["n_significant"] = relevance_table.filter(regex="^relevant_", axis=1).sum(axis=1)
            relevance_table["relevant"] = relevance_table["n_significant"] >= n_significant
            relevance_table.index = relevance_table["feature"]
        else:
            relevance_table = combine_relevance_tables(tables)

        if multiclass:
            for column in relevance_table.filter(regex="^relevant_", axis=1).columns:
                table_const[column] = False
            table_const["n_significant"] = 0
            table_const.drop(columns=["p_value"], inplace=True)
        relevance_table = pd.concat([relevance_table, table_const], axis=0)
        if sum(relevance_table["relevant"]) == 0:
            warnings.warn("No feature was found relevant for {} for fdr level = {} (which corresponds to the maximal percentage "
                          "of irrelevant features, consider using an higher fdr level or add other features."
                          .format(ml_task, fdr_level), RuntimeWarning)
    return relevance_table


def select_features(X, y, test_for_binary_target_binary_feature=TEST_FOR_BINARY_TARGET_BINARY_FEATURE,
                    test_for_binary_target_real_feature=TEST_FOR_BINARY_TARGET_REAL_FEATURE,
                    test_for_real_target_binary_feature=TEST_FOR_REAL_TARGET_BINARY_FEATURE,
                    test_for_real_target_real_feature=TEST_FOR_REAL_TARGET_REAL_FEATURE, fdr_level=FDR_LEVEL,
                    hypotheses_independent=HYPOTHESES_INDEPENDENT, n_jobs=N_PROCESSES, show_warnings=False, chunksize=None,
                    ml_task="auto", multiclass=False, n_significant=1, device=None):
    """GPU implementation of tsfresh.feature_selection.selection.select_features (selection.py:17-200)."""
    assert isinstance(X, pd.DataFrame), "Please pass features in X as pandas.DataFrame."
    assert isinstance(y, (pd.Series, np.ndarray)), "The type of target vector y must be one of: pandas.Series, numpy.ndarray"
    assert len(y) > 1, "y must contain at least two samples."
    assert len(X) == len(y), "X and y must contain the same number of samples."
    assert len(set(y)) > 1, "Feature selection is only possible if more than 1 label/class is provided"
    if isinstance(y, pd.Series) and set(X.index) != set(y.index):
        raise ValueError("Index of X and y must be identical if provided")
    if isinstance(y, np.ndarray):
        y = pd.Series(y, index=X.index)
    relevance_table = calculate_relevance_table(
        X, y, ml_task=ml_task, multiclass=multiclass, n_significant=n_significant, n_jobs=n_jobs, show_warnings=show_warnings,
        chunksize=chunksize, test_for_binary_target_real_feature=test_for_binary_target_real_feature, fdr_level=fdr_level,
        hypotheses_independent=hypotheses_independent, device=device)
    relevant_features = relevance_table[relevance_table.relevant].feature
    return X.loc[:, relevant_features]


# ------------------------------------------------------------------------------------------ feature matrices on the GPU
def _device_args(X, y, columns):
    """The checks of a CUDA matrix's arguments that need no device, and ONE host copy of the targets: a Series with a
    RangeIndex, because X has no index and y is taken positionally (a Series is not aligned by its index).
    That X is on a CUDA device is checked where the matrix is first read (_bound_context), after the checks of the
    target and of ml_task / multiclass the DataFrame path makes, so those errors read the same on any tensor and are
    tested without a device."""
    import torch
    if not isinstance(X, torch.Tensor):
        raise TypeError("X must be a torch.Tensor, not %s" % type(X).__name__)
    if X.dtype != torch.float64:
        raise TypeError("X must be float64, not %s" % X.dtype)
    if X.ndim != 2:
        raise ValueError("X must be a 2-D [N, F] matrix, got shape %s" % (tuple(X.shape),))
    columns = list(columns)
    if len(columns) != X.shape[1]:
        raise ValueError("%d columns named for %d in X" % (len(columns), X.shape[1]))
    if len(set(columns)) != len(columns):
        raise ValueError("columns must be distinct feature names")
    if isinstance(y, torch.Tensor):
        if y.is_cuda and y.device != X.device:
            raise ValueError("y is on %s, X on %s" % (y.device, X.device))
        if y.ndim != 1:
            raise ValueError("y must be 1-D, got shape %s" % (tuple(y.shape),))
        if y.dtype.is_complex:
            raise TypeError("y must be bool, integer or floating, not %s" % y.dtype)
        y = y.detach()
        y = pd.Series((y.float() if y.dtype == torch.bfloat16 else y).cpu().numpy())     # float32 holds bfloat16 exactly
    elif isinstance(y, pd.Series):
        y = y.reset_index(drop=True)
    elif isinstance(y, (np.ndarray, list)):
        y = pd.Series(y)
    else:
        raise TypeError("y must be a torch.Tensor, numpy.ndarray, list or pandas.Series, not %s" % type(y).__name__)
    return columns, y


def _same_samples(X, y):
    if len(X) != len(y):                 # a raise, not an assert: the library reads N targets
        raise AssertionError("X and y must contain the same number of samples.")


@contextlib.contextmanager
def _bound_context(dev):
    """The library context of `dev` with its calls enqueued on torch's current stream of the device, as
    extract_features_device runs, so the matrix needs no synchronisation between extraction and selection."""
    import torch
    if dev.type != "cuda":
        raise ValueError("X must be a CUDA tensor, got one on %s" % dev)
    with torch.cuda.device(dev):
        ctx = get_context(dev.index)
        with ctx.lock:
            ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream or _lib.STREAM_LEGACY)
            try:
                yield ctx
            finally:
                ctx.set_stream(None)


def _device_stats(X):
    """(class_stats, regression_stats) of _relevance_table for the CUDA matrix X.  A row-major X (unit column stride,
    row stride F) is read in place; any other layout, such as a column slice of a wider `out=`, is first copied by
    torch into a contiguous scratch of N * F * 8 bytes."""
    def run(select, *target):
        with _bound_context(X.device) as ctx:
            M = X.contiguous()
            return select(ctx, M.data_ptr(), M.shape[0], M.shape[1], *target)
    return (lambda codes, k: run(_lib.Context.select_classification_device, codes, k),
            lambda yv: run(_lib.Context.select_regression_device, yv))


def calculate_relevance_table_device(X, y, columns, *, ml_task="auto", multiclass=False, n_significant=1,
                                     test_for_binary_target_real_feature=TEST_FOR_BINARY_TARGET_REAL_FEATURE,
                                     fdr_level=FDR_LEVEL, hypotheses_independent=HYPOTHESES_INDEPENDENT, show_warnings=False):
    """calculate_relevance_table of a feature matrix on the GPU, without a host copy of the matrix.

    X: float64 CUDA tensor [N, F], rows are samples in positional order (e.g. the matrix extract_features_device
    returns); columns: its F distinct feature names; y: N targets as a CUDA or CPU tensor (bool, integer or floating),
    numpy array, list or pandas Series (taken positionally; string labels come through the host types).

    Returns the table calculate_relevance_table(pd.DataFrame(X.cpu().numpy(), columns=columns), pd.Series(y)) returns,
    with the same warnings and errors.  The statistics are computed on torch's current stream of X's device.  The host
    waits for that stream to read them back: once for a classification target, and once per feature column for a
    regression target (tsfx_select_regression reads each column's run count to choose its test).  A CUDA y adds one
    copy to the host."""
    columns, y = _device_args(X, y, columns)
    _same_samples(X, y)
    return _relevance_table(columns, y, *_device_stats(X), ml_task, multiclass, n_significant, show_warnings,
                            test_for_binary_target_real_feature, fdr_level, hypotheses_independent)


def select_features_device(X, y, columns, *, test_for_binary_target_binary_feature=TEST_FOR_BINARY_TARGET_BINARY_FEATURE,
                           test_for_binary_target_real_feature=TEST_FOR_BINARY_TARGET_REAL_FEATURE,
                           test_for_real_target_binary_feature=TEST_FOR_REAL_TARGET_BINARY_FEATURE,
                           test_for_real_target_real_feature=TEST_FOR_REAL_TARGET_REAL_FEATURE, fdr_level=FDR_LEVEL,
                           hypotheses_independent=HYPOTHESES_INDEPENDENT, n_jobs=N_PROCESSES, show_warnings=False,
                           chunksize=None, ml_task="auto", multiclass=False, n_significant=1):
    """select_features of a feature matrix on the GPU (arguments as calculate_relevance_table_device; the keywords are
    select_features', whose `device` is X's device here).

    Returns (X_sel, kept): X_sel a new float64 CUDA tensor [N, k] holding the relevant columns of X, kept their names,
    in the order select_features gives them (the relevance table's).  With no relevant feature X_sel is [N, 0]."""
    import torch
    columns, y = _device_args(X, y, columns)
    if not len(y) > 1:
        raise AssertionError("y must contain at least two samples.")
    _same_samples(X, y)
    yh = y.to_numpy()
    # len(set(y)) > 1 without boxing every number: NaN differs from everything, as boxed NaNs do in a set
    if not ((yh != yh[0]).any() if yh.dtype.kind in "biuf" else len(set(yh)) > 1):
        raise AssertionError("Feature selection is only possible if more than 1 label/class is provided")
    table = _relevance_table(columns, y, *_device_stats(X), ml_task, multiclass, n_significant, show_warnings,
                             test_for_binary_target_real_feature, fdr_level, hypotheses_independent)
    kept = list(table[table.relevant].feature)
    position = {c: i for i, c in enumerate(columns)}
    index = torch.tensor([position[c] for c in kept], dtype=torch.int64, device=X.device)
    return X.index_select(1, index), kept
