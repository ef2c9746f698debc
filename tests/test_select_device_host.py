"""calculate_relevance_table_device / select_features_device without a GPU: the argument checks raise before the
library is called, and with the library replaced by a stand-in that returns the same sufficient statistics to both
paths, the device path and the DataFrame path build the same relevance table from them."""
import contextlib
import ctypes
import threading
import warnings

import numpy as np
import pandas as pd
import pytest

from tsfresh_b200 import (_lib, calculate_relevance_table, calculate_relevance_table_device, select_features,
                          select_features_device)
from tsfresh_b200 import feature_selection as fs

torch = pytest.importorskip("torch")

N = 40
TYPES = [2, 2, 0, 1, 2, 1, 0, 2, 2, 1]            # real / binary / constant, as the library types the columns
COLUMNS = ["f%d" % i for i in range(len(TYPES))]


class FakeLib:
    """tsfx_select_*: records every call and writes fixed, valid statistics (they need not belong to the matrix)"""

    def __init__(self, nan=False):
        self.calls, self.nan, self.types = [], nan, TYPES

    @staticmethod
    def _array(ptr, count):
        return np.ctypeslib.as_array((ctypes.c_double * count).from_address(ptr.value))

    def _record(self, name, X, n, f, flags):
        matrix = self._array(X, n * f).reshape(n, f).copy() if f else None
        self.calls.append({"name": name, "ptr": X.value, "flags": flags, "matrix": matrix})
        return -6 if self.nan else 0                 # TSFX_E_NAN

    def tsfx_select_classification(self, h, X, n, f, y, k, out, flags):
        rc = self._record("classification", X, n, f, flags)
        codes = np.ctypeslib.as_array((ctypes.c_int32 * n).from_address(y.value))
        o = self._array(out, k * f * 8).reshape(k, f, 8)
        rng = np.random.default_rng(11)
        for c in range(k):
            n1 = int((codes == c).sum())
            n0 = n - n1
            for j, t in enumerate(self.types[:f]):
                a, b = int(rng.integers(0, n1 + 1)), int(rng.integers(0, n0 + 1))
                if t == 2:                          # U1, tie term, KS statistic, distinct values
                    o[c, j] = [2, n1, n0, 0.5 * rng.integers(0, 2 * n1 * n0 + 1), 0, rng.uniform(0.05, 0.9), n, 0]
                elif t == 1:                        # the 2 x 2 table
                    o[c, j] = [1, n1, n0, a, n1 - a, b, n0 - b, 0]
                else:
                    o[c, j] = [0, n1, n0, 0, 0, 0, 1, 0]
        return rc

    def tsfx_select_regression(self, h, X, n, f, y, out, flags):
        rc = self._record("regression", X, n, f, flags)
        o = self._array(out, f * 8 + 4)
        rng = np.random.default_rng(12)
        for j, t in enumerate(self.types[:f]):
            if t == 2:                              # discordant pairs, no ties
                o[j * 8:j * 8 + 8] = [2, n, rng.integers(0, n * (n - 1) // 2 + 1), 0, 0, 0, 0, 0]
            elif t == 1:                            # KS of the target, rows with the larger / smaller value
                m = int(rng.integers(1, n))
                o[j * 8:j * 8 + 8] = [1, n, rng.uniform(0.05, 0.9), m, n - m, 0, 0, 0]
            else:
                o[j * 8:j * 8 + 8] = [0, n, 0, 0, 0, 0, 0, 0]
        o[f * 8:] = [0, 0, 0, n]
        return rc

    def tsfx_last_error(self, h):
        return b"the feature matrix contains NaN"


def fake_context(lib):
    ctx = _lib.Context.__new__(_lib.Context)
    ctx.lib, ctx.h, ctx.lock, ctx._plans, ctx._alive = lib, None, threading.RLock(), {}, {"h": None}
    return ctx


@pytest.fixture
def lib(monkeypatch):
    """both paths reach the stand-in: the DataFrame path through get_context, the device path through the context
    bound to torch's stream (a CPU tensor stands for the CUDA matrix)"""
    fake = FakeLib()
    ctx = fake_context(fake)
    monkeypatch.setattr(fs, "get_context", lambda device=None: ctx)
    monkeypatch.setattr(fs, "_bound_context", lambda dev: contextlib.nullcontext(ctx))
    return fake


class LibraryCalled(Exception):
    pass


@pytest.fixture
def no_library(monkeypatch):
    def called(*a, **k):
        raise LibraryCalled()
    monkeypatch.setattr(fs, "_bound_context", called)


def matrix(seed=0):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((N, len(TYPES))))


Y2 = np.tile([0, 1, 1, 0, 1], N // 5)


@pytest.mark.parametrize("X, y, columns, kw, exc, match", [
    ([[0.0]], Y2, COLUMNS, {}, TypeError, "X must be a torch.Tensor"),
    (matrix().float(), Y2, COLUMNS, {}, TypeError, "X must be float64"),
    (matrix()[:, 0], Y2, COLUMNS, {}, ValueError, "2-D"),
    (matrix()[None], Y2, COLUMNS, {}, ValueError, "2-D"),
    (matrix(), Y2, COLUMNS[:-1], {}, ValueError, "9 columns named for 10"),
    (matrix(), Y2, COLUMNS[:-1] + ["f0"], {}, ValueError, "distinct"),
    (matrix(), {"a": 1}, COLUMNS, {}, TypeError, "y must be a torch.Tensor, numpy.ndarray, list or pandas.Series"),
    (matrix(), torch.zeros((N, 1)), COLUMNS, {}, ValueError, "y must be 1-D"),
    (matrix(), torch.zeros(N, dtype=torch.complex64), COLUMNS, {}, TypeError, "bool, integer or floating"),
    (matrix(), Y2[:-1], COLUMNS, {}, AssertionError, "same number of samples"),
    (matrix(), Y2, COLUMNS, {"ml_task": "clustering"}, ValueError, "ml_task must be one of"),
    (matrix(), Y2.astype(float), COLUMNS, {"ml_task": "regression", "multiclass": True}, AssertionError,
     "ml_task must be classification for multiclass"),
    (matrix(), Y2, COLUMNS, {"multiclass": True, "n_significant": 3}, AssertionError, "n_significant must not exceed"),
    (matrix(), np.where(Y2 == 1, np.nan, 0.5), COLUMNS, {}, ValueError, "Target y contains NaN values"),
])
@pytest.mark.parametrize("fn", [calculate_relevance_table_device, select_features_device])
def test_argument_errors_before_the_library(no_library, fn, X, y, columns, kw, exc, match):
    with pytest.raises(exc, match=match):
        fn(X, y, columns, **kw)


def test_select_features_errors(no_library):
    with pytest.raises(AssertionError, match="at least two samples"):
        select_features_device(matrix()[:1], [1], COLUMNS)
    with pytest.raises(AssertionError, match="more than 1 label/class"):
        select_features_device(matrix(), np.ones(N), COLUMNS)
    with pytest.raises(AssertionError, match="more than 1 label/class"):
        select_features_device(matrix(), ["a"] * N, COLUMNS)
    with pytest.raises(ValueError, match="Target y contains NaN"):      # one NaN is a second value, as in a set
        select_features_device(matrix(), [np.nan] + [1.0] * (N - 1), COLUMNS)
    with pytest.raises(LibraryCalled):               # the table has no two-sample check
        calculate_relevance_table_device(matrix(), np.ones(N, dtype=int), COLUMNS)


def test_cpu_matrix_is_refused_after_the_argument_checks(monkeypatch):
    monkeypatch.setattr(fs, "get_context", lambda device=None: pytest.fail("library called"))
    for fn in (calculate_relevance_table_device, select_features_device):
        with pytest.raises(ValueError, match="X must be a CUDA tensor, got one on cpu"):
            fn(matrix(), Y2, COLUMNS)


def test_nan_in_the_matrix(monkeypatch):
    ctx = fake_context(FakeLib(nan=True))
    monkeypatch.setattr(fs, "_bound_context", lambda dev: contextlib.nullcontext(ctx))
    for y in (Y2, np.linspace(0, 1, N)):
        with pytest.raises(ValueError, match="Feature matrix contains NaN values"):
            calculate_relevance_table_device(matrix(), y, COLUMNS)


def test_nan_status_is_a_typed_value_error():
    ctx = fake_context(FakeLib(nan=True))
    with pytest.raises(_lib.NanValuesError, match="^tsfx_select_regression: the feature matrix contains NaN$") as e:
        ctx.select_regression(np.zeros((N, 3)), np.zeros(N))
    assert isinstance(e.value, ValueError)


def tables(X, y, columns, **kw):
    """(device table, its warnings, DataFrame table, its warnings), with the table's warnings shown"""
    out = []
    for run in (lambda: calculate_relevance_table_device(X, y, columns, show_warnings=True, **kw),
                lambda: calculate_relevance_table(pd.DataFrame(X.numpy(), columns=columns), pd.Series(host(y)),
                                                  show_warnings=True, **kw)):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            out += [run(), [(x.category, str(x.message)) for x in w if x.filename == fs.__file__]]
    return out


def host(y):
    return y.numpy() if isinstance(y, torch.Tensor) else y


CASES = {
    "binary": (Y2, {}),
    "binary_labels": (list(np.where(Y2 == 1, "yes", "no")), {}),
    "binary_smir": (Y2, {"test_for_binary_target_real_feature": "smir", "hypotheses_independent": True}),
    "multiclass": (np.tile([0, 1, 2, 2], N // 4), {"multiclass": True, "n_significant": 2}),
    "three_classes_merged": (np.tile([0, 1, 2, 2], N // 4), {}),
    "regression": (np.linspace(-1.0, 3.0, N), {"fdr_level": 0.3}),
    "bool_tensor": (torch.from_numpy(Y2.astype(bool)), {}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_the_same_table_from_the_same_statistics(lib, case):
    y, kw = CASES[case]
    X = matrix()
    dev, dev_w, df, df_w = tables(X, y, COLUMNS, **kw)
    pd.testing.assert_frame_equal(dev, df)
    for c in dev.columns:
        if c.startswith("p_value"):
            assert (dev[c].to_numpy(dtype=float).view(np.int64) == df[c].to_numpy(dtype=float).view(np.int64)).all()
    assert dev_w == df_w and any("Constant features" in m for _, m in dev_w)
    assert [c["flags"] for c in lib.calls] == [_lib.FLAG_DEVICE_PTRS, 0]
    # select_features_device keeps select_features' columns, in its order, as a copy of those columns of X
    want = select_features(pd.DataFrame(X.numpy(), columns=COLUMNS), np.asarray(host(y)), **kw)
    X_sel, kept = select_features_device(X, y, COLUMNS, **kw)
    assert kept == list(want.columns) and len(kept) > 0
    assert X_sel.data_ptr() != X.data_ptr() and X_sel.is_contiguous()
    assert np.array_equal(X_sel.numpy(), want.to_numpy())


def test_every_feature_constant(lib):
    lib.types = [0, 0, 0]
    dev, dev_w, df, df_w = tables(matrix()[:, :3], Y2, COLUMNS[:3])
    pd.testing.assert_frame_equal(dev, df)
    assert dev_w == df_w and (dev.type == "constant").all()


def test_no_relevant_feature(lib):
    X_sel, kept = select_features_device(matrix(), Y2, COLUMNS, fdr_level=1e-300)
    assert kept == [] and tuple(X_sel.shape) == (N, 0)
    with pytest.warns(RuntimeWarning, match="No feature was found relevant"):
        select_features_device(matrix(), Y2, COLUMNS, fdr_level=1e-300, show_warnings=True)


def test_device_pointer_of_the_matrix(lib):
    """the library gets X's own pointer with TSFX_FLAG_DEVICE_PTRS; a strided X, a row-major copy of it"""
    X = matrix()
    calculate_relevance_table_device(X, Y2, COLUMNS)
    calculate_relevance_table_device(X, np.linspace(0, 1, N), COLUMNS)
    assert [(c["name"], c["ptr"], c["flags"]) for c in lib.calls] == [
        ("classification", X.data_ptr(), _lib.FLAG_DEVICE_PTRS), ("regression", X.data_ptr(), _lib.FLAG_DEVICE_PTRS)]
    wide = torch.from_numpy(np.random.default_rng(3).standard_normal((N, 25)))
    sl = wide[:, 5:5 + len(COLUMNS)]
    lib.calls.clear()
    calculate_relevance_table_device(sl, Y2, COLUMNS)
    (call,) = lib.calls
    assert call["flags"] == _lib.FLAG_DEVICE_PTRS and call["ptr"] != sl.data_ptr()
    assert np.array_equal(call["matrix"], sl.numpy())
    lib.calls.clear()
    calculate_relevance_table(pd.DataFrame(X.numpy(), columns=COLUMNS), pd.Series(Y2))
    (call,) = lib.calls
    assert call["flags"] == 0 and call["ptr"] != X.data_ptr()


def test_target_types_give_one_table(lib):
    """a CPU tensor, numpy, a list and a Series with any index are the same targets, taken by position"""
    X = matrix()
    want = calculate_relevance_table_device(X, Y2, COLUMNS)
    for y in (torch.from_numpy(Y2), list(Y2), pd.Series(Y2, index=np.arange(N)[::-1] * 3)):
        pd.testing.assert_frame_equal(calculate_relevance_table_device(X, y, COLUMNS), want)
    bf = torch.from_numpy(np.linspace(-1.0, 3.0, N)).to(torch.bfloat16)
    pd.testing.assert_frame_equal(calculate_relevance_table_device(X, bf, COLUMNS),
                                  calculate_relevance_table_device(X, bf.float().numpy(), COLUMNS))
