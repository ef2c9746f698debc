"""add_sub_time_series_index against the UNMODIFIED reference (skipped where the reference tree is absent), and the
argument checks of extract_features_sub_device that need no device."""
import warnings

import numpy as np
import pandas as pd
import pytest

from oracle import ref_shim
from tsfresh_b200 import MinimalFCParameters, add_sub_time_series_index, extract_features_sub_device

needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")


def reference():
    ref_shim.load()
    from tsfresh.utilities.dataframe_functions import add_sub_time_series_index as ref
    return ref


def both(make, *args, **kwargs):
    """(the reference's answer, ours) on fresh copies of the input (the reference may write into its input)"""
    out = []
    for f in (reference(), add_sub_time_series_index):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                out.append(f(make(), *args, **kwargs))
            except Exception as e:                # noqa: BLE001  (the exception type is what is compared)
                out.append(type(e))
    return out


def assert_same(ref, mine):
    if isinstance(ref, type) or isinstance(mine, type):
        assert ref is mine
    elif isinstance(ref, dict):
        assert list(ref) == list(mine)
        for k in ref:
            assert_same(ref[k], mine[k])
    else:
        assert list(ref.columns) == list(mine.columns)
        pd.testing.assert_frame_equal(ref, mine, check_dtype=False)


def small():
    return pd.DataFrame({"value": [1, 2, 3, 4, 5, 6, 7, 8, 9], "id": [1, 1, 1, 1, 2, 2, 2, 2, 2],
                         "kind": [0, 1, 0, 1, 0, 1, 0, 1, 0], "sort": [9, 8, 7, 6, 5, 4, 3, 2, 1]})


# AddSubIdTestCase (tests/units/utilities/test_dataframe_functions.py:1531-1614)
REFERENCE_CASES = [
    (lambda: small()[["value"]], dict()),
    (lambda: small()[["value", "id"]], dict(column_id="id")),
    (lambda: small()[["value", "id", "kind"]], dict(column_id="id", column_kind="kind")),
    (small, dict(column_id="id", column_kind="kind", column_sort="sort")),
    (lambda: {"1": small()[["value", "id"]]}, dict(column_id="id")),
]


@needs_reference
@pytest.mark.parametrize("case", range(len(REFERENCE_CASES)))
def test_reference_cases(case):
    make, kw = REFERENCE_CASES[case]
    assert_same(*both(make, 2, **kw))


def random_frame(seed, n_ids=5, n_kinds=3, float_keys=False, id_name="id", unique_keys=False):
    """sort keys distinct inside every (id, kind) series; with unique_keys distinct over the frame.  Equal sort keys
    inside one series are ordered differently: the reference sorts them with an unstable sort"""
    rng = np.random.default_rng(seed)
    parts = []
    offset = 0
    for i in rng.choice(np.arange(-50, 50), n_ids, replace=False):
        for k in range(n_kinds):
            if rng.random() < 0.2:
                continue                         # an (id, kind) series without rows
            n = int(rng.integers(1, 40))
            keys = rng.permutation(n) * 3 + 1 + offset
            offset += 200 if unique_keys else 0
            parts.append(pd.DataFrame({id_name: i, "kind": "k%d" % k, "value": rng.standard_normal(n),
                                       "time": keys * 0.5 if float_keys else keys}))
    df = pd.concat(parts, ignore_index=True)
    return df.iloc[rng.permutation(len(df))].set_index(pd.Index(rng.permutation(len(df)) * 2 + 7))


@needs_reference
@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("sub_length", [1, 3, 7, 100])
def test_random_frames(seed, sub_length):
    float_keys = seed % 2 == 1
    for kw in (dict(column_id="id", column_kind="kind", column_sort="time"), dict(column_id="id", column_kind="kind")):
        assert_same(*both(lambda: random_frame(seed, float_keys=float_keys), sub_length, **kw))
    for kw in (dict(column_kind="kind", column_sort="time"), dict(column_id="id", column_sort="time"),
               dict(column_sort="time"), dict(column_kind="kind"), dict()):
        assert_same(*both(lambda: random_frame(seed, float_keys=float_keys, unique_keys=True), sub_length, **kw))
    # an id column with another name: "id" is added next to it
    assert_same(*both(lambda: random_frame(seed, id_name="ID"), sub_length, column_id="ID", column_sort="time",
                      column_kind="kind"))
    # a dict of frames, one per kind
    frames = lambda: {k: g.drop(columns="kind") for k, g in random_frame(seed).groupby("kind")}  # noqa: E731
    assert_same(*both(frames, sub_length, column_id="id", column_sort="time"))


@needs_reference
@pytest.mark.parametrize("sub_length", [0, -1, -2, 2.5, 1.5, np.int64(0), None, "2", 2.0, True])
@pytest.mark.parametrize("kw", [dict(), dict(column_id="id"), dict(column_id="id", column_kind="kind")])
def test_argument_errors_match_the_reference(sub_length, kw):
    assert_same(*both(small, sub_length, **kw))


@needs_reference
def test_dict_with_kind_column():
    ref, mine = both(lambda: {"a": small()}, 2, column_kind="kind")
    assert ref is ValueError and mine is ValueError


def test_input_frame_is_left_alone():
    df = small()
    before = df.copy()
    out = add_sub_time_series_index(df, 4)
    pd.testing.assert_frame_equal(df, before)
    assert list(out["id"]) == [0, 0, 0, 0, 1, 1, 1, 1, 2]


torch = pytest.importorskip("torch")
I64 = torch.zeros(6, dtype=torch.int64)
F32 = torch.zeros(6)


def call(ids=I64, values=F32, sort=None, kind=None, **kw):
    kw.setdefault("default_fc_parameters", MinimalFCParameters())
    kw.setdefault("sub_length", 2)
    return extract_features_sub_device(ids, values, sort, kind, **kw)


@pytest.mark.parametrize("sub_length, error", [(0, ZeroDivisionError), (-1, AssertionError), (-7, AssertionError),
                                                (2.5, AssertionError), (None, TypeError), ("2", TypeError)])
def test_sub_length_errors(sub_length, error):
    with pytest.raises(error):
        call(sub_length=sub_length)


def test_sub_length_errors_come_before_the_column_checks():
    with pytest.raises(ZeroDivisionError):
        call(ids=[0, 1], sub_length=0)
    with pytest.raises(TypeError, match="ids must be a torch.Tensor"):
        call(ids=[0, 1])
    with pytest.raises(TypeError):
        call(sub_length=None, ids=None, values=None)


def test_long_format_checks_are_shared():
    with pytest.raises(TypeError, match="sort must be int64 or float64"):
        call(sort=F32)
    with pytest.raises(ValueError, match="kind has 5 rows, ids 6"):
        call(kind=I64[:5], kinds=["a"])
    with pytest.raises(ValueError, match="kind has 5 rows, values 6"):
        call(ids=None, kind=I64[:5], kinds=["a"])
    with pytest.raises(ValueError, match="kinds must name the kinds"):
        call(kind=I64)
    with pytest.raises(TypeError, match="values must be a torch.Tensor, not None"):
        call(ids=None, values=None)
    with pytest.raises(TypeError, match="ids must be int64"):
        call(ids=F32)


def test_cpu_tensors_are_refused_after_the_argument_checks():
    with pytest.raises(ValueError, match="values must be a CUDA tensor"):
        call(sub_length=3.0)
    with pytest.raises(ValueError, match="values must be a CUDA tensor"):
        call(ids=None, sub_length=True)
