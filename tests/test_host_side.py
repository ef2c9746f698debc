"""CPU-only checks of the host side: the C-ABI library loads and exports every symbol of include/tsfx.h,
the plan compiler, roll-window views against the reference's roll_time_series (golden), id-sharding with a
world_size-2 gloo group."""
import ctypes
import os
import re

import numpy as np
import pytest

from tsfresh_b200 import _lib
from tsfresh_b200.plan import CALC, DESC_DTYPE, Plan, param_string
from tsfresh_b200.settings import ComprehensiveFCParameters

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "tsfx.h")).read()
    declared = set(re.findall(r"\b(tsfx_[a-z_]+)\s*\(", header))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    lib = ctypes.CDLL(_lib.LIB_PATH) if os.path.exists(_lib.LIB_PATH) else _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert _lib.load().tsfx_version() == 4


def test_plan_descriptor_table():
    p = Plan(ComprehensiveFCParameters())
    assert p.n_cols == 783 and p.descs.dtype == DESC_DTYPE and p.skipped == ["linear_trend_timewise"]
    assert list(p.descs["col"]) == list(range(783))
    i = p.suffixes.index('fft_coefficient__attr_"imag"__coeff_7')
    assert p.descs[i]["calc"] == CALC["TSFX_FFT_COEFFICIENT"] and p.descs[i]["attr"] == 1 and p.descs[i]["i0"] == 7
    i = p.suffixes.index("symmetry_looking__r_0.15000000000000002")          # float repr carried into the name
    assert p.descs[i]["p0"] == 3 * 0.05
    assert "range_count__max_1000000000000.0__min_0" in p.suffixes
    assert "cwt_coefficients__coeff_14__w_20__widths_(2, 5, 10, 20)" in p.suffixes
    tables, off, half = p.cwt_tables()
    assert list(np.diff(off)) == [34, 82, 162, 322] and list(half) == [16, 40, 80, 160]
    assert param_string({"b": "x", "a": 1.5}) == 'a_1.5__b_"x"'


def test_plan_rejects_what_has_no_gpu_path():
    with pytest.raises(NotImplementedError):
        Plan({(lambda x: 0): None})
    with pytest.raises(NotImplementedError):
        Plan({"approximate_entropy": [{"m": 3, "r": 0.1}]})
    with pytest.raises(NotImplementedError):
        Plan({"query_similarity_count": [{"query": [1.0, 2.0, 3.0], "threshold": 0.0}]})
    with pytest.raises(AttributeError):
        Plan({"no_such_calculator": None})
    with pytest.raises(TypeError):
        Plan({"quantile": [{"q": 0.5, "extra": 1}]})
    # per-kind subsets and duplicate-free combiners
    p = Plan({"ar_coefficient": [{"coeff": 1, "k": 3}, {"coeff": 1, "k": 3}], "maximum": None})
    assert p.suffixes == ["ar_coefficient__coeff_1__k_3", "maximum"]


def test_plan_parameter_limits():
    """the largest value the kernels' layouts hold is accepted, the next one refused (DESIGN.md section 1)"""
    from tsfresh_b200 import plan as P
    limited = [
        (lambda v: {"autocorrelation": [{"lag": v}]}, P.MAX_LAG),
        (lambda v: {"agg_autocorrelation": [{"f_agg": "mean", "maxlag": v}]}, P.MAX_LAG),
        (lambda v: {"partial_autocorrelation": [{"lag": 3}, {"lag": v}]}, P.MAX_LAG),
        (lambda v: {"ar_coefficient": [{"coeff": 0, "k": v}]}, P.MAX_AR_K),
        (lambda v: {"number_cwt_peaks": [{"n": v}]}, P.MAX_CWT_PEAKS_N),
        (lambda v: {"friedrich_coefficients": [{"coeff": 0, "m": 3, "r": v}]}, P.MAX_FRIEDRICH_R),
        (lambda v: {"max_langevin_fixed_point": [{"m": 3, "r": v}]}, P.MAX_FRIEDRICH_R),
        (lambda v: {"permutation_entropy": [{"tau": 1, "dimension": v}]}, P.MAX_PERM_DIMENSION),
        (lambda v: {"lempel_ziv_complexity": [{"bins": v}]}, P.MAX_LZ_BINS),
    ]
    assert (P.MAX_LAG, P.MAX_AR_K, P.MAX_CWT_PEAKS_N, P.MAX_FRIEDRICH_R, P.MAX_PERM_DIMENSION, P.MAX_LZ_BINS) == \
        (4096, 32, 16, 256, 8, 65535)
    for make, top in limited:
        assert Plan(make(top)).n_cols >= 1
        for over in (top + 1, 100000):
            with pytest.raises(NotImplementedError, match=r"\(> %d\)" % top):
                Plan(make(over))
    # calculators whose lag, n or bins the kernels do not bound
    p = Plan({"c3": [{"lag": 50000}], "time_reversal_asymmetry_statistic": [{"lag": 50000}], "number_peaks": [{"n": 50000}],
              "fourier_entropy": [{"bins": 100000}], "binned_entropy": [{"max_bins": 100000}]})
    assert p.n_cols == 5
    # the library states the same Lempel-Ziv limit
    header = open(os.path.join(ROOT, "tsfresh_b200", "csrc", "tsfx_kernels.h")).read()
    assert re.search(r"#define TSFX_LZ_MAX_BINS (\d+)", header).group(1) == str(P.MAX_LZ_BINS)


def test_from_columns_round_trip():
    """from_columns(column names) -> settings whose plan produces exactly those columns (settings.py:23-83; the
    reference pins the same round trip in tests/units/feature_extraction/test_settings.py:100-117)."""
    from tsfresh_b200 import ComprehensiveFCParameters, from_columns
    suffixes = Plan(ComprehensiveFCParameters()).suffixes
    k2 = from_columns(["value__" + s for s in suffixes] + ["b__maximum", "b__quantile__q_0.9", "junk"], columns_to_ignore=["junk"])
    assert list(k2) == ["value", "b"] and k2["b"] == {"maximum": None, "quantile": [{"q": 0.9}]}
    assert sorted(Plan(k2["value"]).suffixes) == sorted(suffixes)
    sub = [s for s in suffixes if s.startswith(("fft_coefficient", "agg_linear_trend", "value_count", "mean"))]
    assert sorted(Plan(from_columns(["x__" + s for s in sub])["x"]).suffixes) == sorted(sub)
    cfg = from_columns(["x__value_count__value_nan", "x__range_count__max_inf__min_-inf"])["x"]
    assert np.isnan(cfg["value_count"][0]["value"]) and cfg["range_count"] == [{"max": np.inf, "min": -np.inf}]
    with pytest.raises(ValueError):
        from_columns(["nounderscore"])
    with pytest.raises(TypeError):
        from_columns([3])
    with pytest.raises(ValueError):
        from_columns(["value__not_a_calculator"])


def test_roll_windows_match_reference_roll_time_series():
    z = np.load(os.path.join(G, "roll.npz"))
    lens = z["lens"].astype(np.int32)
    begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    wb, wl, wp, we = _lib.roll_windows(begin, lens, 3, 7, 7)
    # reference ids are (parent id, time of the window's last row); windows of fewer than 8 rows are dropped
    got = sorted(zip(wp.tolist(), we.tolist()))
    want = sorted(zip(z["parent"].tolist(), z["t_end"].tolist()))
    assert got == want
    assert set(wl.tolist()) == {8} and set(z["count"].tolist()) == {8}
    first = {(p, e): b - begin[p] for p, e, b in zip(wp.tolist(), we.tolist(), wb.tolist())}
    for p, e, f in zip(z["parent"].tolist(), z["t_end"].tolist(), z["first_time"].tolist()):
        assert first[(p, e)] == f
    # without min_timeshift the short leading windows are kept too
    wb, wl, wp, we = _lib.roll_windows(begin, lens, 3, 7, 0)
    got = {(p, e): l for p, e, l in zip(wp.tolist(), we.tolist(), wl.tolist())}
    want = {(p, e): c for p, e, c in zip(z["parent_nomin"].tolist(), z["t_end_nomin"].tolist(), z["count_nomin"].tolist())}
    assert got == want
    # the benchmark shape of BASELINE.json configs[4]: 121 windows of 256 rows per length-4096 series, stride 32
    wb, wl, wp, we = _lib.roll_windows(np.array([0, 4096]), np.array([4096, 4096], np.int32), 32, 255, 255)
    assert len(wb) == 242 and set(wl.tolist()) == {256} and we.max() == 4095


def test_roll_windows_both_directions_match_reference_cases():
    """tests/golden/roll_cases.npz (oracle/make_golden_roll.py, unmodified reference): positive and negative
    rolling_direction, with / without min_timeshift, max_timeshift beyond the longest series."""
    z = np.load(os.path.join(G, "roll_cases.npz"))
    lens = z["lens"].astype(np.int32)
    begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    for k, (rd, mx, mn) in enumerate(z["cases"].tolist()):
        wb, wl, wp, we = _lib.roll_windows(begin, lens, rd, mx, mn)
        got = sorted((int(p), int(e), int(b - begin[p]), int(l)) for b, l, p, e in zip(wb, wl, wp, we))
        assert got == [tuple(r) for r in z["case%d" % k].tolist()], (rd, mx, mn)
    with pytest.raises(ValueError):
        _lib.roll_windows(begin, lens, 0, 3, 0)


def test_roll_time_series_views_ids_and_errors():
    """tsfresh_b200.roll_time_series: window ids / extents on the golden cases + the reference's validation errors
    (dataframe_functions.py:455-515)."""
    import pandas as pd
    from tsfresh_b200 import roll_time_series
    z = np.load(os.path.join(G, "roll_cases.npz"))
    lens = z["lens"].tolist()
    df = pd.DataFrame({"id": np.concatenate([np.full(n, i) for i, n in enumerate(lens)]),
                       "time": np.concatenate([np.arange(n) for n in lens]),
                       "value": np.arange(sum(lens), dtype=np.float32)})
    begin = np.concatenate([[0], np.cumsum(lens)[:-1]])
    for k, (rd, mx, mn) in enumerate(z["cases"].tolist()):
        r = roll_time_series(df.sample(frac=1.0, random_state=k), column_id="id", column_sort="time",
                             rolling_direction=rd, max_timeshift=mx, min_timeshift=mn)
        got = sorted((i[0], i[1], int(b - begin[i[0]]), int(n)) for i, b, n in zip(r.ids, r.begin, r.length))
        assert got == [tuple(x) for x in z["case%d" % k].tolist()]
        assert r.ids == sorted(r.ids) and r.kinds == ["value"]
        assert np.array_equal(r.values["value"], df["value"].to_numpy())        # series order restored
    with pytest.raises(ValueError):
        roll_time_series(df, column_id="id", rolling_direction=0)
    with pytest.raises(ValueError):
        roll_time_series(df, column_id="id", max_timeshift=0)
    with pytest.raises(ValueError):
        roll_time_series(df, column_id="id", min_timeshift=-1)
    with pytest.raises(ValueError):
        roll_time_series(df.iloc[:1], column_id="id")
    with pytest.raises(ValueError):
        roll_time_series(df, column_id=None)
    with pytest.raises(AttributeError):
        roll_time_series(df, column_id="nope")
    with pytest.raises(ValueError):
        roll_time_series({"a": df}, column_id="id", column_kind="k")
    assert set(roll_time_series({"a": df, "b": df}, column_id="id", column_sort="time").keys()) == {"a", "b"}


def test_roll_time_series_known_answers_of_the_reference_tests():
    """Constants of the reference's RollingTestCase (tests/units/utilities/test_dataframe_functions.py:148-740)."""
    import pandas as pd
    from tsfresh_b200 import roll_time_series
    first = pd.DataFrame({"a": [1, 2, 3, 4], "b": [5, 6, 7, 8], "time": range(4), "id": 1})
    second = pd.DataFrame({"a": [10, 11], "b": [12, 13], "time": range(20, 22), "id": 2})
    df = pd.concat([first, second], ignore_index=True)
    f = roll_time_series(df, column_id="id", column_sort="time", rolling_direction=1).to_frame()          # :148-230
    assert list(f["id"]) == [(1, 0)] + [(1, 1)] * 2 + [(1, 2)] * 3 + [(1, 3)] * 4 + [(2, 20)] + [(2, 21)] * 2
    assert list(f["a"]) == [1, 1, 2, 1, 2, 3, 1, 2, 3, 4, 10, 10, 11]
    assert list(f["b"]) == [5, 5, 6, 5, 6, 7, 5, 6, 7, 8, 12, 12, 13]
    f = roll_time_series(df, column_id="id", column_sort="time", rolling_direction=2).to_frame()          # :578-625
    assert list(f["id"]) == [(1, 1)] * 2 + [(1, 3)] * 4 + [(2, 21)] * 2
    assert list(f["a"]) == [1, 2, 1, 2, 3, 4, 10, 11]
    f = roll_time_series(df, column_id="id", column_sort="time", rolling_direction=-2).to_frame()         # :627-650
    assert list(f["id"]) == [(1, 0)] * 4 + [(1, 2)] * 2 + [(2, 20)] * 2
    assert list(f["a"]) == [1, 2, 3, 4, 3, 4, 10, 11] and list(f["b"]) == [5, 6, 7, 8, 7, 8, 12, 13]
    stacked = pd.concat([df[["time", "id", "a"]].rename(columns={"a": "_value"}),                         # :652-740
                         df[["time", "id", "b"]].rename(columns={"b": "_value"})], ignore_index=True)
    stacked["kind"] = ["a"] * 6 + ["b"] * 6
    f = roll_time_series(stacked, column_id="id", column_sort="time", column_kind="kind", rolling_direction=-1).to_frame()
    assert list(f["id"]) == ([(1, 0)] * 8 + [(1, 1)] * 6 + [(1, 2)] * 4 + [(1, 3)] * 2 + [(2, 20)] * 4 + [(2, 21)] * 2)
    assert list(f["kind"]) == ["a", "b"] * 13
    assert list(f["_value"]) == [1, 5, 2, 6, 3, 7, 4, 8, 2, 6, 3, 7, 4, 8, 3, 7, 4, 8, 4, 8, 10, 12, 11, 13, 11, 13]


def _gloo_worker(rank, world, port, n_rows, q):
    import torch
    import torch.distributed as dist
    from tsfresh_b200 import distributed as D
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    full_in = torch.arange(n_rows * 3, dtype=torch.float64).reshape(n_rows, 3)
    lo, hi = D.shard_bounds(n_rows, world, rank)
    local = full_in[lo:hi] * 2.0                     # stands in for this rank's extracted rows
    out = D.gather_rows(local, n_rows)
    q.put((rank, lo, hi, bool(torch.equal(out, full_in * 2.0))))
    dist.destroy_process_group()


@pytest.mark.parametrize("n_rows", [10, 7, 1])
def test_id_sharding_and_gather_world_size_2(n_rows):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, n_rows, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert [r[3] for r in res] == [True, True]
    assert res[0][1] == 0 and res[0][2] == res[1][1] and res[1][2] == n_rows      # contiguous, covering


def test_window_sharding_keeps_parents_together():
    """distributed.shard_windows: config-5 layout -- contiguous, complete, no parent split over two ranks."""
    from tsfresh_b200 import distributed as D
    rng = np.random.default_rng(0)
    for world in (1, 2, 3, 8):
        for n_par in (1, 2, 5, 40):
            counts = rng.integers(0, 9, n_par)
            parent = np.repeat(np.arange(n_par), counts)
            spans = [D.shard_windows(parent, n_par, world, r) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == len(parent)
            assert all(spans[r][1] == spans[r + 1][0] for r in range(world - 1))
            owners = {}
            for r, (lo, hi) in enumerate(spans):
                for p in set(parent[lo:hi].tolist()):
                    assert owners.setdefault(p, r) == r
    # the benchmark shape: 10 000 parents x 121 windows over 8 ranks -> 1250 parents each
    parent = np.repeat(np.arange(10000), 121)
    assert [D.shard_windows(parent, 10000, 8, r) for r in range(8)] == [(r * 151250, (r + 1) * 151250) for r in range(8)]


def test_impute_helpers_validate_before_touching_the_device():
    """impute_dataframe_range raises the reference's ValueErrors (dataframe_functions.py:136-156) and the helpers
    return empty frames untouched (:71-72, :93-94, :133-134) -- all before any device call."""
    import pandas as pd
    from tsfresh_b200 import impute, impute_dataframe_range, impute_dataframe_zero
    df = pd.DataFrame({"a": [1.0, np.nan], "b": [np.inf, 2.0]})
    good = {"a": 1.0, "b": 2.0}
    with pytest.raises(ValueError, match="more or less keys"):
        impute_dataframe_range(df, {"a": 1.0}, good, good)
    with pytest.raises(ValueError, match="non finite values"):
        impute_dataframe_range(df, good, {"a": np.nan, "b": 0.0}, good)
    empty = pd.DataFrame(columns=["a", "b"], dtype=float)
    assert impute(empty) is empty and impute_dataframe_zero(empty) is empty
    assert impute_dataframe_range(empty, good, good, good) is empty


def test_input_validation_matches_reference_wrong_input_cases():
    """The pandas cases of the reference's DataAdapterTestCase.test_with_wrong_input
    (tests/units/feature_extraction/test_data.py:459-548) against the adapters of tsfresh_b200.extract_features
    (`_frames`, restating data.py:124-338): every malformed container raises ValueError before any device work."""
    import pandas as pd
    from tsfresh_b200.extraction import _frames

    def to_tsdata(df, column_id, column_kind, column_value, column_sort):
        return _frames(df, column_id, column_kind, column_value, column_sort)

    bad = [
        (pd.DataFrame([{"id": 0, "kind": "a", "value": 3, "sort": np.nan}]), "id", "kind", "value", "sort"),
        (pd.DataFrame([{"id": 0, "kind": "a", "value": 3, "sort": 1}]), "strange_id", "kind", "value", "sort"),
        (pd.DataFrame([{"id": 0, "kind": "a", "value": 3, "value_2": 1, "sort": 1}]), "strange_id", "kind", None, "sort"),
        (pd.DataFrame([{"id": 0, "kind": "a", "value": 3, "sort": 1}]), "id", "strange_kind", "value", "sort"),
        (pd.DataFrame([{"id": np.nan, "kind": "a", "value": 3, "sort": 1}]), "id", "kind", "value", "sort"),
        (pd.DataFrame([{"id": 0, "kind": np.nan, "value": 3, "sort": 1}]), "id", "kind", "value", "sort"),
        (pd.DataFrame([{"id": 2}, {"id": 1}]), None, "a", "b", None),
        (pd.DataFrame([{"id": 2}, {"id": 1}]), None, "a", "b", "a"),
        ({"a": pd.DataFrame([{"id": 2}, {"id": 1}]), "b": pd.DataFrame([{"id": 2}, {"id": 1}])}, None, "a", "b", None),
        ({"a": pd.DataFrame([{"id": 2}, {"id": 1}]), "b": pd.DataFrame([{"id": 2}, {"id": 1}])}, "id", None, None, None),
        ({"a": pd.DataFrame([{"id": 2, "value_a": 3}, {"id": 1, "value_a": 4}]), "b": pd.DataFrame([{"id": 2}, {"id": 1}])},
         "id", None, None, None),
        (pd.DataFrame([{"id": 0, "value": np.nan}]), "id", None, "value", None),
        (pd.DataFrame([{"id": 0, "value": np.nan}]), None, None, "value", None),
        (pd.DataFrame([{"id": 0, "a_": 3, "b": 5, "sort": 1}]), "id", None, None, "sort"),
        (pd.DataFrame([{"id": 0, "a__c": 3, "b": 5, "sort": 1}]), "id", None, None, "sort"),
        (pd.DataFrame([{"id": 0}]), "id", None, None, None),
        (pd.DataFrame([{"id": 0, "sort": 0}]), "id", None, None, "sort"),
        ([1, 2, 3], "a", "b", "c", "d"),
    ]
    for k, case in enumerate(bad):
        with pytest.raises(ValueError):
            to_tsdata(*case)
            pytest.fail("case %d did not raise" % k)


def test_feature_selection_pvalues_match_scipy():
    """host-side finishing of tsfresh_b200.feature_selection: the p-value of every statistic the device returns is the one
    scipy computes from the raw samples (significance_tests.py:43-132)"""
    from scipy import stats
    from tsfresh_b200.feature_selection import benjamini_reject, fisher_pvalue, ks_2samp_pvalue, mannwhitneyu_pvalue
    rng = np.random.default_rng(0)
    for trial in range(120):
        n1, n2 = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        if trial % 2:
            x, y = rng.standard_normal(n1), rng.standard_normal(n2) + 0.4
        else:
            x, y = rng.integers(0, 6, n1).astype(float), rng.integers(0, 6, n2).astype(float)
        ref = stats.mannwhitneyu(x, y, use_continuity=True, alternative="two-sided")
        xy = np.concatenate([x, y])
        U1 = stats.rankdata(xy)[:n1].sum() - n1 * (n1 + 1) / 2
        _, t = np.unique(xy, return_counts=True)
        p = mannwhitneyu_pvalue(U1, n1, n2, float((t ** 3 - t).sum()), len(t))
        assert (np.isnan(p) and np.isnan(ref.pvalue)) or abs(p - ref.pvalue) < 1e-12
        ks = stats.ks_2samp(x, y)
        assert abs(ks_2samp_pvalue(ks.statistic, n1, n2) - ks.pvalue) < 1e-12
    assert abs(fisher_pvalue(8, 2, 1, 5) - stats.fisher_exact([[8, 2], [1, 5]])[1]) < 1e-15
    # Benjamini-Hochberg by hand: m = 4, alpha = 0.05 -> thresholds 0.0125, 0.025, 0.0375, 0.05
    assert list(benjamini_reject([0.03, 0.001, 0.5, 0.02], 0.05, True)) == [True, True, False, True]
    # Benjamini-Yekutieli divides the thresholds by 1 + 1/2 + 1/3 + 1/4
    assert list(benjamini_reject([0.03, 0.001, 0.5, 0.02], 0.05, False)) == [False, True, False, False]


def test_kendall_pvalue_from_sufficient_statistics_matches_scipy():
    """the statistics tsfx_select_regression returns (discordant pairs, tie sums, joint ties) give scipy's asymptotic
    Kendall p-value (significance_tests.py:170-188); the statistics are formed here by brute force"""
    from scipy import stats
    from tsfresh_b200.feature_selection import kendall_pvalue
    rng = np.random.default_rng(5)

    def tie_sums(v):
        _, t = np.unique(v, return_counts=True)
        t = t.astype(np.float64)
        return (t * (t - 1) // 2).sum(), (t * (t - 1) * (t - 2)).sum(), (t * (t - 1) * (2 * t + 5)).sum()

    for trial in range(60):
        n = int(rng.integers(3, 80))
        if trial % 3 == 0:
            x, y = rng.standard_normal(n), rng.standard_normal(n)
        elif trial % 3 == 1:
            x, y = rng.integers(0, 5, n).astype(float), rng.standard_normal(n)
        else:
            x, y = rng.integers(0, 4, n).astype(float), rng.integers(0, 3, n).astype(float)
        dx, dy = x[:, None] - x[None, :], y[:, None] - y[None, :]
        dis = int(np.sum((dx < 0) & (dy > 0)))
        _, joint = np.unique(np.stack([x, y], axis=1), axis=0, return_counts=True)
        ntie = int((joint * (joint - 1) // 2).sum())
        xt, yt = tie_sums(x), tie_sums(y)
        got = kendall_pvalue(n, dis, int(xt[0]), xt[1], xt[2], ntie, int(yt[0]), yt[1], yt[2])
        want = stats.kendalltau(x, y, method="asymptotic").pvalue
        assert (np.isnan(got) and np.isnan(want)) or abs(got - want) < 1e-12


def _gm_worker(rank, world, port, ret):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tsfresh_b200.distributed import GatheredMatrix
        gm = GatheredMatrix(1000, 7, torch.device("cpu"), n_blocks=7)
        assert gm.kind == "nccl" and gm.placement() == "nccl"          # no symmetric memory on the host: exchange of row blocks
        gm.local[:] = torch.arange(1000 * 7, dtype=torch.float64).reshape(1000, 7) + 1e6 * rank
        cuts = gm.block_bounds(gm.rows)
        for lo, hi in zip(cuts[:-1], cuts[1:]):                       # what extract_*_sharded_device does after every block
            gm.block_done(lo, hi, None)
        gm.finish(None)
        want = torch.cat([torch.arange(7000, dtype=torch.float64).reshape(1000, 7) + 1e6 * r for r in range(world)])
        ret[rank] = bool(torch.equal(gm.full, want)), cuts
    finally:
        dist.destroy_process_group()


def test_gathered_matrix_row_blocks_world_size_2_gloo():
    """the product's result placement (tsfresh_b200.distributed.GatheredMatrix) without GPUs: geometric row blocks,
    the same cuts on every rank, block-wise exchange -> every rank holds every rank's rows"""
    import socket
    import torch.multiprocessing as mp
    from tsfresh_b200.distributed import GatheredMatrix
    g = GatheredMatrix.__new__(GatheredMatrix)
    g.world, g.n_blocks = 8, 7
    cuts = g.block_bounds(1_000_000)
    assert cuts == [0, 250000, 500000, 750000, 875000, 937500, 968750, 1000000]
    assert g.block_bounds(100) == [0, 100]                            # tiny shards: one block
    g.world = 1
    assert g.block_bounds(1_000_000) == [0, 1_000_000]
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_gm_worker, args=(2, port, ret), nprocs=2, join=True)
    assert ret[0][0] and ret[1][0] and ret[0][1] == ret[1][1] and len(ret[0][1]) == 8


def test_n_jobs_maps_to_gpus(monkeypatch):
    from tsfresh_b200 import _lib, extraction
    monkeypatch.setattr(_lib, "device_count", lambda: 8)
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    assert extraction._gpus_for(64, None) == list(range(8))          # the reference's default n_jobs: every visible GPU
    assert extraction._gpus_for(2, None) == [0, 1]
    assert extraction._gpus_for(0, None) == [0] and extraction._gpus_for(1, None) == [0]
    assert extraction._gpus_for(64, 5) == [5]                         # explicit device wins
    monkeypatch.setenv("LOCAL_RANK", "3")
    assert extraction._gpus_for(64, None) == [3]                      # one process per GPU under torchrun
