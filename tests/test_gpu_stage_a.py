"""Stage (a) of the hot path through the C ABI (tsfx_extract_long_alloc / tsfx_extract_long / tsfx_extract_long_kinds):
the pipelined path for rows ordered by (id, sort key), the device sort for every other order, the NaN scan, pinned
and pageable host buffers; device rows go through the staged calls.  Restates the reference's adapter behaviour
(tsfresh/feature_extraction/data.py:217-230, 280-291; row-order invariance: test_extraction.py:207-237)."""
import numpy as np
import pytest

from tsfresh_b200 import MinimalFCParameters
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    from tsfresh_b200._lib import Context, DevicePlan
    ctx = Context(0)
    plan = Plan(MinimalFCParameters())
    dp = DevicePlan(ctx, plan)
    yield ctx, dp, plan
    dp.close()
    ctx.close()


def frame(n_series, rng, min_len=3, max_len=12):
    lens = rng.integers(min_len, max_len + 1, n_series)
    ids = np.repeat(np.arange(n_series, dtype=np.int64) * 3 - 7, lens)          # negative and non-contiguous ids
    t = np.concatenate([np.arange(l, dtype=np.int64) for l in lens])
    v = rng.standard_normal(len(ids)).astype(np.float32)
    return ids, t, v, lens


def dense_reference(dp, ids, t, v, times=None, flags=0):
    """the same rows (and row times) through the CSR entry point after a host-side lexsort"""
    order = np.lexsort((t, ids))
    ids_s, v_s = ids[order], v[order]
    uid, start, cnt = np.unique(ids_s, return_index=True, return_counts=True)
    return uid, dp.extract_csr(v_s, start.astype(np.int64), cnt.astype(np.int32), flags=flags,
                               times=None if times is None else times[order])


def test_ordered_rows_take_the_pipelined_path_in_several_blocks(env):
    ctx, dp, plan = env
    rng = np.random.default_rng(1)
    ids, t, v, lens = frame(50_000, rng)                 # > 16 384 series per block -> 4 row blocks
    uid, mat = dp.extract_long(ids, t, v)
    uid_ref, ref = dense_reference(dp, ids, t, v)
    assert np.array_equal(uid, uid_ref) and mat.shape == ref.shape
    assert np.array_equal(mat, ref, equal_nan=True)
    # pinned inputs (straight cudaMemcpyAsync) give the same answer as pageable ones (staging ring)
    pi, pt, pv = ctx.pinned_array(ids.shape, np.int64), ctx.pinned_array(t.shape, np.int64), ctx.pinned_array(v.shape, np.float32)
    pi[:], pt[:], pv[:] = ids, t, v
    uid2, mat2 = dp.extract_long(pi, pt, pv)
    assert np.array_equal(uid2, uid_ref) and np.array_equal(mat2, ref, equal_nan=True)


def test_any_row_order_gives_the_same_matrix(env):
    ctx, dp, plan = env
    rng = np.random.default_rng(2)
    ids, t, v, lens = frame(20_000, rng)
    uid_ref, ref = dense_reference(dp, ids, t, v)
    perm = rng.permutation(len(ids))
    uid, mat = dp.extract_long(ids[perm], t[perm], v[perm])                 # fully shuffled: two radix sorts
    assert np.array_equal(uid, uid_ref) and np.array_equal(mat, ref, equal_nan=True)
    # ids ascending but the sort keys shuffled inside every id: detected while streaming, then sorted in place
    order = np.lexsort((rng.random(len(ids)), ids))
    uid, mat = dp.extract_long(ids[order], t[order], v[order])
    assert np.array_equal(uid, uid_ref) and np.array_equal(mat, ref, equal_nan=True)
    # float sort keys, no sort keys (row order kept)
    uid, mat = dp.extract_long(ids[perm], t[perm].astype(np.float64) * 0.5 - 3.0, v[perm])
    assert np.array_equal(mat, ref, equal_nan=True)
    uid, mat = dp.extract_long(ids, None, v)
    assert np.array_equal(mat, ref, equal_nan=True)
    orders = {"ordered": np.arange(len(ids)), "shuffled": perm, "keys out of order": order}
    # linear_trend_timewise: the row times follow the rows through the sort, also when it runs after the streamed pass
    from tsfresh_b200 import _lib
    from tsfresh_b200._lib import DevicePlan
    tw = DevicePlan(ctx, Plan({"mean": None, "linear_trend_timewise": [{"attr": a} for a in ("slope", "intercept", "stderr")]},
                              has_datetime_index=True))
    times = (t * 3600 + rng.integers(0, 1800, len(t))) * 1_000_000_000              # hours apart, jittered
    uid_tw, ref_tw = dense_reference(tw, ids, t, v, times=times)
    for name, o in orders.items():
        uid, mat = tw.extract_long(ids[o], t[o], v[o], times=times[o])
        assert np.array_equal(uid, uid_tw) and np.array_equal(mat, ref_tw, equal_nan=True), name
    tw.close()
    # TSFX_FLAG_IMPUTE on a matrix with non-finite features (infinite values)
    vi = v.copy()
    vi[rng.choice(len(v), 40, replace=False)] = np.inf
    _, raw = dense_reference(dp, ids, t, vi)
    _, ref_imp = dense_reference(dp, ids, t, vi, flags=_lib.FLAG_IMPUTE)
    assert not np.isfinite(raw).all() and np.isfinite(ref_imp).all()
    for name, o in orders.items():
        uid, mat = dp.extract_long(ids[o], t[o], vi[o], flags=_lib.FLAG_IMPUTE)
        assert np.array_equal(uid, uid_ref) and np.array_equal(mat, ref_imp), name
    # caller buffers (extract_long_into): the spare rows stay untouched, a buffer one row short is refused
    for name, o in orders.items():
        out_ids, out = np.full(len(uid_ref) + 3, -99, np.int64), np.full((len(uid_ref) + 3, plan.n_cols), -99.0)
        assert dp.extract_long_into(ids[o], t[o], v[o], out_ids, out) == len(uid_ref), name
        assert np.array_equal(out_ids[:len(uid_ref)], uid_ref) and np.array_equal(out[:len(uid_ref)], ref, equal_nan=True)
        assert (out_ids[len(uid_ref):] == -99).all() and (out[len(uid_ref):] == -99.0).all()
        with pytest.raises(ValueError, match="out_capacity too small"):
            dp.extract_long_into(ids[o], t[o], v[o], out_ids[:len(uid_ref) - 1], out[:len(uid_ref) - 1])


def test_nan_values_are_an_error(env):
    ctx, dp, plan = env
    rng = np.random.default_rng(3)
    ids, t, v, lens = frame(30_000, rng)
    v = v.copy()
    v[len(v) // 2] = np.nan
    with pytest.raises(ValueError, match="contains NaN"):
        dp.extract_long(ids, t, v)
    perm = rng.permutation(len(ids))
    with pytest.raises(ValueError, match="contains NaN"):
        dp.extract_long(ids[perm], t[perm], v[perm])
    mid = (len(v) // 2 // 10) * 10
    with pytest.raises(ValueError, match="contains NaN"):
        dp.extract_dense(v[mid - 2000:mid + 2000].reshape(400, 10))
    uid, start, cnt = np.unique(ids, return_index=True, return_counts=True)
    with pytest.raises(ValueError, match="contains NaN"):
        dp.extract_csr(v, start.astype(np.int64), cnt.astype(np.int32))
    from tsfresh_b200 import _lib
    out = dp.extract_csr(v, start.astype(np.int64), cnt.astype(np.int32), flags=_lib.FLAG_NO_NAN_CHECK)   # opt out: NaN features, no error
    assert out.shape == (len(uid), plan.n_cols)
    # the context stays usable
    v[len(v) // 2] = 0.0
    uid2, mat = dp.extract_long(ids, t, v)
    assert np.isfinite(mat).all()
    # no ids / values but rows to read is a bad call, whatever the previous call left on the device
    import ctypes
    n = ctypes.c_int64(0)
    out_ids, out = np.empty(len(uid2), np.int64), np.empty((len(uid2), plan.n_cols))
    rc = ctx.lib.tsfx_extract_long(ctx.h, dp.h, None, None, 0, None, len(ids), ctypes.c_void_p(out_ids.ctypes.data),
                                   ctypes.c_void_p(out.ctypes.data), len(uid2), ctypes.byref(n), 0)
    assert rc == -1 and n.value == 0
    with pytest.raises(ValueError, match="tsfx_extract_long: bad arguments"):
        ctx.check(rc, "tsfx_extract_long")


def test_extract_features_reports_the_nan_column():
    import pandas as pd
    from tsfresh_b200 import extract_features
    from tsfresh_b200 import extraction
    rng = np.random.default_rng(4)
    ids, t, v, lens = frame(2_000, rng)
    v = v.copy()
    v[77] = np.nan
    df = pd.DataFrame({"id": ids, "time": t, "val": v})
    old = extraction._HOST_NAN_CHECK_ROWS
    try:
        for limit in (1 << 20, 0):                       # pandas scan / device scan: the same error
            extraction._HOST_NAN_CHECK_ROWS = limit
            with pytest.raises(ValueError, match="Column must not contain NaN values: val"):
                extract_features(df, column_id="id", column_sort="time", default_fc_parameters=MinimalFCParameters())
    finally:
        extraction._HOST_NAN_CHECK_ROWS = old


def test_device_rows_go_through_the_staged_calls(env):
    """device rows of one kind, no kind codes: tsfx_stage_long_stacked + tsfx_extract_staged give the ids and matrix of the
    host path; tsfx_extract_long refuses device pointers"""
    torch = pytest.importorskip("torch")
    import ctypes
    import re
    from tsfresh_b200 import _lib
    ctx, dp, plan = env
    rng = np.random.default_rng(5)
    ids, t, v, lens = frame(20_000, rng)
    uid_ref, ref = dense_reference(dp, ids, t, v)
    dev = torch.device("cuda", 0)
    for order in (np.arange(len(ids)), rng.permutation(len(ids))):
        d_ids, d_t, d_v = (torch.from_numpy(a[order]).to(dev) for a in (ids, t, v))
        torch.cuda.synchronize(dev)
        n_ids, rows, max_len = ctx.stage_long_stacked(d_ids.data_ptr(), d_t.data_ptr(), 0, d_v.data_ptr(), 0, 0, 1, 0, len(ids))
        assert n_ids == len(uid_ref) and rows[0] == len(ids) and max_len[0] == lens.max()
        d_uid = torch.empty(n_ids, dtype=torch.int64, device=dev)
        d_out = torch.empty((n_ids, plan.n_cols), dtype=torch.float64, device=dev)
        ctx.extract_staged([dp], d_uid.data_ptr(), d_out.data_ptr(), plan.n_cols)
        ctx.sync()
        assert np.array_equal(d_uid.cpu().numpy(), uid_ref)
        assert np.array_equal(d_out.cpu().numpy(), ref, equal_nan=True)
    n = ctypes.c_int64(0)
    rc = ctx.lib.tsfx_extract_long(ctx.h, dp.h, ctypes.c_void_p(d_ids.data_ptr()), ctypes.c_void_p(d_t.data_ptr()), 0,
                                   ctypes.c_void_p(d_v.data_ptr()), len(ids), ctypes.c_void_p(d_uid.data_ptr()),
                                   ctypes.c_void_p(d_out.data_ptr()), len(uid_ref), ctypes.byref(n), _lib.FLAG_DEVICE_PTRS)
    assert rc == -1 and n.value == 0
    msg = "tsfx_extract_long takes host pointers (device rows: tsfx_stage_long_stacked, tsfx_extract_staged)"
    with pytest.raises(ValueError, match=re.escape(msg)):
        ctx.check(rc, "tsfx_extract_long")
    uid, mat = dp.extract_long(ids, t, v)                 # the context stays usable
    assert np.array_equal(uid, uid_ref) and np.array_equal(mat, ref, equal_nan=True)


def test_pinned_pool_reuses_blocks(env):
    ctx, dp, plan = env
    shape = (12345, 77)                                   # a size no other test has left in the pool
    a = ctx.pinned_array(shape, np.float64)
    addr = a.ctypes.data
    a[:] = 1.0
    del a
    import gc
    gc.collect()
    b = ctx.pinned_array(shape, np.float64)
    assert b.ctypes.data == addr                          # the freed block came back from the pool


def test_nan_in_a_later_kind_of_a_shuffled_wide_frame(env):
    """wide frame, rows out of order (device sort): the NaN scan of the second kind's column runs after the sort pass
    read its flags; the call must still fail with the reference's error"""
    from tsfresh_b200 import _lib
    ctx, dp, plan = env
    rng = np.random.default_rng(8)
    ids, t, v, lens = frame(3_000, rng)
    w = rng.standard_normal(len(v)).astype(np.float32)
    perm = rng.permutation(len(ids))
    uid, mat = _lib.extract_long_kinds(ctx, [dp, dp], ids[perm], t[perm], [v[perm], w[perm]])
    uid_ref, ref = dense_reference(dp, ids, t, v)
    assert np.array_equal(uid, uid_ref) and np.array_equal(mat[:, :plan.n_cols], ref, equal_nan=True)
    assert np.array_equal(mat[:, plan.n_cols:], dense_reference(dp, ids, t, w)[1], equal_nan=True)
    w[len(w) // 3] = np.nan
    with pytest.raises(ValueError, match="contains NaN"):
        _lib.extract_long_kinds(ctx, [dp, dp], ids[perm], t[perm], [v[perm], w[perm]])
    with pytest.raises(ValueError, match="contains NaN"):
        _lib.extract_long_kinds(ctx, [dp, dp], ids, t, [v, w])                  # ordered rows: caught while streaming
