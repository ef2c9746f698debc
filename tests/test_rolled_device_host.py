"""extract_features_rolled_device: the argument checks that need no device, and the shared window arithmetic of
tsfx_roll_windows against a direct transcription of the reference's shift loop."""
import numpy as np
import pytest

from tsfresh_b200 import MinimalFCParameters, _lib, extract_features_rolled_device

torch = pytest.importorskip("torch")

I64 = torch.zeros(6, dtype=torch.int64)
F32 = torch.zeros(6)


def call(ids=I64, values=F32, sort=None, kind=None, **kw):
    kw.setdefault("default_fc_parameters", MinimalFCParameters())
    return extract_features_rolled_device(ids, values, sort, kind, **kw)


@pytest.mark.parametrize("args, match", [
    (dict(rolling_direction=0), "Rolling direction of 0 is not possible"),
    (dict(max_timeshift=0), "max_timeshift needs to be positive!"),
    (dict(max_timeshift=-3), "max_timeshift needs to be positive!"),
    (dict(min_timeshift=-1), "min_timeshift needs to be positive or zero!"),
    (dict(ids=I64[:1], values=F32[:1]), "zero or one rows"),
    (dict(ids=I64[:0], values=F32[:0]), "zero or one rows"),
])
def test_roll_time_series_errors(args, match):
    with pytest.raises(ValueError, match=match):
        call(**args)


def test_roll_errors_come_before_the_column_checks():
    with pytest.raises(ValueError, match="Rolling direction"):
        call(ids=[0, 1], rolling_direction=0)
    with pytest.raises(TypeError, match="ids must be a torch.Tensor"):
        call(ids=[0, 1])


def test_long_format_checks_are_shared():
    with pytest.raises(TypeError, match="sort must be int64 or float64"):
        call(sort=F32)
    with pytest.raises(ValueError, match="kind has 5 rows, ids 6"):
        call(kind=I64[:5], kinds=["a"])
    with pytest.raises(ValueError, match="kinds must name the kinds"):
        call(kind=I64)


def test_cpu_tensors_are_refused_after_the_argument_checks():
    with pytest.raises(ValueError, match="values must be a CUDA tensor"):
        call(rolling_direction=-3, max_timeshift=2, min_timeshift=1)


def reference_windows(lens, rd, mx, mn):
    """dataframe_functions.py:340-373, 548-562 as a plain loop over every shift of every series"""
    lmax = max(lens)
    shifts = list(reversed(range(lmax, 0, -rd))) if rd > 0 else list(range(1, lmax + 1, -rd))
    out, b0 = [], 0
    for s, n in enumerate(lens):
        for t in shifts:
            if t > n:
                continue
            lo, hi = (max(t - mx - 1, 0), t) if rd > 0 else (t - 1, min(t + mx, n))
            if hi - lo >= mn + 1:
                out.append((b0 + lo, hi - lo, s, t - 1))
        b0 += n
    return out


def test_roll_windows_against_the_reference_loop():
    rng = np.random.default_rng(0)
    for _ in range(300):
        lens = rng.integers(1, 60, rng.integers(1, 6)).astype(np.int32)
        rd = int(rng.choice([1, 2, 3, 7, 32, 100])) * int(rng.choice([1, -1]))
        mx, mn = int(rng.integers(0, 70)), int(rng.integers(0, 70))
        begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        wb, wl, wp, we = _lib.roll_windows(begin, lens, rd, mx, mn)
        got = list(zip(wb.tolist(), wl.tolist(), wp.tolist(), we.tolist()))
        assert got == reference_windows(lens.tolist(), rd, mx, mn), (lens.tolist(), rd, mx, mn)
