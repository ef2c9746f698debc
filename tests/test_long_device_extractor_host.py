"""DeviceLongExtractor: the refusals that need no device -- sizes and length limits in the constructor; layouts, dtypes,
row counts, devices, `out` and `n_rows` at the call -- and its column names."""
import re

import pytest

from tsfresh_b200 import (ComprehensiveFCParameters, DeviceLongExtractor, EfficientFCParameters, MinimalFCParameters,
                          extract_features_long_device)
from tsfresh_b200.device_api import _plans

torch = pytest.importorskip("torch")

MIN = MinimalFCParameters()
META = "meta"


@pytest.fixture
def no_device(monkeypatch):
    """The constructor up to the device: the library context, plans and status words are not created."""
    monkeypatch.setattr(DeviceLongExtractor, "_open", lambda self: None)


def make(*args, **kw):
    kw.setdefault("device", "cuda:0")
    return DeviceLongExtractor(*args, **kw)


def rows(n, device=META, sort=torch.int64, kind=torch.int64):
    """(ids, values, sort, kind) tensors of n rows"""
    return (torch.zeros(n, dtype=torch.int64, device=device), torch.zeros(n, device=device),
            None if sort is None else torch.zeros(n, dtype=sort, device=device),
            None if kind is None else torch.zeros(n, dtype=kind, device=device))


def test_length_limits_in_the_constructor(no_device):
    make(100, 8, 21_000)
    with pytest.raises(ValueError, match="21001 samples exceed the limit of kind 'value''s settings \\(21000 samples\\)"):
        make(100, 8, 21_001)
    with pytest.raises(ValueError, match="limit of kind 'b'"):
        make(100, 8, 30_000, kinds=["a", "b"], default_fc_parameters=EfficientFCParameters(),
             kind_to_fc_parameters={"b": ComprehensiveFCParameters()})
    make(100, 8, 131_072, default_fc_parameters=EfficientFCParameters())
    with pytest.raises(ValueError, match="131073 samples"):
        make(100, 8, 131_073, default_fc_parameters=EfficientFCParameters())
    make(100, 8, 1_000_000, default_fc_parameters=MIN)        # BASIC / SORTED only: no limit


@pytest.mark.parametrize("args, kw, match", [
    ((0, 8, 16), {}, "max_rows must be an integer"),
    ((-5, 8, 16), {}, "max_rows must be an integer"),
    (((1 << 31) - 4097, 8, 16), {}, "max_rows must be an integer in 1 .. 2147479550"),
    ((100, 0, 16), {}, "max_ids must be an integer"),
    ((100, 2.0, 16), {}, "max_ids must be an integer"),
    ((100, 8, 0), {}, "max_length must be an integer"),
    ((100, 8, -1), {}, "max_length must be an integer"),
    ((100, 8, 16), {"kinds": []}, "between 1 and 64 kinds, 0 named"),
    ((100, 8, 16), {"kinds": ["k%d" % i for i in range(65)]}, "between 1 and 64 kinds, 65 named"),
    ((100, 8, 16), {"kinds": ["a", "a"]}, "distinct"),
    ((100, 8, 16), {"kinds": ["a__b"]}, "'__'"),
    ((100, 8, 16), {"device": "cpu"}, "CUDA device"),
])
def test_constructor_arguments(no_device, args, kw, match):
    with pytest.raises(ValueError, match=match):
        make(*args, **kw)


def test_sixty_four_kinds(no_device):
    ex = make(100, 8, 16, kinds=["k%d" % i for i in range(64)], default_fc_parameters=MIN)
    assert len(ex.columns) == 64 * len(_plans(["k0"], MIN, None)[1])


def test_columns_are_every_kinds_names(no_device):
    k2fc = {"b": MIN}
    ex = make(100, 8, 16, kinds=["a", "b"], default_fc_parameters=EfficientFCParameters(), kind_to_fc_parameters=k2fc)
    assert ex.columns == _plans(["a", "b"], EfficientFCParameters(), k2fc)[1]
    assert make(100, 8, 16).columns == _plans(["value"], None, None)[1]


def test_refusals_at_the_call(no_device):
    ex = make(10, 4, 16, kinds=["a", "b"], default_fc_parameters=MIN)
    W = len(ex.columns)
    ids, values, sort, kind = rows(10)
    with pytest.raises(ValueError, match="11 rows, the extractor was built for at most 10"):
        ex(*rows(11))
    with pytest.raises(TypeError, match="values must be float32, float64"):
        ex(ids, torch.zeros(10, dtype=torch.int32, device=META), sort, kind)
    with pytest.raises(TypeError, match="sort must be int64 or float64"):
        ex(ids, values, torch.zeros(10, device=META), kind)
    with pytest.raises(ValueError, match="without kind codes there is one kind, 2 named"):
        ex(ids, values, sort)
    with pytest.raises(ValueError, match="kind has 9 rows, ids 10"):
        ex(ids, values, sort, kind[:9])
    with pytest.raises(ValueError, match="ids is on meta, the extractor on cuda:0"):
        ex(ids, values, sort, kind)
    with pytest.raises(ValueError, match=r"out has shape \(10, %d\), the result is \(4, %d\)" % (W, W)):
        ex(ids, values, sort, kind, out=torch.empty((10, W), dtype=torch.float64, device=META))
    with pytest.raises(TypeError, match="out must be float64"):
        ex(ids, values, sort, kind, out=torch.empty((4, W), dtype=torch.float32, device=META))
    with pytest.raises(ValueError, match="unit column stride"):
        ex(ids, values, sort, kind, out=torch.empty((W, 4), dtype=torch.float64, device=META).t())
    with pytest.raises(TypeError, match="n_rows must be a torch.Tensor"):
        ex(ids, values, sort, kind, n_rows=5)
    with pytest.raises(ValueError, match="n_rows must be a 0-d int64 tensor"):
        ex(ids, values, sort, kind, n_rows=torch.tensor([5], device=META))
    with pytest.raises(ValueError, match="n_rows must be a 0-d int64 tensor"):
        ex(ids, values, sort, kind, n_rows=torch.tensor(5, dtype=torch.int32, device=META))
    ex.device = torch.device(META)               # the rows' device, to reach the checks of the other tensors' devices
    with pytest.raises(ValueError, match="kind is on cpu, the extractor on meta"):
        ex(ids, values, sort, torch.zeros(10, dtype=torch.int64))
    with pytest.raises(ValueError, match="out is on cpu, the extractor on meta"):
        ex(ids, values, sort, kind, out=torch.empty((4, W), dtype=torch.float64))
    with pytest.raises(ValueError, match="n_rows is on cpu, the extractor on meta"):
        ex(ids, values, sort, kind, n_rows=torch.tensor(5))


@pytest.mark.parametrize("args", [
    dict(ids=[0, 1]),
    dict(ids=torch.zeros((2, 3), dtype=torch.int64)),
    dict(ids=torch.zeros(6, dtype=torch.int32)),
    dict(values=torch.zeros((6, 1))),
    dict(values=torch.zeros(6, dtype=torch.int64)),
    dict(sort=torch.zeros(6)),
    dict(sort=torch.zeros(5, dtype=torch.int64)),
    dict(kind=torch.zeros(6, dtype=torch.int16)),
    dict(kind=torch.zeros((3, 2), dtype=torch.int64)),
])
def test_same_layout_checks_as_extract_features_long_device(no_device, args):
    """Every layout error extract_features_long_device raises for the tensors, the call raises with the same message."""
    ex = make(10, 4, 16, kinds=["a"], default_fc_parameters=MIN)
    call = dict(dict(ids=torch.zeros(6, dtype=torch.int64), values=torch.zeros(6), sort=None,
                     kind=torch.zeros(6, dtype=torch.int64)), **args)
    with pytest.raises((TypeError, ValueError)) as want:
        extract_features_long_device(call["ids"], call["values"], call["sort"], call["kind"], kinds=["a"],
                                     default_fc_parameters=MIN)
    with pytest.raises(want.type, match=re.escape(str(want.value))):
        ex(call["ids"], call["values"], call["sort"], call["kind"])
