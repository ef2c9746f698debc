"""DeviceExtractor: the refusals that need no device -- length limits in the constructor, shapes, dtypes, devices and
`out` at the call -- and its column names."""
import re

import pytest

from tsfresh_b200 import (ComprehensiveFCParameters, DeviceExtractor, EfficientFCParameters, MinimalFCParameters,
                          extract_features_device)
from tsfresh_b200.device_api import _plans

torch = pytest.importorskip("torch")

MIN = MinimalFCParameters()


@pytest.fixture
def no_device(monkeypatch):
    """The constructor up to the device: the library context, plans and status words are not created."""
    monkeypatch.setattr(DeviceExtractor, "_open", lambda self: None)


def make(*args, **kw):
    kw.setdefault("device", "cuda:0")
    return DeviceExtractor(*args, **kw)


def test_length_limits_in_the_constructor(no_device):
    make(8, length=21_000)
    with pytest.raises(ValueError, match="21001 samples exceed the limit of kind 0's settings \\(21000 samples\\)"):
        make(8, length=21_001)
    with pytest.raises(ValueError, match="limit of kind 'b'"):
        make(8, max_length=30_000, kinds=["a", "b"], default_fc_parameters=EfficientFCParameters(),
                        kind_to_fc_parameters={"b": ComprehensiveFCParameters()})
    make(8, max_length=131_072, default_fc_parameters=EfficientFCParameters())
    with pytest.raises(ValueError, match="131073 samples"):
        make(8, max_length=131_073, default_fc_parameters=EfficientFCParameters())
    make(8, length=1_000_000, default_fc_parameters=MIN)       # BASIC / SORTED only: no limit


@pytest.mark.parametrize("kw, match", [
    ({}, "exactly one of length"),
    ({"length": 8, "max_length": 8}, "exactly one of length"),
    ({"length": 0}, "length must be an integer"),
    ({"max_length": 2.5}, "max_length must be an integer"),
    ({"length": 8, "kinds": ["a__b"]}, "'__'"),
    ({"length": 8, "kinds": ["a", "a"]}, "distinct"),
    ({"length": 8, "device": "cpu"}, "CUDA device"),
])
def test_constructor_arguments(no_device, kw, match):
    with pytest.raises(ValueError, match=match):
        make(kw.pop("batch_size", 8), **kw)
    with pytest.raises(ValueError, match="batch_size"):
        make(0, length=8)


def test_columns_are_extract_features_device_names(no_device):
    k2fc = {"b": MIN}
    ex = make(8, length=16, kinds=["a", "b"], default_fc_parameters=EfficientFCParameters(),
                         kind_to_fc_parameters=k2fc)
    assert ex.columns == _plans(["a", "b"], EfficientFCParameters(), k2fc)[1]
    assert make(8, length=16).columns == _plans([0], None, None)[1]


def test_refusals_at_the_call(no_device):
    dense = make(8, length=16, default_fc_parameters=MIN)
    W = len(dense.columns)
    x = torch.zeros((8, 16), device="meta")
    with pytest.raises(ValueError, match="9 series, the extractor was built for at most 8"):
        dense(torch.zeros((9, 16), device="meta"))
    with pytest.raises(ValueError, match="series of 15 samples, the extractor was built for length=16"):
        dense(torch.zeros((8, 15), device="meta"))
    with pytest.raises(TypeError, match="float32, float64"):
        dense(torch.zeros((8, 16), dtype=torch.int32, device="meta"))
    with pytest.raises(ValueError, match="1 kinds named for 3"):
        dense(torch.zeros((8, 16, 3), device="meta"))
    with pytest.raises(ValueError, match="takes CSR|takes dense"):
        dense(torch.zeros(100, device="meta"), torch.zeros(8, dtype=torch.int64, device="meta"),
              torch.ones(8, dtype=torch.int32, device="meta"))
    with pytest.raises(ValueError, match="values is on cpu, the extractor on cuda:0"):
        dense(torch.zeros((8, 16)))
    with pytest.raises(ValueError, match="out has shape"):
        dense(x, out=torch.empty((8, W + 1), dtype=torch.float64, device="meta"))
    with pytest.raises(TypeError, match="out must be float64"):
        dense(x, out=torch.empty((8, W), dtype=torch.float32, device="meta"))
    with pytest.raises(ValueError, match="unit column stride"):
        dense(x, out=torch.empty((W, 8), dtype=torch.float64, device="meta").t())

    csr = make(4, max_length=32, default_fc_parameters=MIN)
    v = torch.zeros(100, device="meta")
    b, n = torch.zeros(4, dtype=torch.int64, device="meta"), torch.ones(4, dtype=torch.int32, device="meta")
    with pytest.raises(ValueError, match="takes CSR views"):
        csr(torch.zeros((4, 32), device="meta"))
    with pytest.raises(ValueError, match="5 series"):
        csr(v, torch.zeros(5, dtype=torch.int64, device="meta"), torch.ones(5, dtype=torch.int32, device="meta"))
    with pytest.raises(TypeError, match="begin must be int64"):
        csr(v, b.to(torch.int32), n)
    with pytest.raises(ValueError, match="values is empty"):
        csr(torch.zeros(0, device="meta"), b, n)
    with pytest.raises(ValueError, match="values is on meta, the extractor on cuda:0"):
        csr(v, b, n)


def test_same_layout_checks_as_extract_features_device(no_device):
    """Every layout error extract_features_device raises for a tensor, the call raises with the same message."""
    ex = make(8, length=8, default_fc_parameters=MIN)
    for values in ([[1.0]], torch.zeros(8), torch.zeros((4, 8, 0))):
        with pytest.raises((TypeError, ValueError)) as want:
            extract_features_device(values, default_fc_parameters=MIN)
        with pytest.raises(want.type, match=re.escape(str(want.value))):
            ex(values)
