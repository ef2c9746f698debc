"""extract_features_long_device: the argument checks that need no device."""
import pytest

from tsfresh_b200 import MinimalFCParameters, extract_features_long_device

torch = pytest.importorskip("torch")

I64 = torch.zeros(6, dtype=torch.int64)
F32 = torch.zeros(6)


def call(ids=I64, values=F32, sort=None, kind=None, **kw):
    kw.setdefault("default_fc_parameters", MinimalFCParameters())
    return extract_features_long_device(ids, values, sort, kind, **kw)


@pytest.mark.parametrize("args, exc, match", [
    (dict(ids=[0, 1]), TypeError, "ids must be a torch.Tensor"),
    (dict(ids=None), TypeError, "ids must be a torch.Tensor"),
    (dict(values=None), TypeError, "values must be a torch.Tensor"),
    (dict(values=F32.numpy()), TypeError, "values must be a torch.Tensor"),
    (dict(sort=[0] * 6), TypeError, "sort must be a torch.Tensor"),
    (dict(kind=[0] * 6, kinds=["a"]), TypeError, "kind must be a torch.Tensor"),
    (dict(times=[0] * 6), TypeError, "times must be a torch.Tensor"),
    (dict(ids=I64.reshape(2, 3)), ValueError, "ids must be 1-D"),
    (dict(values=F32.reshape(6, 1)), ValueError, "values must be 1-D"),
    (dict(kind=I64.reshape(3, 2), kinds=["a"]), ValueError, "kind must be 1-D"),
    (dict(ids=I64.to(torch.int32)), TypeError, "ids must be int64"),
    (dict(values=I64), TypeError, "values must be float32, float64"),
    (dict(sort=F32), TypeError, "sort must be int64 or float64"),
    (dict(kind=I64.to(torch.int16), kinds=["a"]), TypeError, "kind must be int32 or int64"),
    (dict(times=F32.double()), TypeError, "times must be int64"),
])
def test_column_types_and_shapes(args, exc, match):
    with pytest.raises(exc, match=match):
        call(**args)


@pytest.mark.parametrize("name", ["values", "sort", "kind", "times"])
def test_length_mismatch(name):
    short = {"values": F32[:5], "sort": I64[:5], "kind": I64[:5], "times": I64[:5]}[name]
    kw = {name: short}
    if name == "kind":
        kw["kinds"] = ["a"]
    with pytest.raises(ValueError, match="%s has 5 rows, ids 6" % name):
        call(**kw)


def test_kinds():
    with pytest.raises(ValueError, match="one kind, 2 named"):
        call(kinds=["a", "b"])
    with pytest.raises(ValueError, match="kinds must name the kinds"):
        call(kind=I64)
    with pytest.raises(ValueError, match="between 1 and 64 kinds, 0 named"):
        call(kind=I64, kinds=[])
    with pytest.raises(ValueError, match="between 1 and 64 kinds, 65 named"):
        call(kind=I64, kinds=["k%d" % i for i in range(65)])
    with pytest.raises(ValueError, match="distinct"):
        call(kind=I64, kinds=["a", "a"])
    with pytest.raises(ValueError, match="'__'"):
        call(kind=I64, kinds=["a__b"])
    with pytest.raises(ValueError, match="'_'"):
        call(kinds=["v_"])


def test_cpu_tensors_are_refused_after_the_argument_checks():
    with pytest.raises(ValueError, match="values must be a CUDA tensor"):
        call()
    with pytest.raises(ValueError, match="values must be a CUDA tensor"):
        call(sort=I64, kind=I64.to(torch.int32), kinds=["a"], times=I64)
