"""extract_features_device: the argument checks that need no device, and the column names of K kinds."""
import pytest

from tsfresh_b200 import ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, extract_features_device
from tsfresh_b200.device_api import _plans
from tsfresh_b200.plan import Plan

torch = pytest.importorskip("torch")

MIN = MinimalFCParameters()
MIN_W = len(Plan(MIN).suffixes)


def call(*args, **kw):
    kw.setdefault("default_fc_parameters", MIN)
    return extract_features_device(*args, **kw)


@pytest.mark.parametrize("values, exc, match", [
    ([[1.0, 2.0]], TypeError, "torch.Tensor"),
    (torch.zeros((4, 8), dtype=torch.int32), TypeError, "float32, float64"),
    (torch.zeros(8), ValueError, r"\[N, L\] or \[N, L, K\]"),
    (torch.zeros((2, 3, 4, 5)), ValueError, r"\[N, L\] or \[N, L, K\]"),
    (torch.zeros((4, 8, 0)), ValueError, "no kind"),
])
def test_dense_layout(values, exc, match):
    with pytest.raises(exc, match=match):
        call(values)


def test_csr_layout():
    v, b, n = torch.zeros(100), torch.zeros(5, dtype=torch.int64), torch.ones(5, dtype=torch.int32)
    with pytest.raises(ValueError, match="together"):
        call(v, b)
    with pytest.raises(ValueError, match="together"):
        call(v, length=n)
    with pytest.raises(TypeError, match="begin must be int64"):
        call(v, b.to(torch.int32), n)
    with pytest.raises(TypeError, match="length must be int32 or int64"):
        call(v, b, n.to(torch.float32))
    with pytest.raises(TypeError, match="begin must be a torch.Tensor"):
        call(v, [0, 1], n)
    with pytest.raises(ValueError, match="begin must be 1-D"):
        call(v, b.reshape(5, 1), n)
    with pytest.raises(ValueError, match="begin has 5 entries, length 4"):
        call(v, b, n[:4])
    with pytest.raises(ValueError, match=r"\[R\] or \[R, K\]"):
        call(torch.zeros((10, 10, 2)), b, n)


def test_kinds():
    x = torch.zeros((4, 8, 2))
    with pytest.raises(ValueError, match="3 kinds named for 2"):
        call(x, kinds=["a", "b", "c"])
    with pytest.raises(ValueError, match="distinct"):
        call(x, kinds=["a", "a"])
    with pytest.raises(ValueError, match="'__'"):
        call(x, kinds=["a__b", "c"])
    with pytest.raises(ValueError, match="'_'"):
        call(x, kinds=["a_", "c"])


def test_out():
    x = torch.zeros((4, 8))
    with pytest.raises(TypeError, match="out must be float64"):
        call(x, out=torch.zeros((4, MIN_W), dtype=torch.float32))
    with pytest.raises(TypeError, match="out must be a torch.Tensor"):
        call(x, out=[[0.0] * MIN_W] * 4)
    with pytest.raises(ValueError, match=r"out has shape \(4, %d\), the result is \(4, %d\)" % (MIN_W + 1, MIN_W)):
        call(x, out=torch.zeros((4, MIN_W + 1), dtype=torch.float64))
    with pytest.raises(ValueError, match="unit column stride"):
        call(x, out=torch.zeros((MIN_W, 4), dtype=torch.float64).t())
    with pytest.raises(ValueError, match="unit column stride"):
        call(x, out=torch.zeros((4, 2 * MIN_W), dtype=torch.float64)[:, ::2])


def test_cpu_tensor_is_refused_after_the_layout_checks():
    with pytest.raises(ValueError, match="must be a CUDA tensor"):
        call(torch.zeros((4, 8)))
    with pytest.raises(ValueError, match="must be a CUDA tensor"):
        call(torch.zeros(10), torch.zeros(2, dtype=torch.int64), torch.ones(2, dtype=torch.int64))


def test_column_names_of_k_kinds():
    # extract_features on a wide frame: "{kind}__{suffix}" per kind in kind order, kind_to_fc_parameters looked up with
    # the raw kind, no DatetimeIndex (linear_trend_timewise skipped)
    plans, cols = _plans([0, 1, 2], None, None)
    comp = Plan(ComprehensiveFCParameters()).suffixes
    assert cols == ["%d__%s" % (k, s) for k in range(3) for s in comp]
    assert not any("linear_trend_timewise" in c for c in cols)
    k2fc = {"b": MIN, 7: {"mean": None}}
    plans, cols = _plans(["a", "b", 7], EfficientFCParameters(), k2fc)
    eff = Plan(EfficientFCParameters()).suffixes
    assert cols == ["a__" + s for s in eff] + ["b__" + s for s in Plan(MIN).suffixes] + ["7__mean"]
    assert [p.n_cols for p in plans] == [len(eff), MIN_W, 1]
    plans, cols = _plans(["a", "b"], None, {"b": MIN})            # no default settings: the other kinds give nothing
    assert cols == ["b__" + s for s in Plan(MIN).suffixes] and plans[0].n_cols == 0
