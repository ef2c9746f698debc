"""The reference's plugin seam #1 (tsfresh/utilities/distribution.py:64-105): a Distributor whose
`map_reduce` evaluates the whole `data` object on the GPU instead of mapping a Python function over chunks.

    from tsfresh import extract_features                 # the unmodified reference driver
    from tsfresh_b200.distributor import B200Distributor
    X = extract_features(df, column_id="id", column_sort="time", distributor=B200Distributor())

`extract_features` calls `distributor.map_reduce(_do_extraction_on_chunk, data=<TsData>, chunk_size=...,
function_kwargs={default_fc_parameters, kind_to_fc_parameters, show_warnings})` (extraction.py:288-299) and
pivots the returned (id, name, value) triples (data.py:86-121).  The Python `map_function` is never called.
"""
import numpy as np


def _reference_base():
    try:
        from tsfresh.utilities.distribution import DistributorBaseClass
        return DistributorBaseClass
    except Exception:
        return object


def is_distributor(obj):
    base = _reference_base()
    return (base is not object and isinstance(obj, base)) or hasattr(obj, "map_reduce")


class B200Distributor(_reference_base()):
    def __init__(self, device=None):
        self.device = device

    def map_reduce(self, map_function, data, function_kwargs=None, chunk_size=None, data_length=None):
        from .extraction import do_extraction_on_chunks
        kw = function_kwargs or {}
        # the adapter already grouped by (id, kind) and sorted by time; all chunks go to the device together
        return do_extraction_on_chunks(data, kw.get("default_fc_parameters") or {}, kw.get("kind_to_fc_parameters") or {},
                                       show_warnings=kw.get("show_warnings", False), device=self.device)

    def close(self):
        pass


def _reference_tsdata_base():
    try:
        from tsfresh.feature_extraction.data import TsData
        return TsData
    except Exception:
        return object


class CsrTsData(_reference_tsdata_base()):
    """The reference's plugin seam #2 (tsfresh/feature_extraction/data.py:60-72, 488-489): `to_tsdata` returns any
    TsData instance unchanged; a non-iterable one is routed to ApplyDistributor, which calls
    `data.apply(map_function, meta=..., **function_kwargs)` and later `data.pivot(result)`
    (extraction.py:276-304, distribution.py:497-509).  This class holds the series already in CSR form
    (`values[begin[s] : begin[s] + length[s]]`, ids ascending) so the unmodified reference driver runs zero-copy:

        X = tsfresh.extract_features(CsrTsData(values, begin, length, ids), default_fc_parameters=...)
    """

    column_id = "id"

    def __init__(self, values, begin, length, ids, kind="value", device=None):
        self.values = np.ascontiguousarray(values, dtype=np.float32)
        self.begin = np.ascontiguousarray(begin, dtype=np.int64)
        self.length = np.ascontiguousarray(length, dtype=np.int32)
        self.ids = np.asarray(ids)
        self.kind = str(kind)
        self.device = device
        if not (len(self.begin) == len(self.length) == len(self.ids)):
            raise ValueError("begin, length and ids must have one entry per series")

    def apply(self, f, meta=None, default_fc_parameters=None, kind_to_fc_parameters=None, **_):
        from .extraction import _device_plan, _kind_plan, get_context
        plan, names = _kind_plan(self.kind, default_fc_parameters or {}, kind_to_fc_parameters)
        return names, _device_plan(get_context(self.device), plan).extract_csr(self.values, self.begin, self.length)

    def pivot(self, results):
        import pandas as pd
        names, mat = results
        frame = pd.DataFrame(mat, index=pd.Index(self.ids), columns=names, copy=False)
        return frame if frame.index.is_monotonic_increasing else frame.sort_index()
