"""tsfresh_b200 -- H100-native (sm_90a) implementation of tsfresh's feature-extraction hot path.

Public surface = the reference's for this path: `extract_features`, the FC-parameter presets and the
imputation helpers that `extract_features(impute_function=...)` takes."""
from .extraction import _do_extraction_on_chunk, do_extraction_on_chunks, extract_features  # noqa: F401
from .dataframe_functions import (add_sub_time_series_index, get_range_values_per_column, impute,  # noqa: F401
                                  impute_dataframe_range, impute_dataframe_zero)
from .device_api import (DeviceExtractor, DeviceLongExtractor, extract_features_device,  # noqa: F401
                         extract_features_forecasting_device, extract_features_long_device, extract_features_rolled_device,
                         extract_features_sub_device)
from .feature_selection import (calculate_relevance_table, calculate_relevance_table_device,  # noqa: F401
                                select_features, select_features_device)
from .rolling import ForecastingFrame, RolledTimeSeries, make_forecasting_frame, roll_time_series  # noqa: F401
from .settings import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters,  # noqa: F401
                       from_columns)

__all__ = ["extract_features", "extract_features_device", "DeviceExtractor", "DeviceLongExtractor", "extract_features_long_device", "extract_features_rolled_device",
           "extract_features_sub_device", "extract_features_forecasting_device", "add_sub_time_series_index", "do_extraction_on_chunks", "impute", "impute_dataframe_zero", "impute_dataframe_range",
           "get_range_values_per_column", "roll_time_series", "RolledTimeSeries", "make_forecasting_frame", "ForecastingFrame", "select_features", "select_features_device", "calculate_relevance_table",
           "calculate_relevance_table_device", "from_columns", "ComprehensiveFCParameters", "EfficientFCParameters", "MinimalFCParameters"]
