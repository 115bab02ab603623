"""urban_road_filter_b200 — H100-native (sm_90a) per-scan road/curb classification behind the C-ABI of include/urf.h."""
from .ctypes_abi import (DEFAULTS, FULL_ROI, LABEL_CURB, LABEL_NONE, LABEL_OUTSIDE, LABEL_ROAD, UrfParams, UrfResult,
                         UrfStrip, make_params)

__all__ = ["DEFAULTS", "FULL_ROI", "LABEL_CURB", "LABEL_NONE", "LABEL_OUTSIDE", "LABEL_ROAD", "UrfParams",
           "UrfResult", "UrfStrip", "make_params"]
