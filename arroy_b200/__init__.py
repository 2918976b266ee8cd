"""arroy_b200 — H100-native (sm_90a) distance / split / re-rank path for arroy (see DESIGN.md).

`arroy_b200._capi.Context` is the 1:1 ctypes view of the C ABI in include/arroy_b200.h.
The compute path is the CUDA library only; importing this package never touches oracle/.
"""
from ._capi import (Arena, ArroyB200Error, Context, Group, COSINE, DOT_PRODUCT, EUCLIDEAN, MANHATTAN, METRICS, METRIC_NAMES, LIB_PATH, SIGNATURES, item_placement_plan, load, stage_delta_plan)  # noqa: F401
from .api import ArroyBuilder, ArroyError, Env, QueryBuilder, Reader, StdRng, Writer, reencode  # noqa: F401,E402
