"""bifromq_b200 — H100-native batched MQTT topic-filter matcher behind apache/bifromq's dist-worker /
retain-store co-processor seams. The product is the CUDA library (csrc/, C-ABI in include/bfq_gpumatch.h);
this package is the thin host-side mirror of the reference's Java interfaces used by tests and bench.py.
"""
from ._native import NativeError, lib, load_library  # noqa: F401
from .matcher import (GpuRouteIndex, GpuTenantRouteMatcher, GroupFanoutThrottled, MatchedRoutes,  # noqa: F401
                      OutOfTenantResource, PersistentFanoutBytesThrottled, PersistentFanoutThrottled, budget_events)

__all__ = ["GpuRouteIndex", "GpuTenantRouteMatcher", "MatchedRoutes", "PersistentFanoutThrottled",
           "GroupFanoutThrottled", "PersistentFanoutBytesThrottled", "OutOfTenantResource", "budget_events",
           "NativeError", "load_library", "lib"]
