"""ctypes binding of libbfq_gpumatch.so (the C-ABI of include/bfq_gpumatch.h).

There is no fallback: if the library is missing this module raises, and every match call needs a CUDA device.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BFQ_LIB") or os.path.join(_HERE, "libbfq_gpumatch.so")   # BFQ_LIB: A/B experiments only
WORKLOAD_LIB_PATH = os.path.join(_HERE, "libbfq_workload.so")


class NativeError(RuntimeError):
    pass


class BfqRange(C.Structure):
    _fields_ = [("first", C.c_uint32), ("count", C.c_uint32)]


class BfqThrottled(C.Structure):
    _fields_ = [("topic", C.c_uint32), ("rank", C.c_uint32), ("kind", C.c_uint32)]


class BfqDeviceResult(C.Structure):
    _fields_ = [("d_span_begin", C.c_void_p), ("d_span_count", C.c_void_p), ("d_route_count", C.c_void_p),
                ("d_ranges", C.c_void_p), ("d_throttled", C.c_void_p), ("n_ranges", C.c_int64),
                ("n_throttled", C.c_int64), ("n_routes", C.c_int64), ("n_overflow_topics", C.c_int64),
                ("n_flagged_topics", C.c_int64), ("n_launches", C.c_int64), ("n_topics", C.c_int64), ("n_distinct_topics", C.c_int64),
                ("tier0_ms", C.c_double), ("generation", C.c_uint64), ("lease", C.c_void_p)]


class BfqRDeviceResult(C.Structure):
    _fields_ = [("d_offsets", C.c_void_p), ("d_ids", C.c_void_p), ("d_total", C.c_void_p), ("n_filters", C.c_int64),
                ("n_ids", C.c_int64), ("n_ranges", C.c_int64), ("n_overflow_filters", C.c_int64), ("generation", C.c_uint64),
                ("device_ms", C.c_double), ("kernel_ms", C.c_double), ("lease", C.c_void_p)]


class BfqGathered(C.Structure):
    _fields_ = [("d_route_count", C.c_void_p), ("d_span_count", C.c_void_p), ("d_ranges", C.c_void_p),
                ("topic_base", C.POINTER(C.c_int64)), ("range_base", C.POINTER(C.c_int64)), ("topic_count", C.POINTER(C.c_int64)),
                ("range_count", C.POINTER(C.c_int64)), ("n_topics_total", C.c_int64),
                ("n_ranges_total", C.c_int64), ("bytes_received", C.c_int64), ("world", C.c_int32)]


class BfqFanoutResult(C.Structure):
    _fields_ = [("d_pack_offsets", C.c_void_p), ("d_pack_topic", C.c_void_p), ("d_pack_rank", C.c_void_p), ("d_pack_member", C.c_void_p),
                ("n_pairs", C.c_int64), ("n_deliverers", C.c_int32), ("ordered_share_id", C.c_int32), ("generation", C.c_uint64)]


class BfqDeliveryResult(C.Structure):
    _fields_ = [("d_package_off", C.c_void_p), ("d_package_tenant", C.c_void_p), ("d_pack_off", C.c_void_p),
                ("d_pack_topic", C.c_void_p), ("d_match_off", C.c_void_p), ("d_match_rank", C.c_void_p),
                ("d_match_member", C.c_void_p), ("n_pairs", C.c_int64), ("n_packages", C.c_int64), ("n_packs", C.c_int64),
                ("n_deliverers", C.c_int32), ("ordered_share_id", C.c_int32), ("generation", C.c_uint64)]


class BfqDeliveryOrderedResult(C.Structure):
    _fields_ = [("d", BfqDeliveryResult), ("d_pack_pub_off", C.c_void_p), ("d_pack_pub", C.c_void_p), ("n_pack_pubs", C.c_int64),
                ("n_ordered_packs", C.c_int64)]


class BfqDeliveryWireResult(C.Structure):
    _fields_ = [("d_req_off", C.c_void_p), ("n_bytes", C.c_int64), ("n_match_infos", C.c_int64), ("n_skipped", C.c_int64),
                ("n_deliverers", C.c_int32), ("ordered_share_id", C.c_int32), ("generation", C.c_uint64)]


class BfqStaleMatch(C.Structure):
    _fields_ = [("deliverer", C.c_int32), ("tenant", C.c_int32), ("rank", C.c_uint32), ("member", C.c_uint32),
                ("reply_off", C.c_int64), ("reply_len", C.c_int32), ("code", C.c_int32)]


class BfqDeliveryReplyResult(C.Structure):
    _fields_ = [("d_pair_code", C.c_void_p), ("d_status", C.c_void_p), ("d_stale", C.c_void_p), ("n_code", C.c_int64 * 8),
                ("n_pairs", C.c_int64), ("n_stale", C.c_int64), ("n_fallback", C.c_int32), ("n_deliverers", C.c_int32),
                ("ordered_share_id", C.c_int32), ("generation", C.c_uint64)]


class BfqBudgetResult(C.Structure):
    _fields_ = [("d_delivered_persistent", C.c_void_p), ("d_topic_flags", C.c_void_p), ("n_delivered", C.c_int64),
                ("n_dropped_bytes", C.c_int64), ("n_dropped_persistent_bandwidth", C.c_int64),
                ("n_dropped_transient_bandwidth", C.c_int64)]


BUDGET_BYTES_THROTTLED, BUDGET_NO_PERSISTENT_BW, BUDGET_NO_TRANSIENT_BW, BUDGET_METERED = 1, 2, 4, 8
EXCHANGE_ID_BYTES, EXCHANGE_COUNTS, EXCHANGE_RANGES = 128, 1, 2
_vp, _i32, _i64 = C.c_void_p, C.c_int32, C.c_int64
_SIGNATURES = {
    "bfq_last_error": (C.c_char_p, []),
    "bfq_index_create": (_i32, [_i32, C.POINTER(_vp)]),
    "bfq_index_destroy": (None, [_vp]),
    "bfq_index_reset": (_i32, [_vp]),
    "bfq_index_load": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64]),
    "bfq_index_apply": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64]),
    "bfq_index_commit": (_i32, [_vp]),
    "bfq_index_generation": (_i32, [_vp, C.POINTER(C.c_uint64)]),
    "bfq_index_set_option": (_i32, [_vp, C.c_char_p, _i64]),
    "bfq_index_stats": (_i32, [_vp, _vp, _i32]),
    "bfq_host_build_stats": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp, _i32]),
    "bfq_index_last_kernel_ms": (_i32, [_vp, C.POINTER(C.c_double)]),
    "bfq_route_lookup": (_i32, [_vp, _i64, _vp, _i64, C.POINTER(_i64), _vp, _i64, C.POINTER(_i64)]),
    "bfq_route_kind": (_i32, [_vp, _i64, C.POINTER(_i32)]),
    "bfq_route_kinds": (_i32, [_vp, _vp, _i64, _vp]),
    "bfq_match": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp, C.POINTER(_vp)]),
    "bfq_result_num_topics": (_i64, [_vp]),
    "bfq_result_span_begin": (_vp, [_vp]),
    "bfq_result_span_count": (_vp, [_vp]),
    "bfq_result_route_count": (_vp, [_vp]),
    "bfq_result_ranges": (_vp, [_vp, C.POINTER(_i64)]),
    "bfq_result_throttled": (_vp, [_vp, C.POINTER(_i64)]),
    "bfq_result_expand": (_i64, [_vp, _vp, _vp, _i64]),
    "bfq_result_route_lookup": (_i32, [_vp, _i64, _vp, _i64, C.POINTER(_i64), _vp, _i64, C.POINTER(_i64)]),
    "bfq_result_route_kinds": (_i32, [_vp, _vp, _i64, _vp]),
    "bfq_result_generation": (C.c_uint64, [_vp]),
    "bfq_result_timings": (_i32, [_vp, _vp, _i32]),
    "bfq_result_free": (None, [_vp]),
    "bfq_match_device": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp, _vp, C.POINTER(BfqDeviceResult)]),
    "bfq_match_device_async": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp, _vp, C.POINTER(BfqDeviceResult)]),
    "bfq_device_result_wait": (_i32, [C.POINTER(BfqDeviceResult)]),
    "bfq_device_result_release": (None, [C.POINTER(BfqDeviceResult)]),
    "bfq_expand_device": (_i32, [C.POINTER(BfqDeviceResult), _vp, _vp, _i64, _vp, C.POINTER(_i64)]),
    "bfq_expand_device_budget": (_i32, [C.POINTER(BfqDeviceResult), _vp, _vp, _vp, _vp, _vp, _i64, _vp, C.POINTER(BfqBudgetResult)]),
    "bfq_range_lookup": (_i32, [_i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "bfq_fanout_device": (_i32, [C.POINTER(BfqDeviceResult), _vp, _vp, _i64, _vp, C.POINTER(BfqFanoutResult)]),
    "bfq_fanout_deliverer": (_i32, [_vp, _i32, C.POINTER(_i32), _vp, _i64, C.POINTER(_i64)]),
    "bfq_delivery_device": (_i32, [C.POINTER(BfqDeviceResult), _vp, _vp, _i64, _vp, _vp, C.POINTER(BfqDeliveryResult)]),
    "bfq_delivery_device_ordered": (_i32, [C.POINTER(BfqDeviceResult), _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp,
                                           C.POINTER(BfqDeliveryOrderedResult)]),
    "bfq_delivery_encode": (_i32, [C.POINTER(BfqDeviceResult), C.POINTER(BfqDeliveryResult), _vp, _vp, _i32, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _i64, _vp, C.POINTER(BfqDeliveryWireResult)]),
    "bfq_delivery_encode_ordered": (_i32, [C.POINTER(BfqDeviceResult), C.POINTER(BfqDeliveryOrderedResult), _vp, _vp, _i32, _vp,
                                           _vp, _vp, _vp, _vp, _vp, _i64, _vp, C.POINTER(BfqDeliveryWireResult)]),
    "bfq_delivery_reply": (_i32, [C.POINTER(BfqDeviceResult), C.POINTER(BfqDeliveryResult), _vp, _vp, _i32, _vp, _vp, _vp,
                                  C.POINTER(BfqDeliveryReplyResult)]),
    "bfq_exchange_unique_id": (_i32, [_vp, _i32]),
    "bfq_exchange_create": (_i32, [_i32, _i32, _i32, _vp, C.POINTER(_vp)]),
    "bfq_exchange_destroy": (None, [_vp]),
    "bfq_exchange_gather": (_i32, [_vp, C.POINTER(BfqDeviceResult), _i32, _vp, C.POINTER(BfqGathered)]),
    "bfq_receiver_url": (_i64, [_i32, C.c_char_p, _i64, C.c_char_p, _i64, _vp, _i64]),
    "bfq_route_key": (_i64, [C.c_char_p, _i64, C.c_char_p, _i64, C.c_char_p, _i64, _vp, _i64]),
    "bfq_tenant_begin_key": (_i64, [C.c_char_p, _i64, _vp, _i64]),
    "bfq_retain_key": (_i64, [C.c_char_p, _i64, C.c_char_p, _i64, _vp, _i64]),
    "bfq_retain_key_prefix": (_i64, [C.c_char_p, _i64, C.c_char_p, _i64, _vp, _i64]),
    "bfq_is_valid_topic": (_i32, [C.c_char_p, _i64, _i32, _i32, _i32]),
    "bfq_is_valid_topic_filter": (_i32, [C.c_char_p, _i64, _i32, _i32, _i32]),
    "bfq_rindex_create": (_i32, [_i32, C.POINTER(_vp)]),
    "bfq_rindex_destroy": (None, [_vp]),
    "bfq_rindex_reset": (_i32, [_vp]),
    "bfq_rindex_add": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp]),
    "bfq_rindex_load_keys": (_i32, [_vp, _vp, _vp, _i64, _vp]),
    "bfq_rresult_retain_keys": (_i64, [_vp, _vp, _vp, _i64, _vp]),
    "bfq_rindex_remove": (_i32, [_vp, C.c_char_p, _i64, C.c_char_p, _i64]),
    "bfq_rindex_commit": (_i32, [_vp]),
    "bfq_rindex_stats": (_i32, [_vp, _vp, _i32]),
    "bfq_rindex_lookup": (_i32, [_vp, _i64, _vp, _i64, C.POINTER(_i64), _vp, _i64, C.POINTER(_i64)]),
    "bfq_rmatch": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, C.POINTER(_vp)]),
    "bfq_rresult_num_filters": (_i64, [_vp]),
    "bfq_rresult_offsets": (_vp, [_vp]),
    "bfq_rresult_ids": (_vp, [_vp, C.POINTER(_i64)]),
    "bfq_rresult_total_matches": (_vp, [_vp]),
    "bfq_rresult_timings": (_i32, [_vp, _vp, _i32]),
    "bfq_rresult_generation": (C.c_uint64, [_vp]),
    "bfq_rresult_free": (None, [_vp]),
    "bfq_rmatch_device": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _vp, C.POINTER(BfqRDeviceResult)]),
    "bfq_rdevice_result_release": (None, [C.POINTER(BfqRDeviceResult)]),
    "bfq_rretain_keys_device": (_i32, [_vp, C.POINTER(BfqRDeviceResult), _vp, _vp, _i64, _vp, C.POINTER(_i64)]),
}

_lib = None


def load_library(path=LIB_PATH):
    """Load the CUDA library and bind every symbol include/bfq_gpumatch.h declares. Raises NativeError when the
    extension has not been built (run `python -c "import __graft_entry__ as g; g.build()"`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise NativeError("%s is missing: build it with __graft_entry__.build() (no CPU fallback exists)" % path)
    lib_ = C.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib_, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib_
    return _lib


class _LazyLib:
    def __getattr__(self, name):
        return getattr(load_library(), name)


lib = _LazyLib()


def check(rc):
    if rc != 0:
        raise NativeError("bfq error %d: %s" % (rc, load_library().bfq_last_error().decode("utf-8", "replace")))


def as_blob(strings):
    """list[str|bytes] -> (uint8 array, int64 offsets[n+1])"""
    bs = [s.encode("utf-8") if isinstance(s, str) else bytes(s) for s in strings]
    off = np.zeros(len(bs) + 1, dtype=np.int64)
    if bs:
        off[1:] = np.cumsum([len(b) for b in bs])
    joined = b"".join(bs)
    data = np.frombuffer(joined, dtype=np.uint8).copy() if joined else np.zeros(1, np.uint8)
    return data, off


def ptr(a):
    return a.ctypes.data if a is not None else None
