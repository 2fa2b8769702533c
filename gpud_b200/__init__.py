"""gpud_b200 — H100-native (sm_90a) telemetry aggregation + Xid scan hot path of gpud behind a C ABI (include/gpud_b200.h).

The product is `libgpud_b200.so` (hand-written sm_90a CUDA, gpud_b200/csrc).  This package is only the Python
binding over that C ABI used by the tests and bench.py; it contains no compute and no CPU fallback: every entry
point raises if the shared library or a CUDA device is missing.
"""
from .capi import (Context, GpudError, Ring, RingWindows, rings_reduce_range_sets, BoxQuery, FabricRaw, FabricLocal, FabricVerdict, XidHit, lib, OPS, EVENT_NAMES,
                   ACTION_WIRE, SCAN_LINES, SCAN_RAW_KMSG, SCAN_FM_LOG, SCAN_EXT_MATCHERS, HIT_FM_TIME, FmLogSyncer, DTYPES, KmsgStateful, KmsgEvent, KmsgDedupDevice, Poller, POLL_FIELDS, IbSnapshot, IbVerdict, ib_reason, Store, Metric, DedupRule, EventRow, xid_build_message, xid_hit_message, xid_detail, Temperature, PollCounters, temperature_check, fabric_reason, hw_slowdown_event_message, hw_slowdown_check, temperature_reason, fabric_report_reason)

__all__ = ["Context", "GpudError", "Ring", "RingWindows", "rings_reduce_range_sets", "BoxQuery", "FabricRaw", "FabricLocal", "FabricVerdict", "XidHit", "lib", "OPS",
           "EVENT_NAMES", "ACTION_WIRE", "SCAN_LINES", "SCAN_RAW_KMSG", "SCAN_FM_LOG", "SCAN_EXT_MATCHERS", "HIT_FM_TIME", "FmLogSyncer", "DTYPES", "KmsgStateful", "KmsgEvent", "KmsgDedupDevice", "Poller", "POLL_FIELDS", "IbSnapshot", "IbVerdict", "ib_reason", "Store", "Metric", "DedupRule", "EventRow", "xid_build_message", "xid_hit_message", "xid_detail", "Temperature", "PollCounters", "temperature_check", "fabric_reason", "hw_slowdown_event_message", "hw_slowdown_check", "temperature_reason", "fabric_report_reason"]
