"""ctypes binding of include/gpud_b200.h (the same surface a cgo shim binds; see INTEGRATION.md)."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GPUD_B200_LIB") or os.path.join(_HERE, "libgpud_b200.so")   # override: another build of the library, e.g. the ASan build of tools/build_asan.sh

OPS = {"min": 0, "max": 1, "mean": 2, "ema": 3, "p99": 4, "n_over": 5}
EVENT_NAMES = ["Unknown", "Info", "Warning", "Critical", "Fatal"]
ACTION_WIRE = {1: "IGNORE_NO_ACTION_REQUIRED", 2: "REBOOT_SYSTEM", 3: "HARDWARE_INSPECTION", 4: "CHECK_USER_APP_AND_GPU"}
SCAN_LINES, SCAN_RAW_KMSG, SCAN_FM_LOG = 0, 1, 2
SCAN_EXT_MATCHERS = 0x100
KIND_FM_NVSWITCH_FATAL, KIND_FM_NVSWITCH_NON_FATAL, KIND_FM_NVLINK_FAILURE, KIND_FM_TOPOLOGY_MISMATCH, KIND_FM_NOTHING_TO_DO = 25, 26, 27, 28, 29
HIT_FM_TIME = 0x10
DTYPES = {"float64": 0, "uint32": 1, "int32": 2, "float32": 3, "int64": 4, "uint64": 5, "uint16": 6, "int16": 7, "uint8": 8}   # GPUD_DT_*
MAX_LINKS, MAX_GPUS = 18, 16


class GpudError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("gpud_b200 error %d: %s" % (code, msg))
        self.code = code


class RingCfg(C.Structure):
    _fields_ = [("n_fields", C.c_int32), ("window", C.c_int32), ("capacity", C.c_int64), ("ema_alpha", C.c_double),
                ("q_num", C.c_int32), ("q_den", C.c_int32), ("thresholds", C.POINTER(C.c_double))]


class XidHit(C.Structure):
    _fields_ = [("unit_index", C.c_int64), ("unit_offset", C.c_int64), ("dev_off", C.c_int64), ("dev_len", C.c_int32),
                ("kind", C.c_int32), ("code", C.c_int32), ("flags", C.c_uint32), ("sub_code", C.c_int32),
                ("kmsg_priority", C.c_int32), ("kmsg_seq", C.c_int64), ("kmsg_usec", C.c_int64), ("link", C.c_int64),
                ("intrinfo", C.c_uint32), ("error_status", C.c_uint32), ("extra", C.c_uint32 * 4), ("n_extra", C.c_int32),
                ("severity_fatal", C.c_int32), ("xc", C.c_int32), ("unit_name_off", C.c_int64), ("unit_name_len", C.c_int32),
                ("pid_off", C.c_int64), ("pid_len", C.c_int32), ("pname_off", C.c_int64), ("pname_len", C.c_int32),
                ("inj_off", C.c_int64), ("inj_len", C.c_int32), ("event_type", C.c_int32), ("n_actions", C.c_int32),
                ("actions", C.c_int32 * 4), ("rule_index", C.c_int32), ("detail_variant", C.c_int32),
                ("device", C.c_char * 40), ("unit_name", C.c_char * 40)]

    def as_dict(self) -> dict:
        na = self.n_actions
        return {"line": self.unit_index, "offset": self.unit_offset, "kind": self.kind, "code": self.code,
                "device": self.device.decode("latin-1"), "event_type": self.event_type,
                "actions": [self.actions[i] for i in range(max(na, 0))], "actions_nil": na < 0,
                "extended": bool(self.flags & 1), "sub_code": self.sub_code, "unit": self.unit_name.decode("latin-1"),
                "error_status": self.error_status, "intrinfo": self.intrinfo, "link": self.link,
                "rule_index": self.rule_index, "variant": self.detail_variant, "flags": self.flags,
                "extra": [self.extra[i] for i in range(self.n_extra)], "severity_fatal": self.severity_fatal, "xc": self.xc,
                "kmsg": (self.kmsg_priority, self.kmsg_seq, self.kmsg_usec)}


class Metric(C.Structure):
    _fields_ = [("unix_ms", C.c_int64), ("component", C.c_char_p), ("name", C.c_char_p), ("labels_json", C.c_char_p), ("value", C.c_double)]


def hw_slowdown_event_message(bitmask: int, gpu_uuid: str) -> str:
    buf = C.create_string_buffer(2048)
    n = lib().gpud_hw_slowdown_event_message(bitmask, gpu_uuid.encode(), buf, 2048)
    if n < 0:
        raise GpudError(n, "gpud_hw_slowdown_event_message")
    return buf.value.decode()


def hw_slowdown_check(event_unix, now_unix: int, window_seconds: int = 600, threshold_per_minute: float = 0.6):
    """-> (health 0/2, freq per minute, hardware_inspection, reason)"""
    arr = (C.c_int64 * max(1, len(event_unix)))(*event_unix)
    h, insp, freq = C.c_int32(), C.c_int32(), C.c_double()
    buf = C.create_string_buffer(512)
    rc = lib().gpud_hw_slowdown_check(arr, len(event_unix), now_unix, window_seconds, threshold_per_minute, C.byref(h), C.byref(freq), C.byref(insp), buf, 512)
    if rc:
        raise GpudError(rc, "gpud_hw_slowdown_check")
    return h.value, freq.value, bool(insp.value), buf.value.decode()


def fabric_reason(verdict, gpu_uuids=()) -> str:
    arr = (C.c_char_p * max(1, len(gpu_uuids)))(*[u.encode() for u in gpu_uuids])
    buf = C.create_string_buffer(2048)
    n = lib().gpud_fabric_reason(C.byref(verdict), arr, len(gpu_uuids), buf, 2048)
    if n < 0:
        raise GpudError(n, "gpud_fabric_reason")
    return buf.value.decode()


def fabric_report_reason(raws, gpu_uuids):
    """collectFabricState -> (healthy, reason)"""
    n = len(raws)
    arr = (FabricRaw * max(1, n))(*raws)
    uu = (C.c_char_p * max(1, n))(*[u.encode() for u in gpu_uuids])
    h = C.c_int32()
    buf = C.create_string_buffer(8192)
    rc = lib().gpud_fabric_report_reason(arr, uu, n, C.byref(h), buf, 8192)
    if rc < 0:
        raise GpudError(rc, "gpud_fabric_report_reason")
    return bool(h.value), buf.value.decode()


def xid_detail(xid: int, sub_code: int = 0, error_status: int = 0):
    """getDetailWithSubCodeAndStatus -> None or dict(event_type, actions (None = nil), description, sub_code)"""
    ev, na, var, sc = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    acts = (C.c_int32 * 4)()
    L = lib()
    if not L.gpud_xid_detail(xid, sub_code, error_status, C.byref(ev), C.byref(na), acts, C.byref(var), C.byref(sc)):
        return None
    return {"event_type": ev.value, "actions": None if na.value < 0 else [acts[i] for i in range(na.value)],
            "description": L.gpud_xid_description(xid, var.value).decode("utf-8"), "sub_code": sc.value}


def xid_build_message(xid: int, sub_code: int = 0, error_status: int = 0, description: str = "", device_uuid: str = "", gpu_uuid: str = "") -> str:
    buf = C.create_string_buffer(1024)
    n = lib().gpud_xid_build_message(xid, sub_code, error_status, description.encode(), device_uuid.encode(), gpu_uuid.encode() if gpu_uuid else None, buf, 1024)
    if n < 0:
        raise GpudError(n, "gpud_xid_build_message")
    return buf.value.decode("utf-8")


def xid_hit_message(hit, gpu_uuid: str = "") -> str:
    buf = C.create_string_buffer(1024)
    n = lib().gpud_xid_hit_message(C.byref(hit), gpu_uuid.encode() if gpu_uuid else None, buf, 1024)
    if n < 0:
        raise GpudError(n, "gpud_xid_hit_message")
    return buf.value.decode("utf-8")


class EventRow(C.Structure):
    _fields_ = [("unix_s", C.c_int64), ("name", C.c_char * 64), ("type", C.c_char * 16), ("message_off", C.c_int32), ("message_len", C.c_int32),
                ("extra_off", C.c_int32), ("extra_len", C.c_int32)]


class DedupRule(C.Structure):
    _fields_ = [("event", C.c_char * 32), ("message_contains", C.c_char * 32), ("window_seconds", C.c_int64)]


class Store:
    """the reference's SQLite event / metrics stores, written by the library (gpud_store_*)"""

    def __init__(self, path: str):
        self._L = lib()
        self._h = C.c_void_p()
        rc = self._L.gpud_store_open(path.encode(), C.byref(self._h))
        if rc:
            raise GpudError(rc, "gpud_store_open")

    def _check(self, rc):
        if rc:
            buf = C.create_string_buffer(512)
            self._L.gpud_store_last_error(self._h, buf, 512)
            raise GpudError(rc, buf.value.decode())

    def event_table(self, component: str) -> str:
        out = C.create_string_buffer(256)
        self._check(self._L.gpud_store_event_table(self._h, component.encode(), out, 256))
        return out.value.decode()

    def insert_event(self, table, unix_s, name, typ, message="", extra_info_json=""):
        self._check(self._L.gpud_store_insert_event(self._h, table.encode(), unix_s, name.encode(), typ.encode(), message.encode(), extra_info_json.encode()))

    def insert_xid_hits(self, table, hits, fallback_unix=0, boot_unix=0, raw_kmsg=False) -> int:
        arr = (XidHit * max(1, len(hits)))(*hits)
        n = C.c_int32()
        self._check(self._L.gpud_store_insert_xid_hits(self._h, table.encode(), arr, len(hits), fallback_unix, boot_unix, 1 if raw_kmsg else 0, C.byref(n)))
        return n.value

    def insert_hw_slowdown(self, table, unix_s: int, bitmask: int, gpu_uuid: str) -> bool:
        f = C.c_int32()
        self._check(self._L.gpud_store_insert_hw_slowdown(self._h, table.encode(), unix_s, bitmask, gpu_uuid.encode(), C.byref(f)))
        return bool(f.value)

    def insert_sxid_hits(self, table, hits, fallback_unix=0, boot_unix=0, raw_kmsg=False) -> int:
        arr = (XidHit * max(1, len(hits)))(*hits)
        n = C.c_int32()
        self._check(self._L.gpud_store_insert_sxid_hits(self._h, table.encode(), arr, len(hits), fallback_unix, boot_unix, 1 if raw_kmsg else 0, C.byref(n)))
        return n.value

    def fm_log_syncer(self) -> "FmLogSyncer":
        return FmLogSyncer(self)

    def fm_nothing_to_do(self, table, now_unix: int) -> bool:
        """hasNothingToDoEvent: a fabricmanager_nvswitch_nothing_to_do row newer than now - 10 min"""
        f = C.c_int32()
        self._check(self._L.gpud_fm_nothing_to_do_from_store(self._h, table.encode(), now_unix, C.byref(f)))
        return bool(f.value)

    def syncer(self, component: str):
        h = C.c_void_p()
        self._check(self._L.gpud_kmsg_syncer_create(self._h, component.encode(), C.byref(h)))
        return h

    @staticmethod
    def _row(r, text):
        return (r.unix_s, r.name.decode(), r.type.decode(), text[r.message_off:r.message_off + r.message_len].decode("utf-8"),
                text[r.extra_off:r.extra_off + r.extra_len].decode("utf-8"))

    def get_events(self, table, since_unix: int, cap_rows: int = 4096, cap_text: int = 1 << 20):
        """Bucket.Get: (unix_s, name, type, message, extra_info_json) newest first"""
        rows = (EventRow * max(1, cap_rows))()
        text = C.create_string_buffer(cap_text)
        n = C.c_int32()
        self._check(self._L.gpud_store_get_events(self._h, table.encode(), since_unix, rows, cap_rows, text, cap_text, C.byref(n)))
        return [self._row(rows[i], text.raw) for i in range(n.value)]

    def latest_event(self, table):
        row, text, f = EventRow(), C.create_string_buffer(1 << 16), C.c_int32()
        self._check(self._L.gpud_store_latest_event(self._h, table.encode(), C.byref(row), text, 1 << 16, C.byref(f)))
        return self._row(row, text.raw) if f.value else None

    def purge_events(self, table, before_unix: int) -> int:
        n = C.c_int32()
        self._check(self._L.gpud_store_purge_events(self._h, table.encode(), before_unix, C.byref(n)))
        return n.value

    def xid_state(self, xid_table, os_table, now_unix: int, lookback_seconds: int = 3 * 24 * 3600, reboot_threshold: int = 2, devices=None):
        """-> (health 0/1/2, first suggested action id or 0, reason)"""
        h, a, buf = C.c_int32(), C.c_int32(), C.create_string_buffer(2048)
        spec = ";".join("%s=%s" % kv for kv in (devices or {}).items()).encode()
        self._check(self._L.gpud_xid_state_from_store(self._h, xid_table.encode(), os_table.encode() if os_table else None, now_unix, lookback_seconds, reboot_threshold,
                                                      spec, C.byref(h), C.byref(a), buf, 2048))
        return h.value, a.value, buf.value.decode("utf-8")

    def sxid_state(self, sxid_table, os_table, now_unix: int, lookback_seconds: int = 3 * 24 * 3600):
        h, a, buf = C.c_int32(), C.c_int32(), C.create_string_buffer(2048)
        self._check(self._L.gpud_sxid_state_from_store(self._h, sxid_table.encode(), os_table.encode() if os_table else None, now_unix, lookback_seconds,
                                                       C.byref(h), C.byref(a), buf, 2048))
        return h.value, a.value, buf.value.decode("utf-8")

    def record_reboot(self, os_table, now_unix: int, boot_unix: int) -> bool:
        f = C.c_int32()
        self._check(self._L.gpud_store_record_reboot(self._h, os_table.encode(), now_unix, boot_unix, C.byref(f)))
        return bool(f.value)

    def find_event(self, table, unix_s, name, typ, message="", extra_info_json="") -> bool:
        f = C.c_int32()
        self._check(self._L.gpud_store_find_event(self._h, table.encode(), unix_s, name.encode(), typ.encode(), message.encode(), extra_info_json.encode(), C.byref(f)))
        return bool(f.value)

    def syncer_configure(self, sy, truncate_seconds=60, disable_dedup=False, rules=()):
        """rules: (event, message_contains, window_seconds)"""
        arr = (DedupRule * max(1, len(rules)))()
        for i, (ev, sub, win) in enumerate(rules):
            arr[i].event, arr[i].message_contains, arr[i].window_seconds = ev.encode(), sub.encode(), win
        self._check(self._L.gpud_kmsg_syncer_configure(sy, truncate_seconds, 1 if disable_dedup else 0, arr, len(rules)))

    def syncer_configure_component(self, sy, kmsg_component: str):
        self._check(self._L.gpud_kmsg_syncer_configure_component(sy, kmsg_component.encode()))

    def syncer_offer(self, sy, unix_s: int, name: str, message: str, now_unix: int) -> bool:
        f = C.c_int32()
        self._check(self._L.gpud_kmsg_syncer_offer(sy, unix_s, name.encode(), message.encode(), now_unix, C.byref(f)))
        return bool(f.value)

    def syncer_feed(self, sy, kmsg_component: str, hits, buf: bytes, boot_unix: int, now_unix: int) -> int:
        arr = (XidHit * max(1, len(hits)))(*hits)
        n = C.c_int32()
        self._check(self._L.gpud_kmsg_syncer_feed(sy, kmsg_component.encode(), arr, len(hits), C.cast(C.c_char_p(buf), C.c_void_p), boot_unix, now_unix, C.byref(n)))
        return n.value

    def metrics_table(self, table: str = ""):
        self._check(self._L.gpud_store_metrics_table(self._h, table.encode()))

    def record_metrics(self, rows, table: str = ""):
        """rows: (unix_ms, component, name, labels_json, value)"""
        arr = (Metric * max(1, len(rows)))()
        keep = []
        for i, (ms, comp, name, labels, val) in enumerate(rows):
            b = (comp.encode(), name.encode(), labels.encode())
            keep.append(b)
            arr[i].unix_ms, arr[i].component, arr[i].name, arr[i].labels_json, arr[i].value = ms, b[0], b[1], b[2], val
        self._check(self._L.gpud_store_record_metrics(self._h, table.encode(), arr, len(rows)))

    def close(self):
        if self._h:
            self._L.gpud_store_close(self._h)
            self._h = None


class FmLogSyncer:
    """gpud_fm_log_syncer: the fabric-manager component's line dedup, event dedup and insert for the hits of SCAN_FM_LOG scans."""

    def __init__(self, store: Store):
        self._store, self._L = store, store._L
        h = C.c_void_p()
        store._check(self._L.gpud_fm_log_syncer_create(store._h, C.byref(h)))
        self._h = h
        tab = C.create_string_buffer(256)
        store._check(self._L.gpud_store_event_table(store._h, b"accelerator-nvidia-fabric-manager", tab, 256))
        self.table = tab.value.decode()

    def feed(self, hits, buf: bytes, now_unix: int) -> int:
        arr = (XidHit * max(1, len(hits)))(*hits)
        n = C.c_int32()
        self._store._check(self._L.gpud_fm_log_syncer_feed(self._h, arr, len(hits), C.cast(C.c_char_p(buf), C.c_void_p), now_unix, C.byref(n)))
        return n.value

    def close(self):
        if self._h:
            self._L.gpud_fm_log_syncer_destroy(self._h)
            self._h = None


class IbSnapshot(C.Structure):
    _fields_ = [("ts", C.c_int64), ("total_link_downed", C.c_uint64), ("down", C.c_int32), ("pad", C.c_int32)]


class IbVerdict(C.Structure):
    _fields_ = [("drop", C.c_int32), ("flap", C.c_int32), ("drop_down_since", C.c_int64), ("drop_index", C.c_int64),
                ("flap_down_since", C.c_int64), ("flap_index", C.c_int64), ("n_reverts", C.c_int64)]


def ib_reason(device: str, port: int, down_since: int, flap: bool) -> str:
    out = C.create_string_buffer(256)
    n = lib().gpud_ib_reason(device.encode(), port, down_since, 1 if flap else 0, out, 256)
    if n < 0:
        raise GpudError(n, "gpud_ib_reason")
    return out.value.decode()


POLL_FIELDS = ["temperature_c", "power_mw", "clock_graphics_mhz", "clock_sm_mhz", "clock_mem_mhz", "util_gpu_pct", "util_mem_pct", "memory_used_mib"]


class Temperature(C.Structure):
    _fields_ = [("current_gpu_core_c", C.c_uint32), ("current_hbm_c", C.c_uint32), ("threshold_shutdown_c", C.c_uint32), ("threshold_slowdown_c", C.c_uint32),
                ("threshold_mem_max_c", C.c_uint32), ("threshold_gpu_max_c", C.c_uint32), ("slowdown_margin_c", C.c_int32),
                ("hbm_supported", C.c_uint8), ("margin_supported", C.c_uint8), ("pad", C.c_uint8 * 2)]


class PollCounters(C.Structure):
    _fields_ = [("clock_event_reasons", C.c_uint64), ("ecc_aggregate_corrected", C.c_uint64), ("ecc_aggregate_uncorrected", C.c_uint64),
                ("ecc_volatile_corrected", C.c_uint64), ("ecc_volatile_uncorrected", C.c_uint64), ("clock_events_supported", C.c_uint32),
                ("ecc_read_mask", C.c_uint32)]


def temperature_check(t: "Temperature", margin_threshold_c: int = 0) -> int:
    bits = C.c_int32()
    rc = lib().gpud_temperature_check(C.byref(t), margin_threshold_c, C.byref(bits))
    if rc:
        raise GpudError(rc, "gpud_temperature_check")
    return bits.value


def temperature_reason(readings, gpu_uuids, margin_threshold_c: int = 0):
    """-> (health 0 / 1, reason) of the temperature component over the box's readings"""
    n = len(readings)
    arr = (Temperature * max(1, n))(*readings)
    uu = (C.c_char_p * max(1, n))(*[u.encode() for u in gpu_uuids])
    h = C.c_int32()
    buf = C.create_string_buffer(4096)
    rc = lib().gpud_temperature_reason(arr, uu, n, margin_threshold_c, C.byref(h), buf, 4096)
    if rc < 0:
        raise GpudError(rc, "gpud_temperature_reason")
    return h.value, buf.value.decode("utf-8")


class NvmlDevice(C.Structure):
    _fields_ = [("index", C.c_int32), ("cuda_device", C.c_int32), ("nvml_rc", C.c_int32), ("pad", C.c_int32), ("uuid", C.c_char * 96), ("bus_id", C.c_char * 32),
                ("name", C.c_char * 96)]


class RemappedRows(C.Structure):
    _fields_ = [("remapped_due_to_correctable_errors", C.c_int32), ("remapped_due_to_uncorrectable_errors", C.c_int32), ("remapping_pending", C.c_uint8),
                ("remapping_failed", C.c_uint8), ("supported", C.c_uint8), ("pad", C.c_uint8)]


class EccCounts(C.Structure):
    _fields_ = [("corrected", C.c_uint64), ("uncorrected", C.c_uint64)]


ECC_LOCATIONS = ("total", "l1_cache", "l2_cache", "dram", "sram", "gpu_device_memory", "gpu_texture_memory", "shared_memory", "gpu_register_file")
FIELD_ROW = ("power_instant_mw", "power_average_mw", "memory_temp_c", "total_energy_mj", "ecc_sbe_volatile", "ecc_dbe_volatile", "ecc_sbe_aggregate",
             "ecc_dbe_aggregate", "nvlink_crc_flit_total", "nvlink_crc_data_total", "nvlink_replay_total", "nvlink_recovery_total", "remapped_correctable",
             "remapped_uncorrectable", "remapped_pending", "remapped_failure", "pcie_replay")


class EccErrors(C.Structure):
    _fields_ = [("aggregate", EccCounts * 9), ("volatile_", EccCounts * 9), ("ecc_mode_current", C.c_uint8), ("ecc_mode_pending", C.c_uint8), ("supported", C.c_uint8),
                ("pad", C.c_uint8 * 5)]


GPM_METRICS = ("sm_occupancy", "integer_util", "any_tensor_util", "dfma_tensor_util", "hmma_tensor_util", "imma_tensor_util", "fp64_util", "fp32_util", "fp16_util")
GPM_METRIC_IDS = (3, 4, 5, 6, 7, 9, 11, 12, 13)          # nvml.GPM_METRIC_* of the names above (gpm/component.go:56-64)


class GpmMetrics(C.Structure):
    _fields_ = [("value", C.c_double * 9), ("nvml_rc", C.c_int32 * 9), ("supported", C.c_int32), ("sample_seconds", C.c_double)]

    def as_dict(self):
        return dict(zip(GPM_METRICS, list(self.value)))


def gpm_check(metrics):
    """gpud_gpm_check: (health, reason)"""
    n = len(metrics)
    arr = (GpmMetrics * max(n, 1))(*metrics)
    health = C.c_int32()
    buf = C.create_string_buffer(256)
    k = lib().gpud_gpm_check(arr, n, C.byref(health), buf, 256)
    if k < 0:
        raise GpudError(k, "gpud_gpm_check")
    return health.value, buf.value.decode()


def nvml_devices(cap: int = 16):
    """gpud_nvml_devices: (list of NvmlDevice, driver version)"""
    arr = (NvmlDevice * cap)()
    n = C.c_int32()
    drv = C.create_string_buffer(96)
    rc = lib().gpud_nvml_devices(arr, cap, C.byref(n), drv, 96)
    if rc not in (0, -4):
        raise GpudError(rc, "gpud_nvml_devices")
    return [arr[i] for i in range(min(n.value, cap))], drv.value.decode()


def nvml_devices_arg() -> str:
    buf = C.create_string_buffer(4096)
    rc = lib().gpud_nvml_devices_arg(buf, 4096)
    if rc < 0:
        raise GpudError(rc, "gpud_nvml_devices_arg")
    return buf.value.decode()


def nvml_bus_id(nvml_bus_id_str: str) -> str:
    buf = C.create_string_buffer(64)
    lib().gpud_nvml_bus_id(nvml_bus_id_str.encode(), buf, 64)
    return buf.value.decode()


def remapped_rows_check(rows, bus_ids):
    """gpud_remapped_rows_check: (health, action, reason)"""
    n = len(rows)
    arr = (RemappedRows * max(n, 1))(*rows)
    ids = (C.c_char_p * max(n, 1))(*[b.encode() for b in bus_ids])
    health, action = C.c_int32(), C.c_int32()
    buf = C.create_string_buffer(4096)
    k = lib().gpud_remapped_rows_check(arr, ids, n, C.byref(health), C.byref(action), buf, 4096)
    if k < 0:
        raise GpudError(k, "gpud_remapped_rows_check")
    return health.value, action.value, buf.value.decode()


def poll_row_hold(fresh, nvml_rc, held):
    """gpud_poll_row_hold: the row that goes to the ring when some getters failed; updates `held` in place.  Returns (row, fail_mask)."""
    n = len(fresh)
    f = (C.c_uint32 * n)(*fresh)
    r = (C.c_int32 * n)(*nvml_rc)
    h = (C.c_uint32 * n)(*held)
    out = (C.c_uint32 * n)()
    mask = C.c_uint32()
    rc = lib().gpud_poll_row_hold(f, r, n, h, out, C.byref(mask))
    if rc:
        raise GpudError(rc, "gpud_poll_row_hold")
    held[:] = list(h)
    return list(out), mask.value


class Poller:
    """host NVML poller feeding a ring with raw uint32 poll rows (gpud_poller_*)"""

    def __init__(self, ctx: "Context", ring: "Ring", dev: Optional[int] = None):
        self.ctx, self._L = ctx, ctx._L
        self._h = C.c_void_p()
        dev = ctx.devices[0] if dev is None else dev
        ctx._check(self._L.gpud_poller_create(ctx._h, dev, ring._h, C.byref(self._h)))

    def poll(self, n_polls: int, interval_us: int = 0):
        self.ctx._check(self._L.gpud_poller_poll(self._h, n_polls, interval_us))

    def last_rows(self, cap_rows: int = 1 << 14):
        rows = np.empty((cap_rows, len(POLL_FIELDS)), dtype=np.uint32)
        n, sec = C.c_int64(), C.c_double()
        self.ctx._check(self._L.gpud_poller_last_rows(self._h, C.c_void_p(rows.ctypes.data), cap_rows, C.byref(n), C.byref(sec)))
        return rows[: min(cap_rows, n.value)], sec.value

    def remapped_rows(self) -> "RemappedRows":
        r = RemappedRows()
        self.ctx._check(self._L.gpud_poller_remapped_rows(self._h, C.byref(r)))
        return r

    def ecc_errors(self) -> "EccErrors":
        e = EccErrors()
        self.ctx._check(self._L.gpud_poller_ecc_errors(self._h, C.byref(e)))
        return e

    def gpm_supported(self) -> bool:
        v = C.c_int32()
        self.ctx._check(self._L.gpud_poller_gpm_supported(self._h, C.byref(v)))
        return bool(v.value)

    def gpm_metrics(self, sample_ms: int = 5000) -> "GpmMetrics":
        m = GpmMetrics()
        self.ctx._check(self._L.gpud_poller_gpm_metrics(self._h, sample_ms, C.byref(m)))
        return m

    def poll_gpm(self, ring: "Ring", n_polls: int, sample_ms: int = 5000) -> float:
        sec = C.c_double()
        self.ctx._check(self._L.gpud_poller_poll_gpm(self._h, ring._h, n_polls, sample_ms, C.byref(sec)))
        return sec.value

    def field_row(self):
        """one nvmlDeviceGetFieldValues call: ({name: value}, {name: nvml return code})"""
        v = (C.c_uint64 * len(FIELD_ROW))()
        rc = (C.c_int32 * len(FIELD_ROW))()
        self.ctx._check(self._L.gpud_poller_field_row(self._h, v, rc))
        return dict(zip(FIELD_ROW, list(v))), dict(zip(FIELD_ROW, list(rc)))

    def poll_fields(self, ring: "Ring", n_polls: int, interval_us: int = 0) -> float:
        sec = C.c_double()
        self.ctx._check(self._L.gpud_poller_poll_fields(self._h, ring._h, n_polls, interval_us, C.byref(sec)))
        return sec.value

    def errors(self):
        """(fail_mask, last NVML return code per column, failures per column): getters that failed since create"""
        mask = C.c_uint32()
        rc = (C.c_int32 * len(POLL_FIELDS))()
        nf = (C.c_uint64 * len(POLL_FIELDS))()
        self.ctx._check(self._L.gpud_poller_errors(self._h, C.byref(mask), rc, nf))
        return mask.value, list(rc), list(nf)

    def fabric_raw(self, gpu_index: int = 0, peer_bus_ids=()) -> "FabricRaw":
        """this GPU's NVLink / fabric record read from NVML (GetNVLink, GetFabricState, P2P status against the peers)"""
        raw = FabricRaw()
        arr = (C.c_char_p * max(1, len(peer_bus_ids)))(*[b.encode() if b else None for b in peer_bus_ids])
        self.ctx._check(self._L.gpud_poller_fabric_raw(self._h, gpu_index, arr, len(peer_bus_ids), C.byref(raw)))
        return raw

    def temperature(self) -> "Temperature":
        t = Temperature()
        self.ctx._check(self._L.gpud_poller_temperature(self._h, C.byref(t)))
        return t

    def counters(self) -> "PollCounters":
        c = PollCounters()
        self.ctx._check(self._L.gpud_poller_counters(self._h, C.byref(c)))
        return c

    def product_name(self) -> str:
        buf = C.create_string_buffer(96)
        self.ctx._check(self._L.gpud_poller_product_name(self._h, buf, 96))
        return buf.value.decode()

    def close(self):
        if self._h:
            self._L.gpud_poller_destroy(self._h)
            self._h = None


class KmsgEvent(C.Structure):
    _fields_ = [("unit_index", C.c_int64), ("component", C.c_char * 16), ("event", C.c_char * 32), ("message", C.c_char * 440)]


class KmsgStateful:
    """the reference's two stateful kmsg matchers (os kernel panic, memory OOM) over the primitives of EXT scans"""

    def __init__(self):
        self._L = lib()
        self._h = C.c_void_p()
        if self._L.gpud_kmsg_stateful_create(C.byref(self._h)):
            raise GpudError(-1, "gpud_kmsg_stateful_create")

    def feed(self, hits, buf: bytes, n_units: int, cap: int = 4096):
        arr = (XidHit * max(1, len(hits)))(*hits)
        out = (KmsgEvent * cap)()
        n = C.c_int32()
        rc = self._L.gpud_kmsg_stateful_feed(self._h, arr, len(hits), C.cast(C.c_char_p(buf), C.c_void_p), n_units, out, cap, C.byref(n))
        if rc:
            raise GpudError(rc, "gpud_kmsg_stateful_feed")
        return [(out[i].unit_index, out[i].component.decode(), out[i].event.decode(), out[i].message.decode("latin-1")) for i in range(n.value)]

    def feed_units(self, hits, buf: bytes, n_units: int, dropped: bytes, cap: int = 4096):
        """gpud_kmsg_stateful_feed_units: feed without the units the watcher's dedup dropped (dropped[u] != 0)"""
        arr = (XidHit * max(1, len(hits)))(*hits)
        out = (KmsgEvent * cap)()
        n = C.c_int32()
        rc = self._L.gpud_kmsg_stateful_feed_units(self._h, arr, len(hits), C.cast(C.c_char_p(buf), C.c_void_p), n_units, C.cast(C.c_char_p(dropped), C.c_void_p),
                                                   out, cap, C.byref(n))
        if rc:
            raise GpudError(rc, "gpud_kmsg_stateful_feed_units")
        return [(out[i].unit_index, out[i].component.decode(), out[i].event.decode(), out[i].message.decode("latin-1")) for i in range(n.value)]

    def close(self):
        if self._h:
            self._L.gpud_kmsg_stateful_destroy(self._h)
            self._h = None


class ComponentCfg(C.Structure):
    _fields_ = [("row_remapping_supported", C.c_int32), ("reboot_threshold", C.c_int32), ("margin_threshold_c", C.c_int32), ("nvlink_at_least", C.c_int32)]


class Component:
    """gpud_component_*: the mirror of components.Component (components/types.go:20-66) for the xid / temperature / nvlink paths"""

    def __init__(self, ctx: "Context", name: str, **cfg):
        import json
        self._json = json
        self.ctx, self._L = ctx, ctx._L
        c = ComponentCfg(**cfg)
        self._h = C.c_void_p()
        ctx._check(self._L.gpud_component_create(ctx._h, name.encode(), C.byref(c), C.byref(self._h)))

    def name(self) -> str:
        b = C.create_string_buffer(128)
        self._L.gpud_component_name(self._h, b, 128)
        return b.value.decode()

    def start(self, interval_ms: int):
        self.ctx._check(self._L.gpud_component_start(self._h, interval_ms))

    def check(self):
        health, b = C.c_int32(), C.create_string_buffer(8192)
        self.ctx._check(self._L.gpud_component_check(self._h, C.byref(health), b, 8192))
        return health.value, b.value.decode()

    def last_health_states(self):
        b = C.create_string_buffer(1 << 16)
        n = self._L.gpud_component_last_health_states(self._h, b, 1 << 16)
        if n < 0:
            raise GpudError(n, "gpud_component_last_health_states")
        return self._json.loads(b.value.decode())

    def events(self, since_unix: int = 0):
        b = C.create_string_buffer(1 << 20)
        n = self._L.gpud_component_events(self._h, since_unix, b, 1 << 20)
        if n < 0:
            raise GpudError(n, "gpud_component_events")
        return self._json.loads(b.value.decode())

    def checks(self) -> int:
        return int(self._L.gpud_component_checks(self._h))

    def xid_set_source(self, buf: bytes, raw_kmsg: bool = False, boot_unix: int = 0):
        self.ctx._check(self._L.gpud_component_xid_set_source(self._h, C.cast(C.c_char_p(buf), C.c_void_p), len(buf), int(raw_kmsg), boot_unix))

    def xid_set_healthy(self, now_unix: int):
        self.ctx._check(self._L.gpud_component_xid_set_healthy(self._h, now_unix))

    def xid_add_reboot(self, unix_s: int):
        self.ctx._check(self._L.gpud_component_xid_add_reboot(self._h, unix_s))

    def xid_set_devices(self, devices: str):
        self.ctx._check(self._L.gpud_component_xid_set_devices(self._h, devices.encode()))

    def stop(self):
        """Close(): stops the ticker; the object stays readable"""
        self.ctx._check(self._L.gpud_component_close(self._h))

    def ring_handle(self, slot: int = 0):
        return self._L.gpud_component_ring(self._h, slot)

    def close(self):
        if self._h:
            self._L.gpud_component_close(self._h)
            self._L.gpud_component_destroy(self._h)
            self._h = None


class KmsgDeduper:
    """the kmsg watcher's duplicate drop (pkg/kmsg/watcher.go:281-286) over the units of a scanned buffer"""

    def __init__(self, ttl_seconds: int = 0, truncate_seconds: int = 0):
        self._L = lib()
        self._L.gpud_kmsg_deduper_create.restype = C.c_void_p
        self._h = C.c_void_p(self._L.gpud_kmsg_deduper_create(C.c_int64(ttl_seconds), C.c_int32(truncate_seconds)))

    def units(self, buf: bytes, n_units: int, mode: int = 0, boot_unix: int = 0, lines_unix: int = 0, now_unix: int = 0) -> bytes:
        dropped = C.create_string_buffer(max(1, n_units))
        nd = C.c_int64()
        rc = self._L.gpud_kmsg_dedup_units(self._h, C.cast(C.c_char_p(buf), C.c_void_p), C.c_int64(len(buf)), C.c_int32(mode), C.c_int64(boot_unix), C.c_int64(lines_unix),
                                           C.c_int64(now_unix), dropped, C.c_int64(n_units), C.byref(nd))
        if rc:
            raise GpudError(rc, "gpud_kmsg_dedup_units")
        return dropped.raw[:n_units]

    def close(self):
        if self._h:
            self._L.gpud_kmsg_deduper_destroy(self._h)
            self._h = None


class KmsgDedupDevice:
    """gpud_kmsg_dedup: the watcher's duplicate drop as a device-resident cache on `dev`, applied in the same call as the scan"""

    def __init__(self, ctx: "Context", dev: Optional[int] = None, ttl_seconds: int = 0, truncate_seconds: int = 0, hash_bits: int = 64):
        self._L = lib()
        self.ctx = ctx
        self.dev = ctx.devices[0] if dev is None else dev
        self._h = C.c_void_p()
        ctx._check(self._L.gpud_kmsg_dedup_create(ctx._h, self.dev, ttl_seconds, truncate_seconds, C.byref(self._h)))
        if hash_bits != 64:
            ctx._check(self._L.gpudh_kmsg_dedup_hash_bits(self._h, hash_bits))
        self.last_n_hits = 0

    def scan(self, buf: bytes, mode: int = SCAN_LINES, boot_unix: int = 0, lines_unix: int = 0, now_unix: int = 0, cap: int = 1 << 16,
             allow_overflow: bool = False):
        """One gpud_kmsg_scan_dedup call; returns (hits, n_units, dropped bytes).  Every call updates the cache, so an overflowing
        hit list is not retried: it raises, or with allow_overflow returns the first `cap` hits (last_n_hits = all kept hits)."""
        n = len(buf)
        dropped = C.create_string_buffer(n + 1)           # n_units <= len + 1
        hits = (XidHit * max(cap, 1))()
        nh, nu, nd = C.c_int64(), C.c_int64(), C.c_int64()
        rc = self._L.gpud_kmsg_scan_dedup(self.ctx._h, self.dev, self._h, C.cast(C.c_char_p(buf), C.c_void_p), n, mode, boot_unix, lines_unix,
                                          now_unix, hits, cap, C.byref(nh), C.byref(nu), dropped, n + 1, C.byref(nd))
        if not (allow_overflow and rc == -4 and nh.value > cap):
            self.ctx._check(rc)
        self.last_n_hits = nh.value
        return [hits[i] for i in range(min(nh.value, cap))], nu.value, dropped.raw[:nu.value]

    def stats(self):
        out, ms = (C.c_int64 * 4)(), C.c_float()
        self.ctx._check(self._L.gpud_kmsg_dedup_stats(self._h, out, C.byref(ms)))
        return {"live": out[0], "arena_bytes": out[1], "slots": out[2], "rebuilds": out[3], "dedup_ms": ms.value}

    def close(self):
        if self._h:
            self._L.gpud_kmsg_dedup_destroy(self._h)
            self._h = None


class FabricRaw(C.Structure):
    _fields_ = [("gpu_index", C.c_uint32), ("nvlink_supported", C.c_uint32), ("system_expected_nvlink", C.c_uint32),
                ("n_links", C.c_uint32), ("link_feature_enabled", C.c_uint8 * MAX_LINKS), ("pad0", C.c_uint8 * 2),
                ("link_replay_errors", C.c_uint64 * MAX_LINKS), ("link_recovery_errors", C.c_uint64 * MAX_LINKS),
                ("link_crc_errors", C.c_uint64 * MAX_LINKS), ("p2p_status", C.c_uint8 * MAX_GPUS), ("fabric_valid", C.c_uint32),
                ("fabric_state", C.c_uint8), ("fabric_summary", C.c_uint8), ("pad1", C.c_uint8 * 2), ("fabric_status", C.c_int32),
                ("fabric_health_mask", C.c_uint32), ("clique_id", C.c_uint32)]


class FabricLocal(C.Structure):
    _fields_ = [("gpu_index", C.c_uint32), ("flags", C.c_uint32), ("n_links", C.c_uint32), ("links_enabled_mask", C.c_uint32),
                ("replay_errors", C.c_uint64), ("recovery_errors", C.c_uint64), ("crc_errors", C.c_uint64),
                ("p2p_status", C.c_uint8 * MAX_GPUS), ("fabric_state", C.c_uint8), ("fabric_summary", C.c_uint8),
                ("fabric_issue_bits", C.c_uint8), ("pad0", C.c_uint8), ("fabric_status", C.c_int32),
                ("fabric_health_mask", C.c_uint32), ("clique_id", C.c_uint32), ("pad1", C.c_uint8 * (128 - 76))]


class FabricVerdict(C.Structure):
    _fields_ = [("n_gpus", C.c_int32), ("nvlink_health", C.c_int32), ("nvlink_reason", C.c_int32), ("required", C.c_int32),
                ("active", C.c_int32), ("inactive", C.c_int32), ("unsupported", C.c_int32), ("p2p_expected_pairs", C.c_int32),
                ("p2p_probed_pairs", C.c_int32), ("p2p_ok_pairs", C.c_int32), ("p2p_ok_gpu_mask", C.c_uint32),
                ("p2p_observed_status_mask", C.c_uint32), ("active_mask", C.c_uint32), ("inactive_mask", C.c_uint32),
                ("unsupported_mask", C.c_uint32), ("fabric_healthy", C.c_int32), ("fabric_unhealthy_gpu_mask", C.c_uint32),
                ("fabric_issue_bits", C.c_uint8 * MAX_GPUS), ("total_replay", C.c_uint64), ("total_recovery", C.c_uint64),
                ("total_crc", C.c_uint64)]

    def as_dict(self) -> dict:
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "fabric_issue_bits"}
        d["fabric_issue_bits"] = list(self.fabric_issue_bits)
        return d


# every symbol include/gpud_b200.h declares (tests check the library exports each one)
SYMBOLS = ["gpud_abi_version", "gpud_sizeof", "gpud_ctx_create", "gpud_ctx_destroy", "gpud_last_error", "gpud_host_alloc",
           "gpud_host_free", "gpud_ring_create", "gpud_ring_destroy", "gpud_ring_set_stream", "gpud_ring_push",
           "gpud_ring_push_device", "gpud_ring_push_raw", "gpud_clock_event_reasons", "gpud_hw_slowdown_event_message", "gpud_hw_slowdown_check", "gpud_store_insert_hw_slowdown", "gpud_store_open", "gpud_store_close", "gpud_store_last_error", "gpud_store_event_table", "gpud_store_insert_event", "gpud_store_insert_xid_hits", "gpud_store_metrics_table", "gpud_store_record_metrics", "gpud_kmsg_syncer_create", "gpud_kmsg_syncer_destroy", "gpud_kmsg_syncer_feed", "gpud_store_find_event", "gpud_store_record_reboot", "gpud_xid_state_from_store", "gpud_sxid_state_from_store", "gpud_store_get_events", "gpud_store_latest_event", "gpud_store_purge_events", "gpud_kmsg_syncer_configure", "gpud_kmsg_syncer_configure_component", "gpud_kmsg_syncer_offer", "gpud_ib_scan", "gpud_ib_reason", "gpud_poller_create", "gpud_poller_destroy", "gpud_poller_poll", "gpud_poller_last_rows", "gpud_poller_errors", "gpud_poll_row_hold", "gpud_nvml_devices", "gpud_nvml_devices_arg", "gpud_nvml_bus_id", "gpud_poller_remapped_rows", "gpud_remapped_rows_check", "gpud_poller_ecc_errors", "gpud_poller_field_row", "gpud_poller_poll_fields", "gpud_poller_gpm_supported", "gpud_poller_gpm_metrics", "gpud_poller_poll_gpm", "gpud_gpm_check", "gpud_poller_fabric_raw", "gpud_poller_product_name", "gpud_poller_temperature", "gpud_temperature_check", "gpud_temperature_reason", "gpud_poller_counters", "gpud_ring_counts", "gpud_ring_reduce", "gpud_ring_sync", "gpud_ring_kernel_ms", "gpud_ring_read",
           "gpud_ring_result_ptr", "gpud_ring_stream_open", "gpud_ring_stream_reduce", "gpud_ring_stream_counts", "gpud_ring_stream_read", "gpud_ring_windows_open", "gpud_ring_windows_open_hop", "gpud_ring_windows_close", "gpud_ring_windows_reduce", "gpud_ring_windows_counts", "gpud_ring_windows_read", "gpud_ring_windows_stats", "gpud_ring_windows_open_fields", "gpud_ring_windows_fields", "gpud_ring_reduce_range", "gpud_ring_range_stats", "gpud_ring_reduce_ranges", "gpud_ring_reduce_range_sets", "gpud_rings_reduce_range_sets", "gpud_rings_reduce_range_sets_fields", "gpud_ring_ranges_stats", "gpud_box_query_create", "gpud_box_query_create_fields", "gpud_box_query_step", "gpud_box_query_result", "gpud_box_query_stats", "gpud_box_query_destroy", "gpud_ring_set_cta_reserve", "gpud_kmsg_scan", "gpud_kmsg_scan_sharded", "gpud_kmsg_scan_device", "gpud_kmsg_scan_kernel_ms", "gpud_kmsg_scan_phase_timing", "gpud_kmsg_scan_stats", "gpud_xid_classify",
           "gpud_hit_detail_json", "gpud_xid_description", "gpud_xid_mnemonic", "gpud_sxid_name", "gpud_nvlink_rule_hint", "gpud_sxid_reason", "gpud_sxid_get_detail", "gpud_store_insert_sxid_hits", "gpud_product_mem_caps", "gpud_product_fm_supported", "gpud_product_fabric_state_supported", "gpud_xid_get_detail", "gpud_xid_detail", "gpud_xid_build_message", "gpud_xid_hit_message", "gpud_xid_device_matches_bus_id", "gpud_kmsg_event_name", "gpud_kmsg_event_message", "gpud_kmsg_component", "gpud_kmsg_hit_message", "gpud_kmsg_stateful_create", "gpud_kmsg_stateful_destroy", "gpud_kmsg_stateful_feed", "gpud_component_create", "gpud_component_destroy", "gpud_component_name", "gpud_component_start", "gpud_component_check", "gpud_component_last_health_states", "gpud_component_events", "gpud_component_close", "gpud_component_checks", "gpud_component_xid_set_source", "gpud_component_xid_set_healthy", "gpud_component_xid_add_reboot", "gpud_component_xid_set_devices", "gpud_component_ring", "gpud_kmsg_stateful_feed_units", "gpud_kmsg_deduper_create", "gpud_kmsg_deduper_destroy", "gpud_kmsg_dedup_units",
           "gpud_kmsg_dedup_create", "gpud_kmsg_dedup_destroy", "gpud_kmsg_scan_dedup", "gpud_kmsg_dedup_stats",
           "gpud_fabric_issues", "gpud_fabric_suggest_reboot", "gpud_set_nvml_error_string", "gpud_nvml_error_strings_from_driver", "gpud_fabric_reason", "gpud_fabric_report_reason", "gpud_fabric_pack", "gpud_fabric_verdict_device", "gpud_comm_unique_id", "gpud_comm_init", "gpud_fabric_gather",
           "gpud_fabric_gather_p2p", "gpud_fm_log_syncer_create", "gpud_fm_log_syncer_destroy", "gpud_fm_log_syncer_feed",
           "gpud_fm_nothing_to_do_from_store", "gpud_ring_checkpoint_bound", "gpud_ring_checkpoint", "gpud_ring_restore",
           "gpud_ring_checkpoint_stats", "gpud_ring_checkpoint_delta_bound", "gpud_ring_checkpoint_delta", "gpud_ring_restore_delta",
           "gpud_ring_tier_open", "gpud_ring_tier_counts", "gpud_ring_tier_stats", "gpud_ring_tier_checkpoint_bound", "gpud_ring_tier_checkpoint",
           "gpud_ring_tier_checkpoint_delta_bound", "gpud_ring_tier_checkpoint_delta", "gpud_ring_tier_restore", "gpud_ring_tier_checkpoint_stats"]

_lib = None


def lib() -> C.CDLL:
    """Load libgpud_b200.so (fails loudly if it has not been built: there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GpudError(-2, "%s is missing: build it with `make` (or __graft_entry__.build())" % LIB_PATH)
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    sig = {
        "gpud_abi_version": (i32, []), "gpud_sizeof": (i32, [i32]),
        "gpud_ctx_create": (i32, [C.POINTER(i32), i32, C.POINTER(vp)]), "gpud_ctx_destroy": (i32, [vp]),
        "gpud_last_error": (i32, [vp, C.c_char_p, i32]),
        "gpud_host_alloc": (i32, [i64, C.POINTER(vp)]), "gpud_host_free": (i32, [vp]),
        "gpud_ring_create": (i32, [vp, i32, C.POINTER(RingCfg), C.POINTER(vp)]), "gpud_ring_destroy": (i32, [vp]),
        "gpud_ring_set_stream": (i32, [vp, vp]), "gpud_ring_push": (i32, [vp, vp, i64]), "gpud_ring_push_device": (i32, [vp, vp, i64]), "gpud_ring_push_raw": (i32, [vp, vp, i64, i32]),
        "gpud_clock_event_reasons": (i32, [C.c_uint64, vp, i32, vp, i32, vp]),
        "gpud_store_open": (i32, [C.c_char_p, vp]), "gpud_store_close": (None, [vp]), "gpud_store_last_error": (i32, [vp, vp, i32]),
        "gpud_store_event_table": (i32, [vp, C.c_char_p, vp, i32]),
        "gpud_store_insert_event": (i32, [vp, C.c_char_p, i64, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p]),
        "gpud_store_insert_xid_hits": (i32, [vp, C.c_char_p, vp, i64, i64, i64, i32, vp]),
        "gpud_kmsg_syncer_create": (i32, [vp, C.c_char_p, vp]), "gpud_kmsg_syncer_destroy": (None, [vp]),
        "gpud_kmsg_syncer_feed": (i32, [vp, C.c_char_p, vp, i64, vp, i64, i64, vp]),
        "gpud_store_get_events": (i32, [vp, C.c_char_p, i64, vp, i32, vp, i32, vp]), "gpud_store_latest_event": (i32, [vp, C.c_char_p, vp, vp, i32, vp]),
        "gpud_store_purge_events": (i32, [vp, C.c_char_p, i64, vp]), "gpud_store_record_reboot": (i32, [vp, C.c_char_p, i64, i64, vp]),
        "gpud_xid_state_from_store": (i32, [vp, C.c_char_p, C.c_char_p, i64, i64, i32, C.c_char_p, vp, vp, vp, i32]),
        "gpud_sxid_state_from_store": (i32, [vp, C.c_char_p, C.c_char_p, i64, i64, vp, vp, vp, i32]),
        "gpud_store_find_event": (i32, [vp, C.c_char_p, i64, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, vp]),
        "gpud_kmsg_syncer_configure": (i32, [vp, i32, i32, vp, i32]), "gpud_kmsg_syncer_configure_component": (i32, [vp, C.c_char_p]),
        "gpud_kmsg_syncer_offer": (i32, [vp, i64, C.c_char_p, C.c_char_p, i64, vp]),
        "gpud_fm_log_syncer_create": (i32, [vp, vp]), "gpud_fm_log_syncer_destroy": (None, [vp]),
        "gpud_fm_log_syncer_feed": (i32, [vp, vp, i64, vp, i64, vp]), "gpud_fm_nothing_to_do_from_store": (i32, [vp, C.c_char_p, i64, vp]),
        "gpud_store_metrics_table": (i32, [vp, C.c_char_p]), "gpud_store_record_metrics": (i32, [vp, C.c_char_p, vp, i64]),
        "gpud_ib_scan": (i32, [vp, i32, vp, vp, i64, i64, i64, i32, vp]), "gpud_ib_reason": (i32, [C.c_char_p, C.c_uint32, i64, i32, vp, i32]),
        "gpud_poller_create": (i32, [vp, i32, vp, vp]), "gpud_poller_destroy": (None, [vp]), "gpud_poller_poll": (i32, [vp, i64, i64]),
        "gpud_poller_last_rows": (i32, [vp, vp, i64, vp, vp]), "gpud_poller_errors": (i32, [vp, vp, vp, vp]),
        "gpud_poll_row_hold": (i32, [vp, vp, i32, vp, vp, vp]),
        "gpud_nvml_devices": (i32, [vp, i32, vp, vp, i32]), "gpud_nvml_devices_arg": (i32, [vp, i32]), "gpud_nvml_bus_id": (i32, [C.c_char_p, vp, i32]),
        "gpud_poller_remapped_rows": (i32, [vp, vp]), "gpud_remapped_rows_check": (i32, [vp, vp, i32, vp, vp, vp, i32]),
        "gpud_poller_ecc_errors": (i32, [vp, vp]), "gpud_poller_field_row": (i32, [vp, vp, vp]), "gpud_poller_poll_fields": (i32, [vp, vp, i64, i64, vp]),
        "gpud_poller_gpm_supported": (i32, [vp, vp]), "gpud_poller_gpm_metrics": (i32, [vp, i64, vp]), "gpud_poller_poll_gpm": (i32, [vp, vp, i64, i64, vp]),
        "gpud_gpm_check": (i32, [vp, i32, vp, vp, i32]),
        "gpud_poller_temperature": (i32, [vp, C.POINTER(Temperature)]), "gpud_temperature_check": (i32, [C.POINTER(Temperature), i32, vp]),
        "gpud_temperature_reason": (i32, [vp, vp, i32, i32, vp, vp, i32]),
        "gpud_poller_counters": (i32, [vp, C.POINTER(PollCounters)]),
        "gpud_poller_fabric_raw": (i32, [vp, C.c_uint32, vp, i32, C.POINTER(FabricRaw)]), "gpud_poller_product_name": (i32, [vp, vp, i32]),
        "gpud_ring_counts": (i32, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]),
        "gpud_ring_reduce": (i32, [vp]), "gpud_ring_sync": (i32, [vp]),
        "gpud_ring_kernel_ms": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]), "gpud_ring_read": (i32, [vp, i32, vp, i64]),
        "gpud_ring_result_ptr": (i32, [vp, i32, C.POINTER(vp)]), "gpud_ring_reduce_range": (i32, [vp, i64, vp, vp]),
        "gpud_ring_set_cta_reserve": (i32, [vp, i32]),
        "gpud_ring_stream_open": (i32, [vp, i64]), "gpud_ring_stream_reduce": (i32, [vp, C.POINTER(i64), C.POINTER(i64)]),
        "gpud_ring_stream_counts": (i32, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]), "gpud_ring_stream_read": (i32, [vp, i32, i64, i64, vp, i64]),
        "gpud_ring_range_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int32), vp]),
        "gpud_ring_reduce_ranges": (i32, [vp, vp, vp, i64, vp, vp]),
        "gpud_ring_reduce_range_sets": (i32, [vp, vp, vp, i64, vp, i64, vp, vp]),
        "gpud_rings_reduce_range_sets": (i32, [vp, i32, vp, vp, vp, i64, vp, i64, vp, vp]),
        "gpud_rings_reduce_range_sets_fields": (i32, [vp, i32, vp, vp, i32, vp, vp, i64, vp, i64, vp, vp]),
        "gpud_ring_ranges_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(i64), vp]),
        "gpud_box_query_create": (i32, [vp, i32, i32, vp, vp, vp, i64, vp, i64, C.POINTER(vp)]),
        "gpud_box_query_create_fields": (i32, [vp, i32, i32, vp, vp, i32, vp, vp, i64, vp, i64, C.POINTER(vp)]),
        "gpud_box_query_step": (i32, [vp, vp, C.POINTER(vp), C.POINTER(i64)]), "gpud_box_query_result": (i32, [vp, vp, vp]),
        "gpud_box_query_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(i64), C.POINTER(i64), vp]),
        "gpud_box_query_destroy": (None, [vp]),
        "gpudh_box_query_plan": (i32, [i32, vp, i64, i32, i32, i32, vp, vp, vp, i64, vp, i64, vp, vp, vp, vp, vp, vp, vp, C.c_char_p, i32]),
        "gpudh_box_query_plan_fields": (i32, [i32, vp, i64, i32, vp, i32, i32, i32, vp, vp, vp, i64, vp, i64, vp, vp, vp, vp, vp, vp, vp, C.c_char_p, i32]),
        "gpudh_box_query_pivots": (i32, [vp, vp, i64, C.POINTER(i64)]),
        "gpud_ring_windows_open": (i32, [vp, i64, i64, C.POINTER(vp)]),
        "gpud_ring_windows_open_hop": (i32, [vp, i64, i64, i64, C.POINTER(vp)]), "gpud_ring_windows_close": (i32, [vp]),
        "gpud_ring_windows_reduce": (i32, [vp, C.POINTER(i64), C.POINTER(i64)]),
        "gpud_ring_windows_counts": (i32, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]),
        "gpud_ring_windows_read": (i32, [vp, i32, i64, i64, vp, i64]),
        "gpud_ring_windows_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(i64), vp]),
        "gpud_ring_windows_open_fields": (i32, [vp, i64, i64, i64, vp, i32, C.POINTER(vp)]),
        "gpud_ring_windows_fields": (i32, [vp, vp, i32, C.POINTER(i32)]),
        "gpud_ring_checkpoint_bound": (i32, [vp, C.POINTER(i64)]), "gpud_ring_checkpoint": (i32, [vp, vp, i64, C.POINTER(i64)]),
        "gpud_ring_restore": (i32, [vp, vp, i64, vp, i32, C.POINTER(C.c_int32)]),
        "gpud_ring_checkpoint_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), vp]),
        "gpud_ring_checkpoint_delta_bound": (i32, [vp, C.POINTER(i64)]),
        "gpud_ring_checkpoint_delta": (i32, [vp, vp, i64, C.POINTER(i64)]), "gpud_ring_restore_delta": (i32, [vp, vp, i64]),
        "gpudh_ring_windows_sub": (i32, [i32, i64]), "gpudh_ring_ckpt_grid": (i32, [vp, i32]),
        "gpud_ring_tier_open": (i32, [vp, i64]),
        "gpud_ring_tier_counts": (i32, [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]),
        "gpud_ring_tier_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), vp]),
        "gpudh_ring_tier_plan": (i32, [i64, i32, i64, i64, vp, i64, vp, i64, vp, vp]),
        "gpudh_ring_tier_split": (i32, [i64, i64, i32, i64, i64, vp, vp, i64, vp, i64, vp, vp, vp, i64, C.POINTER(i64), C.POINTER(i64)]),
        "gpudh_rings_tier_split": (i32, [vp, i32, i64, vp, vp, vp, vp, vp, i64, vp, i64, vp, vp, vp, C.POINTER(C.c_int32), vp, vp, vp, vp, vp, i64,
                                         C.POINTER(i64)]),
        "gpudh_ring_tier_row": (i32, [vp, i64, vp, i64, C.POINTER(i64)]), "gpudh_ring_tier_group": (i32, [vp, i32]),
        "gpud_ring_tier_checkpoint_bound": (i32, [vp, C.POINTER(i64)]), "gpud_ring_tier_checkpoint": (i32, [vp, vp, i64, C.POINTER(i64)]),
        "gpud_ring_tier_checkpoint_delta_bound": (i32, [vp, C.POINTER(i64)]),
        "gpud_ring_tier_checkpoint_delta": (i32, [vp, vp, i64, C.POINTER(i64)]),
        "gpud_ring_tier_restore": (i32, [vp, i64, vp, vp, i32]),
        "gpud_ring_tier_checkpoint_stats": (i32, [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(i64)]),
        "gpudh_ring_tier_chain_plan": (i32, [i32, i32, i64, i64, i64, vp, vp, i32, vp, i64, C.POINTER(i64), vp, C.c_char_p, i32]),
        "gpud_kmsg_scan": (i32, [vp, i32, vp, i64, i32, C.POINTER(XidHit), i64, C.POINTER(i64), C.POINTER(i64)]),
        "gpud_kmsg_scan_sharded": (i32, [vp, vp, i64, i32, C.POINTER(XidHit), i64, C.POINTER(i64), C.POINTER(i64)]),
        "gpud_kmsg_scan_device": (i32, [vp, i32, vp, i64, i32, C.POINTER(XidHit), i64, C.POINTER(i64), C.POINTER(i64), vp]),
        "gpud_kmsg_scan_kernel_ms": (i32, [vp, i32, C.POINTER(C.c_float)]),
        "gpud_kmsg_scan_phase_timing": (i32, [vp, i32, i32]),
        "gpud_kmsg_scan_stats": (i32, [vp, i32, C.POINTER(i64)]),
        "gpud_xid_classify": (i32, [vp, i32, C.POINTER(XidHit), i64]),
        "gpud_hit_detail_json": (i32, [C.POINTER(XidHit), i64, C.c_char_p, i32]),
        "gpud_xid_description": (C.c_char_p, [i32, i32]), "gpud_xid_mnemonic": (C.c_char_p, [i32]),
        "gpud_sxid_name": (C.c_char_p, [i32]), "gpud_nvlink_rule_hint": (C.c_char_p, [i32]),
        "gpud_sxid_reason": (i32, [i64, C.c_char_p, vp, i32]),
        "gpud_hw_slowdown_event_message": (i32, [C.c_uint64, C.c_char_p, vp, i32]),
        "gpud_hw_slowdown_check": (i32, [vp, i32, i64, i64, C.c_double, vp, vp, vp, vp, i32]),
        "gpud_store_insert_hw_slowdown": (i32, [vp, C.c_char_p, i64, C.c_uint64, C.c_char_p, vp]),
        "gpud_xid_get_detail": (i32, [i32, vp, vp, vp]), "gpud_sxid_get_detail": (i32, [i32, vp, vp, vp]),
        "gpud_store_insert_sxid_hits": (i32, [vp, C.c_char_p, vp, i64, i64, i64, i32, vp]),
        "gpud_product_mem_caps": (i32, [C.c_char_p]), "gpud_product_fm_supported": (i32, [C.c_char_p]), "gpud_product_fabric_state_supported": (i32, [C.c_char_p]),
        "gpud_xid_detail": (i32, [i32, i32, C.c_uint32, vp, vp, vp, vp, vp]),
        "gpud_xid_build_message": (i32, [C.c_uint64, i32, C.c_uint32, C.c_char_p, C.c_char_p, C.c_char_p, vp, i32]),
        "gpud_xid_hit_message": (i32, [C.POINTER(XidHit), C.c_char_p, vp, i32]), "gpud_xid_device_matches_bus_id": (i32, [C.c_char_p, C.c_char_p]), "gpud_kmsg_event_name": (C.c_char_p, [i32]), "gpud_kmsg_event_message": (C.c_char_p, [i32]),
        "gpud_kmsg_component": (C.c_char_p, [i32]), "gpud_kmsg_hit_message": (i32, [vp, vp, vp, i32]),
        "gpud_kmsg_stateful_create": (i32, [vp]), "gpud_kmsg_stateful_destroy": (None, [vp]),
        "gpud_kmsg_stateful_feed": (i32, [vp, vp, i64, vp, i64, vp, i32, vp]),
        "gpud_component_create": (i32, [vp, C.c_char_p, vp, vp]), "gpud_component_destroy": (None, [vp]), "gpud_component_name": (i32, [vp, vp, i32]),
        "gpud_component_start": (i32, [vp, i64]), "gpud_component_check": (i32, [vp, vp, vp, i32]), "gpud_component_last_health_states": (i32, [vp, vp, i32]),
        "gpud_component_events": (i32, [vp, i64, vp, i32]), "gpud_component_close": (i32, [vp]), "gpud_component_checks": (i64, [vp]),
        "gpud_component_xid_set_source": (i32, [vp, vp, i64, i32, i64]), "gpud_component_xid_set_healthy": (i32, [vp, i64]),
        "gpud_component_xid_add_reboot": (i32, [vp, i64]), "gpud_component_xid_set_devices": (i32, [vp, C.c_char_p]), "gpud_component_ring": (vp, [vp, i32]),
        "gpud_kmsg_stateful_feed_units": (i32, [vp, vp, i64, vp, i64, vp, vp, i32, vp]), "gpud_kmsg_deduper_create": (vp, [i64, i32]),
        "gpud_kmsg_deduper_destroy": (None, [vp]), "gpud_kmsg_dedup_units": (i32, [vp, vp, i64, i32, i64, i64, i64, vp, i64, vp]),
        "gpud_kmsg_dedup_create": (i32, [vp, i32, i64, i32, vp]), "gpud_kmsg_dedup_destroy": (None, [vp]),
        "gpud_kmsg_scan_dedup": (i32, [vp, i32, vp, vp, i64, i32, i64, i64, i64, C.POINTER(XidHit), i64, C.POINTER(i64), C.POINTER(i64), vp, i64,
                                       C.POINTER(i64)]),
        "gpud_kmsg_dedup_stats": (i32, [vp, C.POINTER(i64), C.POINTER(C.c_float)]), "gpudh_kmsg_dedup_hash_bits": (i32, [vp, i32]),
        "gpud_fabric_pack": (i32, [vp, i32, C.POINTER(FabricRaw), vp, vp]),
        "gpud_fabric_verdict_device": (i32, [vp, i32, vp, i32, i32, C.POINTER(FabricVerdict), vp]),
        "gpud_comm_unique_id": (i32, [vp]), "gpud_comm_init": (i32, [vp, i32, i32, i32, vp]),
        "gpud_fabric_issues": (i32, [vp, vp, i32]), "gpud_fabric_suggest_reboot": (i32, [vp]), "gpud_fabric_reason": (i32, [vp, vp, i32, vp, i32]), "gpud_set_nvml_error_string": (None, [vp]), "gpud_nvml_error_strings_from_driver": (i32, []), "gpud_fabric_report_reason": (i32, [vp, vp, i32, vp, vp, i32]),
        "gpud_fabric_gather": (i32, [vp, i32, C.POINTER(FabricRaw), i32, C.POINTER(FabricLocal), C.POINTER(FabricVerdict)]),
        "gpud_fabric_gather_p2p": (i32, [vp, C.POINTER(FabricRaw), i32, C.POINTER(FabricLocal), C.POINTER(FabricVerdict)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    for which, st in enumerate((XidHit, FabricRaw, FabricLocal, FabricVerdict, RingCfg, KmsgEvent, IbSnapshot, IbVerdict, Metric, DedupRule, Temperature, PollCounters, EventRow, NvmlDevice, RemappedRows, EccErrors, GpmMetrics)):
        if L.gpud_sizeof(which) != C.sizeof(st):
            raise GpudError(-1, "ABI layout mismatch for %s: C %d vs ctypes %d" % (st.__name__, L.gpud_sizeof(which), C.sizeof(st)))
    _lib = L
    return L


class Context:
    """gpud_ctx: one per process, naming the CUDA devices it drives."""

    def __init__(self, devices: Sequence[int] = (0,)):
        self._L = lib()
        self.devices = list(devices)
        arr = (C.c_int32 * len(self.devices))(*self.devices)
        h = C.c_void_p()
        rc = self._L.gpud_ctx_create(arr, len(self.devices), C.byref(h))
        if rc:
            raise GpudError(rc, "gpud_ctx_create failed (no CUDA device? this path has no CPU fallback)")
        self._h = h

    def _check(self, rc: int):
        if rc:
            buf = C.create_string_buffer(512)
            self._L.gpud_last_error(self._h, buf, 512)
            raise GpudError(rc, buf.value.decode("utf-8", "replace"))

    def close(self):
        if self._h:
            self._L.gpud_ctx_destroy(self._h)
            self._h = None

    # ---- kmsg scan ----
    def kmsg_scan(self, buf: bytes, mode: int = SCAN_LINES, dev: Optional[int] = None, cap: int = 1 << 16):
        """Scan host bytes; returns (hits: List[XidHit], n_units)."""
        dev = self.devices[0] if dev is None else dev
        n = len(buf)
        src = C.c_char_p(buf)                     # no copy: the library only reads the bytes during the call
        while True:
            hits = (XidHit * cap)()
            nh, nu = C.c_int64(), C.c_int64()
            rc = self._L.gpud_kmsg_scan(self._h, dev, C.cast(src, C.c_void_p), n, mode, hits, cap, C.byref(nh), C.byref(nu))
            if rc == -4 and nh.value > cap:
                cap = int(nh.value)
                continue
            self._check(rc)
            self.last_scan_raw = (hits, nh.value)
            return [hits[i] for i in range(nh.value)], nu.value

    def kmsg_scan_c(self, buf: bytes, hits, cap: int, mode: int = SCAN_LINES, dev: Optional[int] = None):
        """The bare C call (preallocated XidHit array): what a cgo caller pays.  Returns (n_hits, n_units)."""
        dev = self.devices[0] if dev is None else dev
        nh, nu = C.c_int64(), C.c_int64()
        self._check(self._L.gpud_kmsg_scan(self._h, dev, C.cast(C.c_char_p(buf), C.c_void_p), len(buf), mode, hits, cap, C.byref(nh), C.byref(nu)))
        return nh.value, nu.value

    def kmsg_scan_sharded(self, buf: bytes, mode: int = SCAN_LINES, cap: int = 1 << 16):
        """gpud_kmsg_scan_sharded: the buffer split over every GPU of this context.  Returns (hits, n_units)."""
        hits = (XidHit * cap)()
        nh, nu = C.c_int64(), C.c_int64()
        self._check(self._L.gpud_kmsg_scan_sharded(self._h, C.cast(C.c_char_p(buf), C.c_void_p), len(buf), mode, hits, cap, C.byref(nh), C.byref(nu)))
        return [hits[i] for i in range(min(nh.value, cap))], nu.value

    def kmsg_scan_sharded_c(self, buf: bytes, hits, cap: int, mode: int = SCAN_LINES):
        """the bare C call with a preallocated XidHit array.  Returns (n_hits, n_units)."""
        nh, nu = C.c_int64(), C.c_int64()
        self._check(self._L.gpud_kmsg_scan_sharded(self._h, C.cast(C.c_char_p(buf), C.c_void_p), len(buf), mode, hits, cap, C.byref(nh), C.byref(nu)))
        return nh.value, nu.value

    def kmsg_scan_device(self, dev_ptr: int, length: int, mode: int = SCAN_LINES, dev: Optional[int] = None, cap: int = 1 << 16,
                         stream: int = 0):
        dev = self.devices[0] if dev is None else dev
        hits = (XidHit * cap)()
        nh, nu = C.c_int64(), C.c_int64()
        rc = self._L.gpud_kmsg_scan_device(self._h, dev, C.c_void_p(dev_ptr), length, mode, hits, cap, C.byref(nh), C.byref(nu),
                                           C.c_void_p(stream))
        self._check(rc)
        return [hits[i] for i in range(nh.value)], nu.value

    def scan_kernel_ms(self, dev: Optional[int] = None):
        dev = self.devices[0] if dev is None else dev
        ms = (C.c_float * 3)()
        self._check(self._L.gpud_kmsg_scan_kernel_ms(self._h, dev, ms))
        return list(ms)

    def scan_phase_timing(self, on: bool, dev: Optional[int] = None):
        """on: plain launches split by events (scan_kernel_ms -> [filter, prefix, match]); off (default): one overlapped chain
        (scan_kernel_ms -> [whole device time, 0, 0])"""
        dev = self.devices[0] if dev is None else dev
        self._check(self._L.gpud_kmsg_scan_phase_timing(self._h, dev, 1 if on else 0))

    def scan_stats(self, dev: Optional[int] = None):
        dev = self.devices[0] if dev is None else dev
        out = (C.c_int64 * 3)()
        self._check(self._L.gpud_kmsg_scan_stats(self._h, dev, out))
        return {"candidates": out[0], "hits": out[1], "separators": out[2]}

    def classify(self, hits: List[XidHit], dev: Optional[int] = None) -> List[XidHit]:
        dev = self.devices[0] if dev is None else dev
        arr = (XidHit * len(hits))(*hits)
        self._check(self._L.gpud_xid_classify(self._h, dev, arr, len(hits)))
        return [arr[i] for i in range(len(hits))]

    def hit_json(self, hit: XidHit, unix_seconds: int = 0) -> str:
        buf = C.create_string_buffer(4096)
        rc = self._L.gpud_hit_detail_json(C.byref(hit), unix_seconds, buf, 4096)
        if rc:
            raise GpudError(rc, "gpud_hit_detail_json")
        return buf.value.decode("utf-8")

    def hit_message(self, hit: XidHit, gpu_uuid: str = "") -> str:
        return xid_hit_message(hit, gpu_uuid)

    def ib_scan(self, series, drop_threshold: int, flap_down_interval: int, flap_back_threshold: int, dev: Optional[int] = None):
        """series: list of lists of (ts, down, total_link_downed); returns one IbVerdict per series"""
        dev = self.devices[0] if dev is None else dev
        total = sum(len(s) for s in series)
        snaps = (IbSnapshot * max(1, total))()
        offs = (C.c_int64 * (len(series) + 1))()
        k = 0
        for i, s in enumerate(series):
            offs[i] = k
            for ts, down, tld in s:
                snaps[k].ts, snaps[k].down, snaps[k].total_link_downed = ts, 1 if down else 0, tld
                k += 1
        offs[len(series)] = k
        out = (IbVerdict * max(1, len(series)))()
        self._check(self._L.gpud_ib_scan(self._h, dev, snaps, offs, len(series), drop_threshold, flap_down_interval, flap_back_threshold, out))
        return [out[i] for i in range(len(series))]

    def kmsg_message(self, hit: XidHit, buf: bytes = None) -> str:
        """(eventName, message) of an extra-matcher hit exactly as the component's Match returns it"""
        out = C.create_string_buffer(4096)
        n = self._L.gpud_kmsg_hit_message(C.byref(hit), C.cast(C.c_char_p(buf), C.c_void_p) if buf is not None else None, out, 4096)
        if n < 0:
            raise GpudError(n, "gpud_kmsg_hit_message")
        return out.raw[:n].decode("latin-1")

    # ---- fabric ----
    def fabric_pack(self, raw: FabricRaw, dev_send_ptr: int, dev: Optional[int] = None, stream: int = 0):
        dev = self.devices[0] if dev is None else dev
        self._check(self._L.gpud_fabric_pack(self._h, dev, C.byref(raw), C.c_void_p(dev_send_ptr), C.c_void_p(stream)))

    def fabric_verdict(self, dev_all_ptr: int, n: int, at_least: int = 0, dev: Optional[int] = None, stream: int = 0) -> FabricVerdict:
        dev = self.devices[0] if dev is None else dev
        v = FabricVerdict()
        self._check(self._L.gpud_fabric_verdict_device(self._h, dev, C.c_void_p(dev_all_ptr), n, at_least, C.byref(v), C.c_void_p(stream)))
        return v

    def fabric_gather_p2p(self, raws: Sequence[FabricRaw], at_least: int = 0):
        n = len(self.devices)
        arr = (FabricRaw * n)(*raws)
        allrec = (FabricLocal * n)()
        vs = (FabricVerdict * n)()
        self._check(self._L.gpud_fabric_gather_p2p(self._h, arr, at_least, allrec, vs))
        return [allrec[i] for i in range(n)], [vs[i] for i in range(n)]

    def comm_init(self, n_ranks: int, rank: int, unique_id: bytes, dev: Optional[int] = None):
        dev = self.devices[0] if dev is None else dev
        b = C.create_string_buffer(unique_id, 128)
        self._check(self._L.gpud_comm_init(self._h, dev, n_ranks, rank, b))

    def fabric_gather(self, raw: FabricRaw, n_ranks: int, at_least: int = 0, dev: Optional[int] = None):
        dev = self.devices[0] if dev is None else dev
        allrec = (FabricLocal * n_ranks)()
        v = FabricVerdict()
        self._check(self._L.gpud_fabric_gather(self._h, dev, C.byref(raw), at_least, allrec, C.byref(v)))
        return [allrec[i] for i in range(n_ranks)], v


def comm_unique_id() -> bytes:
    b = C.create_string_buffer(128)
    rc = lib().gpud_comm_unique_id(b)
    if rc:
        raise GpudError(rc, "gpud_comm_unique_id (libnccl.so.2 not loadable?)")
    return b.raw


def rings_reduce_range_sets(rings, ring_of, first, length, set_off, fields=None) -> dict:
    """Range sets over several rings of one Context (gpud_rings_reduce_range_sets): range i is samples [first[i], first[i] + length[i])
    of rings[ring_of[i]] in that ring's own push order, set s is ranges set_off[s] .. set_off[s + 1] - 1, its samples theirs
    concatenated in that order, whichever rings hold them.  rings[0] is the home ring whose device runs the call.  {op: [F][n_sets]}
    as Ring.reduce_range_sets returns; with a list of fields, only those are read (gpud_rings_reduce_range_sets_fields) and row g
    of each result is field fields[g]: {op: [len(fields)][n_sets]}."""
    rings = list(rings)
    assert len(rings) >= 1
    home = rings[0]
    ring_of = np.ascontiguousarray(ring_of, dtype=np.int32).reshape(-1)
    first = np.ascontiguousarray(first, dtype=np.int64).reshape(-1)
    length = np.ascontiguousarray(length, dtype=np.int64).reshape(-1)
    set_off = np.ascontiguousarray(set_off, dtype=np.int64).reshape(-1)
    assert first.shape == length.shape == ring_of.shape and set_off.shape[0] >= 1
    n_sets = set_off.shape[0] - 1
    hs = (C.c_void_p * len(rings))(*[r._h.value if r is not None else None for r in rings])
    if fields is not None:
        return _range_sets_fields(home, C.cast(hs, C.c_void_p), len(rings), C.c_void_p(ring_of.ctypes.data), fields, first, length, set_off)
    f64 = np.empty((5, home.F, n_sets), dtype=np.float64)
    nov = np.empty((home.F, n_sets), dtype=np.uint32)
    home.ctx._check(home._L.gpud_rings_reduce_range_sets(C.cast(hs, C.c_void_p), len(rings), C.c_void_p(ring_of.ctypes.data),
                                                         C.c_void_p(first.ctypes.data), C.c_void_p(length.ctypes.data), first.shape[0],
                                                         C.c_void_p(set_off.ctypes.data), n_sets, C.c_void_p(f64.ctypes.data),
                                                         C.c_void_p(nov.ctypes.data)))
    return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}


def _range_sets_fields(home, rings_p, n_rings, ring_of_p, fields, first, length, set_off) -> dict:
    """gpud_rings_reduce_range_sets_fields over the rings at rings_p (ring_of_p: NULL for one ring): {op: [len(fields)][n_sets]}"""
    fields = np.ascontiguousarray(fields, dtype=np.int32).reshape(-1)
    n_sets = set_off.shape[0] - 1
    f64 = np.empty((5, fields.shape[0], n_sets), dtype=np.float64)
    nov = np.empty((fields.shape[0], n_sets), dtype=np.uint32)
    home.ctx._check(home._L.gpud_rings_reduce_range_sets_fields(rings_p, n_rings, ring_of_p, C.c_void_p(fields.ctypes.data), fields.shape[0],
                                                                C.c_void_p(first.ctypes.data), C.c_void_p(length.ctypes.data), first.shape[0],
                                                                C.c_void_p(set_off.ctypes.data), n_sets, C.c_void_p(f64.ctypes.data),
                                                                C.c_void_p(nov.ctypes.data)))
    return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}


def _box_args(rank_of, first, length, set_off):
    rank_of = np.ascontiguousarray(rank_of, dtype=np.int32).reshape(-1)
    first = np.ascontiguousarray(first, dtype=np.int64).reshape(-1)
    length = np.ascontiguousarray(length, dtype=np.int64).reshape(-1)
    set_off = np.ascontiguousarray(set_off, dtype=np.int64).reshape(-1)
    assert first.shape == length.shape == rank_of.shape and set_off.shape[0] >= 2
    return rank_of, first, length, set_off


class BoxQuery:
    """gpud_box_query: range sets across processes, this process holding ring `rank` of n_ranks (include/gpud_b200.h).  Every rank
    makes the same query over its own ring and drives it with its own all-gather:

        send, nbytes = q.step()            # then, while nbytes: recv = all-gather of every rank's nbytes at send, in rank order
        send, nbytes = q.step(recv_ptr)    # recv_ptr: device memory on the ring's device, complete
    and reads q.result() ({op: [F][n_sets]}, as rings_reduce_range_sets) and q.stats() at the end.  With a list of fields
    (gpud_box_query_create_fields), only those are read and exchanged and row g of each result is field fields[g]:
    {op: [len(fields)][n_sets]}."""

    def __init__(self, ring, rank: int, n_ranks: int, rank_of, first, length, set_off, fields=None):
        self.ring, self._L = ring, ring._L
        self._args = _box_args(rank_of, first, length, set_off)   # kept alive: the query copies them, but keep them for the caller
        ro, fi, ln, so = self._args
        self.n_sets = so.shape[0] - 1
        self.G = ring.F
        h = C.c_void_p()
        if fields is None:
            ring.ctx._check(self._L.gpud_box_query_create(ring._h, rank, n_ranks, C.c_void_p(ro.ctypes.data), C.c_void_p(fi.ctypes.data),
                                                          C.c_void_p(ln.ctypes.data), fi.shape[0], C.c_void_p(so.ctypes.data), self.n_sets, C.byref(h)))
        else:
            fl = np.ascontiguousarray(fields, dtype=np.int32).reshape(-1)
            self.G = fl.shape[0]
            ring.ctx._check(self._L.gpud_box_query_create_fields(ring._h, rank, n_ranks, C.c_void_p(ro.ctypes.data), C.c_void_p(fl.ctypes.data),
                                                                 fl.shape[0], C.c_void_p(fi.ctypes.data), C.c_void_p(ln.ctypes.data), fi.shape[0],
                                                                 C.c_void_p(so.ctypes.data), self.n_sets, C.byref(h)))
        self._h = h

    def step(self, recv_ptr: int = 0):
        """-> (send_ptr, nbytes); nbytes == 0: done"""
        send, nb = C.c_void_p(), C.c_int64()
        self.ring.ctx._check(self._L.gpud_box_query_step(self._h, C.c_void_p(recv_ptr or None), C.byref(send), C.byref(nb)))
        return (send.value or 0), nb.value

    def result(self) -> dict:
        f64 = np.empty((5, self.G, self.n_sets), dtype=np.float64)
        nov = np.empty((self.G, self.n_sets), dtype=np.uint32)
        self.ring.ctx._check(self._L.gpud_box_query_result(self._h, C.c_void_p(f64.ctypes.data), C.c_void_p(nov.ctypes.data)))
        return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}

    def stats(self) -> dict:
        ms, rounds, sent, radix = C.c_float(), C.c_int32(), C.c_int64(), C.c_int64()
        reasons = np.zeros(8, dtype=np.int32)
        self.ring.ctx._check(self._L.gpud_box_query_stats(self._h, C.byref(ms), C.byref(rounds), C.byref(sent), C.byref(radix),
                                                          C.c_void_p(reasons.ctypes.data)))
        return {"device_ms": ms.value, "rounds": rounds.value, "bytes_sent": sent.value, "segments_by_radix": radix.value,
                "reasons": reasons[:len(RANGE_OPEN_REASONS)].copy()}

    def pivots(self) -> np.ndarray:
        """the pivots {lo, hi} of the last batch of long spread sets, [F][n_long][2], or [len(fields)][n_long][2] (gpudh_box_query_pivots)"""
        n = C.c_int64()
        self._L.gpudh_box_query_pivots(self._h, None, 0, C.byref(n))
        out = np.empty(2 * max(n.value, 1), dtype=np.float64)
        self.ring.ctx._check(self._L.gpudh_box_query_pivots(self._h, C.c_void_p(out.ctypes.data), n.value, C.byref(n)))
        return out[:2 * n.value].reshape(self.G, -1, 2)

    def close(self):
        if self._h:
            self._L.gpud_box_query_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def box_query_plan(totals, cap, rank_of, first, length, set_off, F=4, q=(99, 100), headers=None, fields=None):
    """gpudh_box_query_plan: (rc, message, route [n_sets], owner [n_sets], send_bytes [3], consistent headers [n_ranks][16],
    pivot reads per set [n_sets], the rank of each pivot read [n_sets][8192]); with a list of fields, gpudh_box_query_plan_fields for
    a query over those fields of rings of F fields"""
    L = lib()
    totals = np.ascontiguousarray(totals, dtype=np.int64)
    ro, fi, ln, so = _box_args(rank_of, first, length, set_off)
    n_sets = so.shape[0] - 1
    hdr = np.zeros((totals.shape[0], 16), dtype=np.int64)
    hin = None if headers is None else np.ascontiguousarray(headers, dtype=np.int64)
    route, owner, sb = np.zeros(n_sets, np.int32), np.zeros(n_sets, np.int32), np.zeros(3, np.int64)
    piv_n = np.zeros(n_sets, np.int32)
    piv_owner = np.full((n_sets, 8192), -1, np.int32) if n_sets <= 4096 else None    # the owners only for calls of a few sets
    msg = C.create_string_buffer(512)
    rest = (C.c_void_p(ro.ctypes.data), C.c_void_p(fi.ctypes.data), C.c_void_p(ln.ctypes.data), fi.shape[0], C.c_void_p(so.ctypes.data), n_sets,
            C.c_void_p(hdr.ctypes.data), C.c_void_p(hin.ctypes.data) if hin is not None else None,
            C.c_void_p(route.ctypes.data), C.c_void_p(owner.ctypes.data), C.c_void_p(sb.ctypes.data),
            C.c_void_p(piv_n.ctypes.data), C.c_void_p(piv_owner.ctypes.data) if piv_owner is not None else None, msg, 512)
    if fields is None:
        rc = L.gpudh_box_query_plan(totals.shape[0], C.c_void_p(totals.ctypes.data), cap, F, q[0], q[1], *rest)
    else:
        fl = np.ascontiguousarray(fields, dtype=np.int32).reshape(-1)
        rc = L.gpudh_box_query_plan_fields(totals.shape[0], C.c_void_p(totals.ctypes.data), cap, F, C.c_void_p(fl.ctypes.data), fl.shape[0],
                                           q[0], q[1], *rest)
    return rc, msg.value.decode(), route, owner, sb, hdr, piv_n, piv_owner


class Ring:
    """gpud_ring: device-resident [F][CAP] sample ring with fused windowed aggregates."""

    def __init__(self, ctx: Context, n_fields: int, capacity: int, window: int, thresholds: Optional[np.ndarray] = None,
                 ema_alpha: float = 0.0, q_num: int = 0, q_den: int = 0, dev: Optional[int] = None):
        self.ctx, self._L = ctx, ctx._L
        self.F, self.cap, self.W = n_fields, capacity, window
        self.dev = ctx.devices[0] if dev is None else dev
        cfg = RingCfg(n_fields, window, capacity, ema_alpha, q_num, q_den, None)
        if thresholds is not None:
            self._thr = np.ascontiguousarray(thresholds, dtype=np.float64)
            assert self._thr.shape == (n_fields,)
            cfg.thresholds = self._thr.ctypes.data_as(C.POINTER(C.c_double))
        h = C.c_void_p()
        ctx._check(self._L.gpud_ring_create(ctx._h, ctx.devices[0] if dev is None else dev, C.byref(cfg), C.byref(h)))
        self._h = h

    def close(self):
        if self._h:
            self._L.gpud_ring_destroy(self._h)
            self._h = None

    def set_cta_reserve(self, n_ctas: int):
        self.ctx._check(self._L.gpud_ring_set_cta_reserve(self._h, n_ctas))

    def set_stream(self, cuda_stream: int):
        self.ctx._check(self._L.gpud_ring_set_stream(self._h, C.c_void_p(cuda_stream)))

    def push(self, rows: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=np.float64)
        assert rows.ndim == 2 and rows.shape[1] == self.F
        self.ctx._check(self._L.gpud_ring_push(self._h, C.c_void_p(rows.ctypes.data), rows.shape[0]))

    def push_ptr(self, host_ptr: int, n_rows: int):
        self.ctx._check(self._L.gpud_ring_push(self._h, C.c_void_p(host_ptr), n_rows))

    def push_raw(self, rows: np.ndarray):
        """rows [n][F] of raw counter samples in the getter's own type (uint32 / int32 / float32 / int64 / uint64 / float64)"""
        rows = np.ascontiguousarray(rows)
        assert rows.ndim == 2 and rows.shape[1] == self.F
        self.ctx._check(self._L.gpud_ring_push_raw(self._h, C.c_void_p(rows.ctypes.data), rows.shape[0], DTYPES[rows.dtype.name]))

    def push_raw_ptr(self, host_ptr: int, n_rows: int, dtype: int):
        self.ctx._check(self._L.gpud_ring_push_raw(self._h, C.c_void_p(host_ptr), n_rows, dtype))

    def push_device(self, dev_ptr: int, n_rows: int):
        self.ctx._check(self._L.gpud_ring_push_device(self._h, C.c_void_p(dev_ptr), n_rows))

    def counts(self):
        t, c, w = C.c_int64(), C.c_int64(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_counts(self._h, C.byref(t), C.byref(c), C.byref(w)))
        return t.value, c.value, w.value

    def reduce(self):
        self.ctx._check(self._L.gpud_ring_reduce(self._h))

    def sync(self):
        self.ctx._check(self._L.gpud_ring_sync(self._h))

    def kernel_ms(self):
        a, b = C.c_float(), C.c_float()
        self.ctx._check(self._L.gpud_ring_kernel_ms(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def read(self, op: str) -> np.ndarray:
        _, _, nw = self.counts()
        dt = np.uint32 if op == "n_over" else np.float64
        out = np.empty((self.F, nw), dtype=dt)
        self.ctx._check(self._L.gpud_ring_read(self._h, OPS[op], C.c_void_p(out.ctypes.data), out.nbytes))
        return out

    def result_ptr(self, op: str) -> int:
        p = C.c_void_p()
        self.ctx._check(self._L.gpud_ring_result_ptr(self._h, OPS[op], C.byref(p)))
        return p.value

    def reduce_all(self) -> dict:
        self.reduce()
        return {k: self.read(k) for k in OPS}

    # ---- stream windows: window k = samples [kW, (k+1)W) of the whole push order, reduced once into a history ----
    def stream_open(self, history_windows: int = 0):
        """history_windows <= 0: ceil(capacity / window)"""
        self.ctx._check(self._L.gpud_ring_stream_open(self._h, history_windows))

    def stream_reduce(self):
        """reduce every complete window not reduced yet (asynchronous); -> (windows reduced, windows lost before this call)"""
        a, b = C.c_int64(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_stream_reduce(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def stream_counts(self):
        """-> (first, next, lost_total): the history holds windows [first, next)"""
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_stream_counts(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def stream_read(self, op: str, first: int, n: int) -> np.ndarray:
        """windows [first, first + n) of one aggregate of the history, [F][n]"""
        out = np.empty((self.F, n), dtype=np.uint32 if op == "n_over" else np.float64)
        self.ctx._check(self._L.gpud_ring_stream_read(self._h, OPS[op], first, n, C.c_void_p(out.ctypes.data), out.nbytes))
        return out

    def windows(self, span: int, history: int = 0, hop: int = None, fields=None) -> "RingWindows":
        """stream windows of span x window samples each, one every hop x window samples (gpud_ring_windows_open_hop; hop None or
        span: tumbling windows); history <= 0: ceil(capacity / (hop x window)).  With a list of fields the handle reduces, keeps and
        checkpoints only those (gpud_ring_windows_open_fields): its row g is field fields[g]."""
        return RingWindows(self, span, history, hop, fields)

    def reduce_range(self, last_n: int = 0) -> dict:
        f64 = np.empty((5, self.F), dtype=np.float64)
        nov = np.empty((self.F,), dtype=np.uint32)
        self.ctx._check(self._L.gpud_ring_reduce_range(self._h, last_n, C.c_void_p(f64.ctypes.data), C.c_void_p(nov.ctypes.data)))
        return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}

    def range_stats(self):
        """Device ms of the last single-pass reduce_range (fused pass alone, whole device side) and the number of fields the
        radix select had to redo."""
        a, b, n = C.c_float(), C.c_float(), C.c_int32()
        why = (C.c_int32 * 7)()
        self.ctx._check(self._L.gpud_ring_range_stats(self._h, C.byref(a), C.byref(b), C.byref(n), why))
        self.range_open_reasons = {k: int(why[i]) for i, k in enumerate(("", "short", "nan", "pivots", "above", "below", "overflow")) if i and why[i]}
        return float(a.value), float(b.value), int(n.value)

    def reduce_ranges(self, first, length, fields=None) -> dict:
        """Aggregates of samples [first[i], first[i] + length[i]) of the push order (sample 0 = the first ever pushed), each range one
        window with the definitions of reduce_range: {op: [F][n]}; with a list of fields, only those ({op: [len(fields)][n]}, row g
        field fields[g], as reduce_range_sets(fields=...) over one range per set)"""
        first = np.ascontiguousarray(first, dtype=np.int64).reshape(-1)
        length = np.ascontiguousarray(length, dtype=np.int64).reshape(-1)
        assert first.shape == length.shape
        n = first.shape[0]
        if fields is not None:
            return self.reduce_range_sets(first, length, np.arange(n + 1, dtype=np.int64), fields=fields)
        f64 = np.empty((5, self.F, n), dtype=np.float64)
        nov = np.empty((self.F, n), dtype=np.uint32)
        self.ctx._check(self._L.gpud_ring_reduce_ranges(self._h, C.c_void_p(first.ctypes.data), C.c_void_p(length.ctypes.data), n,
                                                        C.c_void_p(f64.ctypes.data), C.c_void_p(nov.ctypes.data)))
        return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}

    def reduce_range_sets(self, first, length, set_off, fields=None) -> dict:
        """Aggregates of sets of ranges: set s is ranges set_off[s] .. set_off[s + 1] - 1 of (first, length), its samples theirs
        concatenated in that order, reduced as one window with the definitions of reduce_range (the EMA runs across the joins):
        {op: [F][n_sets]}; with a list of fields, only those are read (gpud_rings_reduce_range_sets_fields on this ring alone) and
        row g is field fields[g]: {op: [len(fields)][n_sets]}"""
        first = np.ascontiguousarray(first, dtype=np.int64).reshape(-1)
        length = np.ascontiguousarray(length, dtype=np.int64).reshape(-1)
        set_off = np.ascontiguousarray(set_off, dtype=np.int64).reshape(-1)
        assert first.shape == length.shape and set_off.shape[0] >= 1
        if fields is not None:
            hs = (C.c_void_p * 1)(self._h.value)
            return _range_sets_fields(self, C.cast(hs, C.c_void_p), 1, None, fields, first, length, set_off)
        n_sets = set_off.shape[0] - 1
        f64 = np.empty((5, self.F, n_sets), dtype=np.float64)
        nov = np.empty((self.F, n_sets), dtype=np.uint32)
        self.ctx._check(self._L.gpud_ring_reduce_range_sets(self._h, C.c_void_p(first.ctypes.data), C.c_void_p(length.ctypes.data), first.shape[0],
                                                            C.c_void_p(set_off.ctypes.data), n_sets, C.c_void_p(f64.ctypes.data),
                                                            C.c_void_p(nov.ctypes.data)))
        return {"min": f64[0], "max": f64[1], "mean": f64[2], "ema": f64[3], "p99": f64[4], "n_over": nov}

    def ranges_stats(self):
        """the last reduce_ranges or reduce_range_sets: (device ms, segments sent to the radix select, {reason: segments})"""
        ms, n = C.c_float(), C.c_int64()
        why = (C.c_int32 * len(RANGE_OPEN_REASONS))()
        self.ctx._check(self._L.gpud_ring_ranges_stats(self._h, C.byref(ms), C.byref(n), why))
        return float(ms.value), int(n.value), {k: int(why[i]) for i, k in enumerate(RANGE_OPEN_REASONS) if i and why[i]}

    # ---- checkpoints: samples, push count, config and handles as bytes that outlive the process ----
    def checkpoint_bound(self) -> int:
        n = C.c_int64()
        self.ctx._check(self._L.gpud_ring_checkpoint_bound(self._h, C.byref(n)))
        return n.value

    def _write_blob(self, write, bound, out):
        """one checkpoint call, full or delta: out None -> the bytes, sized by bound(); otherwise into out -> their length"""
        n = C.c_int64()
        if out is None:
            buf = bytearray(bound())
            cbuf = (C.c_char * max(1, len(buf))).from_buffer(buf)
            self.ctx._check(write(self._h, C.cast(cbuf, C.c_void_p), len(buf), C.byref(n)))
            del cbuf
            return bytes(memoryview(buf)[:n.value])
        mv = memoryview(out).cast("B")
        cbuf = (C.c_char * len(mv)).from_buffer(mv)
        self.ctx._check(write(self._h, C.cast(cbuf, C.c_void_p), len(mv), C.byref(n)))
        return n.value

    def checkpoint(self, out=None):
        """gpud_ring_checkpoint.  out None: -> the checkpoint as bytes.  Otherwise a writable buffer (bytearray, numpy array, pinned
        memory as a ctypes array) that receives it: -> its length in bytes."""
        return self._write_blob(self._L.gpud_ring_checkpoint, self.checkpoint_bound, out)

    def restore(self, blob) -> List["RingWindows"]:
        """gpud_ring_restore into this ring (just created with the checkpoint's config, never pushed into, no handle open): -> the
        windows handles in the order they had been opened.  The stream handle, if there was one, is open again on the ring."""
        mv, src = _blob_ptr(blob)
        recs = checkpoint_handles(mv)
        cap = sum(1 for kind, _, _ in recs if kind != 0)
        hs = (C.c_void_p * max(1, cap))()
        n = C.c_int32()
        self.ctx._check(self._L.gpud_ring_restore(self._h, src, len(mv), hs, cap, C.byref(n)))
        wins = [(span, hop) for kind, span, hop in recs if kind != 0]
        return [RingWindows._adopt(self, hs[i], span, hop) for i, (span, hop) in enumerate(wins[:n.value])]

    # ---- delta checkpoints: only what changed since the last checkpoint written or loaded, full or delta ----
    def checkpoint_delta_bound(self) -> int:
        n = C.c_int64()
        self.ctx._check(self._L.gpud_ring_checkpoint_delta_bound(self._h, C.byref(n)))
        return n.value

    def checkpoint_delta(self, out=None):
        """gpud_ring_checkpoint_delta: everything since the ring's chain marker, which then moves to this delta.  out None: -> the
        delta as bytes.  Otherwise a writable buffer (bytearray, numpy array, pinned memory as a ctypes array): -> its length."""
        return self._write_blob(self._L.gpud_ring_checkpoint_delta, self.checkpoint_delta_bound, out)

    def restore_delta(self, blob) -> None:
        """gpud_ring_restore_delta: apply the next delta of the chain onto this ring (a base restored, the deltas before it applied)"""
        mv, src = _blob_ptr(blob)
        self.ctx._check(self._L.gpud_ring_restore_delta(self._h, src, len(mv)))

    def checkpoint_stats(self):
        """the last checkpoint / restore, full or delta: (encode device ms, decode device ms, {"raw": blocks, "int": blocks})"""
        enc, dec = C.c_float(), C.c_float()
        blocks = (C.c_int64 * 2)()
        self.ctx._check(self._L.gpud_ring_checkpoint_stats(self._h, C.byref(enc), C.byref(dec), blocks))
        return float(enc.value), float(dec.value), {"raw": int(blocks[0]), "int": int(blocks[1])}

    # ---- the tier: older samples kept delta-coded on the device, reached by reduce_ranges / reduce_range_sets ----
    def tier_open(self, tier_bytes: int):
        """gpud_ring_tier_open: keep block rows of 1024 samples, coded as checkpoint blocks, in tier_bytes of device memory"""
        self.ctx._check(self._L.gpud_ring_tier_open(self._h, tier_bytes))

    def tier_counts(self):
        """-> (first_sample, next_sample, bytes_used, rows_lost_total): the tier holds samples [first_sample, next_sample)"""
        v = [C.c_int64() for _ in range(4)]
        self.ctx._check(self._L.gpud_ring_tier_counts(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def tier_stats(self):
        """-> (device ms of the last encode, device ms of the last range call's decode, {"raw": blocks, "int": blocks} of that encode)"""
        enc, dec = C.c_float(), C.c_float()
        blocks = (C.c_int64 * 2)()
        self.ctx._check(self._L.gpud_ring_tier_stats(self._h, C.byref(enc), C.byref(dec), blocks))
        return float(enc.value), float(dec.value), {"raw": int(blocks[0]), "int": int(blocks[1])}

    def tier_row(self, row: int) -> bytes:
        """test hook gpudh_ring_tier_row: block row `row` as it lies in the tier (record, then the blocks)"""
        n = C.c_int64()
        rc = self._L.gpudh_ring_tier_row(self._h, row, None, 0, C.byref(n))
        if rc not in (0, -4):
            self.ctx._check(rc)
        buf = np.empty(n.value, dtype=np.uint8)
        self.ctx._check(self._L.gpudh_ring_tier_row(self._h, row, C.c_void_p(buf.ctypes.data), n.value, C.byref(n)))
        return buf.tobytes()

    def tier_group(self, max_fields: int):
        """test hook gpudh_ring_tier_group: at most max_fields fields per decoded group (0: the default)"""
        self.ctx._check(self._L.gpudh_ring_tier_group(self._h, max_fields))

    # ---- tier checkpoints: the tier's rows as bytes that outlive the process, with a marker of their own ----
    def tier_checkpoint_bound(self) -> int:
        n = C.c_int64()
        self.ctx._check(self._L.gpud_ring_tier_checkpoint_bound(self._h, C.byref(n)))
        return n.value

    def tier_checkpoint(self, out=None):
        """gpud_ring_tier_checkpoint: the rows the tier holds; the tier marker moves to this blob.  out as for checkpoint()."""
        return self._write_blob(self._L.gpud_ring_tier_checkpoint, self.tier_checkpoint_bound, out)

    def tier_checkpoint_delta_bound(self) -> int:
        n = C.c_int64()
        self.ctx._check(self._L.gpud_ring_tier_checkpoint_delta_bound(self._h, C.byref(n)))
        return n.value

    def tier_checkpoint_delta(self, out=None):
        """gpud_ring_tier_checkpoint_delta: the tier's rows since its marker, which then moves to this delta.  out as for checkpoint()."""
        return self._write_blob(self._L.gpud_ring_tier_checkpoint_delta, self.tier_checkpoint_delta_bound, out)

    def tier_restore(self, tier_bytes: int, blobs) -> None:
        """gpud_ring_tier_restore: open this ring's tier of tier_bytes from a chain, a full tier checkpoint then its deltas in order"""
        views = [_blob_ptr(b) for b in blobs]
        ptrs = (C.c_void_p * max(1, len(views)))(*[src for _, src in views])
        sizes = (C.c_int64 * max(1, len(views)))(*[len(mv) for mv, _ in views])
        self.ctx._check(self._L.gpud_ring_tier_restore(self._h, tier_bytes, ptrs, sizes, len(views)))

    def tier_checkpoint_stats(self):
        """the last tier checkpoint or tier restore: (export + check device ms, check + load device ms, rows written or loaded)"""
        enc, dec, rows = C.c_float(), C.c_float(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_tier_checkpoint_stats(self._h, C.byref(enc), C.byref(dec), C.byref(rows)))
        return float(enc.value), float(dec.value), int(rows.value)


def _blob_ptr(blob):
    """a checkpoint's bytes as a byte view and the pointer the restore calls take (None for no bytes)"""
    mv = memoryview(blob).cast("B")
    return mv, C.c_void_p(np.frombuffer(mv, dtype=np.uint8).ctypes.data) if len(mv) else None


def checkpoint_handles(blob) -> List[tuple]:
    """(kind, span, hop) of each handle record of a checkpoint (kind 0: the stream handle, 1: a windows handle, 2: a windows handle
    over chosen fields), read from its header and handle section (DESIGN.md "Ring checkpoint format"); [] for bytes too short to hold
    them"""
    import struct
    mv = memoryview(blob).cast("B")
    if len(mv) < 128:
        return []
    F, n_rec = struct.unpack_from("<I4xI", mv, 12)
    thr, dirb, pay, sm = struct.unpack_from("<4q", mv, 64)
    off, out = 128 + thr + dirb + pay + sm, []
    for _ in range(n_rec):
        if off < 0 or off + 64 > len(mv):
            break
        kind, span, hop, _, first, nxt = struct.unpack_from("<6q", mv, off)
        n, nf = nxt - first, F
        out.append((kind, span, hop))
        off += 64
        if kind == 2:
            if off + 8 > len(mv):
                break
            nf = struct.unpack_from("<q", mv, off)[0]
            off += 8 + ((4 * nf + 7) & ~7)
        off += 40 * nf * n + ((4 * nf * n + 7) & ~7) + 8 * nf
    return out


RANGE_OPEN_REASONS = ("", "short", "nan", "pivots", "above", "below", "overflow")


class RingWindows:
    """gpud_ring_windows: window k = samples [kP, kP + L) of the ring's push order, L = span x window, P = hop x window, reduced once
    into a history.  The ring frees a handle that is still open when it is closed itself."""

    def __init__(self, ring: Ring, span: int, history: int = 0, hop: int = None, fields=None):
        self.ring, self.ctx, self._L = ring, ring.ctx, ring._L
        self.hop = span if hop is None else hop
        self.span, self.L, self.P = span, span * ring.W, self.hop * ring.W
        h = C.c_void_p()
        if fields is not None:
            f = np.ascontiguousarray(fields, dtype=np.int32).reshape(-1)
            self.ctx._check(self._L.gpud_ring_windows_open_fields(ring._h, span, self.hop, history, C.c_void_p(f.ctypes.data),
                                                                  f.shape[0], C.byref(h)))
        elif hop is None:
            self.ctx._check(self._L.gpud_ring_windows_open(ring._h, span, history, C.byref(h)))
        else:
            self.ctx._check(self._L.gpud_ring_windows_open_hop(ring._h, span, hop, history, C.byref(h)))
        self._h = h
        self.n_fields = ring.F if fields is None else len(f)

    @classmethod
    def _adopt(cls, ring: Ring, handle, span: int, hop: int) -> "RingWindows":
        """wrap a handle the library opened itself (Ring.restore)"""
        self = cls.__new__(cls)
        self.ring, self.ctx, self._L = ring, ring.ctx, ring._L
        self.span, self.hop, self.L, self.P = span, hop, span * ring.W, hop * ring.W
        self._h = C.c_void_p(handle)
        self.n_fields = len(self.fields())
        return self

    def fields(self) -> np.ndarray:
        """the ring field of each row of the history (gpud_ring_windows_fields): the list of a handle over chosen fields, else 0 .. F - 1"""
        n = C.c_int32()
        rc = self._L.gpud_ring_windows_fields(self._h, None, 0, C.byref(n))
        if rc not in (0, -4):
            self.ctx._check(rc)
        out = np.empty(n.value, dtype=np.int32)
        self.ctx._check(self._L.gpud_ring_windows_fields(self._h, C.c_void_p(out.ctypes.data), n.value, C.byref(n)))
        return out

    def close(self):
        if self._h and self.ring._h:
            self.ctx._check(self._L.gpud_ring_windows_close(self._h))
        self._h = None

    def reduce(self):
        """reduce every complete window not reduced yet; -> (windows reduced, windows lost before this call)"""
        a, b = C.c_int64(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_windows_reduce(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def counts(self):
        """-> (first, next, lost_total): the history holds windows [first, next)"""
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        self.ctx._check(self._L.gpud_ring_windows_counts(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def read(self, op: str, first: int, n: int) -> np.ndarray:
        """windows [first, first + n) of one aggregate of the history, [n_fields][n] (n_fields = F for an all-field handle)"""
        out = np.empty((self.n_fields, n), dtype=np.uint32 if op == "n_over" else np.float64)
        self.ctx._check(self._L.gpud_ring_windows_read(self._h, OPS[op], first, n, C.c_void_p(out.ctypes.data), out.nbytes))
        return out

    def stats(self):
        """the last reduce that reduced windows: (device ms, segments sent to the radix select, {reason: segments})"""
        ms, n = C.c_float(), C.c_int64()
        why = (C.c_int32 * len(RANGE_OPEN_REASONS))()
        self.ctx._check(self._L.gpud_ring_windows_stats(self._h, C.byref(ms), C.byref(n), why))
        return float(ms.value), int(n.value), {k: int(why[i]) for i, k in enumerate(RANGE_OPEN_REASONS) if i and why[i]}
