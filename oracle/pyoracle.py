"""CPU restatement of gpud's Xid/SXid match-and-classify path and the windowed aggregates.

TEST INFRASTRUCTURE ONLY.  Nothing under gpud_b200/ may import this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it, as the checker.

Every function cites the reference file:line it follows (paths relative to the reference root).
The regex strings are the reference's verbatim patterns run through Python `re` on *bytes*
(so `\\d`, `\\s` are ASCII like Go RE2; both engines are leftmost-first).  Parity status:
  * match / classify / health-state / thresholds / fabric: PINNED by the reference's own test
    vectors in tests/golden/ (extracted by tools/gen_golden.py).
  * windowed min/max/mean/EMA/p99/n_over: the reference has no implementation -> PARITY UNPINNED;
    the definitions are ours (oracle/SPEC.md).
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
CATALOG = json.load(open(os.path.join(_HERE, "catalog.json")))

EV_UNKNOWN, EV_INFO, EV_WARNING, EV_CRITICAL, EV_FATAL = 0, 1, 2, 3, 4
EVENT_NAMES = ["Unknown", "Info", "Warning", "Critical", "Fatal"]
ACT_IGNORE, ACT_REBOOT, ACT_HW_INSPECTION, ACT_CHECK_APP = 1, 2, 3, 4
ACTION_WIRE = {1: "IGNORE_NO_ACTION_REQUIRED", 2: "REBOOT_SYSTEM", 3: "HARDWARE_INSPECTION", 4: "CHECK_USER_APP_AND_GPU"}
ACTION_NAMES = {1: "IgnoreNoActionRequired", 2: "RebootSystem", 3: "HardwareInspection", 4: "CheckUserAppAndGPU"}

# --------------------------------------------------------------------------------------------
# regexes: components/accelerator/nvidia/xid/kmsg.go:22,29,38,43 ; sxid/kmsg.go:17,20  (verbatim)
# --------------------------------------------------------------------------------------------
R1 = re.compile(rb"NVRM: Xid \(((?:PCI:)?[0-9a-fA-F:]+)\).*?: (\d+),")
R2 = re.compile(rb"NVRM: Xid \(PCI:([0-9a-fA-F:]+)\): (\d+)(?:, pid=(\d+), name=([^,]+))?, ([A-Z_]+(?:/[A-Z_]+)?)[\t\n\f\r ]+(Nonfatal|Fatal)[\t\n\f\r ]+(XC[01])[\t\n\f\r ]+(i\d+)[\t\n\f\r ]+Link[\t\n\f\r ]+(-?\d+)[\t\n\f\r ]+\((0x[0-9a-fA-F]+)[\t\n\f\r ]+(0x[0-9a-fA-F]+)(?:[\t\n\f\r ]+(0x[0-9a-fA-F]+))?(?:[\t\n\f\r ]+(0x[0-9a-fA-F]+))?(?:[\t\n\f\r ]+(0x[0-9a-fA-F]+))?(?:[\t\n\f\r ]+(0x[0-9a-fA-F]+))?")
R3 = re.compile(rb"(?s)NVRM:[\t\n\f\r ]+The NVIDIA GPU ((?:[0-9a-fA-F]{4}:)?[0-9a-fA-F]{2}:[0-9a-fA-F]{2})\.0.*?fallen off the bus and is not responding to commands\.")
R4 = re.compile(rb"NVRM:[\t\n\f\r ]+GPU ((?:[0-9a-fA-F]{4}:)?[0-9a-fA-F]{2}:[0-9a-fA-F]{2})\.0:[\t\n\f\r ]+GPU has fallen off the bus\.?")
R5 = re.compile(rb"SXid.*?: (\d+),")
R6 = re.compile(rb"SXid \((PCI:[0-9a-fA-F:\.]+)\)")
# next matchers riding the same scanner (SURVEY §8f.1): the stateless line patterns, regex strings verbatim.
# (kind, component, eventName, message, regex, capture group appended to the message or None) -- reference file:line
EXT_PATTERNS = [
    (3, "nccl", "nvidia_nccl_segfault_in_libnccl", "NCCL communication error (segfault in libnccl.so)",
     rb".*segfault at.*in libnccl\.so.*", None),                                           # nccl/kmsg_matcher.go:11-13
    (4, "peermem", "nvidia_peermem_invalid_context", "peermem error detected (possible GPU communication issue)",
     rb".*ERROR detected invalid context, skipping further processing", None),            # peermem/kmsg_matcher.go:13-15
    (5, "infiniband", "pci_power_insufficient", "Insufficient power on MLX5 PCIe slot",
     rb"Detected insufficient power on the PCIe slot \(([0-9]+W)\)", None),                # infiniband/kmsg_matcher.go:14-16
    (6, "infiniband", "port_module_high_temperature", "Overheated MLX5 adapter",
     rb"Port module event.*High Temperature", None),                                      # infiniband/kmsg_matcher.go:24-26
    (7, "infiniband", "access_reg_failed", "MLX5 ACCESS_REG command failed - device may have restricted PF access",
     rb"mlx5_cmd_out_err.*ACCESS_REG.*failed", None),                                     # infiniband/kmsg_matcher.go:56-58
    (8, "cpu", "cpu_blocked_too_long", "CPU task blocked for more than 120 seconds",
     rb"(?:INFO: )?task ([^:]+:[\d]+).+blocked for more than \d+ seconds", 1),             # cpu/kmsg_matcher.go:17-19
    (9, "cpu", "cpu_soft_lockup", "CPU soft lockup detected, not releasing for a period of time",
     rb"soft lockup - CPU#\d+ stuck for \d+s! \[([^:]+:[\d]+)\]", 1),                      # cpu/kmsg_matcher.go:29-31
    (10, "os", "vfs_file_max_limit_reached", "VFS file-max limit reached", rb"VFS: file-max limit \d+ reached", None),   # os/kmsg_matcher.go:17-19
    (11, "disk", "raid_array_failure", "RAID array has failed due to disk failure",
     rb"md/raid.*: Disk failure on .* detected, failing array", None),                    # disk/kmsg_matcher.go:10-12
    (12, "disk", "filesystem_read_only", "filesystem remounted as read-only due to errors", rb".*Remounting filesystem read-only", None),   # :18-20
    (13, "disk", "nvme_path_failure", "NVMe device has no available path, I/O failing", rb"block nvme.*: no available path - failing I/O", None),   # :24-26
    (14, "disk", "nvme_controller_timeout", "NVME controller I/O timeout detected, attempting reset",
     rb"nvme nvme[0-9]+: I/O .* timeout, reset controller", None),                         # :30-32
    (15, "disk", "nvme_device_disabled", "NVME device disabled after reset failure", rb"nvme nvme[0-9]+: Disabling device after reset failure", None),   # :36-38
    (16, "disk", "beyond_end_of_device", "I/O attempt beyond device boundaries detected", rb"attempt to access beyond end of device", None),   # :42-44
    (17, "disk", "buffer_io_error", "Buffer I/O error detected on device", rb"Buffer I/O error on dev [^ ]+, logical block [0-9]+", None),   # :48-50
    (18, "disk", "superblock_write_error", "I/O error while writing superblock", rb"I/O error while writing superblock", None),   # :54-56
    # line primitives of the two STATEFUL matchers (their events are assembled by KernelPanicMatcher / OOMMatcher below)
    (19, "os", "", "", rb"Kernel [Pp]anic", None),                                        # os/kmsg_matcher.go:35
    (20, "os", "", "", rb"CPU: (\d+) PID: (\d+) Comm: (\S+)", None),                      # os/kmsg_matcher.go:39
    (21, "memory", "", "", rb"invoked oom-killer:", None),                                # memory/kmsg_matcher.go:156
    (22, "memory", "", "", rb"oom-kill:constraint=(.*),nodemask=(.*),cpuset=(.*),mems_allowed=(.*),oom_memcg=(.*),task_memcg=(.*),task=(.*),pid=(.*),uid=(.*)", None),   # :148
    (23, "memory", "", "", rb"Task in (.*) killed as a result of limit of (.*)", None),   # memory/kmsg_matcher.go:143
    (24, "memory", "", "", rb"Killed process ([0-9]+) \((.+)\)", None),                   # memory/kmsg_matcher.go:152
]
N_STATELESS_KINDS = 19          # kinds 3..18 are complete matchers; 19..24 are primitives
# which capture groups of a primitive the product reports, in the order of the hit's span slots
# (dev, unit_name, pid, pname, inj): os/kmsg_matcher.go:133-157, memory/kmsg_matcher.go:159-208
PRIM_GROUPS = {20: (1, None, 2, 3, None), 22: (1, 5, 8, 7, 6), 23: (1, 2, None, None, None), 24: (None, None, 1, 2, None)}
EXT_RE = {k: re.compile(rx) for k, _c, _e, _m, rx, _g in EXT_PATTERNS}
EXT_BY_KIND = {k: (c, e, m, g) for k, c, e, m, _rx, g in EXT_PATTERNS}
R_PCI_DEVICE = re.compile(rb"\b[0-9a-fA-F]{4}:[0-9a-fA-F]{2}:[0-9a-fA-F]{2}\.[0-7]\b")       # infiniband/kmsg_matcher.go:59
# NOTE: Go/RE2 `\s` is [\t\n\f\r ] (no \v); Python bytes `\s` also matches \v, hence the explicit class.

INT64_MAX = (1 << 63) - 1


def go_atoi(b: bytes) -> Optional[int]:
    """strconv.Atoi: optional sign, then ASCII digits only; None on syntax or range error (int is 64-bit)."""
    if not re.fullmatch(rb"[+-]?[0-9]+", b):
        return None
    v = int(b)
    if v > INT64_MAX or v < -INT64_MAX - 1:
        return None
    return v


def go_parse_uint32_base0(b: bytes) -> Optional[int]:
    """strconv.ParseUint(s, 0, 32) for the `0x[0-9a-fA-F]+` strings the regex admits."""
    v = int(b, 16)
    return v if v <= 0xFFFFFFFF else None


# --------------------------------------------------------------------------------------------
# catalog tables + NVLink sub-code detail maps   (xid/xid.go:74-117, 2954-3343)
# --------------------------------------------------------------------------------------------
@dataclass
class Detail:
    code: int
    description: str
    event_type: int
    actions: Optional[List[int]]          # None == SuggestedActionsByGPUd nil
    sub_code: int = 0
    sub_code_description: str = ""
    error_status: int = 0
    investigatory_hint: str = ""

    def copy(self) -> "Detail":
        return Detail(self.code, self.description, self.event_type,
                      None if self.actions is None else list(self.actions),
                      self.sub_code, self.sub_code_description, self.error_status, self.investigatory_hint)


XID_DETAILS: Dict[int, Detail] = {
    d["code"]: Detail(d["code"], d["description"], d["event_type"], list(d["actions"]) if d["actions"] else None)
    for d in CATALOG["xid"]}
MNEMONIC = {e["Code"]: e["Mnemonic"] for e in CATALOG["catalog_entries"]}
NVLINK_RULES = CATALOG["nvlink_rules"]
SXID_DETAILS = {d["sxid"]: d for d in CATALOG["sxid"]}


def get_detail(code: int) -> Optional[Detail]:                      # xid.go:74-77
    d = XID_DETAILS.get(code)                                          # a copy, like Go's &e of the map value: callers
    return None if d is None else d.copy()                             # (detailFromNVLinkInfo) edit what they get


def event_type_from_severity(s: str) -> int:                         # xid.go:3263-3272
    s = s.strip().lower()
    if s in ("fatal", "fatal**", "link fatal", "link fatal?"):
        return EV_FATAL
    if s in ("non-fatal", "non-fatal*"):
        return EV_WARNING
    return EV_UNKNOWN


def event_type_from_log_severity(s: str) -> int:                     # xid.go:3274-3283
    s = s.strip().lower()
    if s == "fatal":
        return EV_FATAL
    if s in ("nonfatal", "non-fatal"):
        return EV_WARNING
    return EV_UNKNOWN


_FATAL_BUCKETS = {"CONTACT_SUPPORT", "CHECK_MECHANICALS", "WORKFLOW_NVLINK_ERR", "WORKFLOW_NVLINK5_ERR", "XID_154",
                  "XID_154_EVAL", "RESTART_BM"}
_CRIT_BUCKETS = {"RESET_GPU", "RESTART_APP", "RESTART_VM", "CHECK_UVM", "WORKFLOW_XID_48", "WORKFLOW_XID_45", "UPDATE_SWFW"}


def event_type_from_immediate_bucket(b: str) -> int:                 # xid.go:3222-3246
    if b in _FATAL_BUCKETS:
        return EV_FATAL
    if b in _CRIT_BUCKETS:
        return EV_CRITICAL
    if b in ("IGNORE", ""):
        return EV_INFO
    return EV_WARNING


def suggested_actions_from_bucket(b: str) -> Optional[List[int]]:    # xid.go:3248-3261
    if b in ("CONTACT_SUPPORT", "CHECK_MECHANICALS", "WORKFLOW_NVLINK_ERR", "WORKFLOW_NVLINK5_ERR", "XID_154", "XID_154_EVAL"):
        return [ACT_HW_INSPECTION]
    if b in ("RESET_GPU", "RESTART_BM", "RESTART_VM", "CHECK_UVM"):
        return [ACT_REBOOT]
    if b in ("RESTART_APP", "WORKFLOW_XID_45", "WORKFLOW_XID_48", "UPDATE_SWFW"):
        return [ACT_CHECK_APP]
    if b in ("IGNORE", ""):
        return [ACT_IGNORE]
    return None


def max_event_type(a: int, b: int) -> int:                           # xid.go:3285-3305 (rank == numeric id)
    return b if b > a else a


def merge_actions(base, add):                                        # xid.go:3317-3336 (sorted by wire string)
    if base is None:
        return None if add is None else list(add)
    if add is None:
        return list(base)
    return sorted(set(base) | set(add), key=lambda a: ACTION_WIRE[a])


def sample_from_pattern(p: str) -> Optional[int]:                    # xid.go:3127-3145
    if len(p) != 32:
        return None
    v = 0
    for i, ch in enumerate(p):
        if ch == "1":
            v |= 1 << (31 - i)
        elif ch not in "0-":
            return None
    return v


def pattern_matches(p: str, intrinfo: int) -> bool:                  # xid.go:3147-3172
    if p == "":
        return True
    if len(p) != 32:
        return False
    for i, ch in enumerate(p):
        bit = (intrinfo >> (31 - i)) & 1
        if ch == "1":
            if bit == 0:
                return False
        elif ch == "0":
            if bit == 1:
                return False
        elif ch != "-":
            return False
    return True


def normalize_unit(s: str) -> str:                                   # xid.go:3203-3218
    s = s.strip().upper().replace("-", "_")
    return "".join(c for c in s if ("A" <= c <= "Z") or ("0" <= c <= "9") or c == "_")


def unit_aliases(u: str) -> List[str]:                               # xid.go:3188-3201
    al = [x for x in re.split(r"[/,() ]", u) if x]
    if not al:
        al = [u]
    return al + [u]


def unit_matches(rule_unit: str, log_unit: str) -> bool:             # xid.go:3174-3186
    c = normalize_unit(log_unit)
    if c == "":
        return False
    return any(normalize_unit(a) == c for a in unit_aliases(rule_unit))


def sub_code_from_rule(r) -> Optional[int]:                          # xid.go:3117-3125
    for k in ("IntrinfoPatternV2", "IntrinfoPatternV1"):
        if r[k] != "":
            v = sample_from_pattern(r[k])
            if v is not None:
                return (v >> 20) & 0x3F
    return None


def _build_nvlink_maps():                                            # xid.go:2997-3090
    result: Dict[int, Dict[int, Detail]] = {}
    by_status: Dict[int, Dict[int, Dict[int, Detail]]] = {}
    for r in NVLINK_RULES:
        if r["Xid"] < 144 or r["Xid"] > 150:
            continue
        sc = sub_code_from_rule(r)
        if sc is None:
            continue
        result.setdefault(r["Xid"], {})
        by_status.setdefault(r["Xid"], {}).setdefault(sc, {})
        base = get_detail(r["Xid"])
        if base is None:
            continue
        d = base.copy()
        d.sub_code, d.sub_code_description, d.error_status = sc, r["Unit"], r["ErrorStatus"]
        ev = event_type_from_severity(r["Severity"])
        if ev == EV_UNKNOWN:
            ev = event_type_from_immediate_bucket(r["Resolution"])
        if ev != EV_UNKNOWN:
            d.event_type = ev
        acts = suggested_actions_from_bucket(r["Resolution"])
        if acts is not None:
            d.actions = list(acts)
        ex = by_status[r["Xid"]][sc].get(r["ErrorStatus"])
        if ex is not None:
            d.event_type = max_event_type(ex.event_type, d.event_type)
            d.actions = merge_actions(ex.actions, d.actions)
        by_status[r["Xid"]][sc][r["ErrorStatus"]] = d
        agg = result[r["Xid"]].get(sc)
        if agg is None:
            agg = base.copy()
            agg.sub_code, agg.sub_code_description = sc, r["Unit"]
        agg.actions = merge_actions(agg.actions, d.actions)
        result[r["Xid"]][sc] = agg
    # applyOperationalOverrides  (xid.go:3062-3089)
    for sc, sdesc, desc in ((4, "NETIR_LINK_EVT/NETIR_LINK_DOWN (cartridge error)",
                             "NVLINK: NETIR Link Event - Possible NVLink cartridge error (contact provider)"),
                            (10, "NETIR_LINK_EVT/NETIR_LINK_DOWN (PHY timeout)",
                             "NVLINK: NETIR Link Event - Physical layer retransmission timeout (contact provider)")):
        if 149 in result and sc in result[149]:
            d = result[149][sc]
            d.event_type, d.sub_code_description, d.description, d.actions = EV_FATAL, sdesc, desc, [ACT_HW_INSPECTION]
            if sc in by_status.get(149, {}):
                for st in list(by_status[149][sc]):
                    by_status[149][sc][st] = d.copy()
    return result, by_status


DETAILS_WITH_SUBCODES, DETAILS_BY_STATUS = _build_nvlink_maps()


def get_detail_with_sub_code(xid: int, sc: int) -> Optional[Detail]:           # xid.go:79-93
    sm = DETAILS_WITH_SUBCODES.get(xid)
    if sm is not None:
        if sc in sm:
            return sm[sc].copy()
        if 0 in sm:
            return sm[0].copy()
    return get_detail(xid)


def get_detail_with_sub_code_and_status(xid: int, sc: int, st: int) -> Optional[Detail]:   # xid.go:97-107
    d = DETAILS_BY_STATUS.get(xid, {}).get(sc, {}).get(st)
    if d is not None:
        return d.copy()
    return get_detail_with_sub_code(xid, sc)


@dataclass
class ExtractedInfo:                                                  # xid/kmsg.go:84-98
    device: str
    xid: int
    pid: str
    process_name: str
    unit: str
    severity: str
    xc: str
    injected: str
    link: int
    intrinfo: int
    error_status: int
    extra: List[int]
    sub_code: int


def lookup_nvlink_rule(info: ExtractedInfo):                         # xid.go:3099-3114
    for idx, r in enumerate(NVLINK_RULES):
        if r["Xid"] != info.xid:
            continue
        if not unit_matches(r["Unit"], info.unit):
            continue
        if r["ErrorStatus"] != info.error_status:
            continue
        if pattern_matches(r["IntrinfoPatternV2"], info.intrinfo) or pattern_matches(r["IntrinfoPatternV1"], info.intrinfo):
            return idx, r
    return -1, None


def detail_from_nvlink_info(info: ExtractedInfo) -> Optional[Detail]:           # xid.go:2954-2995
    base = get_detail(info.xid)
    if base is None:
        return None
    d = get_detail_with_sub_code_and_status(info.xid, info.sub_code, info.error_status) or base.copy()
    _, rule = lookup_nvlink_rule(info)
    if rule is not None:
        ev = event_type_from_severity(rule["Severity"])
        if ev == EV_UNKNOWN:
            ev = event_type_from_immediate_bucket(rule["Resolution"])
        if ev != EV_UNKNOWN:
            d.event_type = ev
        acts = suggested_actions_from_bucket(rule["Resolution"])
        if acts is not None:
            d.actions = list(acts)
        d.error_status = rule["ErrorStatus"]
        if rule["Investigatory"] not in ("", "IGNORE", "CONTACT_SUPPORT"):
            d.investigatory_hint = rule["Investigatory"]
    d.sub_code = info.sub_code
    d.sub_code_description = info.unit
    d.error_status = info.error_status
    d.event_type = max_event_type(d.event_type, event_type_from_log_severity(info.severity))
    if d.actions is None:
        d.actions = None if base.actions is None else list(base.actions)
    return d


# --------------------------------------------------------------------------------------------
# xid.Match / sxid.Match     (xid/kmsg.go:73-80,116-183,202-268 ; sxid/kmsg.go:28-73)
# --------------------------------------------------------------------------------------------
def extract_nvrm_xid_info(line: bytes) -> Tuple[int, str]:            # kmsg.go:73-80
    m = R1.search(line)
    if m:
        v = go_atoi(m.group(2))
        if v is not None:
            return v, m.group(1).decode("latin-1")
    return 0, ""


def extract_nvrm_xid_info_extended(line: bytes) -> Optional[ExtractedInfo]:     # kmsg.go:116-183
    m = R2.search(line)
    if not m:
        return None
    code = go_atoi(m.group(2))
    if code is None:
        return None
    intr = go_parse_uint32_base0(m.group(10))
    if intr is None:
        return None
    es = go_parse_uint32_base0(m.group(11))
    if es is None:
        return None
    link = go_atoi(m.group(9))
    if link is None:
        return None
    extra = []
    for i in range(12, 16):
        g = m.group(i)
        if not g:
            continue
        v = go_parse_uint32_base0(g)
        if v is not None:
            extra.append(v)
    s = lambda i: (m.group(i) or b"").decode("latin-1")
    return ExtractedInfo(s(1), code, s(3), s(4), s(5), s(6), s(7), s(8), link, intr, es, extra, (intr >> 20) & 0x3F)


def normalize_pci_bdf(s: str) -> str:                                 # kmsg.go:259-268
    if s.startswith("PCI:"):
        s = s[4:]
    s = s.strip()
    if s.count(":") == 1:
        s = "0000:" + s
    if s == "":
        return ""
    return "PCI:" + s


def extract_fallen_off_bus(line: bytes) -> Tuple[int, str]:           # kmsg.go:247-257
    m = R4.search(line)
    if m:
        return 79, normalize_pci_bdf(m.group(1).decode("latin-1"))
    m = R3.search(line)
    if m:
        return 79, normalize_pci_bdf(m.group(1).decode("latin-1"))
    return 0, ""


@dataclass
class XidError:                                                       # kmsg.go:194-198
    xid: int
    device: str
    detail: Detail
    info: Optional[ExtractedInfo] = None


def xid_match(line: bytes) -> Optional[XidError]:                     # kmsg.go:202-245
    info = extract_nvrm_xid_info_extended(line)
    if info is not None:
        d = detail_from_nvlink_info(info)
        if d is not None:
            dev = info.device
            if dev != "" and not dev.startswith("PCI:"):
                dev = "PCI:" + dev
            return XidError(info.xid, dev, d, info)
    code, dev = extract_nvrm_xid_info(line)
    if code != 0:
        d = get_detail(code)
        if d is None:
            return None
        return XidError(code, dev, d.copy())
    code, dev = extract_fallen_off_bus(line)
    if code != 0:
        d = get_detail(code)
        if d is None:
            return None
        return XidError(code, dev, d.copy())
    return None


def extract_sxid(line: bytes) -> int:                                 # sxid/kmsg.go:31-38
    m = R5.search(line)
    if m:
        v = go_atoi(m.group(1))
        if v is not None:
            return v
    return 0


def extract_sxid_device(line: bytes) -> str:                          # sxid/kmsg.go:42-47
    m = R6.search(line)
    return m.group(1).decode("latin-1") if m else ""


def sxid_match(line: bytes):                                          # sxid/kmsg.go:58-73
    code = extract_sxid(line)
    if code == 0:
        return None
    d = SXID_DETAILS.get(code)
    if d is None:
        return None
    return {"sxid": code, "device": extract_sxid_device(line), "detail": d}


def ext_match(line: bytes):
    """kinds of the extra line patterns that fire on this line, ascending (FindStringSubmatch != nil, e.g.
    nccl/kmsg_matcher.go:20-25, disk/kmsg_matcher.go:70-125)."""
    return [k for k, *_ in EXT_PATTERNS if EXT_RE[k].search(line)]


def ext_capture(kind: int, line: bytes) -> bytes:
    """the text the component appends to its message: cpu process info (cpu/kmsg_matcher.go:38-52), the first PCI BDF of an
    ACCESS_REG line (infiniband/kmsg_matcher.go:136-142), else empty"""
    g = EXT_BY_KIND[kind][3]
    if g is not None:
        return EXT_RE[kind].search(line).group(g)
    if kind in PRIM_GROUPS:
        return prim_spans(kind, line)[0]
    if kind == 7:
        m = R_PCI_DEVICE.search(line)
        return m.group(0) if m else b""
    return b""


def ext_message(kind: int, line: bytes) -> str:
    """the message string `Match` returns for a line on which pattern `kind` fires"""
    msg = EXT_BY_KIND[kind][2]
    cap = ext_capture(kind, line).decode("latin-1")
    if kind in (8, 9):
        return msg + " (" + cap + ")"
    if kind == 7 and cap:
        return msg + " (PCI device " + cap + ")"
    return msg


def component_match(component: str, line: bytes):
    """(eventName, message) of the first STATELESS pattern of `component` that fires, in the component's own order
    (e.g. disk/kmsg_matcher.go:127-134, 143-154); ("", "") if none"""
    for k, c, e, _m, _rx, _g in EXT_PATTERNS:
        if k < N_STATELESS_KINDS and c == component and EXT_RE[k].search(line):
            return e, ext_message(k, line)
    return "", ""


def prim_spans(kind: int, line: bytes):
    """the capture spans a primitive hit reports, as bytes per span slot (b"" = slot unused)"""
    m = EXT_RE[kind].search(line)
    return [m.group(g) if g is not None else b"" for g in PRIM_GROUPS.get(kind, (None,) * 5)]


def go_path_join_root(x: str) -> str:
    """path.Join("/", x) (memory/kmsg_matcher.go:165-166): Clean("/" + x) - collapse slashes, drop ".", resolve ".." at the root"""
    out = []
    for part in x.split("/"):
        if part in ("", "."):
            continue
        if part == "..":
            if out:
                out.pop()
            continue
        out.append(part)
    return "/" + "/".join(out)


def stateful_events(lines):
    """(line index, component, eventName, message) of the two stateful matchers run line by line over `lines`, as the
    os and memory components' Match would return them"""
    pm, om, out = KernelPanicMatcher(), OOMMatcher(), []
    for i, l in enumerate(lines):
        ev = pm.feed(l)
        if ev[0]:
            out.append((i, "os") + ev)
        ev = om.feed(l)
        if ev[0]:
            out.append((i, "memory") + ev)
    return out


class KernelPanicMatcher:
    """createKernelPanicMatchFunc (os/kmsg_matcher.go:60-125): one call per line, returns (eventName, message)"""
    MAX_LINES = 10

    def __init__(self):
        self.reading, self.lines = False, 0

    def feed(self, line: bytes):
        if EXT_RE[19].search(line):                                   # checkIfStartOfPanicMessages (:127-134)
            ev = ("kernel_panic", "Kernel panic detected (no CPU/PID info found)") if self.reading else ("", "")
            self.reading, self.lines = True, 0
            return ev
        if not self.reading:
            return "", ""
        self.lines += 1
        m = EXT_RE[20].search(line)                                   # extractCPUandPID (:136-157)
        if m:
            cpu, pid = go_atoi(m.group(1)), go_atoi(m.group(2))
            if cpu is not None and pid is not None and pid >= 0:
                self.reading, self.lines = False, 0
                return "kernel_panic", "Kernel panic detected - CPU: %d, PID: %d, Process: %s" % (cpu, pid, m.group(3).decode("latin-1"))
        if self.lines >= self.MAX_LINES:
            self.reading, self.lines = False, 0
            return "kernel_panic", "Kernel panic detected (no CPU/PID info found)"
        return "", ""


class OOMMatcher:
    """createMatchFunc (memory/kmsg_matcher.go:29-109): one call per line, returns (eventName, message)"""

    def __init__(self):
        self.cur = None

    @staticmethod
    def summary(o) -> str:                                            # OOMInstance.Summary (:124-137)
        msg = "System OOM encountered" if o["victim"] == "/" else "OOM encountered"
        if o["process"] != "" and o["pid"] != 0:
            msg = "%s, victim process: %s, pid: %d" % (msg, o["process"], o["pid"])
        return msg

    def feed(self, line: bytes):
        if EXT_RE[21].search(line):
            self.cur = {"pid": 0, "process": "", "container": "/", "victim": "/", "constraint": ""}
            return "", ""
        if self.cur is None:
            return "", ""
        o = self.cur
        found = False
        m = EXT_RE[22].search(line)                                   # getContainerName (:169-189)
        if m is None:
            lm = EXT_RE[23].search(line)                              # getLegacyContainerName (:159-167)
            if lm:
                o["container"] = go_path_join_root(lm.group(1).decode("latin-1"))
                o["victim"] = go_path_join_root(lm.group(2).decode("latin-1"))
        else:
            o["container"], o["victim"], o["constraint"] = m.group(6).decode("latin-1"), m.group(5).decode("latin-1"), m.group(1).decode("latin-1")
            pid = go_atoi(m.group(8))
            if pid is None:
                self.cur = None
                return "", ""
            o["pid"], o["process"] = pid, m.group(7).decode("latin-1")
            found = True
        if found and o["pid"] != 0:
            self.cur = None
            return "OOM", self.summary(o)
        if not found:
            km = EXT_RE[24].search(line)                              # getProcessNamePid (:191-208)
            if km:
                pid = go_atoi(km.group(1))
                if pid is None:
                    self.cur = None
                    return "", ""
                o["pid"], o["process"] = pid, km.group(2).decode("latin-1")
                self.cur = None
                return "OOM", self.summary(o)
        return "", ""


def scan_lines(buf: bytes, ext: bool = False):
    """The reference's buffer-scan form: split on '\\n', Match each line (xid/kmsg_test.go:252-267).
    Returns hit dicts in (line, kind) order; kind 1 = xid, 2 = sxid."""
    hits = []
    off = 0
    for ln, line in enumerate(buf.split(b"\n")):
        x = xid_match(line)
        if x is not None:
            hits.append({"line": ln, "offset": off, "kind": 1, "code": x.xid, "device": x.device,
                         "event_type": x.detail.event_type, "actions": x.detail.actions or [],
                         "extended": x.info is not None,
                         "sub_code": x.detail.sub_code, "unit": x.detail.sub_code_description,
                         "error_status": x.detail.error_status,
                         "intrinfo": x.info.intrinfo if x.info else 0, "link": x.info.link if x.info else 0,
                         "hint": x.detail.investigatory_hint, "description": x.detail.description})
        s = sxid_match(line)
        if s is not None:
            hits.append({"line": ln, "offset": off, "kind": 2, "code": s["sxid"], "device": s["device"],
                         "event_type": s["detail"]["event_type"], "actions": s["detail"]["actions"],
                         "extended": False, "sub_code": 0, "unit": "", "error_status": 0, "intrinfo": 0, "link": 0,
                         "hint": "", "description": ""})
        if ext:
            for kind in ext_match(line):
                hits.append({"line": ln, "offset": off, "kind": kind, "code": 0, "device": ext_capture(kind, line).decode("latin-1")[:39],
                             "capture": ext_capture(kind, line), "message": ext_message(kind, line), "event_type": EV_WARNING, "actions": [],
                             "spans": prim_spans(kind, line) if kind in PRIM_GROUPS else None,
                             "extended": False, "sub_code": 0, "unit": "", "error_status": 0, "intrinfo": 0, "link": 0, "hint": "", "description": ""})
        off += len(line) + 1
    return hits


# --------------------------------------------------------------------------------------------
# /dev/kmsg record parsing + dedup      (pkg/kmsg/watcher.go:292-332 ; pkg/kmsg/deduper.go:63-125)
# --------------------------------------------------------------------------------------------
def parse_kmsg_line(boot_unix_us: int, line: str):
    """Returns (priority, seq, ts_unix_us, message) or raises ValueError, like parseLine."""
    parts = line.split(";", 1)                                        # watcher.go:294 SplitN(line, ";", 2)
    if len(parts) < 2:
        raise ValueError("invalid kmsg; must contain a ';'")
    meta = parts[0].split(",")
    if len(meta) < 3:
        raise ValueError("invalid kmsg: must contain at least 3 ',' separated pieces at the start")
    def atoi(s):
        if not re.fullmatch(r"[+-]?\d+", s):
            raise ValueError("could not parse %r" % s)
        v = int(s)
        if not (-(1 << 63) <= v < (1 << 63)):
            raise ValueError("range")
        return v
    prio, seq, usec = atoi(meta[0]), atoi(meta[1]), atoi(meta[2])
    return prio, seq, boot_unix_us + usec, parts[1]


def dedup_key(ts_unix_s: int, message: str) -> str:                   # deduper.go:63-74
    return "%d-%s" % (ts_unix_s - ts_unix_s % 60, message)


def infiniband_dedup_window(name: str, message: str):
    """(*component).kmsgEventDedupWindow (infiniband/component.go:166-179) -> (window seconds, ok)"""
    if name != "access_reg_failed":
        return 0, False
    if "(PCI device " not in message:                     # pciDeviceMessagePrefix (kmsg_matcher.go:63)
        return 5 * 60, True                               # defaultKmsgEventDedupWindow (component.go:38)
    return 24 * 3600, True                                # defaultAccessRegEventDedupWindow (component.go:43)


class KmsgSyncerModel:
    """pkg/kmsg Syncer.sync loop body (syncer.go:84-140) + newSyncer's option handling (:30-59) + dedupParams (:145-155) +
    deduper.addCacheWithWindow (deduper.go:111-125, go-cache: live while now <= expiration) over an in-memory bucket whose Find
    is findEvent (eventstore/database.go:277-324) for events without ExtraInfo."""

    def __init__(self, truncate_seconds: int = 60, disable_dedup: bool = False, window_func=None):
        self.window_func = window_func
        self.has_deduper = (not disable_dedup) or window_func is not None
        self.truncate = 60 if disable_dedup else (truncate_seconds if truncate_seconds > 0 else 60)
        self.cache: Dict[str, Tuple[int, int]] = {}
        self.rows: List[Tuple[int, str, str, str]] = []

    def dedup_params(self, name: str, message: str):
        if self.window_func is not None:
            w, ok = self.window_func(name, message)
            if ok and w > 0:
                return w, w
        return self.truncate, 15 * 60

    def offer(self, t: int, name: str, message: str, now: int) -> bool:
        if not name:
            return False
        if self.has_deduper:
            trunc, ttl = self.dedup_params(name, message)
            key = "%d-%s" % (t - t % trunc, name + "_" + message)
            cnt, exp = self.cache.get(key, (0, -1))
            freq = cnt + 1 if (cnt and exp >= now) else 1
            self.cache[key] = (freq, now + ttl)
            if freq > 1:
                return False
        for (rt, rn, ry, rm) in self.rows:                # Find: same (timestamp, name, type) and, for a non-empty message, same message
            if rt == t and rn == name and ry == "Warning" and (message == "" or rm == message):
                return False
        self.rows.append((t, name, "Warning", message))
        return True


# --------------------------------------------------------------------------------------------
# health evolution     (xid/health_state.go:57-128 ; xid/component.go:614-642)
# events: list of dicts newest-first: {"name": "error_xid"|"reboot"|"SetHealthy", "type": "Fatal"..,
#         "xid": int, "actions": [ids] or None}
# --------------------------------------------------------------------------------------------
def trim_events_after_set_healthy(events):                            # component.go:630-642
    for i, e in enumerate(events):
        if e["name"] == "SetHealthy":
            return events[:i] if i else []
    return events


def sxid_reason(sxid, device: str, name: str = "") -> str:
    """the Reason string of sxid's evolveHealthyState (sxid/health_state.go:93-106); name = GetDetail(sxid).Name or "" """
    if sxid is None:
        return "SXIDComponent is healthy"
    return ("SXID %d(%s) detected on %s" % (sxid, name, device)) if name else ("SXID %d detected on %s" % (sxid, device))


def evolve_healthy_state(events, reboot_threshold: int = 2, event_name: str = "error_xid"):
    """xid/health_state.go:57-128 ; the sxid twin (sxid/health_state.go:38-111) differs in the event name and the fixed threshold 2.
    "last_index" = index into `events` of the event that ends up as lastXidErr (None: healthy reason)."""
    last_action = None
    last_xid = None
    last_index = None
    last_health = 0
    reboot_map: Dict[int, int] = {}
    for i in range(len(events) - 1, -1, -1):
        e = events[i]
        if e["name"] == event_name:
            cur = {"Critical": 1, "Fatal": 2}.get(e.get("type", ""), 0)
            if cur < last_health:
                continue
            last_health = cur
            last_xid = e["xid"]
            last_index = i
            acts = e.get("actions")
            if acts:
                acts = list(acts)
                if acts[0] == ACT_REBOOT:
                    if e["xid"] not in reboot_map:
                        reboot_map[e["xid"]] = 0
                    elif reboot_map[e["xid"]] >= reboot_threshold:
                        acts[0] = ACT_HW_INSPECTION
                last_action = acts[:1]
        elif e["name"] == "reboot":
            if last_action and last_action[0] in (ACT_REBOOT, ACT_CHECK_APP):
                last_health, last_action, last_xid, last_index = 0, None, None, None
            for k in reboot_map:
                reboot_map[k] += 1
    return {"health": ["Healthy", "Degraded", "Unhealthy"][last_health], "actions": last_action, "xid": last_xid, "last_index": last_index}


def xid_build_message(xid: int, sub_code: int = 0, error_status: int = 0, description: str = "", device_uuid: str = "", gpu_uuid: str = "") -> str:
    """(*xidErrorEventDetail).buildMessage (xid/health_state.go:130-169); gpu_uuid = the result of convertBusIDToUUID ("" none)"""
    header = "XID %d" % xid
    if 144 <= xid <= 150:
        header = "XID %d.%d (err status 0x%08x)" % (xid, sub_code, error_status)
    if xid > (1 << 63) - 1:                               # intFromUint64 fails
        return "%s detected on GPU %s" % (header, device_uuid)
    desc = MNEMONIC.get(xid, "")
    if desc == "":
        desc = description
    elif description not in ("", "Unused") and desc != description:
        desc += " " + description
    gpu = "GPU %s" % device_uuid
    if gpu_uuid:
        gpu = "GPU %s UUID:%s" % (device_uuid, gpu_uuid)
    return "%s %s detected on %s" % (header, desc, gpu)


def convert_bus_id_to_uuid(bus_id: str, devices: Dict[str, str]) -> str:
    """convertBusIDToUUID (xid/health_state.go:171-182); devices: NVML uuid -> PCIBusID()"""
    want = (bus_id[4:] if bus_id.startswith("PCI:") else bus_id) + "."
    for uuid, pci in devices.items():
        if pci.startswith(want):
            return uuid
    return ""


def resolve_xid_event(event_type: str, raw_data: str, device_uuid: str = "", devices: Optional[Dict[str, str]] = None):
    """resolveXIDEvent + addEventDetails (xid/health_state.go:184-281) for the "data" payload of a stored error_xid event:
    -> (type, message, payload dict) or None where the reference leaves the event unresolved.  The payload dict uses the JSON
    keys of xidErrorEventDetail; "actions" is a list of ids or None."""
    devices = devices or {}
    p = None
    try:
        j = json.loads(raw_data)
        if isinstance(j, dict) and int(j.get("xid", 0)) != 0:
            acts = j.get("suggested_actions_by_gpud")
            p = {"xid": int(j["xid"]), "device_uuid": j.get("device_uuid", ""), "sub_code": int(j.get("sub_code", 0)),
                 "sub_code_description": j.get("sub_code_description", ""), "error_status": int(j.get("error_status", 0)),
                 "description": j.get("description", ""),
                 "actions": None if acts is None else [{v: k for k, v in ACTION_WIRE.items()}[a] for a in (acts.get("repair_actions") or [])]}
    except (ValueError, TypeError):
        p = None
    if p is None:                                          # legacy rows keep only the decimal code
        try:
            code = go_atoi(raw_data.encode("utf-8"))
        except ValueError:
            return None
        d = get_detail(code)
        if d is None or code < 0:
            return None
        p = {"xid": code, "device_uuid": device_uuid, "sub_code": 0, "sub_code_description": "", "error_status": 0, "description": "",
             "actions": None if d.actions is None else list(d.actions)}
    typ = event_type
    d = get_detail_with_sub_code_and_status(p["xid"], p["sub_code"], p["error_status"]) if p["xid"] <= (1 << 63) - 1 else None
    if d is not None:
        if typ == "" and d.event_type != EV_UNKNOWN:
            typ = EVENT_NAMES[d.event_type]
        if p["description"] == "":
            p["description"] = d.description
        if p["sub_code"] == 0:
            p["sub_code"] = d.sub_code
        if p["sub_code_description"] == "":
            p["sub_code_description"] = d.sub_code_description
        if p["actions"] is None and d.actions is not None:
            p["actions"] = list(d.actions)
    elif typ == "":
        typ = "Unknown"
    msg = xid_build_message(p["xid"], p["sub_code"], p["error_status"], p["description"], p["device_uuid"], convert_bus_id_to_uuid(p["device_uuid"], devices))
    return typ, msg, p


def evolve_healthy_state_stored(events, devices: Optional[Dict[str, str]] = None, reboot_threshold: int = 2):
    """evolveHealthyState over STORED events (xid/health_state.go:57-128): events newest first, each
    {"name", "type", "data": payload string, "device_uuid"}; resolves every error_xid event like the reference and returns
    {"health", "actions", "reason"}."""
    views, payloads = [], {}
    for i, e in enumerate(events):
        if e["name"] != "error_xid":
            views.append({"name": e["name"]})
            continue
        r = resolve_xid_event(e.get("type", ""), e.get("data", ""), e.get("device_uuid", ""), devices)
        if r is None:
            continue                                       # json.Unmarshal of the unresolved payload fails -> the event is skipped (:71-74)
        typ, _msg, p = r
        payloads[i] = p
        views.append({"name": "error_xid", "type": typ, "xid": p["xid"], "actions": p["actions"], "_i": i})
    st = evolve_healthy_state(views, reboot_threshold)
    reason = "XIDComponent is healthy"
    if st["last_index"] is not None:
        p = payloads[views[st["last_index"]]["_i"]]
        reason = xid_build_message(p["xid"], p["sub_code"], p["error_status"], p["description"], p["device_uuid"],
                                   convert_bus_id_to_uuid(p["device_uuid"], devices or {}))
    return {"health": st["health"], "actions": st["actions"], "reason": reason}


def resolve_sxid_event(event_type: str, raw_data: str, device_uuid: str = ""):
    """resolveSXIDEvent (sxid/health_state.go:113-142) + the Unmarshal evolveHealthyState does next (:50-54):
    -> (type, message or None, payload dict) or None when the event is skipped"""
    try:
        code = go_atoi(raw_data.encode("utf-8"))
    except ValueError:
        code = None
    if code is not None:
        d = SXID_DETAILS.get(code)
        if d is None or code < 0:
            return None                                    # payload stays the decimal string, which does not unmarshal into the struct
        name = d["name"]
        return (EVENT_NAMES[d["event_type"]], sxid_reason(code, device_uuid, name),
                {"sxid": code, "device_uuid": device_uuid, "actions": list(d["actions"]) if d["actions"] else None})
    try:
        j = json.loads(raw_data)
        if not isinstance(j, dict):
            return None
        acts = j.get("suggested_actions_by_gpud")
        return (event_type, None, {"sxid": int(j.get("sxid", 0)), "device_uuid": j.get("device_uuid", "") or "",
                                   "actions": None if acts is None else [{v: k for k, v in ACTION_WIRE.items()}[a] for a in (acts.get("repair_actions") or [])]})
    except (ValueError, TypeError, KeyError):
        return None


def evolve_sxid_stored(events):
    """sxid evolveHealthyState over stored events, newest first: {"name", "type", "data", "device_uuid"} -> health / actions / reason"""
    views, payloads = [], {}
    for i, e in enumerate(events):
        if e["name"] != "error_sxid":
            views.append({"name": e["name"]})
            continue
        r = resolve_sxid_event(e.get("type", ""), e.get("data", ""), e.get("device_uuid", ""))
        if r is None:
            continue
        payloads[i] = r[2]
        views.append({"name": "error_sxid", "type": r[0], "xid": r[2]["sxid"], "actions": r[2]["actions"], "_i": i})
    st = evolve_healthy_state(views, 2, "error_sxid")
    reason = "SXIDComponent is healthy"
    if st["last_index"] is not None:
        p = payloads[views[st["last_index"]]["_i"]]
        d = SXID_DETAILS.get(p["sxid"])
        reason = sxid_reason(p["sxid"], p["device_uuid"], d["name"] if d else "")
    return {"health": st["health"], "actions": st["actions"], "reason": reason}


# GPU product capabilities (pkg/nvidia/product/capabilities.go:6-137)
PRODUCT_MEM_CAPS = {"a100": 7, "b100": 7, "b200": 7, "gb200": 7, "h100": 7, "h200": 7, "a10": 4}      # :15-23; 1 containment | 2 offlining | 4 row remapping
PRODUCT_FM = {"a100": True, "b100": True, "b200": True, "gb200": False, "gh200": False, "h100": True, "h200": True, "a10": False}   # :25-50


def _longest_key(p: str, table: dict):
    best = ""
    for k in table:
        if k in p and len(best) < len(k):
            best = k
    return best


def product_mem_caps(name: str) -> int:                               # SupportedMemoryMgmtCapsByGPUProduct :119-137
    k = _longest_key(name.lower(), PRODUCT_MEM_CAPS)
    return PRODUCT_MEM_CAPS[k] if k else 0


def product_fm_supported(name: str) -> bool:                          # SupportedFMByGPUProduct :56-76
    p = name.lower()
    if "pcie" in p:
        return False
    k = _longest_key(p, PRODUCT_FM)
    return PRODUCT_FM[k] if k else False


def product_fabric_state_supported(name: str) -> bool:                # SupportFabricStateByGPUProduct :93-116
    p = name.lower()
    if "pcie" in p or "gh200" in p:
        return False
    return "gb200" in p or "h100" in p or "h200" in p


# --------------------------------------------------------------------------------------------
# threshold rules
# --------------------------------------------------------------------------------------------
def temperature_check(t: dict, margin_threshold: int = 0):
    """the per-GPU rules of the temperature component's Check (temperature/component.go:206-248) and the priority of its reasons
    (:273-287): returns (health, reason class) with class in {"margin", "gpu", "hbm", ""}; default margin threshold 0 = disabled
    (temperature/threshold.go:13)."""
    margin = (t.get("ThresholdCelsiusSlowdown", 0) > 0 and t.get("MarginTemperatureSupported", False) and margin_threshold > 0
              and t.get("ThresholdCelsiusSlowdownMargin", 0) > 0 and t["ThresholdCelsiusSlowdownMargin"] <= margin_threshold)
    gpu = t.get("ThresholdCelsiusGPUMax", 0) > 0 and t.get("CurrentCelsiusGPUCore", 0) > t["ThresholdCelsiusGPUMax"]
    hbm = t.get("ThresholdCelsiusMemMax", 0) > 0 and t.get("HBMTemperatureSupported", False) and t.get("CurrentCelsiusHBM", 0) > t["ThresholdCelsiusMemMax"]
    if margin:
        return "Degraded", "margin"
    if gpu:
        return "Degraded", "gpu"
    if hbm:
        return "Degraded", "hbm"
    return "Healthy", ""


def temperature_reason(temps: List[dict], uuids: List[str], margin_threshold: int = 0):
    """the check result of the temperature component (temperature/component.go:190-287) -> (health, reason); per-GPU findings in the
    order given"""
    margin, gpu, hbm = [], [], []
    for t, u in zip(temps, uuids):
        _h, cls_all = temperature_check(t, margin_threshold), None
        if (t.get("ThresholdCelsiusSlowdown", 0) > 0 and t.get("MarginTemperatureSupported", False) and margin_threshold > 0
                and 0 < t.get("ThresholdCelsiusSlowdownMargin", 0) <= margin_threshold):
            margin.append("%s has only %d \u00b0C margin left to slowdown (threshold %d \u00b0C)" % (u, t["ThresholdCelsiusSlowdownMargin"], margin_threshold))
        if t.get("ThresholdCelsiusGPUMax", 0) > 0 and t.get("CurrentCelsiusGPUCore", 0) > t["ThresholdCelsiusGPUMax"]:
            gpu.append("%s current temperature is %d \u00b0C exceeding the threshold %d \u00b0C" % (u, t["CurrentCelsiusGPUCore"], t["ThresholdCelsiusGPUMax"]))
        if t.get("ThresholdCelsiusMemMax", 0) > 0 and t.get("HBMTemperatureSupported", False) and t.get("CurrentCelsiusHBM", 0) > t["ThresholdCelsiusMemMax"]:
            hbm.append("%s HBM temperature is %d \u00b0C exceeding the threshold %d \u00b0C" % (u, t["CurrentCelsiusHBM"], t["ThresholdCelsiusMemMax"]))
    if margin:
        return "Degraded", "margin threshold exceeded: " + ", ".join(margin)
    if gpu:
        return "Degraded", "GPU temperature anomalies detected: " + ", ".join(gpu)
    if hbm:
        return "Degraded", "HBM temperature anomalies detected: " + ", ".join(hbm)
    return "Healthy", "all %d GPU(s) were checked, no temperature issue found" % len(temps)


# clockEventReasonsToInclude (hw-slowdown/clock_events.go:192-264): (flag, isHWSlowdown, description)
CLOCK_EVENT_REASONS = [
    (0x1, False, 'GPU is idle and clocks are dropping to Idle state'),
    (0x2, False, 'GPU clocks are limited by current setting of applications clocks'),
    (0x4, False, "Clocks have been optimized to not exceed currently set power limits ('SW Power Cap: Active' in nvidia-smi --query)"),
    (0x8, True, "HW Slowdown is engaged due to high temperature, power brake assertion, or high power draw ('HW Slowdown: Active' in nvidia-smi --query)"),
    (0x10, False, 'GPU is part of a Sync boost group to maximize performance per watt'),
    (0x20, False, 'SW Thermal Slowdown is active to keep GPU and memory temperatures within operating limits'),
    (0x40, True, "HW Thermal Slowdown (reducing the core clocks by a factor of 2 or more) is engaged (temperature being too high) ('HW Thermal Slowdown' in nvidia-smi --query)"),
    (0x80, True, "HW Power Brake Slowdown (reducing the core clocks by a factor of 2 or more) is engaged (External Power Brake Assertion being triggered) ('HW Power Brake Slowdown' in nvidia-smi --query)"),
    (0x100, False, 'GPU clocks are limited by current setting of Display clocks'),
]


def clock_event_reasons(bitmask: int):
    """getClockEventReasons (hw-slowdown/clock_events.go:168-190): (sorted HW-slowdown descriptions, sorted other descriptions)"""
    hw = sorted(d for f, is_hw, d in CLOCK_EVENT_REASONS if bitmask & f and is_hw)
    other = sorted(d for f, is_hw, d in CLOCK_EVENT_REASONS if bitmask & f and not is_hw)
    return hw, other


def hw_slowdown_event(bitmask: int, uuid: str, unix_s: int):
    """ClockEvents.HWSlowdownEvent (hw-slowdown/clock_events.go:87-102) for one reading: None or (time, name, type, message, extra_info)"""
    hw, _other = clock_event_reasons(bitmask)
    if not hw:
        return None
    return (unix_s, "hw_slowdown", "Warning", ", ".join("%s: %s" % (uuid, r) for r in hw), {"data_source": "nvml", "gpu_uuid": uuid})


def go_duration_seconds(sec: int) -> str:
    """time.Duration.String() of a whole number of seconds."""
    if sec == 0:
        return "0s"
    u = abs(sec)
    h, m, s_ = u // 3600, (u // 60) % 60, u % 60
    return ("-" if sec < 0 else "") + (f"{h}h" if h else "") + (f"{m}m" if h or m else "") + f"{s_}s"


def hw_slowdown_state(event_unix_s: List[int], now_unix: int, window_seconds: int, threshold_freq_per_min: float):
    """hw-slowdown/component.go:352-407: distinct event-minutes since (now - window) / window minutes >= threshold -> Unhealthy.
    The bucket read is `timestamp > since` (pkg/eventstore/database.go:327-335)."""
    return hw_slowdown_check(event_unix_s, now_unix, window_seconds, threshold_freq_per_min)[:3]


def hw_slowdown_check(event_unix_s: List[int], now_unix: int, window_seconds: int, threshold_freq_per_min: float):
    """-> (health, freq, distinct minutes, reason, hardware_inspection) with the reason strings of component.go:352-401."""
    if window_seconds == 0:
        return "Healthy", 0.0, 0, "no time window to evaluate states", False
    mins = {t // 60 for t in event_unix_s if t > now_unix - window_seconds}
    if not mins:
        return "Healthy", 0.0, 0, "no clock events found", False
    freq = len(mins) / (window_seconds / 60.0)
    head = "hw slowdown events frequency per minute %.2f (total events per minute count %d) " % (freq, len(mins))
    tail = " threshold %.2f for the last %s" % (threshold_freq_per_min, go_duration_seconds(window_seconds))
    if freq < threshold_freq_per_min:
        return "Healthy", freq, len(mins), head + "is less than" + tail, False
    return "Unhealthy", freq, len(mins), head + "exceeded" + tail, True


# --------------------------------------------------------------------------------------------
# windowed aggregates  -- PARITY UNPINNED (no reference implementation), definitions in oracle/SPEC.md
# --------------------------------------------------------------------------------------------
def total_order_key(x: np.ndarray) -> np.ndarray:
    """IEEE-754 totalOrder as an unsigned key: flip all bits of negatives, flip the sign bit of positives."""
    b = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    neg = (b >> np.uint64(63)).astype(bool)
    return np.where(neg, ~b, b | np.uint64(1 << 63))


def key_to_f64(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, dtype=np.uint64)
    pos = (k >> np.uint64(63)).astype(bool)
    return np.where(pos, k & np.uint64((1 << 63) - 1), ~k).view(np.float64)


def quantile_rank(m: int, q_num: int = 99, q_den: int = 100) -> int:
    """1-based nearest rank ceil(m*q_num/q_den), clamped to [1, m]."""
    r = (m * q_num + q_den - 1) // q_den
    return max(1, min(m, r))


def window_aggregates(x: np.ndarray, W: int, thr: float, alpha: float = 0.0, q_num: int = 99, q_den: int = 100):
    """x: [n] f64 chronological samples of one field.  Returns dict of arrays [ceil(n/W)]."""
    n = x.shape[0]
    nw = (n + W - 1) // W
    if alpha <= 0.0:
        alpha = min(2.0 / (W + 1.0), 0.9999)
    out = {k: np.zeros(nw, dtype=np.float64) for k in ("min", "max", "mean", "ema", "p99")}
    out["n_over"] = np.zeros(nw, dtype=np.uint64)
    e = float(x[0]) if n else 0.0
    for w in range(nw):
        seg = x[w * W:min(n, (w + 1) * W)]
        m = seg.shape[0]
        k = np.sort(total_order_key(seg))
        out["min"][w] = key_to_f64(k[:1])[0]
        out["max"][w] = key_to_f64(k[-1:])[0]
        out["p99"][w] = key_to_f64(k[quantile_rank(m, q_num, q_den) - 1:][:1])[0]
        out["mean"][w] = float(np.sum(seg)) / m
        out["n_over"][w] = int(np.count_nonzero(seg > thr))
        for v in seg:                                   # ema_t = a*x_t + (1-a)*ema_{t-1}, ema_{-1} = x_0
            e = alpha * float(v) + (1.0 - alpha) * e
        out["ema"][w] = e
    return out


# --------------------------------------------------------------------------------------------
# whole-box NVLink / fabric verdict  (nvlink/evaluate_threshold.go:77-188 ; device/fabric_state.go:115-177)
# implemented in oracle/fabric.py to keep this file focused on the scan path
# --------------------------------------------------------------------------------------------


def scan_raw_kmsg(buf: bytes, ext: bool = False):
    """Buffer of concatenated /dev/kmsg records (a record continues on lines that start with ' ').  Each record goes
    through parseLine (records that fail to parse are skipped, pkg/kmsg/watcher.go:161-165) and Match runs on the
    message part (xid/component.go:274-299)."""
    hits = []
    off = 0
    recs = re.split(rb"\n(?! )", buf)
    for idx, rec in enumerate(recs):
        try:
            prio, seq, usec, msg = parse_kmsg_line(0, rec.decode("latin-1"))
        except ValueError:
            off += len(rec) + 1
            continue
        m = msg.encode("latin-1")
        x = xid_match(m)
        if x is not None:
            hits.append({"line": idx, "offset": off, "kind": 1, "code": x.xid, "device": x.device,
                         "event_type": x.detail.event_type, "actions": x.detail.actions or [], "kmsg": (prio, seq, usec),
                         "extended": x.info is not None, "sub_code": x.detail.sub_code, "error_status": x.detail.error_status})
        s = sxid_match(m)
        if s is not None:
            hits.append({"line": idx, "offset": off, "kind": 2, "code": s["sxid"], "device": s["device"],
                         "event_type": s["detail"]["event_type"], "actions": s["detail"]["actions"], "kmsg": (prio, seq, usec),
                         "extended": False, "sub_code": 0, "error_status": 0})
        if ext:
            for kind in ext_match(m):
                hits.append({"line": idx, "offset": off, "kind": kind, "code": 0, "device": ext_capture(kind, m).decode("latin-1")[:39],
                             "capture": ext_capture(kind, m), "message": ext_message(kind, m), "event_type": EV_WARNING, "actions": [],
                             "spans": prim_spans(kind, m) if kind in PRIM_GROUPS else None,
                             "kmsg": (prio, seq, usec), "extended": False, "sub_code": 0, "error_status": 0})
        off += len(rec) + 1
    return hits, len(recs)


def xid_event_detail_json(x: "XidError", unix_seconds: int = 0) -> str:
    """json.Marshal(xidErrorEventDetail) as built in xid/component.go:503-521 (struct at health_state.go:284-315)."""
    import datetime
    d = x.detail
    parts = ['"time":' + ("null" if unix_seconds == 0 else json.dumps(
        datetime.datetime.fromtimestamp(unix_seconds, datetime.timezone.utc).strftime("%Y-%m-%dT%H:%M:%SZ"))),
        '"data_source":"kmsg"', '"device_uuid":' + _go_json_str(x.device), '"xid":%d' % x.xid]
    if d.sub_code:
        parts.append('"sub_code":%d' % d.sub_code)
    if d.sub_code_description:
        parts.append('"sub_code_description":' + _go_json_str(d.sub_code_description))
    if d.error_status:
        parts.append('"error_status":%d' % d.error_status)
    if d.investigatory_hint:
        parts.append('"investigatory_hint":' + _go_json_str(d.investigatory_hint))
    if d.description:
        parts.append('"description":' + _go_json_str(d.description))
    if d.actions is not None:
        # apiv1.SuggestedActions{Description, RepairActions}: neither field is omitempty (api/v1/types.go:206-212); the catalog never sets a description
        parts.append('"suggested_actions_by_gpud":{"description":"","repair_actions":[' + ",".join('"%s"' % ACTION_WIRE[a] for a in d.actions) + "]}")
    return "{" + ",".join(parts) + "}"


def _go_json_str(s: str) -> str:
    out = ['"']
    for ch in s:
        o = ord(ch)
        if ch == '"':
            out.append('\\"')
        elif ch == "\\":
            out.append("\\\\")
        elif ch == "\n":
            out.append("\\n")
        elif ch == "\r":
            out.append("\\r")
        elif ch == "\t":
            out.append("\\t")
        elif ch in "<>&" or o < 0x20:
            out.append("\\u%04x" % o)
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)
