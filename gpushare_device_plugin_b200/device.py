"""Thin Python face of the C ABI's device layer (inventory, arena, probe, cycle, health events).

Everything here is a direct call into ``libgpushare_b200.so``; nothing is computed or cached in Python (the
library keeps NVML's (re)start-time inventory snapshot; see include/gpushare_b200.h). Names follow the header.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence

from . import _abi
from ._abi import (CycleResult, DeviceInfo, Event, FaultRecord, FaultReport, GsbError, ProbeCfg, ProbeResult, check, lib)

GiB = 1 << 30
MiB = 1 << 20


def init() -> None:
    """nvml.Init equivalent (gpumanager.go:36). Raises GsbError; never degrades to a CPU path."""
    check(lib.gsb_init(), "gsb_init")


def shutdown() -> None:
    check(lib.gsb_shutdown(), "gsb_shutdown")


def device_count() -> int:
    n = C.c_uint32(0)
    check(lib.gsb_device_count(C.byref(n)), "gsb_device_count")
    return n.value


@dataclass
class Info:
    index: int
    uuid: str
    bus_id: str
    minor: int
    cuda_ordinal: int
    sm_count: int
    cc: tuple
    total_bytes: int
    total_mib: int
    free_bytes: int
    cuda_total_bytes: int

    @staticmethod
    def of(s: DeviceInfo) -> "Info":
        return Info(s.index, s.uuid.decode(), s.bus_id.decode(), s.minor, s.cuda_ordinal, s.sm_count,
                    (s.cc_major, s.cc_minor), s.total_bytes, s.total_mib, s.free_bytes, s.cuda_total_bytes)


def device_info(idx: int) -> Info:
    s = DeviceInfo()
    check(lib.gsb_device_info_get(idx, C.byref(s)), f"gsb_device_info_get({idx})")
    return Info.of(s)


def inventory_refresh(idx: int = _abi.GSB_ALL_DEVICES) -> None:
    """Live NVML query -> snapshot; what NewNvidiaDevicePlugin's getDevices does at every (re)start (server.go:39)."""
    check(lib.gsb_inventory_refresh(idx), f"gsb_inventory_refresh({idx})")


def inventory_snapshot(idx: int):
    """(Info, age_ns): NVML's last answer as the cycle serves it, identity re-validated on the CUDA side."""
    s, age = DeviceInfo(), C.c_uint64(0)
    check(lib.gsb_inventory_snapshot(idx, C.byref(s), C.byref(age)), f"gsb_inventory_snapshot({idx})")
    return Info.of(s), age.value


def set_option(key: int, value: int) -> None:
    check(lib.gsb_set_option(key, value), f"gsb_set_option({key})")


def get_option(key: int) -> int:
    v = C.c_uint64(0)
    check(lib.gsb_get_option(key, C.byref(v)), f"gsb_get_option({key})")
    return v.value


def test_stall(idx: int, ms: int) -> None:
    """Test hook: keep the device's probe stream busy for `ms` ms (a stand-in for a wedged GPU)."""
    check(lib.gsb_test_stall(idx, ms), f"gsb_test_stall({idx})")


test_stall.__test__ = False  # not a pytest case


def slices(total_mib: int, unit_gib: bool = True) -> int:
    return lib.gsb_slices(total_mib, 1 if unit_gib else 0)


def fake_device_id(uuid: str, j: int) -> str:
    buf = C.create_string_buffer(128)
    n = check(lib.gsb_fake_device_id(uuid.encode(), j, buf, len(buf)), "gsb_fake_device_id")
    return buf.raw[:n].decode()


def real_device_id(fake_id: str) -> str:
    buf = C.create_string_buffer(max(128, len(fake_id) + 1))
    n = check(lib.gsb_real_device_id(fake_id.encode(), buf, len(buf)), "gsb_real_device_id")
    return buf.raw[:n].decode()


def encode_list_and_watch(uuids: Sequence[str], n_slices: int, unhealthy_bits: Optional[bytes] = None) -> bytes:
    arr = (C.c_char_p * len(uuids))(*[u.encode() for u in uuids])
    bits = C.cast(C.c_char_p(unhealthy_bits), C.c_void_p) if unhealthy_bits is not None else None
    need = lib.gsb_encode_list_and_watch(arr, len(uuids), n_slices, bits, None, 0)
    check(int(need), "gsb_encode_list_and_watch(size)")
    buf = C.create_string_buffer(int(need) or 1)
    n = lib.gsb_encode_list_and_watch(arr, len(uuids), n_slices, bits, buf, int(need))
    check(int(n), "gsb_encode_list_and_watch")
    return buf.raw[: int(n)]


def encode_register_request(version: str, endpoint: str, resource_name: str) -> bytes:
    buf = C.create_string_buffer(512)
    n = lib.gsb_encode_register_request(version.encode(), endpoint.encode(), resource_name.encode(), buf, len(buf))
    check(int(n), "gsb_encode_register_request")
    return buf.raw[: int(n)]


def arena_create(idx: int, max_bytes: int = 0, keep_free_bytes: int = 0) -> int:
    out = C.c_uint64(0)
    check(lib.gsb_arena_create(idx, max_bytes, keep_free_bytes, C.byref(out)), f"gsb_arena_create({idx})")
    return out.value


def arena_destroy(idx: int) -> None:
    check(lib.gsb_arena_destroy(idx), f"gsb_arena_destroy({idx})")


def arena_bytes(idx: int) -> int:
    out = C.c_uint64(0)
    check(lib.gsb_arena_bytes(idx, C.byref(out)), f"gsb_arena_bytes({idx})")
    return out.value


def probe(idx: int, op: int, *, variant: int = _abi.GSB_VARIANT_AUTO, offset: int = 0, nbytes: int = 0,
          seed_expect: int = 0, seed_write: int = 0, grid: int = 0, flags: int = _abi.GSB_PROBE_TIMED,
          raise_on_error: bool = True) -> ProbeResult:
    cfg = ProbeCfg(op, variant, offset, nbytes, seed_expect, seed_write, grid, flags)
    res = ProbeResult()
    rc = lib.gsb_probe(idx, C.byref(cfg), C.byref(res))
    if raise_on_error:
        check(rc, f"gsb_probe({idx})")
    return res


def probe_all(idxs: Sequence[int], op: int, **kw) -> List[ProbeResult]:
    cfg = ProbeCfg(op, kw.get("variant", 0), kw.get("offset", 0), kw.get("nbytes", 0), kw.get("seed_expect", 0),
                   kw.get("seed_write", 0), kw.get("grid", 0), kw.get("flags", _abi.GSB_PROBE_TIMED))
    arr = (C.c_uint32 * len(idxs))(*idxs)
    res = (ProbeResult * len(idxs))()
    check(lib.gsb_probe_all(len(idxs), arr, C.byref(cfg), res), "gsb_probe_all")
    return list(res)


def arena_read(idx: int, offset: int, nbytes: int) -> bytes:
    buf = C.create_string_buffer(nbytes)
    check(lib.gsb_arena_read(idx, offset, buf, nbytes), "gsb_arena_read")
    return buf.raw


def arena_write(idx: int, offset: int, data: bytes) -> None:
    check(lib.gsb_arena_write(idx, offset, data, len(data)), "gsb_arena_write")


class Cycler:
    """Reusable buffers around gsb_cycle: one inventory + health-probe cycle of one device."""

    def __init__(self, idx: int, window_bytes: int = GiB, unit_gib: bool = True,
                 variant: int = _abi.GSB_VARIANT_AUTO, lw_cap: int = 1 << 16):
        self.idx, self.window_bytes, self.unit_gib, self.variant = idx, window_bytes, unit_gib, variant
        self.buf = C.create_string_buffer(lw_cap)
        self.res = CycleResult()
        self.cycle_no = 0

    def step(self, raise_on_error: bool = True) -> CycleResult:
        rc = lib.gsb_cycle(self.idx, self.cycle_no, self.window_bytes, 1 if self.unit_gib else 0, self.variant,
                           self.buf, len(self.buf), C.byref(self.res))
        self.rc = rc
        if raise_on_error:
            check(rc, f"gsb_cycle({self.idx})")
        self.cycle_no += 1
        return self.res

    def list_and_watch_bytes(self) -> bytes:
        return self.buf.raw[: self.res.lw_len]


class NodeCycler:
    """gsb_cycle_all: every listed device's cycle concurrently (one persistent native thread per device)
    and the concatenated ListAndWatchResponse of the node."""

    def __init__(self, idxs: Sequence[int], window_bytes: int = GiB, unit_gib: bool = True,
                 variant: int = _abi.GSB_VARIANT_AUTO, lw_cap: int = 1 << 20):
        self.idxs = (C.c_uint32 * len(idxs))(*idxs)
        self.n, self.window_bytes, self.unit_gib, self.variant = len(idxs), window_bytes, unit_gib, variant
        self.buf = C.create_string_buffer(lw_cap)
        self.res = (CycleResult * len(idxs))()
        self.cycle_no, self.lw_len = 0, 0

    def step(self):
        n = lib.gsb_cycle_all(self.n, self.idxs, self.cycle_no, self.window_bytes, 1 if self.unit_gib else 0,
                              self.variant, self.buf, len(self.buf), self.res)
        check(int(n), "gsb_cycle_all")
        self.lw_len = int(n)
        self.cycle_no += 1
        return self.res

    def list_and_watch_bytes(self) -> bytes:
        return self.buf.raw[: self.lw_len]


def health_start(probe_period_ms: int = 0, window_bytes: int = GiB) -> None:
    check(lib.gsb_health_start(probe_period_ms, window_bytes), "gsb_health_start")


def health_stop() -> None:
    check(lib.gsb_health_stop(), "gsb_health_stop")


def health_wait(timeout_ms: int) -> Optional[Event]:
    """≙ nvml.WaitForEvent(set, timeout): an Event, or None on timeout."""
    ev = Event()
    rc = lib.gsb_health_wait(timeout_ms, C.byref(ev))
    if rc in (_abi.GSB_ERR_TIMEOUT, _abi.GSB_ERR_STOPPED):
        return None
    check(rc, "gsb_health_wait")
    return ev


def health_stats(idx: int) -> "_abi.HealthStats":
    """What the prober thread of device `idx` has done since health_start: cycles, sweeps, skips, faults, last sizes."""
    st = _abi.HealthStats()
    check(lib.gsb_health_stats_get(idx, C.byref(st)), f"gsb_health_stats_get({idx})")
    return st


def health_inject(uuid: str, etype: int, edata: int) -> None:
    ev = Event(uuid.encode(), etype, edata)
    check(lib.gsb_health_inject(C.byref(ev)), "gsb_health_inject")


def fault_report(idx: int, which: int = _abi.GSB_FAULT_REPORT_LAST) -> FaultReport:
    """The FIRST or LAST HBM fault report of device `idx` (``valid == 0``: none yet)."""
    r = FaultReport()
    check(lib.gsb_fault_report_get(idx, which, C.byref(r)), f"gsb_fault_report_get({idx})")
    return r


def fault_report_text(report: FaultReport, uuid: str) -> str:
    """The one log line both daemons print for a report."""
    need = lib.gsb_fault_report_text(C.byref(report), uuid.encode(), None, 0)
    check(int(need), "gsb_fault_report_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_fault_report_text(C.byref(report), uuid.encode(), buf, int(need))
    check(int(n), "gsb_fault_report_text")
    return buf.raw[: int(n)].decode()


def ecc_status(idx: int) -> "_abi.EccStatus":
    """Live ECC / row-remapper status of device `idx` (fields whose ``valid`` bit is clear are unknown, not zero)."""
    st = _abi.EccStatus()
    check(lib.gsb_ecc_status_get(idx, C.byref(st)), f"gsb_ecc_status_get({idx})")
    return st


def ecc_stats(idx: int) -> "_abi.EccStats":
    """What the prober of device `idx` attributed since health_start with GSB_OPT_ECC_HEALTH = 1."""
    st = _abi.EccStats()
    check(lib.gsb_ecc_stats_get(idx, C.byref(st)), f"gsb_ecc_stats_get({idx})")
    return st


def ecc_conditions(baseline: "_abi.EccStatus", now: "_abi.EccStatus") -> int:
    """GSB_ECC_* bits `now` raises against `baseline`."""
    return lib.gsb_ecc_conditions(C.byref(baseline), C.byref(now))


def ecc_status_text(st: "_abi.EccStatus", uuid: str) -> str:
    """The one log line both daemons print for an ECC status."""
    need = lib.gsb_ecc_status_text(C.byref(st), uuid.encode(), None, 0)
    check(int(need), "gsb_ecc_status_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_ecc_status_text(C.byref(st), uuid.encode(), buf, int(need))
    check(int(n), "gsb_ecc_status_text")
    return buf.raw[: int(n)].decode()


def test_ecc_override(idx: int, st: Optional["_abi.EccStatus"]) -> None:
    """Test hook: device `idx`'s ECC queries answer `st` until called with None."""
    check(lib.gsb_test_ecc_override(idx, C.byref(st) if st is not None else None), f"gsb_test_ecc_override({idx})")


test_ecc_override.__test__ = False  # not a pytest case


def memtest(idx: int, *, offset: int = 0, nbytes: int = 0, first_element: int = 0, n_elements: int = 0,
            raise_on_error: bool = True) -> "_abi.MemtestResult":
    """March C- of device `idx`: elements first_element .. first_element + n_elements - 1 (0 = through element 5) over
    [offset, +nbytes) of the standing arena, or over a transient window of up to nbytes when there is none (0 = all
    allocatable HBM minus the keep-free margin). Mismatches are a result, not an error; with raise_on_error=False a
    failed element is too (``status`` < 0)."""
    cfg = _abi.MemtestCfg(offset, nbytes, first_element, n_elements)
    r = _abi.MemtestResult()
    rc = lib.gsb_memtest(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_memtest({idx})")
    return r


def test_march_probe(idx: int, op: int, *, offset: int = 0, nbytes: int = 0, seed_expect: int = 0,
                     seed_write: int = 0, grid: int = 0) -> ProbeResult:
    """Test hook: one March C- element's kernel (op = GSB_OP_MARCH_*) over [offset, +nbytes) with `grid` CTAs (0 = the
    default), launched as probe() launches a probe op; the seeds are the solid backgrounds' lane values."""
    cfg = ProbeCfg(op, _abi.GSB_VARIANT_AUTO, offset, nbytes, seed_expect, seed_write, grid, _abi.GSB_PROBE_TIMED)
    res = ProbeResult()
    check(lib.gsb_test_march_probe(idx, C.byref(cfg), C.byref(res)), f"gsb_test_march_probe({idx})")
    return res


test_march_probe.__test__ = False  # not a pytest case


def memtest_text(r: "_abi.MemtestResult", uuid: str) -> str:
    """The one log line both daemons print for a memtest result."""
    need = lib.gsb_memtest_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_memtest_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_memtest_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_memtest_text")
    return buf.raw[: int(n)].decode()


def link_probe(idx: int, *, buffer_bytes: int = 0, passes: int = 0, seed_a: int = 0, seed_b: int = 0,
               raise_on_error: bool = True) -> "_abi.LinkResult":
    """PCIe link probe of device `idx`: up A, then down A while up B (`passes` times), then down B, through two pinned
    host buffers of `buffer_bytes` each (0 = 32 MiB), with NVML's link readings at idle and under load. Mismatches are a
    result, not an error; with raise_on_error=False a failed phase is too (``status`` < 0)."""
    cfg = _abi.LinkCfg(buffer_bytes, passes, seed_a, seed_b, 0)
    r = _abi.LinkResult()
    rc = lib.gsb_link_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_link_probe({idx})")
    return r


def link_status(idx: int) -> "_abi.LinkStatus":
    """Live PCIe link status of device `idx` (fields whose ``valid`` bit is clear are unknown, not zero)."""
    st = _abi.LinkStatus()
    check(lib.gsb_link_status_get(idx, C.byref(st)), f"gsb_link_status_get({idx})")
    return st


def link_stats(idx: int) -> "_abi.LinkStats":
    """Link probes of device `idx` since health_start: count, faults, NVML queries, replays, the last result."""
    st = _abi.LinkStats()
    check(lib.gsb_link_stats_get(idx, C.byref(st)), f"gsb_link_stats_get({idx})")
    return st


def link_conditions(r: "_abi.LinkResult") -> int:
    """GSB_LINK_* bits a link probe result raises."""
    return lib.gsb_link_conditions(C.byref(r))


def link_rate_gbps(gen: int, width: int) -> float:
    """Theoretical GB/s per direction of a PCIe link of generation `gen` and `width` lanes."""
    return lib.gsb_link_rate_gbps(gen, width)


def link_text(r: "_abi.LinkResult", uuid: str) -> str:
    """The one log line both daemons print for a link probe result."""
    need = lib.gsb_link_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_link_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_link_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_link_text")
    return buf.raw[: int(n)].decode()


def test_link_override(idx: int, st: Optional["_abi.LinkStatus"]) -> None:
    """Test hook: device `idx`'s link queries answer `st` until called with None."""
    check(lib.gsb_test_link_override(idx, C.byref(st) if st is not None else None), f"gsb_test_link_override({idx})")


def test_link_corrupt(idx: int, phase: int, offset: int, xr) -> None:
    """Test hook: the next link probe of `idx` XORs `xr` (4 lanes) into the word at `offset` of the buffer phase
    `phase` (2 or 3) reads, on the CPU, right before that phase."""
    check(lib.gsb_test_link_corrupt(idx, phase, offset, (C.c_uint32 * 4)(*xr)), f"gsb_test_link_corrupt({idx})")


test_link_override.__test__ = False  # not pytest cases
test_link_corrupt.__test__ = False


def copy_probe(idx: int, *, buffer_bytes: int = 0, src_offset: Optional[int] = None, dst_offset: Optional[int] = None,
               copy_bytes: Optional[int] = None, seed_src: int = 0, seed_host: int = 0, seed_bg: int = 0,
               raise_on_error: bool = True) -> "_abi.CopyResult":
    """Copy-engine probe of device `idx`: H2D, D2H and D2D DMA copies at once between buffers of `buffer_bytes`
    (0 = 32 MiB), then every byte of every destination checked on the GPU. Without offsets and length the copy is
    aligned with a 64-byte guard at each end; with them (all three) any byte geometry that fits. Mismatches are a
    result, not an error; with raise_on_error=False a failed direction is too (``status`` < 0)."""
    given = (src_offset, dst_offset, copy_bytes)
    if any(v is not None for v in given) and not all(v is not None for v in given):
        raise ValueError("give src_offset, dst_offset and copy_bytes together")
    geometry = given[0] is not None
    cfg = _abi.CopyCfg(buffer_bytes, src_offset or 0, dst_offset or 0, copy_bytes or 0, seed_src, seed_host, seed_bg,
                       _abi.GSB_COPY_GEOMETRY if geometry else 0)
    r = _abi.CopyResult()
    rc = lib.gsb_copy_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_copy_probe({idx})")
    return r


def copy_stats(idx: int) -> "_abi.CopyStats":
    """Copy probes of device `idx` since health_start: count, faults, skipped, the last result."""
    st = _abi.CopyStats()
    check(lib.gsb_copy_stats_get(idx, C.byref(st)), f"gsb_copy_stats_get({idx})")
    return st


def copy_conditions(r: "_abi.CopyResult") -> int:
    """GSB_COPY_* bits a copy probe result raises."""
    return lib.gsb_copy_conditions(C.byref(r))


def copy_text(r: "_abi.CopyResult", uuid: str) -> str:
    """The one log line both daemons print for a copy probe result."""
    need = lib.gsb_copy_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_copy_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_copy_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_copy_text")
    return buf.raw[: int(n)].decode()


def test_copy_corrupt(idx: int, op: int, offset: int, xr) -> None:
    """Test hook: the next copy probe of `idx` XORs `xr` (4 lanes) into the word at `offset` of direction `op`'s
    (GSB_OP_COPY_*) destination after its copy and before its verify."""
    check(lib.gsb_test_copy_corrupt(idx, op, offset, (C.c_uint32 * 4)(*xr)), f"gsb_test_copy_corrupt({idx})")


def test_copy_skip(idx: int, op: int) -> None:
    """Test hook: the next copy probe of `idx` does not issue direction `op`'s (GSB_OP_COPY_*) copy."""
    check(lib.gsb_test_copy_skip(idx, op), f"gsb_test_copy_skip({idx})")


test_copy_corrupt.__test__ = False
test_copy_skip.__test__ = False


def sm_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0,
             raise_on_error: bool = True) -> "_abi.SmResult":
    """SM compute probe of device `idx`: known-answer checks of every SM's shared memory, integer, FP32 and FP64 pipes
    and tensor cores (`units`: a mask of 1 << GSB_SM_UNIT_*, 0 = all), compared bit for bit with the answers for
    `seed_expect` (0 = `seed`; `seed` 0 = fresh). Mismatches are a result, not an error; with raise_on_error=False a
    failed launch is too (``status`` < 0)."""
    cfg = _abi.SmCfg(seed, seed_expect, units, 0)
    r = _abi.SmResult()
    rc = lib.gsb_sm_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_sm_probe({idx})")
    return r


def sm_stats(idx: int) -> "_abi.SmStats":
    """SM probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.SmStats()
    check(lib.gsb_sm_stats_get(idx, C.byref(st)), f"gsb_sm_stats_get({idx})")
    return st


def sm_expected(unit: int, seed: int) -> List[int]:
    """The exact answers of SM unit `unit` for `seed`, one per result word of a CTA (none for SMEM)."""
    n = check(int(lib.gsb_sm_expected(unit, seed, None, 0)), "gsb_sm_expected(size)")
    out = (C.c_uint64 * max(n, 1))()
    check(int(lib.gsb_sm_expected(unit, seed, out, n)), "gsb_sm_expected")
    return list(out[:n])


def sm_conditions(r: "_abi.SmResult") -> int:
    """GSB_SM_* bits an SM probe result raises."""
    return lib.gsb_sm_conditions(C.byref(r))


def sm_text(r: "_abi.SmResult", uuid: str) -> str:
    """The one log line both daemons print for an SM probe result."""
    need = lib.gsb_sm_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_sm_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_sm_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_sm_text")
    return buf.raw[: int(n)].decode()


def test_sm_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next SM probe of `idx`, the CTA on SM `smid` XORs `xr` into its result word `index` of `unit`
    just before the compare (SMEM: into that shared-memory word between March elements 1 and 2); once."""
    check(lib.gsb_test_sm_corrupt(idx, smid, unit, index, xr), f"gsb_test_sm_corrupt({idx})")


test_sm_corrupt.__test__ = False


def test_sm_operands(idx: int, unit: int, a=None, b=None, sa=None, sb=None, expected=None) -> None:
    """Test hook: the next SM probe of `idx` that runs tensor unit `unit` runs it on A'[64][K] `a`, B'[K][128] `b` and
    the scales `sa[64]`, `sb[128]` (integer sequences, row-major) and compares D with `expected` (8192 words, row-major:
    FP32 bits, or S32 two's complement); once. `a` None disarms it."""
    if a is None:
        check(lib.gsb_test_sm_operands(idx, unit, None, None, None, None, None), f"gsb_test_sm_operands({idx})")
        return

    def arr(ctype, xs):
        xs = [int(x) for x in (xs.reshape(-1) if hasattr(xs, "reshape") else xs)]
        return (ctype * len(xs))(*xs)
    i32 = C.c_int32
    a_, b_, sa_, sb_ = arr(i32, a), arr(i32, b), arr(i32, sa), arr(i32, sb)
    exp = arr(C.c_uint32, [int(x) & 0xFFFFFFFF for x in expected])
    K = 64 if unit == _abi.GSB_SM_UNIT_E4M3 else 256  # the library reads 64 x K of a and K x 128 of b
    if len(sa_) != 64 or len(sb_) != 128 or len(exp) != 8192 or len(a_) != 64 * K or len(b_) != K * 128:
        raise ValueError("test_sm_operands: a is 64 x K, b is K x 128, sa 64, sb 128, expected 8192 words")
    check(lib.gsb_test_sm_operands(idx, unit, a_, b_, sa_, sb_, exp), f"gsb_test_sm_operands({idx})")


test_sm_operands.__test__ = False


def sm_stress(idx: int, duration_ms: int, *, units: int = 0, slice_ms: int = 0, seed: int = 0, seed_expect: int = 0,
              raise_on_error: bool = True) -> "_abi.StressResult":
    """SM stress of device `idx`: the tensor units (`units`: a mask of 1 << GSB_SM_UNIT_{F16, BF16, E4M3, S8}, 0 = all)
    at full rate on every SM for `duration_ms`, in slices of `slice_ms` (0 = 50, at most 100), every D word compared
    bit for bit with the answers for `seed_expect` (0 = `seed`; `seed` 0 = fresh). Mismatches are a result, not an
    error; with raise_on_error=False a failed slice is too (``status`` < 0)."""
    cfg = _abi.StressCfg(duration_ms, units, slice_ms, seed, seed_expect, 0)
    r = _abi.StressResult()
    rc = lib.gsb_sm_stress(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_sm_stress({idx})")
    return r


def stress_fold(unit: int, seed: int) -> List[int]:
    """The 128 per-thread folds of the D tile gsb_sm_expected(unit, seed) returns (tensor units only)."""
    n = check(int(lib.gsb_stress_fold(unit, seed, None, 0)), "gsb_stress_fold(size)")
    out = (C.c_uint32 * n)()
    check(int(lib.gsb_stress_fold(unit, seed, out, n)), "gsb_stress_fold")
    return list(out)


def stress_conditions(r: "_abi.StressResult") -> int:
    """GSB_STRESS_* bits an SM stress result raises."""
    return lib.gsb_stress_conditions(C.byref(r))


def stress_text(r: "_abi.StressResult", uuid: str) -> str:
    """The one log line both daemons print for an SM stress result."""
    need = lib.gsb_stress_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_stress_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_stress_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_stress_text")
    return buf.raw[: int(n)].decode()


def test_stress_corrupt(idx: int, smid: int, unit: int, index: int, xr: int, slice_: int) -> None:
    """Test hook: in slice `slice_` of the next SM stress of `idx`, if that slice runs `unit`, the CTA on SM `smid`
    XORs `xr` into D word `index` of its first iteration just before the check; once."""
    check(lib.gsb_test_stress_corrupt(idx, smid, unit, index, xr, slice_), f"gsb_test_stress_corrupt({idx})")


test_stress_corrupt.__test__ = False


def cluster_probe(idx: int, *, paths: int = 0, sizes: int = 0, seed: int = 0, seed_expect: int = 0,
                  raise_on_error: bool = True) -> "_abi.ClusterResult":
    """SM-to-SM probe of device `idx`: bit-exact transfers between the CTAs of thread-block clusters over `paths` (a
    mask of 1 << GSB_CLUSTER_PATH_*, 0 = all) at cluster sizes `sizes` (a mask of 1 << k for n = 2 << k; 0 = n = 2 and
    the largest of 16 and 8 that can be scheduled), checked against `seed_expect` (0 = `seed`; `seed` 0 = fresh).
    Mismatches and timeouts are a result, not an error; with raise_on_error=False a failed launch is too."""
    cfg = _abi.ClusterCfg(paths, sizes, seed, seed_expect)
    r = _abi.ClusterResult()
    rc = lib.gsb_cluster_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_cluster_probe({idx})")
    return r


def cluster_stats(idx: int) -> "_abi.ClusterStats":
    """SM-to-SM probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.ClusterStats()
    check(lib.gsb_cluster_stats_get(idx, C.byref(st)), f"gsb_cluster_stats_get({idx})")
    return st


def cluster_conditions(r: "_abi.ClusterResult") -> int:
    """GSB_CLUSTER_* bits an SM-to-SM probe result raises."""
    return lib.gsb_cluster_conditions(C.byref(r))


def cluster_classify(seed: int, smem_bytes: int, rec: "_abi.ClusterRecord") -> "_abi.ClusterClass":
    """What the wrong word of `rec` holds (GSB_CLUSTER_CLASS_*), for a launch that sent under `seed`."""
    out = _abi.ClusterClass()
    check(lib.gsb_cluster_classify(seed, smem_bytes, C.byref(rec), C.byref(out)), "gsb_cluster_classify")
    return out


def cluster_text(r: "_abi.ClusterResult", uuid: str) -> str:
    """The one log line both daemons print for an SM-to-SM probe result."""
    need = lib.gsb_cluster_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_cluster_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_cluster_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_cluster_text")
    return buf.raw[: int(n)].decode()


def test_cluster_corrupt(idx: int, smid: int, path: int, index: int, xr: int) -> None:
    """Test hook: in the first launch of `path` of the next SM-to-SM probe of `idx`, the CTA on SM `smid` XORs `xr`
    into lanes 0-1 of the `index`th word it checks, before the compare; once."""
    check(lib.gsb_test_cluster_corrupt(idx, smid, path, index, xr), f"gsb_test_cluster_corrupt({idx})")


def test_cluster_skip(idx: int, smid: int, path: int) -> None:
    """Test hook: in the first launch of `path` of the next SM-to-SM probe of `idx`, the CTA on SM `smid` sends
    nothing; once."""
    check(lib.gsb_test_cluster_skip(idx, smid, path), f"gsb_test_cluster_skip({idx})")


def test_cluster_script(idx: int, path: int, n: int, region_words: int, route) -> None:
    """Test hook: the first launch of (`path`, clusters of `n`) in the next SM-to-SM probe of `idx` that runs that pair
    is the path's twin on a script: regions of `region_words` words, and the words of rank s for rank d in slot
    route[s][d] of their area (n x n, or n * n flat; GSB_CLUSTER_UNROUTED: nowhere); once. route=None disarms it."""
    import numpy as np
    if route is None:
        check(lib.gsb_test_cluster_script(idx, path, n, region_words, None), f"gsb_test_cluster_script({idx})")
        return
    r = np.ascontiguousarray(route, dtype=np.uint8).reshape(-1)
    if r.size != n * n:
        raise ValueError(f"test_cluster_script: route has {r.size} entries, not {n} x {n}")
    check(lib.gsb_test_cluster_script(idx, path, n, region_words, r.ctypes.data_as(C.POINTER(C.c_uint8))),
          f"gsb_test_cluster_script({idx})")


test_cluster_corrupt.__test__ = False
test_cluster_skip.__test__ = False
test_cluster_script.__test__ = False


def atomic_probe(idx: int, *, ops: int = 0, seed: int = 0, seed_expect: int = 0,
                 raise_on_error: bool = True) -> "_abi.AtomicResult":
    """L2 atomic probe of device `idx`: global-memory atomics of every op in `ops` (a mask of 1 << GSB_ATOMIC_OP_*, 0 =
    all) from one CTA per SM, every word checked against the words gsb_atomic_expected gives for `seed_expect` (0 =
    `seed`; `seed` 0 = fresh). Mismatches, ticket faults and CAS timeouts are a result, not an error; with
    raise_on_error=False a failed launch is too."""
    cfg = _abi.AtomicCfg(ops, seed, seed_expect, 0)
    r = _abi.AtomicResult()
    rc = lib.gsb_atomic_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_atomic_probe({idx})")
    return r


def atomic_stats(idx: int) -> "_abi.AtomicStats":
    """L2 atomic probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.AtomicStats()
    check(lib.gsb_atomic_stats_get(idx, C.byref(st)), f"gsb_atomic_stats_get({idx})")
    return st


def atomic_expected(op: int, seed: int, sm_count: int) -> bytes:
    """The GSB_ATOMIC_BYTES a clean run of `op` under `seed` with `sm_count` CTAs leaves, as the device holds them."""
    buf = C.create_string_buffer(_abi.GSB_ATOMIC_BYTES)
    check(int(lib.gsb_atomic_expected(op, seed, sm_count, buf, len(buf))), "gsb_atomic_expected")
    return buf.raw


def atomic_conditions(r: "_abi.AtomicResult") -> int:
    """GSB_ATOMIC_* bits an L2 atomic probe result raises."""
    return lib.gsb_atomic_conditions(C.byref(r))


def atomic_text(r: "_abi.AtomicResult", uuid: str) -> str:
    """The one log line both daemons print for an L2 atomic probe result."""
    need = lib.gsb_atomic_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_atomic_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_atomic_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_atomic_text")
    return buf.raw[: int(n)].decode()


def test_atomic_corrupt(idx: int, op: int, word: int, xr: int) -> None:
    """Test hook: the first check launch of `op` in the next L2 atomic probe of `idx` XORs `xr` into observed word
    `word` before the compare; once."""
    check(lib.gsb_test_atomic_corrupt(idx, op, word, xr), f"gsb_test_atomic_corrupt({idx})")


def test_atomic_skip(idx: int, smid: int, op: int) -> None:
    """Test hook: in the first run launch of `op` in the next L2 atomic probe of `idx`, the CTA on SM `smid` issues
    none of its atomics; once."""
    check(lib.gsb_test_atomic_skip(idx, smid, op), f"gsb_test_atomic_skip({idx})")


def test_atomic_values(idx: int, op: int, ctas: int, init, values, expected) -> None:
    """Test hook: the next L2 atomic probe of `idx` that runs `op` starts from words `init`, takes every operand's raw
    bits from `values` (gsb_atomic_value_index) and compares with `expected` (one uint64 per word); once. init=None
    disarms it."""
    import numpy as np
    if init is None:
        check(lib.gsb_test_atomic_values(idx, op, ctas, None, None, 0, None), f"gsb_test_atomic_values({idx})")
        return
    i, v, e = (np.ascontiguousarray(x, dtype=np.uint64) for x in (init, values, expected))
    if len(i) != len(e):
        raise ValueError("test_atomic_values: init and expected differ in length")
    check(lib.gsb_test_atomic_values(idx, op, ctas, _u64p(i), _u64p(v), len(v), _u64p(e)),
          f"gsb_test_atomic_values({idx})")


test_atomic_corrupt.__test__ = False
test_atomic_skip.__test__ = False
test_atomic_values.__test__ = False


def tensor_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0,
                 raise_on_error: bool = True) -> "_abi.TensorResult":
    """Tensor-core format probe of device `idx`: one D per unit (`units`: a mask of 1 << GSB_TENSOR_UNIT_*, 0 = all)
    on every SM, compared bit for bit with the answers for `seed_expect` (0 = `seed`; `seed` 0 = fresh). Mismatches
    are a result, not an error; with raise_on_error=False a failed launch is too (``status`` < 0)."""
    cfg = _abi.TensorCfg(seed, seed_expect, units, 0)
    r = _abi.TensorResult()
    rc = lib.gsb_tensor_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_tensor_probe({idx})")
    return r


def tensor_stats(idx: int) -> "_abi.TensorStats":
    """Tensor probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.TensorStats()
    check(lib.gsb_tensor_stats_get(idx, C.byref(st)), f"gsb_tensor_stats_get({idx})")
    return st


def tensor_expected(unit: int, seed: int) -> List[int]:
    """The 8192 D words of tensor unit `unit` for `seed`, row-major (FP64 bits for DMMA, else zero-extended)."""
    n = check(int(lib.gsb_tensor_expected(unit, seed, None, 0)), "gsb_tensor_expected(size)")
    out = (C.c_uint64 * n)()
    check(int(lib.gsb_tensor_expected(unit, seed, out, n)), "gsb_tensor_expected")
    return list(out)


def tensor_conditions(r: "_abi.TensorResult") -> int:
    """GSB_TENSOR_* bits a tensor probe result raises."""
    return lib.gsb_tensor_conditions(C.byref(r))


def tensor_text(r: "_abi.TensorResult", uuid: str) -> str:
    """The one log line both daemons print for a tensor probe result."""
    need = lib.gsb_tensor_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_tensor_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_tensor_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_tensor_text")
    return buf.raw[: int(n)].decode()


def test_tensor_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next tensor probe of `idx`, the CTA on SM `smid` XORs `xr` into its D word `index` of `unit`
    just before the compare; once."""
    check(lib.gsb_test_tensor_corrupt(idx, smid, unit, index, xr), f"gsb_test_tensor_corrupt({idx})")


def test_tensor_operands(idx: int, unit: int, a=None, b=None, sa=None, sb=None, expected=None) -> None:
    """Test hook: the next tensor probe of `idx` that runs `unit` runs it on A'[64][K] `a`, B'[K][128] `b` and the
    scales `sa[64]`, `sb[128]` (integer sequences, row-major) and compares D with `expected` (8192 words, row-major,
    as gsb_tensor_expected gives them); once. `a` None disarms it."""
    if a is None:
        check(lib.gsb_test_tensor_operands(idx, unit, None, None, None, None, None), f"gsb_test_tensor_operands({idx})")
        return

    def arr(ctype, xs):
        xs = [int(x) for x in (xs.reshape(-1) if hasattr(xs, "reshape") else xs)]
        return (ctype * len(xs))(*xs)
    i32 = C.c_int32
    a_, b_, sa_, sb_ = arr(i32, a), arr(i32, b), arr(i32, sa), arr(i32, sb)
    exp = arr(C.c_uint64, expected)
    K = {_abi.GSB_TENSOR_UNIT_DMMA: 64, _abi.GSB_TENSOR_UNIT_TF32: 128, _abi.GSB_TENSOR_UNIT_HMMA: 256,
         _abi.GSB_TENSOR_UNIT_F16_RS: 256}.get(unit, 64)
    if len(sa_) != 64 or len(sb_) != 128 or len(exp) != 8192 or len(a_) != 64 * K or len(b_) != K * 128:
        raise ValueError("test_tensor_operands: a is 64 x K, b is K x 128, sa 64, sb 128, expected 8192 words")
    check(lib.gsb_test_tensor_operands(idx, unit, a_, b_, sa_, sb_, exp), f"gsb_test_tensor_operands({idx})")


test_tensor_corrupt.__test__ = False
test_tensor_operands.__test__ = False


def sparse_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0,
                 raise_on_error: bool = True) -> "_abi.SparseResult":
    """Sparse tensor-core probe of device `idx`: one D per unit (`units`: a mask of 1 << GSB_SPARSE_UNIT_*, 0 = all)
    on every SM, compared bit for bit with the answers for `seed_expect` (0 = `seed`; `seed` 0 = fresh). Mismatches
    are a result, not an error; with raise_on_error=False a failed launch is too (``status`` < 0)."""
    cfg = _abi.SparseCfg(seed, seed_expect, units, 0)
    r = _abi.SparseResult()
    rc = lib.gsb_sparse_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_sparse_probe({idx})")
    return r


def sparse_stats(idx: int) -> "_abi.SparseStats":
    """Sparse probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.SparseStats()
    check(lib.gsb_sparse_stats_get(idx, C.byref(st)), f"gsb_sparse_stats_get({idx})")
    return st


def sparse_expected(unit: int, seed: int) -> List[int]:
    """The 8192 D words of sparse unit `unit` for `seed`, row-major (FP32 bits, S8_SP's S32)."""
    n = check(int(lib.gsb_sparse_expected(unit, seed, None, 0)), "gsb_sparse_expected(size)")
    out = (C.c_uint32 * n)()
    check(int(lib.gsb_sparse_expected(unit, seed, out, n)), "gsb_sparse_expected")
    return list(out)


def sparse_conditions(r: "_abi.SparseResult") -> int:
    """GSB_SPARSE_* bits a sparse probe result raises."""
    return lib.gsb_sparse_conditions(C.byref(r))


def sparse_text(r: "_abi.SparseResult", uuid: str) -> str:
    """The one log line both daemons print for a sparse probe result."""
    need = lib.gsb_sparse_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_sparse_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_sparse_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_sparse_text")
    return buf.raw[: int(n)].decode()


def test_sparse_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next sparse probe of `idx`, the CTA on SM `smid` XORs `xr` into its D word `index` of `unit`
    just before the compare; once."""
    check(lib.gsb_test_sparse_corrupt(idx, smid, unit, index, xr), f"gsb_test_sparse_corrupt({idx})")


def test_sparse_operands(idx: int, unit: int, a=None, pattern=None, b=None, sa=None, sb=None, expected=None) -> None:
    """Test hook: the next sparse probe of `idx` that runs `unit` runs it on the compressed A'[64][K/2] `a`, its
    patterns `pattern[64][groups]`, B'[K][128] `b` and the scales `sa[64]`, `sb[128]` (integer sequences, row-major)
    and compares D with `expected` (8192 words, row-major, as gsb_sparse_expected gives them); once. `a` None disarms
    it."""
    if a is None:
        check(lib.gsb_test_sparse_operands(idx, unit, None, None, None, None, None, None),
              f"gsb_test_sparse_operands({idx})")
        return

    def arr(ctype, xs):
        xs = [int(x) for x in (xs.reshape(-1) if hasattr(xs, "reshape") else xs)]
        return (ctype * len(xs))(*xs)
    i32 = C.c_int32
    K = _abi.SPARSE_UNIT_K[unit]
    groups = K // 2 if unit == _abi.GSB_SPARSE_UNIT_TF32_SP else K // 4
    a_, p_, b_, sa_, sb_ = arr(i32, a), arr(C.c_uint8, pattern), arr(i32, b), arr(i32, sa), arr(i32, sb)
    exp = arr(C.c_uint64, expected)
    if (len(a_) != 64 * K // 2 or len(p_) != 64 * groups or len(b_) != K * 128 or len(sa_) != 64 or len(sb_) != 128
            or len(exp) != 8192):
        raise ValueError("test_sparse_operands: a is 64 x K/2, pattern 64 x groups, b K x 128, sa 64, sb 128, "
                         "expected 8192 words")
    check(lib.gsb_test_sparse_operands(idx, unit, a_, p_, b_, sa_, sb_, exp), f"gsb_test_sparse_operands({idx})")


test_sparse_corrupt.__test__ = False
test_sparse_operands.__test__ = False


def shared_atomic_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0,
                        raise_on_error: bool = True) -> "_abi.SharedAtomicResult":
    """Shared-memory atomic probe of device `idx`: each unit (`units`: a mask of 1 << GSB_SHARED_ATOMIC_UNIT_*, 0 =
    all) on every SM, its area compared bit for bit with the words for `seed_expect` (0 = `seed`; `seed` 0 = fresh).
    Mismatches and slot faults are a result, not an error; with raise_on_error=False a failed launch is too
    (``status`` < 0)."""
    cfg = _abi.SharedAtomicCfg(units, seed, seed_expect, 0)
    r = _abi.SharedAtomicResult()
    rc = lib.gsb_shared_atomic_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_shared_atomic_probe({idx})")
    return r


def shared_atomic_stats(idx: int) -> "_abi.SharedAtomicStats":
    """Shared-memory atomic probes of device `idx` since health_start: count, faults, skipped, incomplete, the last
    result."""
    st = _abi.SharedAtomicStats()
    check(lib.gsb_shared_atomic_stats_get(idx, C.byref(st)), f"gsb_shared_atomic_stats_get({idx})")
    return st


def shared_atomic_expected(unit: int, seed: int, cluster: int = 1, rank: int = 0) -> List[int]:
    """The 3072 4-byte words of one CTA's area after a clean run of shared-memory atomic unit `unit` under `seed`
    (DSMEM, REDAS: of rank `rank` of a cluster of `cluster` CTAs)."""
    n = check(int(lib.gsb_shared_atomic_expected(unit, seed, cluster, rank, None, 0)),
              "gsb_shared_atomic_expected(size)")
    out = (C.c_uint32 * n)()
    check(int(lib.gsb_shared_atomic_expected(unit, seed, cluster, rank, out, n)), "gsb_shared_atomic_expected")
    return list(out)


def shared_atomic_conditions(r: "_abi.SharedAtomicResult") -> int:
    """GSB_SHARED_ATOMIC_* bits a shared-memory atomic probe result raises."""
    return lib.gsb_shared_atomic_conditions(C.byref(r))


def shared_atomic_text(r: "_abi.SharedAtomicResult", uuid: str) -> str:
    """The one log line both daemons print for a shared-memory atomic probe result."""
    need = lib.gsb_shared_atomic_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_shared_atomic_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_shared_atomic_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_shared_atomic_text")
    return buf.raw[: int(n)].decode()


def test_shared_atomic_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next shared-memory atomic probe of `idx`, in the first launch of `unit`, the CTA on SM `smid`
    XORs `xr` into its area word `index` just before the compare; once."""
    check(lib.gsb_test_shared_atomic_corrupt(idx, smid, unit, index, xr), f"gsb_test_shared_atomic_corrupt({idx})")


def test_shared_atomic_skip(idx: int, smid: int, unit: int) -> None:
    """Test hook: on the next shared-memory atomic probe of `idx`, in the first launch of `unit`, the CTA on SM `smid`
    issues none of the unit's atomics; once."""
    check(lib.gsb_test_shared_atomic_skip(idx, smid, unit), f"gsb_test_shared_atomic_skip({idx})")


test_shared_atomic_corrupt.__test__ = False
test_shared_atomic_skip.__test__ = False


def sfu_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0,
              raise_on_error: bool = True) -> "_abi.SfuResult":
    """SM special-function probe of device `idx`: every instruction of each unit (`units`: a mask of
    1 << GSB_SFU_UNIT_*, 0 = all) on every SM; the exact units compared bit for bit with the folds for `seed_expect`
    (0 = `seed`; `seed` 0 = fresh), MUFU voted across SMs. Mismatches are a result, not an error; with
    raise_on_error=False a failed launch is too (``status`` < 0)."""
    cfg = _abi.SfuCfg(seed, seed_expect, units, 0)
    r = _abi.SfuResult()
    rc = lib.gsb_sfu_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_sfu_probe({idx})")
    return r


def sfu_stats(idx: int) -> "_abi.SfuStats":
    """SFU probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.SfuStats()
    check(lib.gsb_sfu_stats_get(idx, C.byref(st)), f"gsb_sfu_stats_get({idx})")
    return st


def sfu_expected(unit: int, seed: int) -> List[int]:
    """The exact folds of SFU unit `unit` (not MUFU) for `seed`, index op * 256 + thread."""
    n = check(int(lib.gsb_sfu_expected(unit, seed, None, 0)), "gsb_sfu_expected(size)")
    out = (C.c_uint64 * n)()
    check(int(lib.gsb_sfu_expected(unit, seed, out, n)), "gsb_sfu_expected")
    return list(out)


def sfu_model(unit: int, op: int, a, b=None) -> "np.ndarray":
    """The host's answer (gsb_sfu_model) of exact SFU instruction (unit, op) for operand bits a[i] (and b[i]: the
    second f32 of an x2 pack, or the divisor), as a uint64 numpy array."""
    import numpy as np
    a_ = np.ascontiguousarray(a, dtype=np.uint64)
    b_ = None if b is None else np.ascontiguousarray(b, dtype=np.uint64)
    if b_ is not None and b_.shape != a_.shape:
        raise ValueError("sfu_model: a and b differ in length")
    out = np.zeros(len(a_), dtype=np.uint64)
    check(int(lib.gsb_sfu_model(unit, op, _u64p(a_), _u64p(b_), len(a_), _u64p(out))), "gsb_sfu_model")
    return out


def _u64p(x):
    return None if x is None else x.ctypes.data_as(C.POINTER(C.c_uint64))


def sfu_vote(seed: int, folds, raw, smid, r: Optional["_abi.SfuResult"] = None) -> "_abi.SfuResult":
    """gsb_sfu_vote over len(smid) CTAs: folds[cta][op][thread] and raw[cta][op][thread][GSB_SFU_RAW] (numpy arrays
    or flat sequences) and smid[cta], added into `r` (a fresh result by default), which is returned."""
    r = _abi.SfuResult() if r is None else r
    ctas = len(smid)
    f = _words(C.c_uint64, "<u8", folds, ctas * _abi.GSB_SFU_MUFU_FOLDS)
    w = _words(C.c_uint32, "<u4", raw, ctas * _abi.GSB_SFU_MUFU_FOLDS * _abi.GSB_SFU_RAW)
    s = _words(C.c_uint32, "<u4", smid, ctas)
    check(lib.gsb_sfu_vote(seed, ctas, f, w, s, C.byref(r)), "gsb_sfu_vote")
    return r


def _words(ctype, dtype, xs, n):
    """n words of ctype from a numpy array (any shape) or a flat sequence."""
    if hasattr(xs, "astype"):
        data = xs.astype(dtype).tobytes()
        if len(data) != n * C.sizeof(ctype):
            raise ValueError(f"expected {n} words, got {len(data) // C.sizeof(ctype)}")
        return (ctype * n).from_buffer_copy(data)
    xs = [int(x) for x in xs]
    if len(xs) != n:
        raise ValueError(f"expected {n} words, got {len(xs)}")
    return (ctype * n)(*xs)


def sfu_conditions(r: "_abi.SfuResult") -> int:
    """GSB_SFU_* bits an SFU probe result raises."""
    return lib.gsb_sfu_conditions(C.byref(r))


def sfu_text(r: "_abi.SfuResult", uuid: str) -> str:
    """The one log line both daemons print for an SFU probe result."""
    need = lib.gsb_sfu_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_sfu_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_sfu_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_sfu_text")
    return buf.raw[: int(n)].decode()


def test_sfu_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next SFU probe of `idx`, the CTA on SM `smid` XORs `xr` into its fold `index`
    (op * 256 + thread) of `unit` just before the compare (MUFU: the write); once."""
    check(lib.gsb_test_sfu_corrupt(idx, smid, unit, index, xr), f"gsb_test_sfu_corrupt({idx})")


test_sfu_corrupt.__test__ = False


def test_sfu_inputs(idx: int, unit: int, op: int, a, b=None):
    """Test hook, synchronous: SFU instruction (unit, op) on operand bits a[i] (and b[i]) on every SM of `idx`, at
    most GSB_SFU_INPUTS_MAX pairs. Returns (results, sms): results[k] holds the raw results of SM sms[k], a uint64
    numpy array of shape (len(sms), n)."""
    import numpy as np
    a_ = np.ascontiguousarray(a, dtype=np.uint64)
    b_ = None if b is None else np.ascontiguousarray(b, dtype=np.uint64)
    if b_ is not None and b_.shape != a_.shape:
        raise ValueError("test_sfu_inputs: a and b differ in length")
    n = len(a_)
    results = np.zeros((_abi.GSB_SM_MAX, max(n, 1)), dtype=np.uint64)
    covered = (C.c_uint32 * (_abi.GSB_SM_MAX // 32))()
    check(lib.gsb_test_sfu_inputs(idx, unit, op, _u64p(a_), _u64p(b_), n, _u64p(results), covered),
          f"gsb_test_sfu_inputs({idx})")
    sms = [sm for sm in range(_abi.GSB_SM_MAX) if covered[sm >> 5] >> (sm & 31) & 1]
    return results[sms], sms


test_sfu_inputs.__test__ = False


def l1_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0, passes: int = 0,
             raise_on_error: bool = True) -> "_abi.L1Result":
    """L1 and constant-cache probe of device `idx`: each unit (`units`: a mask of 1 << GSB_L1_UNIT_*, 0 = all) on
    every SM, every word compared on the SM with the pattern for `seed_expect` (0 = `seed`; `seed` 0 = fresh);
    `passes` per L1_LOAD and NC form (0 = 8). Mismatches are a result, not an error; with raise_on_error=False a failed
    launch is too (``status`` < 0)."""
    cfg = _abi.L1Cfg(seed, seed_expect, units, passes)
    r = _abi.L1Result()
    rc = lib.gsb_l1_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_l1_probe({idx})")
    return r


def l1_stats(idx: int) -> "_abi.L1Stats":
    """L1 probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.L1Stats()
    check(lib.gsb_l1_stats_get(idx, C.byref(st)), f"gsb_l1_stats_get({idx})")
    return st


def l1_schedule(unit: int, form: int, pass_: int, cta: int, ctas: int, thread: int, step: int) -> int:
    """gsb_l1_schedule: the word that read of the L1 probe returns (GSB_L1_ZERO_TEXEL: a border texel), or a negative
    status for a read the unit does not make."""
    return int(lib.gsb_l1_schedule(unit, form, pass_, cta, ctas, thread, step))


def l1_conditions(r: "_abi.L1Result") -> int:
    """GSB_L1_* bits an L1 probe result raises."""
    return lib.gsb_l1_conditions(C.byref(r))


def l1_text(r: "_abi.L1Result", uuid: str) -> str:
    """The one log line both daemons print for an L1 probe result."""
    need = lib.gsb_l1_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_l1_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_l1_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_l1_text")
    return buf.raw[: int(n)].decode()


def test_l1_corrupt(idx: int, smid: int, unit: int, index: int, xr: int) -> None:
    """Test hook: on the next L1 probe of `idx`, the CTA on SM `smid` XORs `xr` into lanes 0-1 of its observed word
    `index` of `unit` just before the compare, in the unit's first launch; once."""
    check(lib.gsb_test_l1_corrupt(idx, smid, unit, index, xr), f"gsb_test_l1_corrupt({idx})")


def test_l1_skip(idx: int, smid: int) -> None:
    """Test hook: in the next L1 probe of `idx`, the first L1_STORE launch's CTA on SM `smid` stores nothing."""
    check(lib.gsb_test_l1_skip(idx, smid), f"gsb_test_l1_skip({idx})")


def test_l1_table(idx: int, unit: int, table, expected=None, region_words: int = 0) -> None:
    """Test hook: the next L1 probe of `idx` that runs `unit` runs its test-only twin on `table` (uint32 entries, as
    gsb_test_l1_table lays them out) against `expected` (L1_STORE: the region words after the last round, every CTA's;
    TEX: the texel each read returns, -1 for 0), with CTA regions of `region_words` words; once. table=None disarms
    it."""
    import numpy as np
    if table is None:
        check(lib.gsb_test_l1_table(idx, unit, None, 0, None, 0, 0), f"gsb_test_l1_table({idx})")
        return
    t = np.ascontiguousarray(np.asarray(table).astype(np.uint32))
    e = None if expected is None else np.ascontiguousarray(np.asarray(expected).astype(np.int64).astype(np.uint32))
    ptr = lambda x: None if x is None else x.ctypes.data_as(C.POINTER(C.c_uint32))  # noqa: E731
    check(lib.gsb_test_l1_table(idx, unit, ptr(t), len(t), ptr(e), 0 if e is None else len(e), region_words),
          f"gsb_test_l1_table({idx})")


test_l1_corrupt.__test__ = False
test_l1_skip.__test__ = False
test_l1_table.__test__ = False


def order_probe(idx: int, *, seed: int = 0, seed_expect: int = 0, units: int = 0, observations: int = 0,
                raise_on_error: bool = True) -> "_abi.OrderResult":
    """Memory-ordering probe of device `idx`: each unit (`units`: a mask of 1 << GSB_ORDER_UNIT_*, 0 = all) at three
    distances, `observations` per CTA and launch (0 = 1024), every word's hash checked against `seed_expect` (0 =
    `seed`; `seed` 0 = fresh). Outcomes are a result, not an error; with raise_on_error=False a failed launch is too
    (``status`` < 0)."""
    cfg = _abi.OrderCfg(seed, seed_expect, units, observations)
    r = _abi.OrderResult()
    rc = lib.gsb_order_probe(idx, C.byref(cfg), C.byref(r))
    if raise_on_error:
        check(rc, f"gsb_order_probe({idx})")
    return r


def order_stats(idx: int) -> "_abi.OrderStats":
    """Memory-ordering probes of device `idx` since health_start: count, faults, skipped, incomplete, the last result."""
    st = _abi.OrderStats()
    check(lib.gsb_order_stats_get(idx, C.byref(st)), f"gsb_order_stats_get({idx})")
    return st


def order_pairing(unit: int, n: int, d: int, rank: int) -> list:
    """gsb_order_pairing: the ranks CTA `rank` of `n` reads in `unit` at distance `d` ([] for a bad argument)."""
    out = (C.c_uint32 * 3)()
    k = lib.gsb_order_pairing(unit, n, d, rank, out)
    return list(out[:k])


def order_classify(unit: int, seed: int, keys, words, iteration: int = 0) -> int:
    """gsb_order_classify: the GSB_ORDER_CLS_* class of one observation."""
    k = (C.c_uint32 * _abi.GSB_ORDER_WORDS)(*list(keys)[:_abi.GSB_ORDER_WORDS])
    w = (C.c_uint64 * _abi.GSB_ORDER_WORDS)(*list(words)[:_abi.GSB_ORDER_WORDS])
    return int(lib.gsb_order_classify(unit, seed, k, w, iteration))


def order_conditions(r: "_abi.OrderResult") -> int:
    """GSB_ORDER_* bits a memory-ordering probe result raises."""
    return lib.gsb_order_conditions(C.byref(r))


def order_text(r: "_abi.OrderResult", uuid: str) -> str:
    """The one log line both daemons print for a memory-ordering probe result."""
    need = lib.gsb_order_text(C.byref(r), uuid.encode(), None, 0)
    check(int(need), "gsb_order_text(size)")
    buf = C.create_string_buffer(int(need))
    n = lib.gsb_order_text(C.byref(r), uuid.encode(), buf, int(need))
    check(int(n), "gsb_order_text")
    return buf.raw[: int(n)].decode()


def test_order_inject(idx: int, smid: int, unit: int, index: int) -> None:
    """Test hook: on the next memory-ordering probe of `idx`, the consumer on SM `smid` reports observation `index` of
    `unit`'s first launch as a forbidden outcome with valid hashes; once. The next probe takes it whatever its
    observations; an index at or past them injects nothing."""
    check(lib.gsb_test_order_inject(idx, smid, unit, index), f"gsb_test_order_inject({idx})")


def test_order_skip(idx: int, smid: int) -> None:
    """Test hook: in the next memory-ordering probe of `idx`, the producer on SM `smid` stores nothing in the first
    MP_RELACQ launch; once."""
    check(lib.gsb_test_order_skip(idx, smid), f"gsb_test_order_skip({idx})")


test_order_inject.__test__ = False
test_order_skip.__test__ = False


def fault_classify(offset: int, expected, observed) -> FaultRecord:
    """gsb_fault_classify of one word: cls, alias_bit, seed_key and flipped_bits filled in."""
    rec = FaultRecord(offset, (C.c_uint32 * 4)(*expected), (C.c_uint32 * 4)(*observed))
    check(lib.gsb_fault_classify(C.byref(rec)), "gsb_fault_classify")
    return rec
