"""ctypes binding of include/gpushare_b200.h — the Python twin of the cgo stub in INTEGRATION.md.

Loads the in-tree ``libgpushare_b200.so`` (built by ``build.sh`` / ``__graft_entry__.build()``).
There is no fallback of any kind: if the library is missing this module raises ImportError, and if
the CUDA driver / NVML / an sm_90 device is missing every device entry point returns a negative
``gsb_status`` which :func:`check` turns into :class:`GsbError`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgpushare_b200.so")

GSB_UUID_BUFFER_SIZE = 80
GSB_BUSID_BUFFER_SIZE = 32

GSB_OK = 0
GSB_ERR_NOT_INITIALIZED = -1
GSB_ERR_INVALID_ARGUMENT = -2
GSB_ERR_LIBRARY_NOT_FOUND = -3
GSB_ERR_DRIVER = -4
GSB_ERR_NVML = -5
GSB_ERR_NO_DEVICE = -6
GSB_ERR_IDENTITY_MISMATCH = -7
GSB_ERR_BUFFER_TOO_SMALL = -8
GSB_ERR_OUT_OF_MEMORY = -9
GSB_ERR_UNSUPPORTED_ARCH = -10
GSB_ERR_TIMEOUT = -11
GSB_ERR_NO_ARENA = -12
GSB_ERR_MALFORMED = -13
GSB_ERR_STOPPED = -14

GSB_OP_FILL, GSB_OP_VERIFY, GSB_OP_VERIFY_REFILL = 1, 2, 3
GSB_VARIANT_AUTO, GSB_VARIANT_DIRECT, GSB_VARIANT_CPASYNC, GSB_VARIANT_BULK, GSB_VARIANT_BULKW, GSB_VARIANT_BULKD = 0, 1, 2, 3, 4, 5
VARIANT_NAMES = {0: "auto", 1: "direct", 2: "cpasync", 3: "bulk", 4: "bulkw", 5: "bulkd"}
GSB_PROBE_TIMED, GSB_PROBE_SEED_TABLE = 1, 2
GSB_EVENT_XID, GSB_EVENT_PROBE, GSB_EVENT_INVENTORY = 8, 0x100, 0x200
GSB_PROBE_FAULT_MISMATCH, GSB_PROBE_FAULT_LAUNCH, GSB_PROBE_RECOVERED, GSB_PROBE_FAULT_WEDGED = 1, 2, 3, 4
GSB_INVENTORY_IDENTITY_CHANGED, GSB_INVENTORY_TOTAL_CHANGED = 1, 2
GSB_ABI_VERSION = 3
GSB_FAULT_RECORDS = 64
GSB_FAULT_ZERO, GSB_FAULT_STALE, GSB_FAULT_ALIASED, GSB_FAULT_BITS = 1, 2, 3, 4
FAULT_CLASS_NAMES = {1: "zero", 2: "stale", 3: "aliased", 4: "bits"}
GSB_FAULT_NO_ALIAS = 0xFFFFFFFF
GSB_FAULT_REPORT_FIRST, GSB_FAULT_REPORT_LAST = 0, 1
GSB_ALL_DEVICES = 0xFFFFFFFF
GSB_OPT_INVENTORY_POLICY, GSB_OPT_WAIT_SPIN_US, GSB_OPT_WATCHDOG_MS, GSB_OPT_INVENTORY_REFRESH_MS, \
    GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, GSB_OPT_SWEEP_EVERY_CYCLES = 1, 2, 3, 4, 5, 6
GSB_INVENTORY_SNAPSHOT, GSB_INVENTORY_LIVE = 0, 1
GSB_ALLOC_MATCHED, GSB_ALLOC_SINGLE_GPU, GSB_ALLOC_ERR_RESPONSE = 1, 2, 3
UINT64_MAX = (1 << 64) - 1

# every symbol include/gpushare_b200.h declares (tests/test_abi.py checks header <-> this list <-> .so)
SYMBOLS = [
    "gsb_abi_version", "gsb_init", "gsb_shutdown", "gsb_strerror", "gsb_last_error",
    "gsb_device_count", "gsb_device_info_get", "gsb_inventory_refresh", "gsb_inventory_snapshot",
    "gsb_set_option", "gsb_get_option", "gsb_slices", "gsb_fake_device_id", "gsb_real_device_id",
    "gsb_encode_list_and_watch", "gsb_encode_register_request",
    "gsb_arena_create", "gsb_arena_destroy", "gsb_arena_bytes", "gsb_probe", "gsb_probe_all",
    "gsb_arena_read", "gsb_arena_write", "gsb_test_stall", "gsb_test_skew_snapshot", "gsb_cycle", "gsb_cycle_all",
    "gsb_health_start", "gsb_health_stop", "gsb_health_wait", "gsb_health_inject", "gsb_health_set_recovery", "gsb_health_stats_get",
    "gsb_xid_is_benign", "gsb_fault_report_get", "gsb_fault_classify", "gsb_fault_report_text",
    "gsb_allocate", "gsb_allocate_err_response", "gsb_patch_assigned_body",
]


class DeviceInfo(C.Structure):
    _fields_ = [
        ("uuid", C.c_char * GSB_UUID_BUFFER_SIZE),
        ("bus_id", C.c_char * GSB_BUSID_BUFFER_SIZE),
        ("index", C.c_uint32),
        ("minor", C.c_uint32),
        ("cuda_ordinal", C.c_int32),
        ("sm_count", C.c_uint32),
        ("cc_major", C.c_uint32),
        ("cc_minor", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("total_bytes", C.c_uint64),
        ("total_mib", C.c_uint64),
        ("free_bytes", C.c_uint64),
        ("cuda_total_bytes", C.c_uint64),
    ]


class ProbeCfg(C.Structure):
    _fields_ = [
        ("op", C.c_uint32),
        ("variant", C.c_uint32),
        ("window_offset", C.c_uint64),
        ("window_bytes", C.c_uint64),
        ("seed_expect", C.c_uint32),
        ("seed_write", C.c_uint32),
        ("grid_ctas", C.c_uint32),
        ("flags", C.c_uint32),
    ]


class ProbeResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("variant", C.c_uint32),
        ("bytes_walked", C.c_uint64),
        ("bytes_read", C.c_uint64),
        ("bytes_written", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("first_bad_offset", C.c_uint64),
        ("checksum_xor", C.c_uint32),
        ("checksum_sum", C.c_uint32),
        ("kernel_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
        ("grid_ctas", C.c_uint32),
        ("block_threads", C.c_uint32),
    ]


class CycleResult(C.Structure):
    _fields_ = [
        ("info", DeviceInfo),
        ("slices", C.c_uint32),
        ("healthy", C.c_uint32),
        ("lw_len", C.c_int64),
        ("inventory_ns", C.c_uint64),
        ("probe", ProbeResult),
        ("snapshot_age_ns", C.c_uint64),
        ("inventory_live", C.c_uint32),
        ("transient", C.c_uint32),
    ]


class HealthStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("cycles", "sweeps", "skipped", "faults", "last_bytes_walked", "last_kernel_ns",
                                          "last_sweep_bytes", "last_sweep_ns")]


class Event(C.Structure):
    _fields_ = [("uuid", C.c_char * GSB_UUID_BUFFER_SIZE), ("etype", C.c_uint64), ("edata", C.c_uint64)]


class FaultRecord(C.Structure):
    _fields_ = [
        ("offset", C.c_uint64),
        ("expected", C.c_uint32 * 4),
        ("observed", C.c_uint32 * 4),
        ("cls", C.c_uint32),
        ("alias_bit", C.c_uint32),
        ("seed_key", C.c_uint32),
        ("flipped_bits", C.c_uint32),
    ]


class FaultReport(C.Structure):
    _fields_ = [
        ("valid", C.c_uint32),
        ("op", C.c_uint32),
        ("transient", C.c_uint32),
        ("n_records", C.c_uint32),
        ("unix_ns", C.c_uint64),
        ("window_offset", C.c_uint64),
        ("window_bytes", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("first_bad_offset", C.c_uint64),
        ("flips_0to1", C.c_uint64 * 128),
        ("flips_1to0", C.c_uint64 * 128),
        ("records", FaultRecord * GSB_FAULT_RECORDS),
    ]


class Pod(C.Structure):
    _fields_ = [
        ("name", C.c_char_p),
        ("ns", C.c_char_p),
        ("uid", C.c_char_p),
        ("gpu_mem_limit", C.c_uint64),
        ("assume_time", C.c_uint64),
        ("gpu_idx", C.c_int32),
        ("has_assume_time", C.c_uint8),
        ("has_assigned", C.c_uint8),
        ("assigned_is_false", C.c_uint8),
        ("on_node", C.c_uint8),
    ]


class AllocateCtx(C.Structure):
    _fields_ = [
        ("uuids", C.POINTER(C.c_char_p)),
        ("minors", C.POINTER(C.c_uint32)),
        ("n_gpus", C.c_uint32),
        ("slices", C.c_uint32),
        ("unit_gib", C.c_int32),
        ("disable_cgpu_isolation", C.c_int32),
        ("pods_unique", C.c_int32),
    ]


class GsbError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        text = lib.gsb_strerror(status).decode() if lib is not None else str(status)
        super().__init__(f"{where}: {text} ({status}){': ' + detail if detail else ''}")


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run ./build.sh (or __graft_entry__.build()). "
            "gpushare_device_plugin_b200 has no non-CUDA fallback."
        )
    l = C.CDLL(LIB_PATH)
    u8p, u32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    sig = {
        "gsb_abi_version": (C.c_int, []),
        "gsb_init": (C.c_int, []),
        "gsb_shutdown": (C.c_int, []),
        "gsb_strerror": (C.c_char_p, [C.c_int]),
        "gsb_last_error": (C.c_int, [C.c_char_p, C.c_size_t]),
        "gsb_device_count": (C.c_int, [u32p]),
        "gsb_device_info_get": (C.c_int, [C.c_uint32, C.POINTER(DeviceInfo)]),
        "gsb_inventory_refresh": (C.c_int, [C.c_uint32]),
        "gsb_inventory_snapshot": (C.c_int, [C.c_uint32, C.POINTER(DeviceInfo), u64p]),
        "gsb_set_option": (C.c_int, [C.c_uint32, C.c_uint64]),
        "gsb_get_option": (C.c_int, [C.c_uint32, u64p]),
        "gsb_test_stall": (C.c_int, [C.c_uint32, C.c_uint32]),
        "gsb_test_skew_snapshot": (C.c_int, [C.c_uint32, C.c_uint64]),
        "gsb_slices": (C.c_uint32, [C.c_uint64, C.c_int]),
        "gsb_fake_device_id": (C.c_int, [C.c_char_p, C.c_uint32, C.c_char_p, C.c_size_t]),
        "gsb_real_device_id": (C.c_int, [C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_encode_list_and_watch": (C.c_int64, [C.POINTER(C.c_char_p), C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t]),
        "gsb_encode_register_request": (C.c_int64, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t]),
        "gsb_arena_create": (C.c_int, [C.c_uint32, C.c_uint64, C.c_uint64, u64p]),
        "gsb_arena_destroy": (C.c_int, [C.c_uint32]),
        "gsb_arena_bytes": (C.c_int, [C.c_uint32, u64p]),
        "gsb_probe": (C.c_int, [C.c_uint32, C.POINTER(ProbeCfg), C.POINTER(ProbeResult)]),
        "gsb_probe_all": (C.c_int, [C.c_uint32, u32p, C.POINTER(ProbeCfg), C.POINTER(ProbeResult)]),
        "gsb_arena_read": (C.c_int, [C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64]),
        "gsb_arena_write": (C.c_int, [C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64]),
        "gsb_cycle": (C.c_int, [C.c_uint32, C.c_uint64, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(CycleResult)]),
        "gsb_cycle_all": (C.c_int64, [C.c_uint32, u32p, C.c_uint64, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(CycleResult)]),
        "gsb_health_start": (C.c_int, [C.c_uint32, C.c_uint64]),
        "gsb_health_stop": (C.c_int, []),
        "gsb_health_wait": (C.c_int, [C.c_uint32, C.POINTER(Event)]),
        "gsb_health_inject": (C.c_int, [C.POINTER(Event)]),
        "gsb_health_set_recovery": (C.c_int, [C.c_uint32]),
        "gsb_health_stats_get": (C.c_int, [C.c_uint32, C.POINTER(HealthStats)]),
        "gsb_xid_is_benign": (C.c_int, [C.c_uint64]),
        "gsb_fault_report_get": (C.c_int, [C.c_uint32, C.c_uint32, C.POINTER(FaultReport)]),
        "gsb_fault_classify": (C.c_int, [C.POINTER(FaultRecord)]),
        "gsb_fault_report_text": (C.c_int64, [C.POINTER(FaultReport), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_allocate": (C.c_int, [C.POINTER(AllocateCtx), C.POINTER(Pod), C.c_uint32, C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int32), u32p]),
        "gsb_allocate_err_response": (C.c_int, [C.POINTER(AllocateCtx), C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
        "gsb_patch_assigned_body": (C.c_int, [C.c_uint64, C.c_char_p, C.c_size_t]),
    }
    for name in SYMBOLS:
        fn = getattr(l, name)  # AttributeError here == header/.so drift
        fn.restype, fn.argtypes = sig[name]
    return l


lib = None
lib = _load()


def last_error() -> str:
    buf = C.create_string_buffer(512)
    lib.gsb_last_error(buf, len(buf))
    return buf.value.decode(errors="replace")


def check(status: int, where: str) -> int:
    if status < 0:
        raise GsbError(status, where, last_error())
    return status
