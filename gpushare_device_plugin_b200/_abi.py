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
# the L1 and constant-cache check's kernels, a module of their own that LIB_PATH loads
L1_LIB_PATH = os.path.join(_HERE, "libgpushare_b200_l1.so")
# the memory-ordering check's kernel, likewise a module of its own that LIB_PATH loads
ORDER_LIB_PATH = os.path.join(_HERE, "libgpushare_b200_order.so")
# the SM-to-SM check's test-only twins (gsb_test_cluster_script), likewise a module of their own that LIB_PATH loads
CLUSTER_SCRIPT_LIB_PATH = os.path.join(_HERE, "libgpushare_b200_cluster_script.so")

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
GSB_OP_MARCH_FILL, GSB_OP_MARCH_VERIFY, GSB_OP_MARCH_RW_UP, GSB_OP_MARCH_RW_DOWN = 4, 5, 6, 7
GSB_MEMTEST_ELEMENTS = 6
GSB_OP_LINK_UP, GSB_OP_LINK_DOWN, GSB_OP_LINK_DUPLEX = 8, 9, 10
GSB_LINK_PHASES = 3
GSB_LINK_VALID_CUR_GEN, GSB_LINK_VALID_CUR_WIDTH, GSB_LINK_VALID_MAX_GEN, GSB_LINK_VALID_MAX_WIDTH, \
    GSB_LINK_VALID_GPU_MAX_GEN, GSB_LINK_VALID_REPLAY = 1, 2, 4, 8, 16, 32
GSB_LINK_CORRUPT, GSB_LINK_FAILED, GSB_LINK_WIDTH_DEGRADED, GSB_LINK_SPEED_DEGRADED = 1, 2, 4, 8
LINK_CONDITION_NAMES = {1: "corrupted data across the link", 2: "link probe failed", 4: "link width degraded",
                        8: "link speed degraded"}
GSB_OP_COPY_H2D, GSB_OP_COPY_D2H, GSB_OP_COPY_D2D = 11, 12, 13
GSB_COPY_DIRECTIONS = 3
GSB_COPY_GEOMETRY = 1
GSB_COPY_CORRUPT, GSB_COPY_FAILED = 1, 2
COPY_CONDITION_NAMES = {1: "corrupted data after a DMA copy", 2: "copy probe failed"}
GSB_SM_UNIT_SMEM, GSB_SM_UNIT_INT32, GSB_SM_UNIT_FP32, GSB_SM_UNIT_FP64, GSB_SM_UNIT_F16, GSB_SM_UNIT_BF16, \
    GSB_SM_UNIT_E4M3, GSB_SM_UNIT_S8 = range(8)
SM_UNIT_NAMES = ["smem", "int32", "fp32", "fp64", "f16", "bf16", "e4m3", "s8"]
GSB_SM_UNITS, GSB_SM_MAX, GSB_SM_RECORDS, GSB_SM_MAX_LAUNCHES, GSB_SM_SMEM_WORDS_MAX = 8, 256, 64, 3, 29056
GSB_SM_CORRUPT, GSB_SM_FAILED = 1, 2
SM_CONDITION_NAMES = {1: "wrong result on an SM", 2: "SM probe failed"}
GSB_CLUSTER_PATH_DSMEM_ST, GSB_CLUSTER_PATH_DSMEM_LD, GSB_CLUSTER_PATH_ST_ASYNC, GSB_CLUSTER_PATH_BULK_S2S, \
    GSB_CLUSTER_PATH_MULTICAST = range(5)
CLUSTER_PATH_NAMES = ["dsmem_st", "dsmem_ld", "st_async", "bulk_s2s", "multicast"]
GSB_CLUSTER_PATHS, GSB_CLUSTER_SIZES, GSB_CLUSTER_MAX_N, GSB_CLUSTER_RECORDS, GSB_CLUSTER_MAX_LAUNCHES = 5, 4, 16, 64, 3
GSB_CLUSTER_SM_MAX, GSB_CLUSTER_WAIT_NS, GSB_CLUSTER_EVERY_RANK, GSB_CLUSTER_HEADER_BYTES = 256, 100000000, 0xFF, 1024
GSB_CLUSTER_HOOK_INDEX_MAX = 14464
GSB_CLUSTER_UNROUTED = 0xFF
GSB_CLUSTER_CORRUPT, GSB_CLUSTER_FAILED = 1, 2
CLUSTER_CONDITION_NAMES = {1: "wrong word across the SM-to-SM network", 2: "SM-to-SM probe failed"}
GSB_CLUSTER_CLASS_ZERO, GSB_CLUSTER_CLASS_STALE, GSB_CLUSTER_CLASS_MISROUTED, GSB_CLUSTER_CLASS_BITS = 1, 2, 3, 4
GSB_ATOMIC_OP_ADD32, GSB_ATOMIC_OP_ADD64, GSB_ATOMIC_OP_LOGIC, GSB_ATOMIC_OP_MINMAX, GSB_ATOMIC_OP_FADD32, \
    GSB_ATOMIC_OP_FADD64, GSB_ATOMIC_OP_HADD2, GSB_ATOMIC_OP_TICKET, GSB_ATOMIC_OP_CAS = range(9)
ATOMIC_OP_NAMES = ["add32", "add64", "logic", "minmax", "fadd32", "fadd64", "hadd2", "ticket", "cas"]
GSB_ATOMIC_OPS, GSB_ATOMIC_RECORDS, GSB_ATOMIC_MAX_LAUNCHES, GSB_ATOMIC_SM_MAX, GSB_ATOMIC_THREADS = 9, 64, 3, 256, 256
GSB_ATOMIC_LINES, GSB_ATOMIC_LINE_BYTES, GSB_ATOMIC_HOT_WORDS, GSB_ATOMIC_HOT_STRIDE, GSB_ATOMIC_HOT_REPS = \
    8192, 128, 32, 4096, 4
GSB_ATOMIC_REGION_BYTES = GSB_ATOMIC_LINES * GSB_ATOMIC_LINE_BYTES
GSB_ATOMIC_BYTES = GSB_ATOMIC_REGION_BYTES + GSB_ATOMIC_HOT_WORDS * GSB_ATOMIC_HOT_STRIDE
GSB_ATOMIC_CAS_WAIT_NS, GSB_ATOMIC_NO_ID, GSB_ATOMIC_NO_SM = 100000000, 0xFFFFFFFF, 0xFFFFFFFF
GSB_ATOMIC_PHASE_SPREAD, GSB_ATOMIC_PHASE_HOT, GSB_ATOMIC_PHASE_SLOT = 0, 1, 2
GSB_ATOMIC_CORRUPT, GSB_ATOMIC_FAILED = 1, 2
ATOMIC_CONDITION_NAMES = {1: "wrong result of an L2 atomic", 2: "L2 atomic probe failed"}
GSB_TENSOR_UNIT_DMMA, GSB_TENSOR_UNIT_TF32, GSB_TENSOR_UNIT_E5M2, GSB_TENSOR_UNIT_E4M3_E5M2, GSB_TENSOR_UNIT_E5M2_E4M3, \
    GSB_TENSOR_UNIT_F16_ACC, GSB_TENSOR_UNIT_HMMA, GSB_TENSOR_UNIT_F16_RS = range(8)
TENSOR_UNIT_NAMES = ["dmma", "tf32", "e5m2", "e4m3_e5m2", "e5m2_e4m3", "f16_acc", "hmma", "f16_rs"]
GSB_TENSOR_UNITS, GSB_TENSOR_RECORDS, GSB_TENSOR_MAX_LAUNCHES, GSB_TENSOR_WORDS = 8, 64, 3, 8192
GSB_TENSOR_CORRUPT, GSB_TENSOR_FAILED = 1, 2
TENSOR_CONDITION_NAMES = {1: "wrong tensor-core result", 2: "tensor probe failed"}
GSB_SPARSE_UNIT_F16_SP, GSB_SPARSE_UNIT_BF16_SP, GSB_SPARSE_UNIT_TF32_SP, GSB_SPARSE_UNIT_E4M3_SP, \
    GSB_SPARSE_UNIT_E5M2_SP, GSB_SPARSE_UNIT_S8_SP, GSB_SPARSE_UNIT_HMMA_SP = range(7)
SPARSE_UNIT_NAMES = ["f16", "bf16", "tf32", "e4m3", "e5m2", "s8", "hmma"]
SPARSE_UNIT_K = [512, 512, 256, 128, 128, 512, 512]  # logical K of each unit (= gsb_sparse_shape(unit).k)
GSB_SPARSE_UNITS, GSB_SPARSE_RECORDS, GSB_SPARSE_MAX_LAUNCHES, GSB_SPARSE_WORDS = 7, 64, 3, 8192
GSB_SPARSE_CORRUPT, GSB_SPARSE_FAILED = 1, 2
SPARSE_CONDITION_NAMES = {1: "wrong sparse tensor-core result", 2: "sparse probe failed"}
GSB_SHARED_ATOMIC_UNIT_INT32, GSB_SHARED_ATOMIC_UNIT_WIDE, GSB_SHARED_ATOMIC_UNIT_FLOAT, GSB_SHARED_ATOMIC_UNIT_TICKET, \
    GSB_SHARED_ATOMIC_UNIT_CAS, GSB_SHARED_ATOMIC_UNIT_DSMEM, GSB_SHARED_ATOMIC_UNIT_REDAS = range(7)
SHARED_ATOMIC_UNIT_NAMES = ["int32", "wide", "float", "ticket", "cas", "dsmem", "redas"]
GSB_SHARED_ATOMIC_UNITS, GSB_SHARED_ATOMIC_RECORDS, GSB_SHARED_ATOMIC_MAX_LAUNCHES = 7, 64, 3
GSB_SHARED_ATOMIC_AREA_WORDS, GSB_SHARED_ATOMIC_CAS_WAIT_NS, GSB_SHARED_ATOMIC_NO_SM = 3072, 100_000_000, 0xFFFFFFFF
GSB_SHARED_ATOMIC_REC_WORD, GSB_SHARED_ATOMIC_REC_SLOT, GSB_SHARED_ATOMIC_REC_TICKET, GSB_SHARED_ATOMIC_REC_TORN = range(4)
GSB_SHARED_ATOMIC_CORRUPT, GSB_SHARED_ATOMIC_FAILED = 1, 2
SHARED_ATOMIC_CONDITION_NAMES = {1: "wrong shared-memory atomic result", 2: "shared-memory atomic probe failed"}
GSB_SFU_UNIT_CVT_HALF, GSB_SFU_UNIT_CVT_FP8, GSB_SFU_UNIT_CVT_INT, GSB_SFU_UNIT_DIVSQRT, GSB_SFU_UNIT_WARP, \
    GSB_SFU_UNIT_MUFU = range(6)
SFU_UNIT_NAMES = ["cvt_half", "cvt_fp8", "cvt_int", "divsqrt", "warp", "mufu"]
SFU_MUFU_NAMES = ["ex2", "lg2", "rcp", "rsqrt", "sqrt", "sin", "cos", "tanh", "ex2_f16", "ex2_bf16", "tanh_f16",
                  "tanh_bf16"]
GSB_SFU_UNITS, GSB_SFU_THREADS, GSB_SFU_STEPS, GSB_SFU_RAW, GSB_SFU_OPS_MAX, GSB_SFU_MUFU_OPS = 6, 256, 1024, 4, 15, 12
GSB_SFU_RECORDS, GSB_SFU_MAX_LAUNCHES, GSB_SFU_INPUTS_MAX = 64, 3, 1 << 15
GSB_SFU_MUFU_FOLDS = GSB_SFU_MUFU_OPS * GSB_SFU_THREADS
GSB_SFU_MUFU_WORDS = GSB_SFU_MUFU_FOLDS * (1 + GSB_SFU_RAW)
GSB_SFU_CORRUPT, GSB_SFU_BOUND, GSB_SFU_FAILED = 1, 2, 4
SFU_CONDITION_NAMES = {1: "wrong special-function result", 2: "MUFU result outside its envelope",
                       4: "SFU probe failed"}
GSB_L1_UNIT_L1_LOAD, GSB_L1_UNIT_L1_STORE, GSB_L1_UNIT_NC, GSB_L1_UNIT_TEX, GSB_L1_UNIT_CONST, GSB_L1_UNIT_PARAM = range(6)
L1_UNIT_NAMES = ["l1_load", "l1_store", "nc", "tex", "const", "param"]
GSB_L1_FORM_CA, GSB_L1_FORM_PLAIN, GSB_L1_FORM_EVICT_LAST, GSB_L1_FORM_NC = range(4)
L1_FORM_NAMES = ["ca", "plain", "evict_last", "nc"]
GSB_L1_UNITS, GSB_L1_THREADS, GSB_L1_REGION_WORDS, GSB_L1_STEPS, GSB_L1_PASSES_DEFAULT, GSB_L1_PASSES_MAX = \
    6, 1024, 8192, 8, 8, 64
GSB_L1_TEX_WIDTH, GSB_L1_TEX_ROWS, GSB_L1_TEX_2D_READS, GSB_L1_CONST_WORDS, GSB_L1_PARAM_WORDS = 64, 128, 16384, 4096, 2000
GSB_L1_RECORDS, GSB_L1_MAX_LAUNCHES, GSB_L1_FORMS = 64, 3, 4
GSB_L1_ZERO_TEXEL = (1 << 63) - 1
GSB_L1_CORRUPT, GSB_L1_FAILED = 1, 2
L1_CONDITION_NAMES = {1: "wrong word through L1, texture or constant cache", 2: "L1 probe failed"}
GSB_ORDER_UNIT_MP_RELACQ, GSB_ORDER_UNIT_MP_FENCE, GSB_ORDER_UNIT_SB_SC, GSB_ORDER_UNIT_IRIW_SC, GSB_ORDER_UNIT_CORR, \
    GSB_ORDER_UNIT_MP_RELAXED = range(6)
ORDER_UNIT_NAMES = ["mp_relacq", "mp_fence", "sb_sc", "iriw_sc", "corr", "mp_relaxed"]
GSB_ORDER_UNITS, GSB_ORDER_DISTANCES, GSB_ORDER_THREADS, GSB_ORDER_OBS_DEFAULT, GSB_ORDER_OBS_MAX, GSB_ORDER_WORDS, \
    GSB_ORDER_RECORDS = 6, 3, 256, 1024, 65536, 5, 64
GSB_ORDER_WAIT_NS, GSB_ORDER_WAIT_NS_PER_OBS = 100000000, 5000
GSB_ORDER_CLS_ALLOWED, GSB_ORDER_CLS_OVERLAP, GSB_ORDER_CLS_WEAK, GSB_ORDER_CLS_FORBIDDEN, GSB_ORDER_CLS_CORRUPT, \
    GSB_ORDER_CLS_LOST = range(6)
GSB_ORDER_CORRUPT, GSB_ORDER_FORBIDDEN, GSB_ORDER_LOST, GSB_ORDER_TIMEOUT, GSB_ORDER_FAILED = 1, 2, 4, 8, 16
ORDER_CONDITION_NAMES = {1: "word read back that no writer stored", 2: "outcome the memory model forbids",
                         4: "store lost after the grid barrier", 8: "grid barrier ran out",
                         16: "memory-ordering probe failed"}
# gsb_test_l1_table
GSB_L1_TABLE_MAX, GSB_L1_TABLE_EXPECTED_MAX, GSB_L1_TABLE_REGION_MAX, GSB_L1_TABLE_ROUNDS_MAX = 1 << 20, 1 << 24, 131072, 8
GSB_L1_STORE_WORD_BITS, GSB_L1_TABLE_RESIDENT, GSB_L1_TABLE_READ_OWN, GSB_L1_TEX_1D = 17, 1, 2, 0x80000000
GSB_STRESS_UNITS, GSB_STRESS_SETS_MAX, GSB_STRESS_FOLD_THREADS = 4, 4, 128
GSB_STRESS_DURATION_MAX_MS, GSB_STRESS_SLICE_MAX_MS, GSB_STRESS_SLICE_DEFAULT_MS, GSB_STRESS_SAMPLE_MS = 600000, 100, 50, 25
GSB_STRESS_UNIT_MASK = 0xF0
STRESS_UNIT_NAMES = ["f16", "bf16", "e4m3", "s8"]  # unit[k] of a result is GSB_SM_UNIT_F16 + k
GSB_STRESS_VALID_ENERGY, GSB_STRESS_VALID_POWER, GSB_STRESS_VALID_TEMP, GSB_STRESS_VALID_SM_CLOCK, \
    GSB_STRESS_VALID_REASONS, GSB_STRESS_VALID_POWER_LIMIT = 1, 2, 4, 8, 16, 32
GSB_STRESS_SLOWDOWN_REASONS = 0xC8
GSB_STRESS_CORRUPT, GSB_STRESS_FAILED = 1, 2
STRESS_CONDITION_NAMES = {1: "wrong tensor-core result under load", 2: "SM stress failed"}
GSB_VARIANT_AUTO, GSB_VARIANT_DIRECT, GSB_VARIANT_CPASYNC, GSB_VARIANT_BULK, GSB_VARIANT_BULKW, GSB_VARIANT_BULKD = 0, 1, 2, 3, 4, 5
VARIANT_NAMES = {0: "auto", 1: "direct", 2: "cpasync", 3: "bulk", 4: "bulkw", 5: "bulkd"}
GSB_PROBE_TIMED, GSB_PROBE_SEED_TABLE = 1, 2
GSB_EVENT_XID, GSB_EVENT_PROBE, GSB_EVENT_INVENTORY, GSB_EVENT_ECC, GSB_EVENT_LINK, GSB_EVENT_COPY, GSB_EVENT_SM, \
    GSB_EVENT_CLUSTER, GSB_EVENT_ATOMIC, GSB_EVENT_TENSOR, GSB_EVENT_SFU, GSB_EVENT_L1, GSB_EVENT_ORDER, \
    GSB_EVENT_SPARSE, GSB_EVENT_SHARED_ATOMIC = 8, 0x100, 0x200, 0x400, 0x800, 0x1000, 0x2000, 0x4000, 0x8000, \
    0x10000, 0x20000, 0x40000, 0x80000, 0x100000, 0x200000
GSB_PROBE_FAULT_MISMATCH, GSB_PROBE_FAULT_LAUNCH, GSB_PROBE_RECOVERED, GSB_PROBE_FAULT_WEDGED = 1, 2, 3, 4
GSB_INVENTORY_IDENTITY_CHANGED, GSB_INVENTORY_TOTAL_CHANGED = 1, 2
GSB_ECC_VALID_MODE, GSB_ECC_VALID_VOLATILE, GSB_ECC_VALID_AGGREGATE, GSB_ECC_VALID_DRAM, GSB_ECC_VALID_REMAP, \
    GSB_ECC_VALID_HISTOGRAM = 1, 2, 4, 8, 16, 32
GSB_ECC_REMAP_PENDING, GSB_ECC_REMAP_FAILURE, GSB_ECC_UNCORRECTED = 1, 2, 4
ECC_CONDITION_NAMES = {1: "row remap pending (the GPU needs a reset)", 2: "row remap failure (no spare rows left)",
                       4: "uncorrected ECC error"}
GSB_ABI_VERSION = 4
GSB_FAULT_RECORDS = 64
GSB_FAULT_ZERO, GSB_FAULT_STALE, GSB_FAULT_ALIASED, GSB_FAULT_BITS = 1, 2, 3, 4
FAULT_CLASS_NAMES = {1: "zero", 2: "stale", 3: "aliased", 4: "bits"}
GSB_FAULT_NO_ALIAS = 0xFFFFFFFF
GSB_FAULT_REPORT_FIRST, GSB_FAULT_REPORT_LAST = 0, 1
GSB_ALL_DEVICES = 0xFFFFFFFF
GSB_OPT_INVENTORY_POLICY, GSB_OPT_WAIT_SPIN_US, GSB_OPT_WATCHDOG_MS, GSB_OPT_INVENTORY_REFRESH_MS, \
    GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, GSB_OPT_SWEEP_EVERY_CYCLES, GSB_OPT_ECC_HEALTH, GSB_OPT_LINK_PROBE_EVERY_CYCLES, \
    GSB_OPT_COPY_PROBE_EVERY_CYCLES, GSB_OPT_SM_PROBE_EVERY_CYCLES, GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, \
    GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, GSB_OPT_SFU_PROBE_EVERY_CYCLES, \
    GSB_OPT_L1_PROBE_EVERY_CYCLES, GSB_OPT_ORDER_PROBE_EVERY_CYCLES, GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, \
    GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18
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
    "gsb_ecc_status_get", "gsb_ecc_stats_get", "gsb_ecc_conditions", "gsb_ecc_status_text", "gsb_test_ecc_override",
    "gsb_memtest", "gsb_memtest_text", "gsb_test_march_probe",
    "gsb_link_probe", "gsb_link_status_get", "gsb_link_stats_get", "gsb_link_conditions", "gsb_link_rate_gbps",
    "gsb_link_text", "gsb_test_link_override", "gsb_test_link_corrupt",
    "gsb_copy_probe", "gsb_copy_stats_get", "gsb_copy_conditions", "gsb_copy_text", "gsb_test_copy_corrupt",
    "gsb_test_copy_skip",
    "gsb_sm_probe", "gsb_sm_stats_get", "gsb_sm_expected", "gsb_sm_conditions", "gsb_sm_text", "gsb_test_sm_corrupt",
    "gsb_test_sm_operands",
    "gsb_sm_stress", "gsb_stress_fold", "gsb_stress_conditions", "gsb_stress_text", "gsb_test_stress_corrupt",
    "gsb_cluster_probe", "gsb_cluster_stats_get", "gsb_cluster_conditions", "gsb_cluster_classify", "gsb_cluster_text",
    "gsb_test_cluster_corrupt", "gsb_test_cluster_skip", "gsb_test_cluster_script",
    "gsb_atomic_probe", "gsb_atomic_stats_get", "gsb_atomic_expected", "gsb_atomic_conditions", "gsb_atomic_text",
    "gsb_test_atomic_corrupt", "gsb_test_atomic_skip", "gsb_test_atomic_values",
    "gsb_tensor_probe", "gsb_tensor_stats_get", "gsb_tensor_expected", "gsb_tensor_conditions", "gsb_tensor_text",
    "gsb_test_tensor_corrupt", "gsb_test_tensor_operands",
    "gsb_sfu_probe", "gsb_sfu_stats_get", "gsb_sfu_expected", "gsb_sfu_model", "gsb_sfu_vote", "gsb_sfu_conditions",
    "gsb_sfu_text", "gsb_test_sfu_corrupt", "gsb_test_sfu_inputs",
    "gsb_l1_probe", "gsb_l1_stats_get", "gsb_l1_schedule", "gsb_l1_conditions", "gsb_l1_text", "gsb_test_l1_corrupt",
    "gsb_test_l1_skip", "gsb_test_l1_table",
    "gsb_order_probe", "gsb_order_stats_get", "gsb_order_distance", "gsb_order_iriw_distance", "gsb_order_pairing",
    "gsb_order_classify", "gsb_order_conditions", "gsb_order_text", "gsb_test_order_inject", "gsb_test_order_skip",
    "gsb_sparse_probe", "gsb_sparse_stats_get", "gsb_sparse_expected", "gsb_sparse_conditions", "gsb_sparse_text",
    "gsb_test_sparse_corrupt", "gsb_test_sparse_operands",
    "gsb_shared_atomic_probe", "gsb_shared_atomic_stats_get", "gsb_shared_atomic_expected",
    "gsb_shared_atomic_conditions", "gsb_shared_atomic_text", "gsb_test_shared_atomic_corrupt",
    "gsb_test_shared_atomic_skip",
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


class EccStatus(C.Structure):
    _fields_ = [
        ("valid", C.c_uint32),
        ("mode_current", C.c_uint32),
        ("mode_pending", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("unix_ns", C.c_uint64),
        ("corrected_volatile", C.c_uint64),
        ("uncorrected_volatile", C.c_uint64),
        ("corrected_aggregate", C.c_uint64),
        ("uncorrected_aggregate", C.c_uint64),
        ("dram_corrected_volatile", C.c_uint64),
        ("dram_uncorrected_volatile", C.c_uint64),
        ("remapped_correctable", C.c_uint32),
        ("remapped_uncorrectable", C.c_uint32),
        ("remap_pending", C.c_uint32),
        ("remap_failure", C.c_uint32),
        ("hist_max", C.c_uint32),
        ("hist_high", C.c_uint32),
        ("hist_partial", C.c_uint32),
        ("hist_low", C.c_uint32),
        ("hist_none", C.c_uint32),
        ("reserved1", C.c_uint32),
    ]


class EccStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("cycles", "queries", "corrected_in_walks", "uncorrected_in_walks",
                                          "corrected_between_walks", "bytes_walked", "last_corrected",
                                          "last_window_offset", "last_window_bytes", "first_corrected_volatile",
                                          "latest_corrected_volatile")]


class MemtestCfg(C.Structure):
    _fields_ = [
        ("window_offset", C.c_uint64),
        ("window_bytes", C.c_uint64),
        ("first_element", C.c_uint32),
        ("n_elements", C.c_uint32),
    ]


class MemtestElement(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("element", C.c_uint32),
        ("op", C.c_uint32),
        ("descending", C.c_uint32),
        ("expected", C.c_uint32),
        ("written", C.c_uint32),
        ("bytes_read", C.c_uint64),
        ("bytes_written", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("first_bad_offset", C.c_uint64),
        ("kernel_ns", C.c_uint64),
        ("ecc_valid", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("ecc_corrected", C.c_uint64),
        ("ecc_uncorrected", C.c_uint64),
    ]


class MemtestResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("transient", C.c_uint32),
        ("window_offset", C.c_uint64),
        ("window_bytes", C.c_uint64),
        ("wall_ns", C.c_uint64),
        ("n_elements", C.c_uint32),
        ("refilled", C.c_uint32),
        ("elements", MemtestElement * GSB_MEMTEST_ELEMENTS),
    ]


class LinkStatus(C.Structure):
    _fields_ = [
        ("valid", C.c_uint32),
        ("cur_gen", C.c_uint32),
        ("cur_width", C.c_uint32),
        ("max_gen", C.c_uint32),
        ("max_width", C.c_uint32),
        ("gpu_max_gen", C.c_uint32),
        ("replay_counter", C.c_uint64),
        ("unix_ns", C.c_uint64),
    ]


class LinkCfg(C.Structure):
    _fields_ = [
        ("buffer_bytes", C.c_uint64),
        ("passes", C.c_uint32),
        ("seed_a", C.c_uint32),
        ("seed_b", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class LinkPhase(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("op", C.c_uint32),
        ("bytes_read", C.c_uint64),
        ("bytes_written", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("first_bad_offset", C.c_uint64),
        ("checksum_xor", C.c_uint32),
        ("checksum_sum", C.c_uint32),
        ("kernel_ns", C.c_uint64),
    ]


class LinkResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("passes", C.c_uint32),
        ("buffer_bytes", C.c_uint64),
        ("seed_a", C.c_uint32),
        ("seed_b", C.c_uint32),
        ("idle", LinkStatus),
        ("load_valid", C.c_uint32),
        ("load_gen", C.c_uint32),
        ("load_width", C.c_uint32),
        ("polls", C.c_uint32),
        ("replay_valid", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("replays", C.c_uint64),
        ("phases", LinkPhase * GSB_LINK_PHASES),
        ("up_gbps", C.c_double),
        ("down_gbps", C.c_double),
        ("duplex_up_gbps", C.c_double),
        ("duplex_down_gbps", C.c_double),
        ("link_gbps", C.c_double),
        ("wall_ns", C.c_uint64),
    ]


class LinkStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("queries", C.c_uint64),
        ("replays", C.c_uint64),
        ("skipped", C.c_uint64),
        ("last", LinkResult),
    ]


class CopyCfg(C.Structure):
    _fields_ = [
        ("buffer_bytes", C.c_uint64),
        ("src_offset", C.c_uint64),
        ("dst_offset", C.c_uint64),
        ("copy_bytes", C.c_uint64),
        ("seed_src", C.c_uint32),
        ("seed_host", C.c_uint32),
        ("seed_bg", C.c_uint32),
        ("flags", C.c_uint32),
    ]


class CopyDirection(C.Structure):
    _fields_ = [
        ("op", C.c_uint32),
        ("copied", C.c_uint32),
        ("copy_status", C.c_int32),
        ("verify_status", C.c_int32),
        ("bytes", C.c_uint64),
        ("copy_ns", C.c_uint64),
        ("gbps", C.c_double),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("first_bad_offset", C.c_uint64),
        ("checksum_xor", C.c_uint32),
        ("checksum_sum", C.c_uint32),
        ("kernel_ns", C.c_uint64),
    ]


class CopyResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("async_engines", C.c_uint32),
        ("buffer_bytes", C.c_uint64),
        ("src_offset", C.c_uint64),
        ("dst_offset", C.c_uint64),
        ("copy_bytes", C.c_uint64),
        ("seed_src", C.c_uint32),
        ("seed_host", C.c_uint32),
        ("seed_bg", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("dirs", CopyDirection * GSB_COPY_DIRECTIONS),
        ("wall_ns", C.c_uint64),
    ]


class CopyStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("reserved0", C.c_uint64),
        ("last", CopyResult),
    ]


class SmCfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class SmRecord(C.Structure):
    _fields_ = [
        ("smid", C.c_uint32),
        ("unit", C.c_uint32),
        ("index", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("expected", C.c_uint64),
        ("observed", C.c_uint64),
    ]


class SmUnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class SmResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", SmUnitResult * GSB_SM_UNITS),
        ("n_records", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("records", SmRecord * GSB_SM_RECORDS),
        ("expected_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class SmStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", SmResult),
    ]


class StressCfg(C.Structure):
    _fields_ = [
        ("duration_ms", C.c_uint32),
        ("units", C.c_uint32),
        ("slice_ms", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class StressRecord(C.Structure):
    _fields_ = [
        ("smid", C.c_uint32),
        ("unit", C.c_uint32),
        ("index", C.c_uint32),
        ("slice", C.c_uint32),
        ("expected", C.c_uint64),
        ("observed", C.c_uint64),
    ]


class StressUnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("slices", C.c_uint32),
        ("sets", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("iterations", C.c_uint64),
        ("set_iterations", C.c_uint64 * GSB_STRESS_SETS_MAX),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
        ("tera_ops", C.c_double),
    ]


class StressTelemetry(C.Structure):
    _fields_ = [
        ("valid", C.c_uint32),
        ("samples", C.c_uint32),
        ("power_mean_w", C.c_double),
        ("power_peak_w", C.c_double),
        ("power_limit_w", C.c_double),
        ("temp_peak_c", C.c_uint32),
        ("sm_clock_min_mhz", C.c_uint32),
        ("sm_clock_max_mhz", C.c_uint32),
        ("slowdown_samples", C.c_uint32),
        ("reasons", C.c_uint64),
    ]


class StressResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("duration_ms", C.c_uint32),
        ("slice_ms", C.c_uint32),
        ("slices", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("sm_iterations_min_smid", C.c_uint32),
        ("sm_iterations_min", C.c_uint64),
        ("sm_iterations_max", C.c_uint64),
        ("first_mismatch_slice", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("first_mismatch_ms", C.c_uint64),
        ("unit", StressUnitResult * GSB_STRESS_UNITS),
        ("telemetry", StressTelemetry),
        ("n_records", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("records", StressRecord * GSB_SM_RECORDS),
        ("wall_ns", C.c_uint64),
        ("gap_ns", C.c_uint64),
        ("expected_ns", C.c_uint64),
    ]


class ClusterCfg(C.Structure):
    _fields_ = [
        ("paths", C.c_uint32),
        ("sizes", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
    ]


class ClusterRecord(C.Structure):
    _fields_ = [
        ("path", C.c_uint32),
        ("n", C.c_uint32),
        ("src_rank", C.c_uint32),
        ("dst_rank", C.c_uint32),
        ("src_smid", C.c_uint32),
        ("dst_smid", C.c_uint32),
        ("index", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("expected", C.c_uint32 * 4),
        ("observed", C.c_uint32 * 4),
    ]


class ClusterRun(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("timeouts", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class ClusterResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("paths", C.c_uint32),
        ("sizes", C.c_uint32),
        ("smem_bytes", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("max_clusters", C.c_uint32 * GSB_CLUSTER_SIZES),
        ("expect_covered", C.c_uint32 * GSB_CLUSTER_SIZES),
        ("covered", C.c_uint32 * (GSB_CLUSTER_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_CLUSTER_SM_MAX // 32)),
        ("run", (ClusterRun * GSB_CLUSTER_SIZES) * GSB_CLUSTER_PATHS),
        ("n_records", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("records", ClusterRecord * GSB_CLUSTER_RECORDS),
        ("wall_ns", C.c_uint64),
    ]


class ClusterClass(C.Structure):
    _fields_ = [
        ("cls", C.c_uint32),
        ("src_rank", C.c_uint32),
        ("dst_rank", C.c_uint32),
        ("index", C.c_uint32),
        ("flipped_bits", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class ClusterStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", ClusterResult),
    ]


class AtomicCfg(C.Structure):
    _fields_ = [
        ("ops", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class AtomicRecord(C.Structure):
    _fields_ = [
        ("op", C.c_uint32),
        ("phase", C.c_uint32),
        ("word", C.c_uint32),
        ("smid", C.c_uint32),
        ("expected", C.c_uint64),
        ("observed", C.c_uint64),
    ]


class AtomicRun(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("hook_cta", C.c_uint32),
        ("atomics_issued", C.c_uint64),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("ticket_faults", C.c_uint64),
        ("cas_timeouts", C.c_uint64),
        ("cas_max_ns", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class AtomicResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("ops", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_ATOMIC_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_ATOMIC_SM_MAX // 32)),
        ("run", AtomicRun * GSB_ATOMIC_OPS),
        ("n_records", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("records", AtomicRecord * GSB_ATOMIC_RECORDS),
        ("expected_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class AtomicStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", AtomicResult),
    ]


class TensorCfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class TensorUnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class TensorResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", TensorUnitResult * GSB_TENSOR_UNITS),
        ("n_records", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("records", SmRecord * GSB_TENSOR_RECORDS),  # unit: GSB_TENSOR_UNIT_*
        ("expected_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class TensorStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", TensorResult),
    ]


SparseCfg = TensorCfg  # the same four fields


class SparseResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", TensorUnitResult * GSB_SPARSE_UNITS),
        ("n_records", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("records", SmRecord * GSB_SPARSE_RECORDS),  # unit: GSB_SPARSE_UNIT_*
        ("expected_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class SparseStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", SparseResult),
    ]


class SharedAtomicCfg(C.Structure):
    _fields_ = [
        ("units", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class SharedAtomicRecord(C.Structure):
    _fields_ = [
        ("smid", C.c_uint32),
        ("unit", C.c_uint32),
        ("kind", C.c_uint32),  # GSB_SHARED_ATOMIC_REC_*
        ("index", C.c_uint32),
        ("expected", C.c_uint64),
        ("observed", C.c_uint64),
    ]


class SharedAtomicRun(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("hook_cta", C.c_uint32),
        ("cluster_launches", C.c_uint32 * 2),
        ("clusters", C.c_uint32 * 2),
        ("atomics_issued", C.c_uint64),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("ticket_faults", C.c_uint64),
        ("timeouts", C.c_uint64),
        ("cas_max_ns", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class SharedAtomicResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("cluster_n", C.c_uint32 * 2),
        ("run", SharedAtomicRun * GSB_SHARED_ATOMIC_UNITS),
        ("n_records", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("records", SharedAtomicRecord * GSB_SHARED_ATOMIC_RECORDS),
        ("expected_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class SharedAtomicStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", SharedAtomicResult),
    ]


class SfuCfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("reserved0", C.c_uint32),
    ]


class SfuUnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class SfuResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", SfuUnitResult * GSB_SFU_UNITS),
        ("n_records", C.c_uint32),
        ("bound", C.c_uint32),  # bit GSB_SFU_MUFU_*: a voted result outside its envelope
        ("records", SmRecord * GSB_SFU_RECORDS),  # unit: GSB_SFU_UNIT_*
        ("max_err", C.c_double * GSB_SFU_MUFU_OPS),
        ("expected_ns", C.c_uint64),
        ("vote_ns", C.c_uint64),
        ("wall_ns", C.c_uint64),
    ]


class SfuStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", SfuResult),
    ]


class L1Cfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("passes", C.c_uint32),
    ]


class L1Record(C.Structure):
    _fields_ = [
        ("smid", C.c_uint32),
        ("unit", C.c_uint32),
        ("form", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("offset", C.c_uint64),
        ("expected", C.c_uint32 * 4),
        ("observed", C.c_uint32 * 4),
        ("cls", C.c_uint32),
        ("alias_bit", C.c_uint32),
        ("seed_key", C.c_uint32),
        ("flipped_bits", C.c_uint32),
    ]


class L1UnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("ctas_per_sm", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class L1Result(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("passes", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("n_records", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", L1UnitResult * GSB_L1_UNITS),
        ("warm_cold", C.c_double * GSB_L1_FORMS),  # by GSB_L1_FORM_*
        ("records", L1Record * GSB_L1_RECORDS),
        ("wall_ns", C.c_uint64),
    ]


class L1Stats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", L1Result),
    ]


class OrderCfg(C.Structure):
    _fields_ = [
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("observations", C.c_uint32),
    ]


class OrderRecord(C.Structure):
    _fields_ = [
        ("unit", C.c_uint32),
        ("distance", C.c_uint32),
        ("cls", C.c_uint32),
        ("smid", C.c_uint32),
        ("producer", C.c_uint32 * 3),
        ("index", C.c_uint32),
        ("words", C.c_uint64 * GSB_ORDER_WORDS),
    ]


class OrderUnitResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("launches", C.c_uint32),
        ("refused", C.c_uint32),
        ("sms_covered", C.c_uint32),
        ("words_checked", C.c_uint64),
        ("mismatch_words", C.c_uint64),
        ("mismatch_bits", C.c_uint64),
        ("corrupt", C.c_uint64),
        ("forbidden", C.c_uint64),
        ("lost", C.c_uint64),
        ("timeout", C.c_uint64),
        ("overlap", C.c_uint64),
        ("weak", C.c_uint64),
        ("kernel_ns", C.c_uint64),
    ]


class OrderResult(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("sm_count", C.c_uint32),
        ("seed", C.c_uint32),
        ("seed_expect", C.c_uint32),
        ("units", C.c_uint32),
        ("observations", C.c_uint32),
        ("distance", C.c_uint32 * GSB_ORDER_DISTANCES),
        ("sms_covered", C.c_uint32),
        ("n_records", C.c_uint32),
        ("covered", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("faulty", C.c_uint32 * (GSB_SM_MAX // 32)),
        ("unit", OrderUnitResult * GSB_ORDER_UNITS),
        ("records", OrderRecord * GSB_ORDER_RECORDS),
        ("wall_ns", C.c_uint64),
    ]


class OrderStats(C.Structure):
    _fields_ = [
        ("probes", C.c_uint64),
        ("faults", C.c_uint64),
        ("skipped", C.c_uint64),
        ("incomplete", C.c_uint64),
        ("last", OrderResult),
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
    i32p = C.POINTER(C.c_int32)
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
        "gsb_ecc_status_get": (C.c_int, [C.c_uint32, C.POINTER(EccStatus)]),
        "gsb_ecc_stats_get": (C.c_int, [C.c_uint32, C.POINTER(EccStats)]),
        "gsb_ecc_conditions": (C.c_uint32, [C.POINTER(EccStatus), C.POINTER(EccStatus)]),
        "gsb_ecc_status_text": (C.c_int64, [C.POINTER(EccStatus), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_ecc_override": (C.c_int, [C.c_uint32, C.POINTER(EccStatus)]),
        "gsb_memtest": (C.c_int, [C.c_uint32, C.POINTER(MemtestCfg), C.POINTER(MemtestResult)]),
        "gsb_memtest_text": (C.c_int64, [C.POINTER(MemtestResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_march_probe": (C.c_int, [C.c_uint32, C.POINTER(ProbeCfg), C.POINTER(ProbeResult)]),
        "gsb_link_probe": (C.c_int, [C.c_uint32, C.POINTER(LinkCfg), C.POINTER(LinkResult)]),
        "gsb_link_status_get": (C.c_int, [C.c_uint32, C.POINTER(LinkStatus)]),
        "gsb_link_stats_get": (C.c_int, [C.c_uint32, C.POINTER(LinkStats)]),
        "gsb_link_conditions": (C.c_uint32, [C.POINTER(LinkResult)]),
        "gsb_link_rate_gbps": (C.c_double, [C.c_uint32, C.c_uint32]),
        "gsb_link_text": (C.c_int64, [C.POINTER(LinkResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_link_override": (C.c_int, [C.c_uint32, C.POINTER(LinkStatus)]),
        "gsb_test_link_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint64, u32p]),
        "gsb_copy_probe": (C.c_int, [C.c_uint32, C.POINTER(CopyCfg), C.POINTER(CopyResult)]),
        "gsb_copy_stats_get": (C.c_int, [C.c_uint32, C.POINTER(CopyStats)]),
        "gsb_copy_conditions": (C.c_uint32, [C.POINTER(CopyResult)]),
        "gsb_copy_text": (C.c_int64, [C.POINTER(CopyResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_copy_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint64, u32p]),
        "gsb_test_copy_skip": (C.c_int, [C.c_uint32, C.c_uint32]),
        "gsb_sm_probe": (C.c_int, [C.c_uint32, C.POINTER(SmCfg), C.POINTER(SmResult)]),
        "gsb_sm_stats_get": (C.c_int, [C.c_uint32, C.POINTER(SmStats)]),
        "gsb_sm_expected": (C.c_int64, [C.c_uint32, C.c_uint32, u64p, C.c_size_t]),
        "gsb_sm_conditions": (C.c_uint32, [C.POINTER(SmResult)]),
        "gsb_sm_text": (C.c_int64, [C.POINTER(SmResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_sm_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_sm_operands": (C.c_int, [C.c_uint32, C.c_uint32, i32p, i32p, i32p, i32p, u32p]),
        "gsb_sm_stress": (C.c_int, [C.c_uint32, C.POINTER(StressCfg), C.POINTER(StressResult)]),
        "gsb_stress_fold": (C.c_int64, [C.c_uint32, C.c_uint32, u32p, C.c_size_t]),
        "gsb_stress_conditions": (C.c_uint32, [C.POINTER(StressResult)]),
        "gsb_stress_text": (C.c_int64, [C.POINTER(StressResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_stress_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
        "gsb_cluster_probe": (C.c_int, [C.c_uint32, C.POINTER(ClusterCfg), C.POINTER(ClusterResult)]),
        "gsb_cluster_stats_get": (C.c_int, [C.c_uint32, C.POINTER(ClusterStats)]),
        "gsb_cluster_conditions": (C.c_uint32, [C.POINTER(ClusterResult)]),
        "gsb_cluster_classify": (C.c_int, [C.c_uint32, C.c_uint32, C.POINTER(ClusterRecord), C.POINTER(ClusterClass)]),
        "gsb_cluster_text": (C.c_int64, [C.POINTER(ClusterResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_cluster_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_cluster_skip": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32]),
        "gsb_test_cluster_script": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u8p]),
        "gsb_atomic_probe": (C.c_int, [C.c_uint32, C.POINTER(AtomicCfg), C.POINTER(AtomicResult)]),
        "gsb_atomic_stats_get": (C.c_int, [C.c_uint32, C.POINTER(AtomicStats)]),
        "gsb_atomic_expected": (C.c_int64, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
        "gsb_atomic_conditions": (C.c_uint32, [C.POINTER(AtomicResult)]),
        "gsb_atomic_text": (C.c_int64, [C.POINTER(AtomicResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_atomic_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_atomic_skip": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32]),
        "gsb_test_atomic_values": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, u64p, u64p, C.c_size_t, u64p]),
        "gsb_tensor_probe": (C.c_int, [C.c_uint32, C.POINTER(TensorCfg), C.POINTER(TensorResult)]),
        "gsb_tensor_stats_get": (C.c_int, [C.c_uint32, C.POINTER(TensorStats)]),
        "gsb_tensor_expected": (C.c_int64, [C.c_uint32, C.c_uint32, u64p, C.c_size_t]),
        "gsb_tensor_conditions": (C.c_uint32, [C.POINTER(TensorResult)]),
        "gsb_tensor_text": (C.c_int64, [C.POINTER(TensorResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_tensor_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_tensor_operands": (C.c_int, [C.c_uint32, C.c_uint32, i32p, i32p, i32p, i32p, u64p]),
        "gsb_sfu_probe": (C.c_int, [C.c_uint32, C.POINTER(SfuCfg), C.POINTER(SfuResult)]),
        "gsb_sfu_stats_get": (C.c_int, [C.c_uint32, C.POINTER(SfuStats)]),
        "gsb_sfu_expected": (C.c_int64, [C.c_uint32, C.c_uint32, u64p, C.c_size_t]),
        "gsb_sfu_vote": (C.c_int, [C.c_uint32, C.c_uint32, u64p, u32p, u32p, C.POINTER(SfuResult)]),
        "gsb_sfu_conditions": (C.c_uint32, [C.POINTER(SfuResult)]),
        "gsb_sfu_text": (C.c_int64, [C.POINTER(SfuResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_sfu_model": (C.c_int64, [C.c_uint32, C.c_uint32, u64p, u64p, C.c_size_t, u64p]),
        "gsb_test_sfu_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_sfu_inputs": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, u64p, u64p, C.c_size_t, u64p, u32p]),
        "gsb_l1_probe": (C.c_int, [C.c_uint32, C.POINTER(L1Cfg), C.POINTER(L1Result)]),
        "gsb_l1_stats_get": (C.c_int, [C.c_uint32, C.POINTER(L1Stats)]),
        "gsb_l1_schedule": (C.c_int64, [C.c_uint32] * 7),
        "gsb_l1_conditions": (C.c_uint32, [C.POINTER(L1Result)]),
        "gsb_l1_text": (C.c_int64, [C.POINTER(L1Result), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_l1_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_l1_skip": (C.c_int, [C.c_uint32, C.c_uint32]),
        "gsb_test_l1_table": (C.c_int, [C.c_uint32, C.c_uint32, u32p, C.c_size_t, u32p, C.c_size_t, C.c_uint32]),
        "gsb_order_probe": (C.c_int, [C.c_uint32, C.POINTER(OrderCfg), C.POINTER(OrderResult)]),
        "gsb_order_stats_get": (C.c_int, [C.c_uint32, C.POINTER(OrderStats)]),
        "gsb_order_distance": (C.c_uint32, [C.c_uint32] * 3),
        "gsb_order_iriw_distance": (C.c_uint32, [C.c_uint32] * 2),
        "gsb_order_pairing": (C.c_int, [C.c_uint32] * 4 + [u32p]),
        "gsb_order_classify": (C.c_uint32, [C.c_uint32, C.c_uint32, u32p, u64p, C.c_uint32]),
        "gsb_order_conditions": (C.c_uint32, [C.POINTER(OrderResult)]),
        "gsb_order_text": (C.c_int64, [C.POINTER(OrderResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_order_inject": (C.c_int, [C.c_uint32] * 4),
        "gsb_test_order_skip": (C.c_int, [C.c_uint32, C.c_uint32]),
        "gsb_sparse_probe": (C.c_int, [C.c_uint32, C.POINTER(SparseCfg), C.POINTER(SparseResult)]),
        "gsb_sparse_stats_get": (C.c_int, [C.c_uint32, C.POINTER(SparseStats)]),
        "gsb_sparse_expected": (C.c_int64, [C.c_uint32, C.c_uint32, u32p, C.c_size_t]),
        "gsb_sparse_conditions": (C.c_uint32, [C.POINTER(SparseResult)]),
        "gsb_sparse_text": (C.c_int64, [C.POINTER(SparseResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_sparse_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_sparse_operands": (C.c_int, [C.c_uint32, C.c_uint32, i32p, u8p, i32p, i32p, i32p, u64p]),
        "gsb_shared_atomic_probe": (C.c_int, [C.c_uint32, C.POINTER(SharedAtomicCfg), C.POINTER(SharedAtomicResult)]),
        "gsb_shared_atomic_stats_get": (C.c_int, [C.c_uint32, C.POINTER(SharedAtomicStats)]),
        "gsb_shared_atomic_expected": (C.c_int64, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u32p, C.c_size_t]),
        "gsb_shared_atomic_conditions": (C.c_uint32, [C.POINTER(SharedAtomicResult)]),
        "gsb_shared_atomic_text": (C.c_int64, [C.POINTER(SharedAtomicResult), C.c_char_p, C.c_char_p, C.c_size_t]),
        "gsb_test_shared_atomic_corrupt": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64]),
        "gsb_test_shared_atomic_skip": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32]),
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
