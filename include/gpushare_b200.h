/*
 * gpushare_b200.h — C ABI of libgpushare_b200.so.
 *
 * This is the inner drop-in boundary of SURVEY.md §8(b): every entry point replaces one or
 * more `nvml.*` call sites of the reference's inventory + health path (all citations are
 * relative to the reference tree):
 *
 *   pkg/gpu/nvidia/gpumanager.go:36,41      nvml.Init / nvml.Shutdown      -> gsb_init / gsb_shutdown
 *   pkg/gpu/nvidia/nvidia.go:47-51,54       nvml.GetDeviceCount            -> gsb_device_count
 *   pkg/gpu/nvidia/nvidia.go:60-71          nvml.NewDevice (UUID/Path/Mem) -> gsb_device_info_get
 *   pkg/gpu/nvidia/nvidia.go:34-45          setGPUMemory / getGPUMemory    -> gsb_slices
 *   pkg/gpu/nvidia/nvidia.go:26-32          generate/extract fake IDs      -> gsb_fake_device_id / gsb_real_device_id
 *   pkg/gpu/nvidia/nvidia.go:100-152        watchXIDs (NewEventSet, RegisterEventForDevice,
 *                                           WaitForEvent, DeleteEventSet)  -> gsb_health_* + gsb_probe*
 *   pkg/gpu/nvidia/server.go:172-185 + vendor/.../v1beta1/api.pb.go:794-843 (gogo MarshalTo)
 *                                                                          -> gsb_encode_list_and_watch
 *   pkg/gpu/nvidia/server.go:150-169        RegisterRequest                -> gsb_encode_register_request
 *   pkg/gpu/nvidia/allocate.go:24-198       Allocate / buildErrResponse    -> gsb_allocate
 *
 * Conventions (cgo / ctypes friendly): plain C, no callbacks, caller-allocated outputs,
 * `int` return (0 = GSB_OK, negative = gsb_status), text via gsb_strerror(). All functions are
 * thread-safe after gsb_init() returned GSB_OK; gsb_probe() blocks the calling thread only.
 * Nothing returned through a pointer outlives the call. There is no CPU fallback: with no
 * usable sm_90 device / driver every device entry point fails with a negative status.
 */
#ifndef GPUSHARE_B200_H_
#define GPUSHARE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_ABI_VERSION 4u /* 2: inventory snapshot + options, transient window, watchdog; gsb_cycle_result grew;
                              3: HBM fault reports (gsb_fault_*);
                              4: ECC and row-remapper health (gsb_ecc_*, GSB_EVENT_ECC, GSB_OPT_ECC_HEALTH);
                              the March C- memory test (gsb_memtest*, GSB_OP_MARCH_*) was added to 4 without a new
                              number: it only adds, and a client finds it by looking up gsb_memtest; PCIe link
                              health (gsb_link_*, GSB_OP_LINK_*, GSB_EVENT_LINK) likewise, found by gsb_link_probe;
                              copy-engine health (gsb_copy_*, GSB_OP_COPY_*, GSB_EVENT_COPY) likewise, found by
                              gsb_copy_probe; SM compute health (gsb_sm_*, GSB_EVENT_SM) likewise, found by
                              gsb_sm_probe; SM-to-SM health (gsb_cluster_*, GSB_EVENT_CLUSTER) likewise, found by
                              gsb_cluster_probe; L2 atomic health (gsb_atomic_*, GSB_EVENT_ATOMIC) likewise, found
                              by gsb_atomic_probe; tensor-core format health (gsb_tensor_*, GSB_EVENT_TENSOR)
                              likewise, found by gsb_tensor_probe; SM special-function health (gsb_sfu_*,
                              GSB_EVENT_SFU) likewise, found by gsb_sfu_probe; L1 and constant-cache health
                              (gsb_l1_*, GSB_EVENT_L1) likewise, found by gsb_l1_probe; memory-ordering health
                              (gsb_order_*, GSB_EVENT_ORDER) likewise, found by gsb_order_probe; sparse
                              tensor-core health (gsb_sparse_*, GSB_EVENT_SPARSE) likewise, found by
                              gsb_sparse_probe; shared-memory atomic health (gsb_shared_atomic_*,
                              GSB_EVENT_SHARED_ATOMIC) likewise, found by gsb_shared_atomic_probe */

/* = NVML_DEVICE_UUID_BUFFER_SIZE (vendor/.../nvml/nvml.h:1567), used by bindings.go:20 szUUID */
#define GSB_UUID_BUFFER_SIZE 80
#define GSB_BUSID_BUFFER_SIZE 32
#define GSB_MAX_DEVICES 64
/* device-plugin API limit on Device.ID (v1beta1/api.proto:82-85) */
#define GSB_DEVICE_ID_MAX 63

typedef enum gsb_status {
  GSB_OK = 0,
  GSB_ERR_NOT_INITIALIZED = -1,
  GSB_ERR_INVALID_ARGUMENT = -2,
  /* ≙ NVML_ERROR_LIBRARY_NOT_FOUND -> "could not load NVML library" (bindings.go:60-66) */
  GSB_ERR_LIBRARY_NOT_FOUND = -3,
  GSB_ERR_DRIVER = -4,            /* CUDA driver / runtime call failed; see gsb_last_error() */
  GSB_ERR_NVML = -5,              /* NVML call failed; text is "nvml: <nvmlErrorString>" (bindings.go:52-58) */
  GSB_ERR_NO_DEVICE = -6,         /* index out of range / no such UUID ("nvml: device not found", bindings.go:127) */
  GSB_ERR_IDENTITY_MISMATCH = -7, /* CUDA-side and NVML-side identity of one device disagree */
  GSB_ERR_BUFFER_TOO_SMALL = -8,
  GSB_ERR_OUT_OF_MEMORY = -9,
  GSB_ERR_UNSUPPORTED_ARCH = -10, /* device is not compute capability 10.x: no kernel image, no fallback */
  GSB_ERR_TIMEOUT = -11,          /* gsb_health_wait: no event within timeout (≙ NVML_ERROR_TIMEOUT) */
  GSB_ERR_NO_ARENA = -12,         /* gsb_probe before gsb_arena_create */
  GSB_ERR_MALFORMED = -13,        /* protobuf decode failure */
  GSB_ERR_STOPPED = -14           /* health queue closed by gsb_health_stop */
} gsb_status;

/* ---- lifecycle (a1) -------------------------------------------------------------------- */

int gsb_abi_version(void);
/* dlopen libcuda.so.1 + libnvidia-ml.so.1, cuInit, nvmlInit_v2, enumerate devices in PCI-bus
 * (= NVML index) order, cross-check CUDA uuid/bus id against NVML uuid/bus id. Idempotent. */
int gsb_init(void);
int gsb_shutdown(void);
const char *gsb_strerror(int status);
/* thread-local detail of the last failing call on this thread; copies a NUL-terminated string */
int gsb_last_error(char *buf, size_t cap);

/* ---- inventory (a2-a7) ------------------------------------------------------------------ */

typedef struct gsb_device_info {
  char uuid[GSB_UUID_BUFFER_SIZE];     /* "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx" = nvml Device.UUID */
  char bus_id[GSB_BUSID_BUFFER_SIZE];  /* NVML busId form "00000000:1B:00.0" */
  uint32_t index;                      /* NVML index == position in PCI-bus order */
  uint32_t minor;                      /* /dev/nvidia<minor>  (nvidia.go:65) */
  int32_t cuda_ordinal;                /* ordinal the CUDA driver gave this device in this process */
  uint32_t sm_count;
  uint32_t cc_major, cc_minor;
  uint32_t reserved0;
  uint64_t total_bytes;                /* nvmlMemory_t.total (v1 struct, nvml.h:178-183): the reference's source */
  uint64_t total_mib;                  /* total_bytes / (1024*1024)   (bindings.go:346-349) */
  uint64_t free_bytes;                 /* nvmlMemory_t.free at query time */
  uint64_t cuda_total_bytes;           /* cuDeviceTotalMem, informational */
} gsb_device_info;

int gsb_device_count(uint32_t *n);
/* ≙ nvml.NewDevice(idx) at plugin (re)start (server.go:39 -> nvidia.go:60): a LIVE query — UUID, minor and
 * nvmlMemory_t re-read from NVML, identity re-verified against the CUDA driver — nothing served from a cache.
 * It also rewrites the device's inventory snapshot (below). */
int gsb_device_info_get(uint32_t idx, gsb_device_info *out);

/*
 * Inventory snapshot. The reference asks NVML for identity and memory ONCE per plugin (re)start (server.go:39,
 * nvidia.go:53-89) and never again while serving; its steady state is a blocked nvmlEventSetWait. Here gsb_init
 * and every gsb_device_info_get / gsb_inventory_refresh store NVML's answer per device, and the steady-state
 * cycle (gsb_cycle / gsb_cycle_all) reads identity + total from that snapshot, re-validating the identity on every
 * cycle against the CUDA driver (cuDeviceGetUuid: user-mode, no driver-wide lock). nvmlDeviceGetMemoryInfo on a
 * sub-millisecond cadence convoys with every other NVML client of the node (nvidia-smi, dcgm-exporter). While
 * health is running a low-rate refresher (GSB_OPT_INVENTORY_REFRESH_MS) re-asks
 * NVML off the cycle's path and raises GSB_EVENT_INVENTORY if the answer changed.
 */
#define GSB_ALL_DEVICES 0xFFFFFFFFu
int gsb_inventory_refresh(uint32_t idx);  /* idx or GSB_ALL_DEVICES: live NVML query -> snapshot */
/* the snapshot as the cycle sees it (identity re-validated), and how old it is */
int gsb_inventory_snapshot(uint32_t idx, gsb_device_info *out, uint64_t *age_ns);

/* ---- options ------------------------------------------------------------------------------ */
enum {
  GSB_OPT_INVENTORY_POLICY = 1,          /* GSB_INVENTORY_SNAPSHOT (default) | GSB_INVENTORY_LIVE */
  GSB_OPT_WAIT_SPIN_US = 2,              /* completion wait: spin budget before sleeping (default 2000; prober
                                            threads with a period >= 10 ms never spin) */
  GSB_OPT_WATCHDOG_MS = 3,               /* completion watchdog of a probe launch (default 2000, + 1 ns per 10
                                            window bytes); 0 = off (waits for ever) */
  GSB_OPT_INVENTORY_REFRESH_MS = 4,      /* low-rate NVML refresh while health runs (default 5000; 0 = never) */
  GSB_OPT_TRANSIENT_KEEP_FREE_BYTES = 5, /* HBM a transient probe window never takes (default 1 GiB) */
  GSB_OPT_SWEEP_EVERY_CYCLES = 6,        /* prober, devices without a standing arena: every Nth cycle walks ALL the HBM
                                            that is allocatable at that moment (minus the keep-free margin) instead of
                                            one window, then gives it back — SURVEY §7 hard-part 2's "full walk at idle";
                                            0 = never (default) */
  GSB_OPT_ECC_HEALTH = 7,                /* 1 = ECC and row-remapper health while health runs (gsb_ecc_* below); 0 =
                                            off (default): no ECC query is made */
  GSB_OPT_LINK_PROBE_EVERY_CYCLES = 8,   /* N > 0: each prober thread runs gsb_link_probe after its first cycle of a
                                            health session and after every Nth cycle, outside gsb_cycle, and raises
                                            GSB_EVENT_LINK; 0 = off (default): no pinned buffer, no link query */
  GSB_OPT_COPY_PROBE_EVERY_CYCLES = 9,   /* N > 0: each prober thread runs gsb_copy_probe after its first cycle of a
                                            health session and after every Nth cycle, outside gsb_cycle (after the link
                                            probe when both are due), and raises GSB_EVENT_COPY; 0 = off (default): no
                                            stream, no buffer, no allocation */
  GSB_OPT_SM_PROBE_EVERY_CYCLES = 10,    /* N > 0: each prober thread runs gsb_sm_probe after its first cycle of a
                                            health session and after every Nth cycle, outside gsb_cycle (after the link
                                            and copy probes when they are due), and raises GSB_EVENT_SM; 0 = off
                                            (default): no buffer, no launch */
  GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES = 11, /* N > 0: each prober thread runs gsb_cluster_probe after its first cycle of
                                            a health session and after every Nth cycle, outside gsb_cycle (after the
                                            link, copy and SM probes when they are due), and raises GSB_EVENT_CLUSTER;
                                            0 = off (default): no buffer, no launch */
  GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES = 12, /* N > 0: each prober thread runs gsb_atomic_probe after its first cycle of
                                            a health session and after every Nth cycle, outside gsb_cycle (after the
                                            link, copy, SM and SM-to-SM probes when they are due), and raises
                                            GSB_EVENT_ATOMIC; 0 = off (default): no buffer, no launch */
  GSB_OPT_TENSOR_PROBE_EVERY_CYCLES = 13, /* N > 0: each prober thread runs gsb_tensor_probe after its first cycle of
                                            a health session and after every Nth cycle, outside gsb_cycle (after the
                                            link, copy, SM, SM-to-SM and L2 atomic probes when they are due), and
                                            raises GSB_EVENT_TENSOR; 0 = off (default): no buffer, no launch */
  GSB_OPT_SFU_PROBE_EVERY_CYCLES = 14,    /* N > 0: each prober thread runs gsb_sfu_probe after its first cycle of a
                                            health session and after every Nth cycle, outside gsb_cycle (after the
                                            link, copy, SM, SM-to-SM, L2 atomic and tensor-core format probes when
                                            they are due), and raises GSB_EVENT_SFU; 0 = off (default): no buffer, no
                                            launch */
  GSB_OPT_L1_PROBE_EVERY_CYCLES = 15,     /* N > 0: each prober thread runs gsb_l1_probe after its first cycle of a
                                            health session and after every Nth cycle, outside gsb_cycle (after the
                                            link, copy, SM, SM-to-SM, L2 atomic, tensor-core format and SFU probes
                                            when they are due), and raises GSB_EVENT_L1; 0 = off (default): no
                                            buffer, no launch */
  GSB_OPT_ORDER_PROBE_EVERY_CYCLES = 16,  /* N > 0: each prober thread runs gsb_order_probe after its first cycle of
                                            a health session and after every Nth cycle, outside gsb_cycle (after the
                                            link to L1 probes when they are due), and raises GSB_EVENT_ORDER; 0 = off
                                            (default): no buffer, no launch */
  GSB_OPT_SPARSE_PROBE_EVERY_CYCLES = 17, /* N > 0: each prober thread runs gsb_sparse_probe after its first cycle of
                                            a health session and after every Nth cycle, outside gsb_cycle (after the
                                            link to memory-ordering probes when they are due), and raises
                                            GSB_EVENT_SPARSE; 0 = off (default): no buffer, no launch */
  GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES = 18 /* N > 0: each prober thread runs gsb_shared_atomic_probe after its
                                            first cycle of a health session and after every Nth cycle, outside
                                            gsb_cycle (after every other periodic probe that is due), and raises
                                            GSB_EVENT_SHARED_ATOMIC; 0 = off (default): no buffer, no launch */
};
enum {
  GSB_INVENTORY_SNAPSHOT = 0, /* cycle: NVML's (re)start-time answer + per-cycle CUDA-side identity check */
  GSB_INVENTORY_LIVE = 1      /* cycle: fresh NVML UUID/minor/MemoryInfo every cycle (round-1 behaviour) */
};
int gsb_set_option(uint32_t key, uint64_t value);
int gsb_get_option(uint32_t key, uint64_t *value);
/* setGPUMemory (nvidia.go:34-41): unit_gib != 0 -> total_mib / 1024, else total_mib. Pure. */
uint32_t gsb_slices(uint64_t total_mib, int unit_gib);
/* "<uuid>-_-<j>" (nvidia.go:26-28). Returns length written (excluding NUL) or negative status. */
int gsb_fake_device_id(const char *uuid, uint32_t j, char *buf, size_t cap);
/* strings.Split(id, "-_-")[0] (nvidia.go:30-32). Returns length or negative status. */
int gsb_real_device_id(const char *fake_id, char *buf, size_t cap);

/* ---- wire encoders (a7, a9; gogo-identical bytes) ---------------------------------------- */

/*
 * ListAndWatchResponse{devices: for g in [0,n_gpus), j in [0,slices): Device{ID:"<uuid[g]>-_-<j>",
 * health: unhealthy_bits bit (g*slices+j) ? "Unhealthy" : "Healthy"}} — the list getDevices()
 * builds (nvidia.go:73-85) marshalled like api.pb.go:794-843. `unhealthy_bits` may be NULL (all
 * healthy); otherwise it holds ceil(n_gpus*slices/8) bytes, LSB-first. Returns bytes written, or
 * with buf==NULL the size required, or a negative status.
 */
int64_t gsb_encode_list_and_watch(const char *const *uuids, uint32_t n_gpus, uint32_t slices,
                                  const uint8_t *unhealthy_bits, uint8_t *buf, size_t cap);
/* RegisterRequest{version, endpoint, resource_name} (server.go:158-162; api.pb.go:730-792). */
int64_t gsb_encode_register_request(const char *version, const char *endpoint,
                                    const char *resource_name, uint8_t *buf, size_t cap);

/* ---- HBM probe (replaces the passive XID wait with an active walk; SURVEY §8(d)) --------- */

enum {
  GSB_OP_FILL = 1,          /* write pattern(seed_write); traffic = W */
  GSB_OP_VERIFY = 2,        /* read, compare with pattern(seed_expect); traffic = W */
  GSB_OP_VERIFY_REFILL = 3, /* read+compare(seed_expect), write pattern(seed_write); traffic = 2W */
  /* March C- elements (gsb_memtest, and the gsb_test_march_probe hook; gsb_probe refuses them): solid backgrounds,
     see gsb_memtest below */
  GSB_OP_MARCH_FILL = 4,    /* w: store the background; traffic = W */
  GSB_OP_MARCH_VERIFY = 5,  /* r: read, compare with the background; traffic = W */
  GSB_OP_MARCH_RW_UP = 6,   /* ⇑(r, w): tiles in ascending order, each read, compared, then written in place; 2W */
  GSB_OP_MARCH_RW_DOWN = 7  /* ⇓(r, w): the same, tiles in descending order; 2W */
};
enum {
  GSB_VARIANT_AUTO = 0,
  GSB_VARIANT_DIRECT = 1,   /* ld.global.v4 -> registers -> st.global.v4 (control: no staging) */
  GSB_VARIANT_CPASYNC = 2,  /* cp.async 16 B -> shared ring -> ld.shared.v4 -> st.global.v4 */
  GSB_VARIANT_BULK = 3,     /* cp.async.bulk (TMA 1-D) -> shared ring -> ld.shared.v4 / st.shared.v4
                               -> cp.async.bulk shared->global; one ring per CTA, CTA barrier per tile */
  GSB_VARIANT_BULKW = 4,    /* same data path, one private ring + mbarriers per WARP: no CTA barrier */
  GSB_VARIANT_BULKD = 5     /* BULK with a dynamic (atomic-counter) tile scheduler instead of the static stride */
};
enum {
  GSB_PROBE_TIMED = 1u,       /* bracket the launch with CUDA events, fill kernel_ns */
  GSB_PROBE_SEED_TABLE = 2u   /* expected seed per granule from the arena's generation table */
};

typedef struct gsb_probe_cfg {
  uint32_t op;            /* GSB_OP_* */
  uint32_t variant;       /* GSB_VARIANT_* */
  uint64_t window_offset; /* bytes from arena start, multiple of 16 */
  uint64_t window_bytes;  /* multiple of 16; 0 = to the end of the arena */
  uint32_t seed_expect;
  uint32_t seed_write;
  uint32_t grid_ctas;     /* 0 = auto (resident CTAs per SM x SM count) */
  uint32_t flags;         /* GSB_PROBE_* */
} gsb_probe_cfg;

typedef struct gsb_probe_result {
  int32_t status;            /* gsb_status of this device's probe */
  uint32_t variant;          /* variant actually launched */
  uint64_t bytes_walked;     /* window size actually walked */
  uint64_t bytes_read;       /* algorithmic bytes loaded  (0 for FILL) */
  uint64_t bytes_written;    /* algorithmic bytes stored  (0 for VERIFY) */
  uint64_t mismatch_words;   /* 16-byte words with >= 1 differing bit */
  uint64_t mismatch_bits;    /* total differing bits */
  uint64_t first_bad_offset; /* lowest arena byte offset of a mismatching word; UINT64_MAX if none */
  uint32_t checksum_xor;     /* XOR of every 32-bit lane observed (read ops) or written (FILL) */
  uint32_t checksum_sum;     /* wrapping 32-bit sum of the same lanes */
  uint64_t kernel_ns;        /* CUDA-event time of the launch (GSB_PROBE_TIMED), else 0 */
  uint64_t wall_ns;          /* host monotonic time of the whole call */
  uint32_t grid_ctas;
  uint32_t block_threads;
} gsb_probe_result;

/*
 * Arena = the device memory the probe walks: every byte the driver will actually hand out right
 * now (max_bytes == 0), found by mapping physical chunks (cuMemCreate, 2 MiB granularity) into one
 * reserved VA range until the driver refuses; `keep_free_bytes` is left unallocated for tenants.
 * *arena_bytes is the "actually allocatable" figure.
 */
int gsb_arena_create(uint32_t idx, uint64_t max_bytes, uint64_t keep_free_bytes, uint64_t *arena_bytes);
int gsb_arena_destroy(uint32_t idx);
int gsb_arena_bytes(uint32_t idx, uint64_t *arena_bytes);
int gsb_probe(uint32_t idx, const gsb_probe_cfg *cfg, gsb_probe_result *out);
/* Same cfg on n devices concurrently: one host thread, one primary context and one non-blocking
 * stream per device. Returns GSB_OK iff every results[i].status == GSB_OK. */
int gsb_probe_all(uint32_t n, const uint32_t *idxs, const gsb_probe_cfg *cfg, gsb_probe_result *results);
/* test hooks: raw access to arena bytes (fault injection / read-back by the parity tests). The copy runs on the
 * device's probe stream, after every launch before it, and has landed when the call returns; GSB_ERR_TIMEOUT while a
 * wedged launch still holds that stream. */
int gsb_arena_read(uint32_t idx, uint64_t offset, void *dst, uint64_t bytes);
int gsb_arena_write(uint32_t idx, uint64_t offset, const void *src, uint64_t bytes);
/* test hook: enqueue a kernel that keeps the device's probe stream busy for `ms` milliseconds — a stand-in for a
 * wedged GPU, to exercise the completion watchdog */
int gsb_test_stall(uint32_t idx, uint32_t ms);
/* test hook: overwrite the snapshot's total (as if NVML had answered differently at the last (re)start), to exercise the
 * off-path refresher: its next pass must raise GSB_EVENT_INVENTORY / GSB_INVENTORY_TOTAL_CHANGED for this device */
int gsb_test_skew_snapshot(uint32_t idx, uint64_t total_bytes);

/*
 * One inventory + health-probe cycle of one device (the unit of BASELINE.json's metric):
 * identity + total (GSB_OPT_INVENTORY_POLICY: snapshot re-validated on the CUDA side, or a live NVML query)
 * -> slices -> S fake devices -> ListAndWatchResponse bytes into lw_buf -> HBM walk -> verdict.
 *   standing arena (gsb_arena_create was called): VERIFY_REFILL of the arena window that holds slice
 *     (cycle_no mod arena_slices) (window_bytes == 0: the whole arena); traffic 2 * W.
 *   no arena, window_bytes > 0: TRANSIENT window (SURVEY.md §7 hard-part 2) — allocate up to window_bytes
 *     (never the last GSB_OPT_TRANSIENT_KEEP_FREE_BYTES), FILL, VERIFY, free; traffic 2 * W; nothing is held
 *     between cycles. If nothing can be allocated the cycle is inventory-only: rc GSB_OK, healthy unchanged,
 *     probe.status == GSB_ERR_OUT_OF_MEMORY, probe.bytes_walked == 0.
 * A launch that outlives the watchdog returns GSB_ERR_TIMEOUT with healthy == 0.
 */
typedef struct gsb_cycle_result {
  gsb_device_info info;
  uint32_t slices;
  uint32_t healthy;      /* 1 iff this cycle's walk was clean AND no earlier cycle faulted (Unhealthy is sticky,
                            server.go:180) */
  int64_t lw_len;        /* bytes written to lw_buf */
  uint64_t inventory_ns; /* host time of the identity/memory step + encode */
  gsb_probe_result probe;
  uint64_t snapshot_age_ns; /* policy SNAPSHOT: age of NVML's answer the cycle served */
  uint32_t inventory_live;  /* 1 = this cycle queried NVML itself */
  uint32_t transient;       /* 1 = transient window (allocate -> walk -> free) */
} gsb_cycle_result;
int gsb_cycle(uint32_t idx, uint64_t cycle_no, uint64_t window_bytes, int unit_gib, uint32_t variant,
              uint8_t *lw_buf, size_t lw_cap, gsb_cycle_result *out);

/*
 * One NODE cycle: gsb_cycle on every listed device concurrently — one persistent host thread, one
 * primary context and one non-blocking stream per device, no collective (SURVEY.md §8(e)) — then
 * the single host-side join: the per-device lists concatenated in index order into ONE
 * ListAndWatchResponse (what getDevices builds sequentially, nvidia.go:59-86). The slice count of
 * device idxs[0] is applied to every device, as the reference's process-global gpuMemory does
 * (nvidia.go:70-72). results[i] is device idxs[i]'s cycle; returns bytes written to lw_buf or a
 * negative status.
 */
int64_t gsb_cycle_all(uint32_t n, const uint32_t *idxs, uint64_t cycle_no, uint64_t window_bytes, int unit_gib,
                      uint32_t variant, uint8_t *lw_buf, size_t lw_cap, gsb_cycle_result *results);

/* ---- health events (a10, a11) ------------------------------------------------------------ */

enum {
  GSB_EVENT_XID = 8,        /* = nvmlEventTypeXidCriticalError (nvml.h:1082); edata = XID */
  GSB_EVENT_PROBE = 0x100,  /* active probe verdict; edata = GSB_PROBE_FAULT_* */
  GSB_EVENT_INVENTORY = 0x200, /* the low-rate NVML refresh disagrees with the snapshot; edata = GSB_INVENTORY_*_CHANGED */
  GSB_EVENT_ECC = 0x400,       /* GSB_OPT_ECC_HEALTH: an ECC / row-remapper condition; edata = one GSB_ECC_* bit */
  GSB_EVENT_LINK = 0x800,      /* GSB_OPT_LINK_PROBE_EVERY_CYCLES: a PCIe link condition; edata = one GSB_LINK_* bit */
  GSB_EVENT_COPY = 0x1000,     /* GSB_OPT_COPY_PROBE_EVERY_CYCLES: a copy-engine condition; edata = one GSB_COPY_* bit */
  GSB_EVENT_SM = 0x2000,       /* GSB_OPT_SM_PROBE_EVERY_CYCLES: an SM compute condition; edata = one GSB_SM_* bit */
  GSB_EVENT_CLUSTER = 0x4000,  /* GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES: an SM-to-SM condition; edata = one GSB_CLUSTER_* bit */
  GSB_EVENT_ATOMIC = 0x8000,   /* GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES: an L2 atomic condition; edata = one GSB_ATOMIC_* bit */
  GSB_EVENT_TENSOR = 0x10000,  /* GSB_OPT_TENSOR_PROBE_EVERY_CYCLES: a tensor-core format condition; edata = one
                                  GSB_TENSOR_* bit */
  GSB_EVENT_SFU = 0x20000,     /* GSB_OPT_SFU_PROBE_EVERY_CYCLES: an SM special-function condition; edata = one
                                  GSB_SFU_* bit */
  GSB_EVENT_L1 = 0x40000,      /* GSB_OPT_L1_PROBE_EVERY_CYCLES: an L1 or constant-cache condition; edata = one
                                  GSB_L1_* bit */
  GSB_EVENT_ORDER = 0x80000,   /* GSB_OPT_ORDER_PROBE_EVERY_CYCLES: a memory-ordering condition; edata = one
                                  GSB_ORDER_* bit */
  GSB_EVENT_SPARSE = 0x100000, /* GSB_OPT_SPARSE_PROBE_EVERY_CYCLES: a sparse tensor-core condition; edata = one
                                  GSB_SPARSE_* bit */
  GSB_EVENT_SHARED_ATOMIC = 0x200000 /* GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES: a shared-memory atomic condition;
                                        edata = one GSB_SHARED_ATOMIC_* bit */
};
enum { GSB_PROBE_FAULT_MISMATCH = 1, GSB_PROBE_FAULT_LAUNCH = 2, GSB_PROBE_RECOVERED = 3,
       GSB_PROBE_FAULT_WEDGED = 4 /* the launch outlived the completion watchdog */ };
enum { GSB_INVENTORY_IDENTITY_CHANGED = 1, GSB_INVENTORY_TOTAL_CHANGED = 2 };

typedef struct gsb_event {
  char uuid[GSB_UUID_BUFFER_SIZE]; /* empty => applies to all devices (nvidia.go:138-144) */
  uint64_t etype;
  uint64_t edata;
} gsb_event;

/* Start: one NVML event set with XidCriticalError registered once per *GPU* (the reference does
 * it once per fake device, nvidia.go:104-117 — same resulting set) plus, if probe_period_ms > 0, a
 * prober thread per device running gsb_cycle (standing arena if one exists, else transient windows).
 * A registration that fails with anything but NOT_SUPPORTED fails the call with GSB_ERR_NVML and starts
 * nothing (the reference: log.Fatalf, nvidia.go:114-116); NOT_SUPPORTED queues an Unhealthy event for
 * that GPU (nvidia.go:107-112). */
int gsb_health_start(uint32_t probe_period_ms, uint64_t window_bytes);
int gsb_health_stop(void);
/* ≙ nvml.WaitForEvent(set, timeout) (bindings.go:134-146): GSB_OK + event, or GSB_ERR_TIMEOUT. */
int gsb_health_wait(uint32_t timeout_ms, gsb_event *ev);
/* What the prober thread of one device has done since gsb_health_start (counters restart with it). */
typedef struct gsb_health_stats {
  uint64_t cycles;            /* probe cycles run */
  uint64_t sweeps;            /* of which: whole-free-HBM sweeps (GSB_OPT_SWEEP_EVERY_CYCLES) */
  uint64_t skipped;           /* cycles that found nothing allocatable to probe */
  uint64_t faults;            /* cycles whose walk was not clean (mismatch, failed or wedged launch) */
  uint64_t last_bytes_walked; /* of the most recent cycle */
  uint64_t last_kernel_ns;
  uint64_t last_sweep_bytes;  /* bytes the most recent sweep walked = what was actually allocatable then */
  uint64_t last_sweep_ns;     /* host time of that sweep, allocation and release included */
} gsb_health_stats;
int gsb_health_stats_get(uint32_t idx, gsb_health_stats *out);
/* SURVEY.md §8(f) rank 1, optional: after `clean_cycles` consecutive clean probe cycles a GPU that a PROBE
 * verdict had marked unhealthy is reported again with edata = GSB_PROBE_RECOVERED. 0 (default) keeps the
 * reference's behaviour: Unhealthy is sticky (server.go:180 FIXME). XID faults never recover. */
int gsb_health_set_recovery(uint32_t clean_cycles);
/* test hook: enqueue an event as if the driver had delivered it */
int gsb_health_inject(const gsb_event *ev);
/* nvidia.go:134: XIDs 31, 43, 45 are application errors and do not mark the GPU unhealthy. Pure. */
int gsb_xid_is_benign(uint64_t xid);

/* ---- HBM fault reports (not in the reference: the evidence behind a PROBE / MISMATCH verdict) ---- */

/*
 * Every launch that compares (VERIFY, VERIFY_REFILL: gsb_probe, gsb_probe_all, gsb_cycle, gsb_cycle_all, the prober,
 * sweeps) and finds mismatching words leaves a report: a histogram of the flipped bit positions over ALL mismatching
 * words, and up to GSB_FAULT_RECORDS of those words with what was read and what was expected (which ones, when there
 * are more, is unspecified; the exact total is mismatch_words). A clean launch leaves nothing and costs nothing.
 *
 * Because every pattern word depends on its own address and on its generation through bijections (gsb_pattern.h),
 * one observed word tells what went wrong; gsb_fault_classify checks, in this order:
 */
#define GSB_FAULT_RECORDS 64
enum {
  GSB_FAULT_ZERO = 1,    /* the word reads as all zero */
  GSB_FAULT_STALE = 2,   /* an intact pattern word of THIS address under another seed key: a refill never landed */
  GSB_FAULT_ALIASED = 3, /* an intact pattern word of address w ^ 2^k (k = 0..39) under any seed key: the read (or an
                            earlier write) went to another address */
  GSB_FAULT_BITS = 4     /* anything else: bits flipped in the cell */
};
#define GSB_FAULT_NO_ALIAS 0xFFFFFFFFu /* alias_bit of a record that is not ALIASED */
enum { GSB_FAULT_REPORT_FIRST = 0, /* the first HBM fault since the start (or since the prober last reported RECOVERED);
                                      a PCIe link phase's report (GSB_OP_LINK_*) and a copy verify's
                                      (GSB_OP_COPY_*) are only ever LAST */
       GSB_FAULT_REPORT_LAST = 1   /* the most recent faulted launch */ };

typedef struct gsb_fault_record {
  uint64_t offset;       /* arena byte offset of the 16-byte word (a transient window: from the window's start) */
  uint32_t expected[4];  /* lanes 0..3 = bytes 4l..4l+3 of the word */
  uint32_t observed[4];
  uint32_t cls;          /* GSB_FAULT_* */
  uint32_t alias_bit;    /* ALIASED: k; otherwise GSB_FAULT_NO_ALIAS */
  uint32_t seed_key;     /* STALE / ALIASED: the (mixed) seed key the intact word carries; otherwise 0 */
  uint32_t flipped_bits; /* popcount(expected ^ observed) */
} gsb_fault_record;

typedef struct gsb_fault_report {
  uint32_t valid;        /* 0: no such report (yet); every other field is then 0 */
  uint32_t op;           /* GSB_OP_* of the launch */
  uint32_t transient;    /* 1 = a transient window (offsets are relative to its allocation) */
  uint32_t n_records;    /* records[0 .. n_records) are filled, <= GSB_FAULT_RECORDS */
  uint64_t unix_ns;      /* CLOCK_REALTIME when the launch was collected */
  uint64_t window_offset, window_bytes;
  uint64_t mismatch_words, mismatch_bits, first_bad_offset; /* = the launch's gsb_probe_result */
  /* per bit position b = 32 * lane + bit, over every mismatching word of the launch */
  uint64_t flips_0to1[128]; /* expected 0, observed 1 */
  uint64_t flips_1to0[128]; /* expected 1, observed 0 */
  gsb_fault_record records[GSB_FAULT_RECORDS];
} gsb_fault_report;

/* Copy the FIRST or LAST report of device idx; out->valid = 0 when there is none. */
int gsb_fault_report_get(uint32_t idx, uint32_t which, gsb_fault_report *out);
/* Pure: fill cls, alias_bit, seed_key and flipped_bits of *rec from offset, expected and observed. */
int gsb_fault_classify(gsb_fault_record *rec);
/* Pure: the one-line text both daemons log for a report (counts, window, op, first bad offset, 0->1 / 1->0 totals,
 * the up to 8 most-hit bit positions, records per class, unrecorded faults). uuid may be NULL. Returns the line's
 * length (excluding the NUL it also writes), or with buf == NULL the size required (including the NUL), or a
 * negative status. */
int64_t gsb_fault_report_text(const gsb_fault_report *r, const char *uuid, char *buf, size_t cap);

/* ---- ECC and row-remapper health (not in the reference; opt-in: GSB_OPT_ECC_HEALTH) ------------------------------ */

/*
 * HBM3 ECC corrects a weak or flipped cell before the probe kernel loads the word, so the walk's mismatch count never
 * sees that error; NVML's counters do. And the row remapper's state (a remap pending a reset, no spare rows left) is
 * level-triggered: it survives a plugin restart that an XID event does not. gsb_ecc_status_get reads both.
 *
 * A query NVML answers with anything but success (NOT_SUPPORTED, NO_PERMISSION, ...) leaves its group's `valid` bit
 * clear and its fields 0: a cleared bit means "unknown", never "zero".
 */
enum {
  GSB_ECC_VALID_MODE = 1u,            /* mode_current, mode_pending (nvmlDeviceGetEccMode) */
  GSB_ECC_VALID_VOLATILE = 2u,        /* corrected_volatile, uncorrected_volatile (nvmlDeviceGetTotalEccErrors) */
  GSB_ECC_VALID_AGGREGATE = 4u,       /* corrected_aggregate, uncorrected_aggregate (nvmlDeviceGetTotalEccErrors) */
  GSB_ECC_VALID_DRAM = 8u,            /* dram_*_volatile (nvmlDeviceGetMemoryErrorCounter, NVML_MEMORY_LOCATION_DRAM) */
  GSB_ECC_VALID_REMAP = 16u,          /* remapped_*, remap_pending, remap_failure (nvmlDeviceGetRemappedRows) */
  GSB_ECC_VALID_HISTOGRAM = 32u       /* hist_* (nvmlDeviceGetRowRemapperHistogram) */
};
typedef struct gsb_ecc_status {
  uint32_t valid;                     /* GSB_ECC_VALID_* */
  uint32_t mode_current, mode_pending; /* 1 = ECC enabled */
  uint32_t reserved0;
  uint64_t unix_ns;                   /* CLOCK_REALTIME of the query */
  uint64_t corrected_volatile, uncorrected_volatile;   /* since the driver last loaded */
  uint64_t corrected_aggregate, uncorrected_aggregate; /* over the device's lifetime */
  uint64_t dram_corrected_volatile, dram_uncorrected_volatile;
  uint32_t remapped_correctable, remapped_uncorrectable; /* rows remapped for correctable / uncorrectable errors */
  uint32_t remap_pending;             /* 1 = a remap waits for a GPU reset */
  uint32_t remap_failure;             /* 1 = a remap failed: no spare rows left */
  uint32_t hist_max, hist_high, hist_partial, hist_low, hist_none; /* banks by spare rows left */
  uint32_t reserved1;
} gsb_ecc_status;

/* Conditions (gsb_ecc_conditions): each one counts only when its fields are valid in both structs. Corrected errors
 * are never a condition: the row remapper retires rows that keep failing; they are counted (gsb_ecc_stats). */
enum {
  GSB_ECC_REMAP_PENDING = 1u,         /* now: a row remap is pending (the GPU needs a reset) */
  GSB_ECC_REMAP_FAILURE = 2u,         /* now: a row remap failed (no spare rows: replace the GPU) */
  GSB_ECC_UNCORRECTED = 4u            /* now's uncorrected_volatile is above the baseline's */
};

/* What the prober thread of one device has seen since gsb_health_start with GSB_OPT_ECC_HEALTH = 1 (counters restart
 * with it). The prober reads the volatile corrected / uncorrected totals right before and right after each cycle it
 * runs; the difference across a cycle is the walk's, the difference between two cycles everyone else's. */
typedef struct gsb_ecc_stats {
  uint64_t cycles;                    /* prober cycles run with ECC health on */
  uint64_t queries;                   /* ECC reads the health session made for this device: status queries (start,
                                         refresher) and the prober's pre- and post-cycle counter reads */
  uint64_t corrected_in_walks;        /* corrected errors that appeared while a cycle ran */
  uint64_t uncorrected_in_walks;
  uint64_t corrected_between_walks;   /* corrected errors that appeared between two cycles: tenants, the driver */
  uint64_t bytes_walked;              /* Σ bytes the bracketed cycles walked */
  uint64_t last_corrected;            /* corrected count of the most recent walk that had any, with its window: */
  uint64_t last_window_offset;        /*   arena byte offset (a transient window: 0, from its own start) */
  uint64_t last_window_bytes;
  uint64_t first_corrected_volatile;  /* the total at the first pre-cycle read, and at the latest post-cycle read: */
  uint64_t latest_corrected_volatile; /*   in + between = latest - first */
} gsb_ecc_stats;

/* Live query of device idx (up to nine NVML calls; made whatever GSB_OPT_ECC_HEALTH says). */
int gsb_ecc_status_get(uint32_t idx, gsb_ecc_status *out);
int gsb_ecc_stats_get(uint32_t idx, gsb_ecc_stats *out);
/* Pure: GSB_ECC_* bits that hold for `now` against `baseline` (see above). */
uint32_t gsb_ecc_conditions(const gsb_ecc_status *baseline, const gsb_ecc_status *now);
/* Pure: the one-line text both daemons log for a status (ECC mode, volatile / aggregate / DRAM corrected and
 * uncorrected counts, remapped rows, pending, failure; "unknown" where not valid). uuid may be NULL. Returns like
 * gsb_fault_report_text: the line's length, or with buf == NULL the size required (NUL included), or a negative status. */
int64_t gsb_ecc_status_text(const gsb_ecc_status *st, const char *uuid, char *buf, size_t cap);
/* test hook: until called again with st == NULL, every ECC query of device idx answers *st (unix_ns set at the query),
 * as if NVML had — drives the ECC events and the attribution without a faulty card */
int gsb_test_ecc_override(uint32_t idx, const gsb_ecc_status *st);

/* ---- March C- memory test (not in the reference; on demand or at daemon start-up) ---------------------------------- */

/*
 * March C- over a window of W bytes, "0" the all-zero 16-byte word and "1" the all-ones word:
 *
 *   element 0 ⇕(w0); 1 ⇑(r0,w1); 2 ⇑(r1,w0); 3 ⇓(r0,w1); 4 ⇓(r1,w0); 5 ⇕(r0)
 *
 * Traffic 10 * W: W for elements 0 and 5, 2 * W for each of 1-4. An (r, w) element reads, compares and writes each
 * tile in place before it moves on. ⇑ and ⇓ hold at tile granularity (32 KiB): tiles are claimed in ascending or
 * descending order, and the words of one tile are in flight together. Each element is one launch under the completion
 * watchdog, and the call holds the device for its whole run (a prober cycle waits).
 *
 *   standing arena: the window [window_offset, +window_bytes) of the arena (window_bytes 0 = to its end). A run that
 *     includes element 5 then rewrites the window with the steady-state pattern (a new generation, recorded in the
 *     generation table, for the granules the window covers completely; the generation already recorded for the
 *     others), so the next gsb_cycle over it is clean. Running a sub-range of elements leaves the background instead.
 *   no arena: a transient window of up to window_bytes (0 = all allocatable HBM minus
 *     GSB_OPT_TRANSIENT_KEEP_FREE_BYTES; window_offset must be 0), freed afterwards.
 *
 * A faulted element leaves a fault report like any comparing launch (op = its GSB_OP_MARCH_*, expected = the solid
 * word); a word still holding the previous element's background shows all 128 bits flipped: that write never landed.
 * Mismatches, a failed or a wedged element mark the device faulted, as a cycle does. With GSB_OPT_ECC_HEALTH = 1 the
 * volatile ECC totals are read before and after each element; with it off no ECC query is made and ecc_valid is 0.
 */
#define GSB_MEMTEST_ELEMENTS 6
typedef struct gsb_memtest_cfg {
  uint64_t window_offset;  /* bytes from arena start, multiple of 16 */
  uint64_t window_bytes;   /* multiple of 16; 0 = see above */
  uint32_t first_element;  /* 0..5 */
  uint32_t n_elements;     /* elements first_element .. first_element + n_elements - 1; 0 = through element 5 */
} gsb_memtest_cfg;

typedef struct gsb_memtest_element {
  int32_t status;            /* gsb_status of this element's launch */
  uint32_t element;          /* 0..5 */
  uint32_t op;               /* GSB_OP_MARCH_* */
  uint32_t descending;       /* 1 = tiles in descending order */
  uint32_t expected;         /* lane value of the background read (0 or 0xFFFFFFFF); 0 when the element reads nothing */
  uint32_t written;          /* lane value of the background written; 0 when the element writes nothing */
  uint64_t bytes_read, bytes_written;
  uint64_t mismatch_words, mismatch_bits;
  uint64_t first_bad_offset; /* arena byte offset (transient: from the window's start); UINT64_MAX if none */
  uint64_t kernel_ns;        /* CUDA-event time of the launch */
  uint32_t ecc_valid;        /* 1 = the two fields below are known */
  uint32_t reserved0;
  uint64_t ecc_corrected, ecc_uncorrected; /* rise of the volatile totals across the element */
} gsb_memtest_element;

typedef struct gsb_memtest_result {
  int32_t status;            /* GSB_OK iff every element ran (mismatches are a result, not an error) */
  uint32_t transient;        /* 1 = a transient window */
  uint64_t window_offset, window_bytes; /* the window actually tested */
  uint64_t wall_ns;          /* host time of the whole call, allocation and refill included */
  uint32_t n_elements;       /* elements[0 .. n_elements) were run */
  uint32_t refilled;         /* 1 = the standing window was rewritten with the steady-state pattern afterwards */
  gsb_memtest_element elements[GSB_MEMTEST_ELEMENTS];
} gsb_memtest_result;

int gsb_memtest(uint32_t idx, const gsb_memtest_cfg *cfg, gsb_memtest_result *out);
/* test hook: one March C- element's kernel (cfg->op a GSB_OP_MARCH_*) launched as gsb_probe launches a probe op, so the
 * parity tests reach it with any window and grid. seed_expect / seed_write are the lane values of the background read
 * and written. GSB_ERR_INVALID_ARGUMENT for any other op and for GSB_PROBE_SEED_TABLE (the generation table records
 * pattern generations, never a solid background). A faulted launch leaves a fault report as any probe does; the device
 * is not marked faulted. */
int gsb_test_march_probe(uint32_t idx, const gsb_probe_cfg *cfg, gsb_probe_result *out);
/* Pure: the one-line text both daemons log for a result (window, mismatching words per element, corrected errors per
 * element or "unknown"). uuid may be NULL. Returns like gsb_fault_report_text: the line's length, or with buf == NULL
 * the size required (NUL included), or a negative status. */
int64_t gsb_memtest_text(const gsb_memtest_result *r, const char *uuid, char *buf, size_t cap);

/* ---- PCIe link health (not in the reference; opt-in: GSB_OPT_LINK_PROBE_EVERY_CYCLES) --------------------------- */

/*
 * The probe pattern carried across the GPU's host link in both directions, and NVML's link readings taken while that
 * traffic flows. gsb_link_probe pins two transient, device-mapped host buffers A and B of buffer_bytes each (one link
 * probe's buffers exist at a time in the process) and runs three launches under the completion watchdog (4 ns per
 * byte moved: a link trained at Gen1 x1 is slow, not wedged), holding the device while it runs:
 *
 *   phase 1  GSB_OP_LINK_UP      the GPU writes pattern(seed_a) into A
 *   phase 2  GSB_OP_LINK_DUPLEX  the GPU reads A back and compares it with pattern(seed_a) while it writes
 *                                pattern(seed_b) into B, `passes` times over in one launch
 *   phase 3  GSB_OP_LINK_DOWN    the GPU reads B back and compares it with pattern(seed_b)
 *
 * So what was checked is what landed in host DRAM; the CPU never writes or checks probe data. A mismatching word
 * leaves a fault report like an HBM one (op = its GSB_OP_LINK_*, transient = 1, offsets from the buffer's start).
 * The link status is read once at idle before phase 1; during phase 2 the current generation and width are polled
 * until the launch completes, and the highest of each is kept (an idle GPU may train its link down to save power).
 * Bandwidth is reported, never judged: tenants share the link.
 */
enum {
  GSB_OP_LINK_UP = 8,     /* GPU -> host: store pattern(seed_write); traffic = W */
  GSB_OP_LINK_DOWN = 9,   /* host -> GPU: load, compare with pattern(seed_expect); traffic = W */
  GSB_OP_LINK_DUPLEX = 10 /* both at once, on separate CTAs; traffic = passes * W each way */
};
/* A link phase's fault report becomes the device's LAST report, never its FIRST, which stays the first HBM fault. */
enum {
  GSB_LINK_VALID_CUR_GEN = 1u,     /* cur_gen (nvmlDeviceGetCurrPcieLinkGeneration) */
  GSB_LINK_VALID_CUR_WIDTH = 2u,   /* cur_width (nvmlDeviceGetCurrPcieLinkWidth) */
  GSB_LINK_VALID_MAX_GEN = 4u,     /* max_gen (nvmlDeviceGetMaxPcieLinkGeneration: the GPU and the system) */
  GSB_LINK_VALID_MAX_WIDTH = 8u,   /* max_width (nvmlDeviceGetMaxPcieLinkWidth) */
  GSB_LINK_VALID_GPU_MAX_GEN = 16u, /* gpu_max_gen (nvmlDeviceGetGpuMaxPcieLinkGeneration: the GPU alone) */
  GSB_LINK_VALID_REPLAY = 32u      /* replay_counter (nvmlDeviceGetPcieReplayCounter) */
};
typedef struct gsb_link_status {
  uint32_t valid;                  /* GSB_LINK_VALID_*: a clear bit means "unknown", never "zero" */
  uint32_t cur_gen, cur_width;
  uint32_t max_gen, max_width;     /* below gpu_max_gen: the system limits the link, not a fault */
  uint32_t gpu_max_gen;
  uint64_t replay_counter;         /* TLP replays since the driver loaded */
  uint64_t unix_ns;                /* CLOCK_REALTIME of the query */
} gsb_link_status;

typedef struct gsb_link_cfg {
  uint64_t buffer_bytes;  /* each of A and B; multiple of 16; 0 = 32 MiB */
  uint32_t passes;        /* phase 2 repetitions; 0 = 8 */
  uint32_t seed_a, seed_b; /* raw seeds of A and B; 0 = the library picks a fresh pair */
  uint32_t reserved0;
} gsb_link_cfg;

typedef struct gsb_link_phase {
  int32_t status;            /* gsb_status of this phase's launch */
  uint32_t op;               /* GSB_OP_LINK_* */
  uint64_t bytes_read;       /* host -> GPU */
  uint64_t bytes_written;    /* GPU -> host */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t first_bad_offset; /* byte offset from the read buffer's start; UINT64_MAX if none */
  uint32_t checksum_xor;     /* XOR / wrapping sum of every lane read and written */
  uint32_t checksum_sum;
  uint64_t kernel_ns;        /* CUDA-event time of the launch */
} gsb_link_phase;

#define GSB_LINK_PHASES 3
typedef struct gsb_link_result {
  int32_t status;              /* GSB_OK iff every phase ran (mismatches are a result, not an error) */
  uint32_t passes;
  uint64_t buffer_bytes;
  uint32_t seed_a, seed_b;
  gsb_link_status idle;        /* before phase 1 */
  uint32_t load_valid;         /* GSB_LINK_VALID_CUR_GEN / _CUR_WIDTH: a poll during phase 2 answered */
  uint32_t load_gen, load_width; /* the highest generation and width seen during phase 2 */
  uint32_t polls;              /* status polls made during phase 2 */
  uint32_t replay_valid;       /* 1 = replays is known (read before phase 1 and after phase 3) */
  uint32_t reserved0;
  uint64_t replays;            /* rise of the replay counter across the probe */
  gsb_link_phase phases[GSB_LINK_PHASES];
  double up_gbps;              /* phase 1: GB/s GPU -> host, alone */
  double down_gbps;            /* phase 3: GB/s host -> GPU, alone */
  double duplex_up_gbps, duplex_down_gbps; /* phase 2, each direction while the other runs */
  double link_gbps;            /* theoretical rate per direction of load_gen x load_width (gsb_link_rate_gbps) */
  uint64_t wall_ns;            /* host time of the whole call, pinning and freeing included */
} gsb_link_result;

/* Conditions (gsb_link_conditions), from the phases that ran only: a probe that ran none (its status says why, e.g.
 * GSB_ERR_OUT_OF_MEMORY when the host buffers could not be pinned) raises none. A replay-counter rise is counted
 * (gsb_link_stats) and logged, never a condition. */
enum {
  GSB_LINK_CORRUPT = 1u,         /* a phase read a word that is not what the GPU wrote */
  GSB_LINK_FAILED = 2u,          /* a phase failed or outlived the watchdog */
  GSB_LINK_WIDTH_DEGRADED = 4u,  /* load_width < idle.max_width (both known) */
  GSB_LINK_SPEED_DEGRADED = 8u   /* load_gen < idle.max_gen (both known) */
};

/* Link probes of one device since gsb_health_start (counters restart with it; gsb_link_probe calls count too). */
typedef struct gsb_link_stats {
  uint64_t probes;   /* link probes run */
  uint64_t faults;   /* of which raised at least one GSB_LINK_* condition */
  uint64_t queries;  /* NVML link query rounds made (idle reads, polls, replay reads, gsb_link_status_get) */
  uint64_t replays;  /* Σ replays over the probes where it was known */
  uint64_t skipped;  /* probes that ran no phase (the host buffers could not be pinned): no condition, no event */
  gsb_link_result last;
} gsb_link_stats;

int gsb_link_probe(uint32_t idx, const gsb_link_cfg *cfg, gsb_link_result *out);
/* Live query of device idx (up to six NVML calls; made whatever the option says). */
int gsb_link_status_get(uint32_t idx, gsb_link_status *out);
int gsb_link_stats_get(uint32_t idx, gsb_link_stats *out);
/* Pure: GSB_LINK_* bits that hold for a result (see above). */
uint32_t gsb_link_conditions(const gsb_link_result *now);
/* Pure: GB/s per direction of a link at generation gen (2.5 / 5 GT/s with 8b/10b, 8 / 16 / 32 GT/s with 128b/130b)
 * and `width` lanes; 0 for an unknown generation. */
double gsb_link_rate_gbps(uint32_t gen, uint32_t width);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_fault_report_text: the
 * line's length, or with buf == NULL the size required (NUL included), or a negative status. */
int64_t gsb_link_text(const gsb_link_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: until called again with st == NULL, every link query of device idx answers *st (unix_ns set at the
 * query), as if NVML had, except that the replay counter advances by one at every query that reads it */
int gsb_test_link_override(uint32_t idx, const gsb_link_status *st);
/* test hook: the next gsb_link_probe of device idx XORs xr into the 16-byte word at `offset` of the buffer that phase
 * `phase` (2: A, 3: B) reads, on the CPU, right before that phase; once. Host memory only. */
int gsb_test_link_corrupt(uint32_t idx, uint32_t phase, uint64_t offset, const uint32_t xr[4]);

/* ---- Copy-engine health (not in the reference; opt-in: GSB_OPT_COPY_PROBE_EVERY_CYCLES) ------------------------- */

/*
 * The probe pattern moved by the GPU's DMA copy engines, the path every cudaMemcpy* a tenant makes takes, and checked
 * on the GPU, every byte of every destination. gsb_copy_probe allocates three transient HBM buffers of buffer_bytes
 * each (source S, destinations D_h2d and D_d2d; never the last GSB_OPT_TRANSIENT_KEEP_FREE_BYTES) and pins two
 * device-mapped host buffers (source H_s, destination H_d; under the same process-wide lock as the link probe's), and
 * holds the device while it runs:
 *
 *   prepare  FILL writes pattern(seed_src) into S, the link kernel's up side pattern(seed_host) into H_s, and every
 *            destination is filled with its own background pattern(seed_bg)
 *   copy     three cudaMemcpyAsync on three streams at once: H2D H_s -> D_h2d, D2H S -> H_d, D2D S -> D_d2d, each of
 *            copy_bytes from src + src_offset to dst + dst_offset, timed with events on its own stream, under the
 *            completion watchdog (4 ns per byte copied)
 *   verify   one launch per destination (GSB_OP_COPY_*) compares every 16-byte word of it with what it must hold:
 *            inside [dst_offset, dst_offset + copy_bytes) the source's bytes, elsewhere its background; a word that
 *            straddles an end is a byte-wise merge of the two. H_d is read through its device mapping.
 *
 * Every pattern is keyed by the word index from its own buffer's start and the seeds are fresh per probe, so a copy
 * that never landed leaves background words (GSB_FAULT_STALE). A mismatching word leaves a fault report (op =
 * GSB_OP_COPY_*, transient = 1, offsets from the destination's start) that becomes the device's LAST report, never its
 * FIRST. Bandwidth is reported, never judged: tenants share the engines. Which engine the driver uses for a direction
 * is the driver's choice; the probe checks the engines it picks.
 */
enum {
  GSB_OP_COPY_H2D = 11, /* verify D_h2d after host -> device; traffic = W (HBM) */
  GSB_OP_COPY_D2H = 12, /* verify H_d after device -> host; traffic = W (host link) */
  GSB_OP_COPY_D2D = 13  /* verify D_d2d after device -> device; traffic = W (HBM) */
};
#define GSB_COPY_DIRECTIONS 3 /* dirs[k] of a result: k = op - GSB_OP_COPY_H2D */
enum { GSB_COPY_GEOMETRY = 1u /* gsb_copy_cfg.flags: src_offset, dst_offset and copy_bytes are used as given */ };

typedef struct gsb_copy_cfg {
  uint64_t buffer_bytes;        /* each of the five buffers; a multiple of 16 below 4 GiB; 0 = 32 MiB */
  /* with GSB_COPY_GEOMETRY any byte offsets and length with src_offset + copy_bytes and dst_offset + copy_bytes
   * <= buffer_bytes (copy_bytes 0 included); without it src_offset = dst_offset = 64 and copy_bytes = buffer_bytes -
   * 128: an aligned copy with a 64-byte guard at each end */
  uint64_t src_offset, dst_offset, copy_bytes;
  uint32_t seed_src, seed_host; /* raw seeds of S and H_s; 0 = fresh */
  uint32_t seed_bg;             /* raw seed of the destinations' background; 0 = fresh */
  uint32_t flags;               /* GSB_COPY_* */
} gsb_copy_cfg;

typedef struct gsb_copy_direction {
  uint32_t op;               /* GSB_OP_COPY_*; 0 = the direction did not run */
  uint32_t copied;           /* 1 = the copy was issued (0 after gsb_test_copy_skip) */
  int32_t copy_status;       /* gsb_status of the copy (GSB_ERR_TIMEOUT: it outlived the watchdog) */
  int32_t verify_status;     /* gsb_status of the verify launch; the copy's when the copy failed (no verify ran) */
  uint64_t bytes;            /* bytes copied */
  uint64_t copy_ns;          /* CUDA-event time of the copy on its own stream */
  double gbps;               /* bytes / copy_ns, while the other directions copy too */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t first_bad_offset; /* byte offset from the destination's start; UINT64_MAX if none */
  uint32_t checksum_xor;     /* XOR / wrapping sum of every lane of the destination as read */
  uint32_t checksum_sum;
  uint64_t kernel_ns;        /* CUDA-event time of the verify launch */
} gsb_copy_direction;

typedef struct gsb_copy_result {
  int32_t status;            /* GSB_OK iff every direction copied and verified (mismatches are a result) */
  uint32_t async_engines;    /* cudaDevAttrAsyncEngineCount (informational) */
  uint64_t buffer_bytes, src_offset, dst_offset, copy_bytes;
  uint32_t seed_src, seed_host, seed_bg;
  uint32_t reserved0;
  gsb_copy_direction dirs[GSB_COPY_DIRECTIONS];
  uint64_t wall_ns;          /* host time of the whole call, allocation and freeing included */
} gsb_copy_result;

/* Conditions (gsb_copy_conditions), from the directions that ran only: a probe that ran none (its status says why,
 * e.g. GSB_ERR_OUT_OF_MEMORY when the HBM could not be allocated or the host buffers pinned) raises none. */
enum {
  GSB_COPY_CORRUPT = 1u, /* a destination byte differs from what the copy must have left, inside the range or out */
  GSB_COPY_FAILED = 2u   /* a copy or a verify failed or outlived the watchdog */
};

/* Copy probes of one device since gsb_health_start (counters restart with it; gsb_copy_probe calls count too). */
typedef struct gsb_copy_stats {
  uint64_t probes;   /* copy probes run */
  uint64_t faults;   /* of which raised at least one GSB_COPY_* condition */
  uint64_t skipped;  /* probes that ran no direction (nothing allocatable or pinnable): no condition, no event */
  uint64_t reserved0;
  gsb_copy_result last;
} gsb_copy_stats;

int gsb_copy_probe(uint32_t idx, const gsb_copy_cfg *cfg, gsb_copy_result *out);
int gsb_copy_stats_get(uint32_t idx, gsb_copy_stats *out);
/* Pure: GSB_COPY_* bits that hold for a result (see above). */
uint32_t gsb_copy_conditions(const gsb_copy_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_fault_report_text: the
 * line's length, or with buf == NULL the size required (NUL included), or a negative status. */
int64_t gsb_copy_text(const gsb_copy_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: the next gsb_copy_probe of device idx XORs xr into the 16-byte word at `offset` of direction op's
 * (GSB_OP_COPY_*) destination after its copy and before its verify; once. The CPU does it for H_d, a 16-byte
 * read-modify-write on the device's stream for an HBM destination. */
int gsb_test_copy_corrupt(uint32_t idx, uint32_t op, uint64_t offset, const uint32_t xr[4]);
/* test hook: the next gsb_copy_probe of device idx does not issue direction op's copy (its destination keeps its
 * background); once */
int gsb_test_copy_skip(uint32_t idx, uint32_t op);

/* ---- SM compute health (not in the reference; opt-in: GSB_OPT_SM_PROBE_EVERY_CYCLES) ----------------------------- */

/*
 * Known-answer checks of what every SM computes: its tensor cores (wgmma), its FMA and integer pipes and its shared
 * memory. Each unit is one launch with one CTA per SM (grid = the SM count, each CTA asking for the opt-in maximum of
 * dynamic shared memory, so no two fit on one SM); every CTA records %smid in a coverage bitmap, and a launch that left
 * an SM uncovered is repeated, up to GSB_SM_MAX_LAUNCHES launches of that unit. Results are compared bit for bit with
 * answers computed exactly on the host (gsb_sm_expected), never with a tolerance and never across SMs:
 *
 *   SMEM   March C- (as gsb_memtest, solid 0 then all-ones) over the CTA's whole dynamic shared memory with 128-bit
 *          accesses, ascending and descending at row granularity (256 threads x 16 B); words are 64-bit
 *   INT32  per thread, a dependent chain of IMAD, IADD3, LOP3, funnel shift, POPC, BREV and PRMT
 *   FP32   per thread, a dependent FFMA chain (IEEE round to nearest, no FTZ; every value normal and finite)
 *   FP64   the same with DFMA
 *   F16, BF16  wgmma m64n128k16, FP32 accumulate, K = 256; E4M3 wgmma m64n128k32, K = 64; S8 wgmma m64n128k32 s32, K = 256
 *
 * A chain thread folds every intermediate result into a 64-bit checksum, and that word is compared; a tensor-core thread
 * compares every register of its D fragment. The operands are generated on the device from (unit, seed, row, col); only
 * the expected answers (at most 32 KiB per unit, the same for every SM) are uploaded, into a transient buffer taken only
 * when GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free. A mismatch never touches the HBM fault log or reports.
 */
enum {
  GSB_SM_UNIT_SMEM = 0,
  GSB_SM_UNIT_INT32 = 1,
  GSB_SM_UNIT_FP32 = 2,
  GSB_SM_UNIT_FP64 = 3,
  GSB_SM_UNIT_F16 = 4,
  GSB_SM_UNIT_BF16 = 5,
  GSB_SM_UNIT_E4M3 = 6,
  GSB_SM_UNIT_S8 = 7
};
#define GSB_SM_UNITS 8
#define GSB_SM_MAX 256          /* %smid values a bitmap holds (%smid need not be contiguous) */
#define GSB_SM_RECORDS 64
#define GSB_SM_MAX_LAUNCHES 3
#define GSB_SM_SMEM_WORDS_MAX 29056u /* 64-bit words of the 227 KiB opt-in maximum: the SMEM indices a hook may name */

typedef struct gsb_sm_cfg {
  uint32_t seed;        /* operands' seed; 0 = fresh per probe */
  uint32_t seed_expect; /* seed of the expected answers; 0 = seed (another value makes every chain and tensor word wrong) */
  uint32_t units;       /* mask of 1 << GSB_SM_UNIT_*; 0 = all */
  uint32_t reserved0;
} gsb_sm_cfg;

typedef struct gsb_sm_record {
  uint32_t smid;
  uint32_t unit;     /* GSB_SM_UNIT_* */
  uint32_t index;    /* chains: thread; tensor units: row * 128 + column of D; SMEM: 64-bit word of shared memory */
  uint32_t reserved0;
  uint64_t expected; /* 32-bit results zero-extended */
  uint64_t observed;
} gsb_sm_record;

typedef struct gsb_sm_unit_result {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = the unit did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t reserved0;
  uint64_t words_checked;  /* result words compared, over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_sm_unit_result;

typedef struct gsb_sm_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs with at least one wrong word */
  gsb_sm_unit_result unit[GSB_SM_UNITS];
  uint32_t n_records;      /* records filled (the first GSB_SM_RECORDS mismatches) */
  uint32_t reserved0;
  gsb_sm_record records[GSB_SM_RECORDS];
  uint64_t expected_ns;    /* host time spent computing the expected answers */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_sm_result;

/* Conditions (gsb_sm_conditions), from the units that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_sm_stats.incomplete) and logged, never a condition: another context, such as a tenant's MPS server, may
 * hold SMs. */
enum {
  GSB_SM_CORRUPT = 1u, /* a result word differs from its exact answer on some SM */
  GSB_SM_FAILED = 2u   /* a launch failed or outlived the watchdog */
};

/* SM probes of one device since gsb_health_start (counters restart with it; gsb_sm_probe calls count too). */
typedef struct gsb_sm_stats {
  uint64_t probes;     /* SM probes run */
  uint64_t faults;     /* of which raised at least one GSB_SM_* condition */
  uint64_t skipped;    /* probes that ran no unit (buffers not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_sm_result last;
} gsb_sm_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffers
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_sm_probe(uint32_t idx, const gsb_sm_cfg *cfg, gsb_sm_result *out);
int gsb_sm_stats_get(uint32_t idx, gsb_sm_stats *out);
/* Pure: the exact answers of `unit` for `seed`, one per result word of a CTA (chains: 256 checksums; tensor units: the
 * 8192 words of D in row-major order, zero-extended; SMEM: none, its answers are the solid backgrounds). Returns the
 * count, or with out == NULL the count required, or a negative status (GSB_ERR_BUFFER_TOO_SMALL when cap is short). */
int64_t gsb_sm_expected(uint32_t unit, uint32_t seed, uint64_t *out, size_t cap);
/* Pure: GSB_SM_* bits that hold for a result (see above). */
uint32_t gsb_sm_conditions(const gsb_sm_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_copy_text. */
int64_t gsb_sm_text(const gsb_sm_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_sm_probe of device idx, the CTA running on SM `smid` XORs xr into its result word `index`
 * of `unit` just before the compare, once (SMEM: into that shared-memory word between March elements 1 and 2). */
int gsb_test_sm_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
/* test hook: the next gsb_sm_probe of device idx that runs tensor unit `unit` runs it on chosen operands instead of the
 * seed's: every launch of the unit in that probe (coverage repeats included) computes D = A B with A[i][k] =
 * a[i * K + k] * 2^sa[i] and B[k][j] = b[k * 128 + j] * 2^sb[j] (K = 256, E4M3 64) through the same conversion, layout,
 * wgmma and fragment compare, and compares D with expected[row * 128 + col] (FP32 bits, S8: S32). Once. a == NULL
 * disarms it. Refused with GSB_ERR_INVALID_ARGUMENT before any device is touched: a unit other than F16, BF16, E4M3
 * and S8, an integer outside what the seeded operands can take ([-amp, amp] of A or B; S8 [-128, 127]), or a scale
 * outside its range (S8: 0). In-range operands keep every D exact in FP32 (S32) whatever order the sums take. */
int gsb_test_sm_operands(uint32_t idx, uint32_t unit, const int32_t *a, const int32_t *b, const int32_t *sa,
                         const int32_t *sb, const uint32_t *expected);

/* ---- SM stress (not in the reference; opt-in: a call, or the daemons' --startup-stress-ms) ----------------------- */

/*
 * Sustained tensor-core load with every result bit checked: the tensor units of gsb_sm_probe (F16, BF16, E4M3, S8),
 * their m64n128 D tiles and their operands, run back to back on every SM for duration_ms. Operand set s is the SM
 * probe's operands at seed + s and its answer is gsb_sm_expected(unit, seed_expect + s); at least two sets stay resident
 * in each CTA's shared memory and consecutive iterations use different ones. One CTA per SM (each asks for the opt-in
 * maximum of shared memory); each CTA runs two consumer warpgroups, and each warpgroup computes D with its accumulators
 * zeroed, then checks it, iteration after iteration. A thread folds its 64 D words (gsb_stress_fold) and compares the
 * fold with the set's expected fold; on a difference it compares each word with the full expected D and records the
 * wrong ones. A mismatch never touches the HBM fault log or reports.
 *
 * The run is cut into slices of at most GSB_STRESS_SLICE_MAX_MS, one launch each, that end on their own at a
 * %globaltimer deadline (backed by an iteration cap), so no launch occupies the GPU for long. Slices run back to back
 * on the device's stream, cycle through the selected units, and each runs under the completion watchdog with a budget
 * of its length plus GSB_OPT_WATCHDOG_MS. The expected answers and the log live in one transient buffer, taken only when
 * GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free. While it waits on a slice the calling thread samples read-only NVML
 * telemetry about every GSB_STRESS_SAMPLE_MS; nothing sets a clock or a power limit, and telemetry is never judged.
 */
#define GSB_STRESS_UNITS 4              /* unit[k] of a result: GSB_SM_UNIT_F16 + k */
#define GSB_STRESS_SETS_MAX 4           /* operand sets a unit keeps resident (F16, BF16: 2; E4M3, S8: 4) */
#define GSB_STRESS_DURATION_MAX_MS 600000u
#define GSB_STRESS_SLICE_MAX_MS 100u
#define GSB_STRESS_SLICE_DEFAULT_MS 50u
#define GSB_STRESS_SAMPLE_MS 25u
#define GSB_STRESS_FOLD_THREADS 128     /* the folds of one set: one per thread of a warpgroup */
#define GSB_STRESS_UNIT_MASK 0xF0u      /* 1 << GSB_SM_UNIT_{F16, BF16, E4M3, S8} */

typedef struct gsb_stress_cfg {
  uint32_t duration_ms;  /* required: 1 .. GSB_STRESS_DURATION_MAX_MS */
  uint32_t units;        /* mask of 1 << GSB_SM_UNIT_{F16, BF16, E4M3, S8}; 0 = all four */
  uint32_t slice_ms;     /* 0 = GSB_STRESS_SLICE_DEFAULT_MS; at most GSB_STRESS_SLICE_MAX_MS */
  uint32_t seed;         /* operands' seed; 0 = fresh per run */
  uint32_t seed_expect;  /* seed of the expected answers; 0 = seed */
  uint32_t reserved0;
} gsb_stress_cfg;

typedef struct gsb_stress_record {
  uint32_t smid;
  uint32_t unit;         /* GSB_SM_UNIT_* */
  uint32_t index;        /* row * 128 + column of D */
  uint32_t slice;        /* the run's slice, from 0 */
  uint64_t expected;     /* 32-bit words zero-extended */
  uint64_t observed;
} gsb_stress_record;

typedef struct gsb_stress_unit_result {
  int32_t status;          /* GSB_OK, or the first failed slice's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t slices;         /* 0 = the unit did not run */
  uint32_t sets;           /* operand sets it rotated through */
  uint32_t reserved0;
  uint64_t iterations;     /* D tiles computed and checked, over every warpgroup of every CTA */
  uint64_t set_iterations[GSB_STRESS_SETS_MAX];
  uint64_t words_checked;  /* = 8192 x iterations when every warpgroup finished its iterations */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its slices */
  double tera_ops;         /* 2 * 64 * 128 * K * iterations / kernel_ns / 1e3: TFLOP/s (TOP/s for S8) */
} gsb_stress_unit_result;

enum {
  GSB_STRESS_VALID_ENERGY = 1u,       /* power_mean_w (nvmlDeviceGetTotalEnergyConsumption before and after) */
  GSB_STRESS_VALID_POWER = 2u,        /* power_peak_w (nvmlDeviceGetPowerUsage) */
  GSB_STRESS_VALID_TEMP = 4u,         /* temp_peak_c (nvmlDeviceGetTemperature, GPU sensor) */
  GSB_STRESS_VALID_SM_CLOCK = 8u,     /* sm_clock_min_mhz, sm_clock_max_mhz (nvmlDeviceGetClockInfo, SM) */
  GSB_STRESS_VALID_REASONS = 16u,     /* reasons, slowdown_samples (nvmlDeviceGetCurrentClocksEventReasons) */
  GSB_STRESS_VALID_POWER_LIMIT = 32u  /* power_limit_w (nvmlDeviceGetEnforcedPowerLimit) */
};
/* HW slowdown, HW thermal slowdown and HW power brake: a sample with any of them counts in slowdown_samples */
#define GSB_STRESS_SLOWDOWN_REASONS 0xC8ull

typedef struct gsb_stress_telemetry {
  uint32_t valid;          /* GSB_STRESS_VALID_*: a clear bit means "unknown", never "zero" */
  uint32_t samples;        /* sampling rounds made (one before the first slice, then every GSB_STRESS_SAMPLE_MS) */
  double power_mean_w;     /* energy delta / the time between the two readings */
  double power_peak_w;
  double power_limit_w;
  uint32_t temp_peak_c;
  uint32_t sm_clock_min_mhz, sm_clock_max_mhz;
  uint32_t slowdown_samples;
  uint64_t reasons;        /* OR of every sample's clocks-event reasons (nvmlClocksEventReason*) */
} gsb_stress_telemetry;

typedef struct gsb_stress_result {
  int32_t status;          /* GSB_OK iff every slice ran (mismatches are a result) */
  uint32_t sm_count;       /* the grid of every slice */
  uint32_t seed, seed_expect, units, duration_ms, slice_ms;
  uint32_t slices;         /* slices launched */
  uint32_t sms_covered;    /* SMs that ran in every slice */
  uint32_t covered[GSB_SM_MAX / 32];
  uint32_t faulty[GSB_SM_MAX / 32];    /* SMs with at least one wrong word */
  uint32_t sm_iterations_min_smid;     /* the covered SM with the fewest iterations */
  uint64_t sm_iterations_min, sm_iterations_max;  /* per-SM iterations over the run (covered SMs; reported only) */
  uint32_t first_mismatch_slice;       /* UINT32_MAX: none */
  uint32_t reserved0;
  uint64_t first_mismatch_ms;          /* from the call's start to the end of that slice */
  gsb_stress_unit_result unit[GSB_STRESS_UNITS];
  gsb_stress_telemetry telemetry;
  uint32_t n_records;      /* records filled (the first GSB_SM_RECORDS mismatches) */
  uint32_t reserved1;
  gsb_stress_record records[GSB_SM_RECORDS];
  uint64_t wall_ns;        /* host time of the whole call */
  uint64_t gap_ns;         /* host time of the slices outside their kernels: launch, log copy, sampling */
  uint64_t expected_ns;    /* host time spent computing the expected answers */
} gsb_stress_result;

/* Conditions (gsb_stress_conditions), from the slices that ran only. Coverage short of sm_count is logged, never a
 * condition, for the reason gsb_sm_conditions gives. */
enum {
  GSB_STRESS_CORRUPT = 1u, /* a D word differs from its exact answer on some SM */
  GSB_STRESS_FAILED = 2u   /* a slice failed or outlived the watchdog */
};

/* Holds the device for the whole run. GSB_ERR_INVALID_ARGUMENT for a unit outside GSB_STRESS_UNIT_MASK, a duration of 0
 * or above GSB_STRESS_DURATION_MAX_MS, or a slice above GSB_STRESS_SLICE_MAX_MS; GSB_ERR_OUT_OF_MEMORY (nothing run, a
 * skipped run) when the buffer cannot be taken. */
int gsb_sm_stress(uint32_t idx, const gsb_stress_cfg *cfg, gsb_stress_result *out);
/* Pure: the GSB_STRESS_FOLD_THREADS folds of the D that gsb_sm_expected(unit, seed) returns, for a tensor unit: thread t
 * of a warpgroup (warp w = t / 32, lane l = t % 32) holds, in register r, D[16w + l/4 + 8((r/2) mod 2)][8(r/4) +
 * 2(l mod 4) + (r mod 2)]; its fold is the XOR over r < 64 of that word rotated left by r mod 32, which any one wrong word
 * changes. Returns the count, or with out == NULL the count required, or a negative status. */
int64_t gsb_stress_fold(uint32_t unit, uint32_t seed, uint32_t *out, size_t cap);
/* Pure: GSB_STRESS_* bits that hold for a result (see above). */
uint32_t gsb_stress_conditions(const gsb_stress_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_copy_text. */
int64_t gsb_stress_text(const gsb_stress_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: in slice `slice` of the next gsb_sm_stress of device idx, if that slice runs `unit`, the CTA on SM `smid`
 * XORs xr into D word `index` of its first iteration (first warpgroup) just before the check; once */
int gsb_test_stress_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint32_t xr, uint32_t slice);

/* ---- SM-to-SM health (not in the reference; opt-in: GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES) --------------------------- */

/*
 * Bit-exact checks of the SM-to-SM network inside a GPC, the path thread-block clusters use. Each (path, cluster size n)
 * is one launch of clusters of n CTAs (grid = cudaOccupancyMaxActiveClusters x n), every CTA asking for the opt-in
 * maximum of dynamic shared memory so that each runs on its own SM. A CTA's dynamic shared memory is a 1 KiB header
 * (%smid, %cluster_ctarank, the peers' %smid read through DSMEM, mbarriers) and then its area, which holds one region of
 * GSB_CLUSTER_REGION_WORDS 16-byte words per peer (per rank for MULTICAST; BULK_S2S keeps its send tiles in the area's
 * second half). Every ordered pair of distinct CTAs of a cluster carries data (MULTICAST: every rank to every rank), and
 * every word of every region is written (DSMEM_LD: read) by a peer:
 *
 *   DSMEM_ST   st.shared::cluster.v4 into every peer's region; a cluster barrier; each CTA checks its own area
 *   DSMEM_LD   each CTA fills its own area; a cluster barrier; peers read it with ld.shared::cluster.v4 and check it
 *   ST_ASYNC   st.async ... mbarrier::complete_tx::bytes.v4 into every peer's region, once the peer has said the region
 *              is free with a remote mbarrier.arrive.release.cluster; the receiver waits on its own mbarrier
 *   BULK_S2S   one thread per CTA: cp.async.bulk.shared::cluster.shared::cta of a tile into every peer's region,
 *              completion on the receiver's mbarrier
 *   MULTICAST  rank s: cp.async.bulk.shared::cluster.global ... multicast::cluster of segment s of a buffer in HBM into
 *              region s of every CTA of the cluster; every CTA checks all n regions
 *
 * Word i of what rank s sends rank d on path p is gsb_pattern_word(gsb_cluster_word_addr(p, n, s, d, i)) under the
 * seed key (gsb_cluster.h; MULTICAST's d is GSB_CLUSTER_EVERY_RANK); a region is filled with its receiver's background
 * (gsb_cluster_bg_addr) first, so a transfer that never lands leaves STALE words. Every wait on an mbarrier is bounded
 * by GSB_CLUSTER_WAIT_NS of %globaltimer; a wait that runs out is counted and the region checked anyway. The log of a
 * launch goes to the result only, never to the HBM fault log or reports.
 */
enum {
  GSB_CLUSTER_PATH_DSMEM_ST = 0,
  GSB_CLUSTER_PATH_DSMEM_LD = 1,
  GSB_CLUSTER_PATH_ST_ASYNC = 2,
  GSB_CLUSTER_PATH_BULK_S2S = 3,
  GSB_CLUSTER_PATH_MULTICAST = 4
};
#define GSB_CLUSTER_PATHS 5
#define GSB_CLUSTER_SIZES 4            /* n = 2, 4, 8, 16: size index k is n = 2 << k */
#define GSB_CLUSTER_MAX_N 16
#define GSB_CLUSTER_RECORDS 64
#define GSB_CLUSTER_MAX_LAUNCHES 3
#define GSB_CLUSTER_SM_MAX 256         /* %smid values a bitmap holds */
#define GSB_CLUSTER_WAIT_NS 100000000u /* bound of every mbarrier wait in the kernels: 100 ms */
#define GSB_CLUSTER_EVERY_RANK 0xFFu   /* the destination rank of MULTICAST words: every CTA of the cluster */
#define GSB_CLUSTER_HEADER_BYTES 1024u /* the head of every CTA's dynamic shared memory; the area follows */
#define GSB_CLUSTER_HOOK_INDEX_MAX 14464u /* words of the area at the 227 KiB opt-in maximum: the most a CTA checks */

typedef struct gsb_cluster_cfg {
  uint32_t paths;       /* mask of 1 << GSB_CLUSTER_PATH_*; 0 = all */
  uint32_t sizes;       /* mask of 1 << k for n = 2 << k; 0 = n = 2 and the largest of 16 and 8 that can be scheduled */
  uint32_t seed;        /* 0 = fresh per probe */
  uint32_t seed_expect; /* seed the words are checked against; 0 = seed (another value makes every checked word wrong) */
} gsb_cluster_cfg;

typedef struct gsb_cluster_record {
  uint32_t path, n;           /* GSB_CLUSTER_PATH_*, cluster size */
  uint32_t src_rank, dst_rank;
  uint32_t src_smid, dst_smid;
  uint32_t index;             /* word i of the (src, dst) pair's region */
  uint32_t reserved0;
  uint32_t expected[4], observed[4];
} gsb_cluster_record;

typedef struct gsb_cluster_run {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = this (path, size) did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t timeouts;       /* mbarrier waits that ran out of GSB_CLUSTER_WAIT_NS */
  uint64_t words_checked;  /* 16-byte words compared, over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_cluster_run;

typedef struct gsb_cluster_result {
  int32_t status;          /* GSB_OK iff every launch asked for ran (mismatches and timeouts are a result) */
  uint32_t sm_count;
  uint32_t seed, seed_expect;
  uint32_t paths, sizes;   /* what ran (the defaults resolved) */
  uint32_t smem_bytes;     /* dynamic shared memory of every CTA (header + area) */
  uint32_t reserved0;
  uint32_t max_clusters[GSB_CLUSTER_SIZES]; /* cudaOccupancyMaxActiveClusters per size (0: cannot be scheduled) */
  uint32_t expect_covered[GSB_CLUSTER_SIZES]; /* min(sm_count, max_clusters x n): the coverage a size is held to */
  uint32_t covered[GSB_CLUSTER_SM_MAX / 32];  /* SMs some launch ran on, bit %smid */
  uint32_t faulty[GSB_CLUSTER_SM_MAX / 32];   /* both ends of every wrong word */
  gsb_cluster_run run[GSB_CLUSTER_PATHS][GSB_CLUSTER_SIZES];
  uint32_t n_records;      /* records filled (the first GSB_CLUSTER_RECORDS mismatches) */
  uint32_t reserved1;
  gsb_cluster_record records[GSB_CLUSTER_RECORDS];
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_cluster_result;

/* Conditions (gsb_cluster_conditions), from the runs that ran only. Coverage short of expect_covered after the
 * relaunches is counted (gsb_cluster_stats.incomplete) and logged, never a condition. */
enum {
  GSB_CLUSTER_CORRUPT = 1u, /* a word that crossed the SM-to-SM network differs from its pattern */
  GSB_CLUSTER_FAILED = 2u   /* a launch failed or outlived the watchdog, or a transfer never completed (a wait ran out) */
};

/* What a wrong word holds (gsb_cluster_classify) */
enum {
  GSB_CLUSTER_CLASS_ZERO = 1,      /* all zero */
  GSB_CLUSTER_CLASS_STALE = 2,     /* the receiver's background at that place: the transfer never landed */
  GSB_CLUSTER_CLASS_MISROUTED = 3, /* the intact word of another (src, dst) pair or region of the same launch */
  GSB_CLUSTER_CLASS_BITS = 4       /* none of these: flipped bits */
};
typedef struct gsb_cluster_class {
  uint32_t cls;            /* GSB_CLUSTER_CLASS_* */
  uint32_t src_rank, dst_rank, index; /* MISROUTED: the pair and word whose data it is (MULTICAST: dst_rank = GSB_CLUSTER_EVERY_RANK) */
  uint32_t flipped_bits;   /* popcount(expected ^ observed) */
  uint32_t reserved0;
} gsb_cluster_class;

/* Cluster probes of one device since gsb_health_start (counters restart with it; gsb_cluster_probe calls count too). */
typedef struct gsb_cluster_stats {
  uint64_t probes;
  uint64_t faults;     /* probes that raised at least one GSB_CLUSTER_* condition */
  uint64_t skipped;    /* probes that ran no launch (the buffer was not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some (path, size) covered fewer than expect_covered SMs */
  gsb_cluster_result last;
} gsb_cluster_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_cluster_probe(uint32_t idx, const gsb_cluster_cfg *cfg, gsb_cluster_result *out);
int gsb_cluster_stats_get(uint32_t idx, gsb_cluster_stats *out);
/* Pure: GSB_CLUSTER_* bits that hold for a result (see above). */
uint32_t gsb_cluster_conditions(const gsb_cluster_result *r);
/* Pure: what the wrong word of `rec` holds, for a launch with `seed` (the seed the words were sent under) and
 * `smem_bytes` of dynamic shared memory per CTA. Returns GSB_OK or GSB_ERR_INVALID_ARGUMENT. */
int gsb_cluster_classify(uint32_t seed, uint32_t smem_bytes, const gsb_cluster_record *rec, gsb_cluster_class *out);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_cluster_text(const gsb_cluster_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_cluster_probe of device idx, in the first launch of `path`, the CTA on SM `smid` XORs xr
 * into lanes 0-1 of the `index`th word it checks (slot j = (src - dst - 1) mod n, or src for MULTICAST, holds words
 * j x region_words .. (j + 1) x region_words - 1) before the compare; once */
int gsb_test_cluster_corrupt(uint32_t idx, uint32_t smid, uint32_t path, uint32_t index, uint64_t xr);
/* test hook: on the next gsb_cluster_probe of device idx, in the first launch of `path`, the CTA on SM `smid` sends
 * nothing (DSMEM_LD: leaves its area's background for its readers); its receivers find STALE words and, on the mbarrier
 * paths, a wait that runs out; once */
int gsb_test_cluster_skip(uint32_t idx, uint32_t smid, uint32_t path);
#define GSB_CLUSTER_UNROUTED 0xFFu /* gsb_test_cluster_script: rank s sends rank d nothing */
/* test hook: the first launch of (path, n) in the next gsb_cluster_probe of device idx that runs that pair is the
 * path's test-only twin, run on a script; once. Every region is region_words words (1 up to the path's region words at
 * n with the 227 KiB opt-in maximum) and route[s * n + d] (n x n bytes) is the slot, in the area the words of rank s for
 * rank d land in (d's; DSMEM_LD: s's own), where they go, or GSB_CLUSTER_UNROUTED. A receiver arms and waits on the
 * mbarriers of routed slots only; the compare is the probe's own, so a word routed elsewhere is MISROUTED and a slot
 * nobody fills is STALE. MULTICAST: row s is one slot or GSB_CLUSTER_UNROUTED throughout, and the ranks it names are
 * the multicast mask. Refused before any device is touched: an unknown path, n not 2, 4, 8 or 16, region_words out of
 * range, a slot past the path's slots, s routed to itself (but on MULTICAST), two senders in one slot of one area, a
 * MULTICAST row with two slots. route NULL disarms it. Later launches of the pair (coverage) are the probe's own. */
int gsb_test_cluster_script(uint32_t idx, uint32_t path, uint32_t n, uint32_t region_words, const uint8_t *route);

/* ---- L2 atomic health (not in the reference; opt-in: GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES) ---------------------------- */

/*
 * Bit-exact checks of the atomic units in the L2, which run every atom / red on global memory. Each op is three
 * launches on one transient buffer: an init launch writes the op's starting words from the seed, a run launch of one
 * CTA per SM (GSB_ATOMIC_THREADS threads, the opt-in maximum of dynamic shared memory) issues the atomics, and a check
 * launch compares every word of the buffer with expected words computed on the host (gsb_atomic_expected). The buffer
 * (GSB_ATOMIC_BYTES) is a spread region of GSB_ATOMIC_LINES lines of 128 bytes, then GSB_ATOMIC_HOT_WORDS hot words
 * GSB_ATOMIC_HOT_STRIDE bytes apart. Two phases:
 *
 *   spread  every CTA issues one atomic to every line; in line j CTA b hits word (b + j) mod words-per-line, so every
 *           word gets contributions from several CTAs and every line (and so, by address, every L2 slice) is reached
 *           from every SM. Not for TICKET and CAS, whose spread words keep their starting value and are checked too.
 *   hot     lane l of every hot warp of every CTA hits hot word l, GSB_ATOMIC_HOT_REPS times (HADD2: one warp per CTA,
 *           once; CAS: once), so the lanes of a warp never share an address
 *
 * Every contribution depends on blockIdx, thread and seed, never on %smid. Integer add, and/or/xor and min/max commute;
 * float contributions are integers whose sum of magnitudes per word stays under the type's exact-integer bound, so
 * every order gives the same bits. TICKET (atom.add of 1, return value used) and CAS (a compare-and-swap increment loop
 * that feeds each returned value into the next compare) store each contributor's id at slot[word][ticket]; slots start
 * at GSB_ATOMIC_NO_ID and are checked on the host: every slot must hold a distinct id below the word's contributor
 * count. A returned ticket at or past that count is recorded and never used as an index. Every CAS loop ends at a
 * GSB_ATOMIC_CAS_WAIT_NS %globaltimer deadline. The log goes to the result only, never to the HBM fault log or reports.
 */
enum {
  GSB_ATOMIC_OP_ADD32 = 0,  /* red.add.u32 */
  GSB_ATOMIC_OP_ADD64 = 1,  /* red.add.u64 */
  GSB_ATOMIC_OP_LOGIC = 2,  /* red.and / or / xor .b32 and .b64, by word (8-byte words; b32 forms on the low half) */
  GSB_ATOMIC_OP_MINMAX = 3, /* red.min.s32, max.u32, min.s64, max.u64, by word (8-byte words) */
  GSB_ATOMIC_OP_FADD32 = 4, /* red.add.f32 (lower half of the lines, hot words 0-15), red.add.v4.f32 (the rest) */
  GSB_ATOMIC_OP_FADD64 = 5, /* red.add.f64 */
  GSB_ATOMIC_OP_HADD2 = 6,  /* red.add.noftz.f16x2 (even words) and .bf16x2 (odd words) */
  GSB_ATOMIC_OP_TICKET = 7, /* atom.add.u32 of 1 on the hot words, the returned ticket used */
  GSB_ATOMIC_OP_CAS = 8     /* atom.cas.b32 increment loop on the hot words */
};
#define GSB_ATOMIC_OPS 9
#define GSB_ATOMIC_RECORDS 64
#define GSB_ATOMIC_MAX_LAUNCHES 3
#define GSB_ATOMIC_SM_MAX 256          /* %smid values a bitmap holds; also the most CTAs a run launch has */
#define GSB_ATOMIC_THREADS 256         /* threads of every run CTA */
#define GSB_ATOMIC_LINES 8192u
#define GSB_ATOMIC_LINE_BYTES 128u
#define GSB_ATOMIC_REGION_BYTES (GSB_ATOMIC_LINES * GSB_ATOMIC_LINE_BYTES)
#define GSB_ATOMIC_HOT_WORDS 32u
#define GSB_ATOMIC_HOT_STRIDE 4096u    /* bytes between hot words */
#define GSB_ATOMIC_HOT_REPS 4u         /* atomics per hot lane, but for HADD2 and CAS (1) */
#define GSB_ATOMIC_BYTES (GSB_ATOMIC_REGION_BYTES + GSB_ATOMIC_HOT_WORDS * GSB_ATOMIC_HOT_STRIDE)
#define GSB_ATOMIC_CAS_WAIT_NS 100000000u /* bound of every CAS loop: 100 ms */
#define GSB_ATOMIC_NO_ID 0xFFFFFFFFu   /* what a ticket slot starts as */
#define GSB_ATOMIC_NO_SM 0xFFFFFFFFu   /* a record that no single SM can be named for */
enum {
  GSB_ATOMIC_PHASE_SPREAD = 0, /* record.word: a word of the spread region */
  GSB_ATOMIC_PHASE_HOT = 1,    /* record.word: a word of the hot area (a hot word, or the padding after it) */
  GSB_ATOMIC_PHASE_SLOT = 2    /* record.word: ticket slot hot_word x contributors + ticket */
};

typedef struct gsb_atomic_cfg {
  uint32_t ops;         /* mask of 1 << GSB_ATOMIC_OP_*; 0 = all */
  uint32_t seed;        /* 0 = fresh per probe */
  uint32_t seed_expect; /* seed the expected words are computed from; 0 = seed */
  uint32_t reserved0;
} gsb_atomic_cfg;

/* One wrong word, slot or ticket. A word's `word` is its index in the buffer in the op's word size (8 bytes for ADD64,
 * LOGIC, MINMAX and FADD64, else 4); expected and observed are that word. A slot's expected is the word's contributor
 * count (an id must lie below it, once) and observed its content; a ticket returned at or past that count (phase HOT,
 * `word` the hot word's index) has the count as expected and the ticket as observed. smid names the SM of the CTA
 * whose id or ticket it is, GSB_ATOMIC_NO_SM for a final word or an empty slot. */
typedef struct gsb_atomic_record {
  uint32_t op, phase, word, smid;
  uint64_t expected, observed;
} gsb_atomic_record;

typedef struct gsb_atomic_run {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* run launches (each with its init and check launch); 0 = the op did not run */
  uint32_t sms_covered;    /* distinct %smid over its run launches */
  uint32_t hook_cta;       /* the blockIdx that applied gsb_test_atomic_skip; GSB_ATOMIC_NO_SM when none did */
  uint64_t atomics_issued; /* atomic instructions the run launches issued (CAS: successful compare-and-swaps) */
  uint64_t words_checked;  /* words compared by the check launches */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t ticket_faults;  /* TICKET, CAS: slots without a distinct valid id, plus tickets returned out of range */
  uint64_t cas_timeouts;   /* CAS loops that ran out of GSB_ATOMIC_CAS_WAIT_NS */
  uint64_t cas_max_ns;     /* CAS: the longest loop of any thread, by %globaltimer */
  uint64_t kernel_ns;      /* CUDA-event time of its init, run and check launches */
} gsb_atomic_run;

typedef struct gsb_atomic_result {
  int32_t status;          /* GSB_OK iff every launch asked for ran (mismatches, faults and timeouts are a result) */
  uint32_t sm_count;
  uint32_t seed, seed_expect;
  uint32_t ops;            /* what ran (the default resolved) */
  uint32_t reserved0;
  uint32_t covered[GSB_ATOMIC_SM_MAX / 32];  /* SMs every op's run launches reached, bit %smid */
  uint32_t faulty[GSB_ATOMIC_SM_MAX / 32];   /* SMs a record names */
  gsb_atomic_run run[GSB_ATOMIC_OPS];
  uint32_t n_records;      /* records filled (the first GSB_ATOMIC_RECORDS) */
  uint32_t reserved1;
  gsb_atomic_record records[GSB_ATOMIC_RECORDS];
  uint64_t expected_ns;    /* host time spent on the expected words */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_atomic_result;

/* Conditions (gsb_atomic_conditions), from the ops that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_atomic_stats.incomplete) and logged, never a condition. */
enum {
  GSB_ATOMIC_CORRUPT = 1u, /* a final word, a ticket or a slot is wrong */
  GSB_ATOMIC_FAILED = 2u   /* a launch failed or outlived the watchdog, or a CAS loop ran out of its deadline */
};

/* Atomic probes of one device since gsb_health_start (counters restart with it; gsb_atomic_probe calls count too). */
typedef struct gsb_atomic_stats {
  uint64_t probes;
  uint64_t faults;     /* probes that raised at least one GSB_ATOMIC_* condition */
  uint64_t skipped;    /* probes that ran no launch (the buffer was not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some op covered fewer than sm_count SMs */
  gsb_atomic_result last;
} gsb_atomic_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_atomic_probe(uint32_t idx, const gsb_atomic_cfg *cfg, gsb_atomic_result *out);
int gsb_atomic_stats_get(uint32_t idx, gsb_atomic_stats *out);
/* Pure: the GSB_ATOMIC_BYTES of the buffer after a clean run of `op` under `seed` with `sm_count` CTAs, little-endian
 * words as the device holds them. Returns GSB_ATOMIC_BYTES (with out == NULL too), GSB_ERR_BUFFER_TOO_SMALL when cap is
 * short, or GSB_ERR_INVALID_ARGUMENT for an unknown op, an sm_count of 0 or above GSB_ATOMIC_SM_MAX, or a float word
 * whose sum of magnitudes would reach its type's exact-integer bound. */
int64_t gsb_atomic_expected(uint32_t op, uint32_t seed, uint32_t sm_count, void *out, size_t cap);
/* Pure: GSB_ATOMIC_* bits that hold for a result (see above). */
uint32_t gsb_atomic_conditions(const gsb_atomic_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_atomic_text(const gsb_atomic_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_atomic_probe of device idx, the first check launch of `op` XORs xr into the observed word
 * `word` (in the op's word size) before the compare; once. Refused before any device is touched: op out of range,
 * word past the buffer, or xr wider than a 4-byte op's word. */
int gsb_test_atomic_corrupt(uint32_t idx, uint32_t op, uint32_t word, uint64_t xr);
/* test hook: on the next gsb_atomic_probe of device idx, in the first run launch of `op`, the CTA on SM `smid` issues
 * none of its atomics; once */
int gsb_test_atomic_skip(uint32_t idx, uint32_t smid, uint32_t op);
/* test hook: the next gsb_atomic_probe of device idx that runs `op` runs it on chosen values. Each launch uploads
 * `init` (gsb_atomic_units(op) words, one per uint64_t) as the starting words in place of the init launch, a test-only
 * twin of the run kernel takes each operand's raw bits from `values` (integer operand, FP32 or FP64 bits, or the f16x2 /
 * bf16x2 pair; where each contribution's operand lies is gsb_atomic_value_index in csrc/gsb_atomic.h, n_values is
 * ctas x (GSB_ATOMIC_LINES + 1024) x 4), and the check launch compares the words with `expected`. Geometry, records,
 * counts, the other hooks and relaunches are as in an ordinary probe; the table takes its share of the transient
 * buffer. Once; init == NULL disarms it. Refused before any device is touched: TICKET, CAS or an unknown op, ctas of 0
 * or above GSB_ATOMIC_SM_MAX, a wrong n_values, or a starting, expected or operand word wider than its word (4-byte
 * ops, and the b32, s32 and u32 forms); then refused when ctas is not the device's SM count. */
int gsb_test_atomic_values(uint32_t idx, uint32_t op, uint32_t ctas, const uint64_t *init, const uint64_t *values,
                           size_t n_values, const uint64_t *expected);

/* ---- Tensor-core format health (not in the reference; opt-in: GSB_OPT_TENSOR_PROBE_EVERY_CYCLES) ----------------- */

/*
 * Known-answer checks of the tensor-core forms gsb_sm_probe does not run, on every SM. Each unit is one launch as in
 * the SM check: one CTA per SM, each asking for the opt-in maximum of dynamic shared memory, thread 0 recording %smid,
 * a launch that left an SM uncovered repeated up to GSB_TENSOR_MAX_LAUNCHES times. Each computes one 64 x 128 D and
 * compares every word bit for bit, on the SM, with answers computed exactly on the host (gsb_tensor_expected):
 *
 *   DMMA       mma.sync m16n8k16 FP64 (FP64 tensor cores), K = 64
 *   TF32       wgmma m64n128k8 .f32.tf32.tf32, K = 128
 *   E5M2, E4M3_E5M2, E5M2_E4M3   wgmma m64n128k32 FP32 accumulate, A and B of those types, K = 64
 *   F16_ACC    wgmma m64n128k16 .f16.f16.f16 (FP16 accumulators), K = 64
 *   HMMA       mma.sync m16n8k16 .f32.f16.f16.f32, fragments loaded with ldmatrix, K = 256
 *   F16_RS     wgmma m64n128k16 .f32.f16.f16 with A in registers (loaded with ldmatrix), K = 256
 *
 * HMMA and F16_RS run the SM check's F16 GEMM (its operands at the same seed), so their answer is
 * gsb_sm_expected(GSB_SM_UNIT_F16, seed). The operands are generated on the device from (unit, seed, row, col); only the
 * expected answers are uploaded, into a transient buffer taken only when GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free.
 * A mismatch never touches the HBM fault log or reports.
 */
enum {
  GSB_TENSOR_UNIT_DMMA = 0,
  GSB_TENSOR_UNIT_TF32 = 1,
  GSB_TENSOR_UNIT_E5M2 = 2,
  GSB_TENSOR_UNIT_E4M3_E5M2 = 3, /* A E4M3, B E5M2 */
  GSB_TENSOR_UNIT_E5M2_E4M3 = 4, /* A E5M2, B E4M3 */
  GSB_TENSOR_UNIT_F16_ACC = 5,
  GSB_TENSOR_UNIT_HMMA = 6,
  GSB_TENSOR_UNIT_F16_RS = 7
};
#define GSB_TENSOR_UNITS 8
#define GSB_TENSOR_RECORDS 64
#define GSB_TENSOR_MAX_LAUNCHES 3
#define GSB_TENSOR_WORDS 8192 /* D words of one CTA: 64 x 128 */

typedef struct gsb_tensor_cfg {
  uint32_t seed;        /* operands' seed; 0 = fresh per probe */
  uint32_t seed_expect; /* seed of the expected answers; 0 = seed */
  uint32_t units;       /* mask of 1 << GSB_TENSOR_UNIT_*; 0 = all */
  uint32_t reserved0;
} gsb_tensor_cfg;

typedef struct gsb_tensor_unit_result {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = the unit did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t reserved0;
  uint64_t words_checked;  /* D words compared, over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_tensor_unit_result;

typedef struct gsb_tensor_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs with at least one wrong word */
  gsb_tensor_unit_result unit[GSB_TENSOR_UNITS];
  uint32_t n_records;      /* records filled (the first GSB_TENSOR_RECORDS mismatches) */
  uint32_t reserved0;
  /* unit: GSB_TENSOR_UNIT_*; index: row * 128 + column of D; expected and observed: FP64 bits for DMMA, otherwise
   * zero-extended (F16_ACC: the FP16 bits) */
  gsb_sm_record records[GSB_TENSOR_RECORDS];
  uint64_t expected_ns;    /* host time spent computing the expected answers */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_tensor_result;

/* Conditions (gsb_tensor_conditions), from the units that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_tensor_stats.incomplete) and logged, never a condition, as in the SM check. */
enum {
  GSB_TENSOR_CORRUPT = 1u, /* a D word differs from its exact answer on some SM */
  GSB_TENSOR_FAILED = 2u   /* a launch failed or outlived the watchdog */
};

/* Tensor probes of one device since gsb_health_start (counters restart with it; gsb_tensor_probe calls count too). */
typedef struct gsb_tensor_stats {
  uint64_t probes;     /* tensor probes run */
  uint64_t faults;     /* of which raised at least one GSB_TENSOR_* condition */
  uint64_t skipped;    /* probes that ran no unit (buffers not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_tensor_result last;
} gsb_tensor_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_tensor_probe(uint32_t idx, const gsb_tensor_cfg *cfg, gsb_tensor_result *out);
int gsb_tensor_stats_get(uint32_t idx, gsb_tensor_stats *out);
/* Pure: the exact answers of `unit` for `seed`: the 8192 words of D in row-major order (FP64 bits for DMMA, FP32 bits,
 * F16_ACC's FP16 bits zero-extended). Returns the count, or with out == NULL the count required, or a negative status
 * (GSB_ERR_BUFFER_TOO_SMALL when cap is short, GSB_ERR_INVALID_ARGUMENT for an unknown unit). */
int64_t gsb_tensor_expected(uint32_t unit, uint32_t seed, uint64_t *out, size_t cap);
/* Pure: GSB_TENSOR_* bits that hold for a result (see above). */
uint32_t gsb_tensor_conditions(const gsb_tensor_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_tensor_text(const gsb_tensor_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_tensor_probe of device idx, the CTA running on SM `smid` XORs xr into its D word `index`
 * of `unit` just before the compare; once. Refused before any device is touched: unit, smid or index out of range,
 * or xr wider than the unit's word (16 bits for F16_ACC, 32 for the FP32 units). */
int gsb_test_tensor_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
/* test hook: the next gsb_tensor_probe of device idx that runs `unit` runs it on chosen operands instead of the seed's:
 * every launch of the unit in that probe computes D = A B with A[i][k] = a[i * K + k] * 2^sa[i] and
 * B[k][j] = b[k * 128 + j] * 2^sb[j] (K of the unit) through the same conversion, layout, instruction and fragment
 * compare, and compares D with expected[row * 128 + col] (as gsb_tensor_expected gives them). Once. a == NULL disarms
 * it. Refused with GSB_ERR_INVALID_ARGUMENT before any device is touched: an unknown unit, an integer outside
 * [-amp, amp] of A or B, a scale outside its range, or an expected word wider than the unit's word. */
int gsb_test_tensor_operands(uint32_t idx, uint32_t unit, const int32_t *a, const int32_t *b, const int32_t *sa,
                             const int32_t *sb, const uint64_t *expected);

/* ---- SM special-function health (not in the reference; opt-in: GSB_OPT_SFU_PROBE_EVERY_CYCLES) ------------------ */

/*
 * Known-answer checks of the SM datapaths outside the FMA, integer and tensor pipes, on every SM. Each unit is one
 * launch as in the SM check: one CTA of GSB_SFU_THREADS per SM, each asking for the opt-in maximum of dynamic shared
 * memory, thread 0 recording %smid, a launch that left an SM uncovered repeated up to GSB_SFU_MAX_LAUNCHES times. Every
 * instruction is inline PTX with its rounding, .ftz and .satfinite spelled out. Per instruction ("op"), each thread
 * folds its GSB_SFU_STEPS results into one 64-bit checksum; the inputs are functions of (unit, seed, thread, step,
 * operand) only, drawn from classes (normals, subnormals, zeros and infinities, rounding ties of the destination,
 * saturation edges, integers near 2^24 and 2^53) and never NaN nor yielding NaN:
 *
 *   CVT_HALF  cvt.rn.f16x2.f32, cvt.rn.bf16x2.f32, cvt.f32.f16, cvt.f32.bf16                       4 ops
 *   CVT_FP8   cvt.rn.satfinite.{e4m3x2,e5m2x2}.f32, cvt.rn.f16x2.{e4m3x2,e5m2x2}                     4 ops
 *   CVT_INT   cvt.{rni,rzi,rmi,rpi}.s32.f32, cvt.rn.f32.s32, cvt.rzi.s64.f64, cvt.rn.f64.s64,
 *             cvt.rn.f32.f64, cvt.f64.f32                                                          9 ops
 *   DIVSQRT   div.rn, sqrt.rn, rcp.rn in f32 (no .ftz) and f64                                      6 ops
 *   WARP      shfl.sync idx/up/down/bfly, vote.sync ballot/any/all, match.{any,all}.sync,
 *             redux.sync add/min.s32/max.u32/and/or/xor                                           15 ops
 *   MUFU      {ex2,lg2,rcp,rsqrt,sqrt,sin,cos}.approx.ftz.f32, tanh.approx.f32, ex2.approx.f16x2,
 *             ex2.approx.ftz.bf16x2, tanh.approx.{f16x2,bf16x2}                                   12 ops
 *
 * The first five are exact: each thread's folds are compared bit for bit, on the SM, with folds computed on the host
 * (gsb_sfu_expected); a record's index is op * GSB_SFU_THREADS + thread. PTX bounds MUFU's approximations only, so the
 * MUFU unit's verdict is consensus: every CTA writes its folds, the raw results of its first GSB_SFU_RAW inputs per
 * thread and op, and its %smid, and gsb_sfu_vote takes the value more than half the CTAs hold as each word's answer
 * (every other CTA is a mismatch; with no majority every CTA is), then checks each voted raw result against the
 * host's double-precision libm answer within a loose envelope (GSB_SFU_ENVELOPE_*). A mismatch never touches the HBM
 * fault log or reports.
 */
enum {
  GSB_SFU_UNIT_CVT_HALF = 0,
  GSB_SFU_UNIT_CVT_FP8 = 1,
  GSB_SFU_UNIT_CVT_INT = 2,
  GSB_SFU_UNIT_DIVSQRT = 3,
  GSB_SFU_UNIT_WARP = 4,
  GSB_SFU_UNIT_MUFU = 5
};
#define GSB_SFU_UNITS 6
#define GSB_SFU_THREADS 256
#define GSB_SFU_STEPS 1024
#define GSB_SFU_RAW 4          /* raw MUFU results kept per thread and op: those of steps 0..3 */
#define GSB_SFU_OPS_MAX 15     /* ops of the widest unit (WARP) */
#define GSB_SFU_MUFU_OPS 12
#define GSB_SFU_RECORDS 64
#define GSB_SFU_MAX_LAUNCHES 3
/* Words the vote compares per CTA: the 12 x 256 folds, then the 12 x 256 x 4 raw results. Index of fold (op, t):
 * op * 256 + t; of raw result r of (op, t): GSB_SFU_MUFU_FOLDS + (op * 256 + t) * 4 + r. */
#define GSB_SFU_MUFU_FOLDS (GSB_SFU_MUFU_OPS * GSB_SFU_THREADS)
#define GSB_SFU_MUFU_WORDS (GSB_SFU_MUFU_FOLDS * (1 + GSB_SFU_RAW))

/* MUFU ops, in the order of gsb_sfu_result.max_err */
enum {
  GSB_SFU_MUFU_EX2 = 0, GSB_SFU_MUFU_LG2 = 1, GSB_SFU_MUFU_RCP = 2, GSB_SFU_MUFU_RSQRT = 3, GSB_SFU_MUFU_SQRT = 4,
  GSB_SFU_MUFU_SIN = 5, GSB_SFU_MUFU_COS = 6, GSB_SFU_MUFU_TANH = 7, GSB_SFU_MUFU_EX2_F16 = 8,
  GSB_SFU_MUFU_EX2_BF16 = 9, GSB_SFU_MUFU_TANH_F16 = 10, GSB_SFU_MUFU_TANH_BF16 = 11
};

typedef struct gsb_sfu_cfg {
  uint32_t seed;        /* inputs' seed; 0 = fresh per probe */
  uint32_t seed_expect; /* seed of the exact units' expected folds; 0 = seed (the MUFU vote does not use it) */
  uint32_t units;       /* mask of 1 << GSB_SFU_UNIT_*; 0 = all */
  uint32_t reserved0;
} gsb_sfu_cfg;

typedef struct gsb_sfu_unit_result {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = the unit did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t reserved0;
  uint64_t words_checked;  /* folds compared (MUFU: folds and raw results voted), over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_sfu_unit_result;

typedef struct gsb_sfu_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs with at least one wrong or minority word */
  gsb_sfu_unit_result unit[GSB_SFU_UNITS];
  uint32_t n_records;      /* records filled (the first GSB_SFU_RECORDS mismatches) */
  uint32_t bound;          /* bit GSB_SFU_MUFU_*: a voted raw result of that op lies outside its envelope */
  /* unit: GSB_SFU_UNIT_*; index as above; expected: the host's fold, or the majority (0 when there is none);
   * observed: the CTA's word (raw results zero-extended) */
  gsb_sm_record records[GSB_SFU_RECORDS];
  double max_err[GSB_SFU_MUFU_OPS]; /* worst error of each MUFU op's voted raw results against libm, in its envelope's
                                       unit (relative, absolute, or ulps of the 16-bit output) */
  uint64_t expected_ns;    /* host time spent computing the exact units' folds */
  uint64_t vote_ns;        /* host time spent in gsb_sfu_vote */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_sfu_result;

/* Conditions (gsb_sfu_conditions), from the units that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_sfu_stats.incomplete) and logged, never a condition, as in the SM check. */
enum {
  GSB_SFU_CORRUPT = 1u, /* a fold or raw result differs from its exact answer or from the majority on some SM */
  GSB_SFU_BOUND = 2u,   /* a MUFU result every SM agrees on lies outside its envelope */
  GSB_SFU_FAILED = 4u   /* a launch failed or outlived the watchdog */
};

/* SFU probes of one device since gsb_health_start (counters restart with it; gsb_sfu_probe calls count too). */
typedef struct gsb_sfu_stats {
  uint64_t probes;     /* SFU probes run */
  uint64_t faults;     /* of which raised at least one GSB_SFU_* condition */
  uint64_t skipped;    /* probes that ran no unit (buffers not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_sfu_result last;
} gsb_sfu_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_sfu_probe(uint32_t idx, const gsb_sfu_cfg *cfg, gsb_sfu_result *out);
int gsb_sfu_stats_get(uint32_t idx, gsb_sfu_stats *out);
/* Pure: the exact folds of exact unit `unit` (not MUFU) for `seed`, index op * 256 + thread. Returns the count, or
 * with out == NULL the count required, or a negative status (GSB_ERR_BUFFER_TOO_SMALL when cap is short,
 * GSB_ERR_INVALID_ARGUMENT for MUFU or an unknown unit). */
int64_t gsb_sfu_expected(uint32_t unit, uint32_t seed, uint64_t *out, size_t cap);
/* Pure: the host's answer of exact SFU instruction (unit, op) for n operand pairs; a[i], b[i] hold the operand bits
 * as the kernel takes them (b: the second f32 of an x2 pack, or the divisor; unused otherwise, and may be NULL). Units
 * CVT_HALF, CVT_FP8, CVT_INT and DIVSQRT. Returns n, or GSB_ERR_INVALID_ARGUMENT for WARP, MUFU, an op past the unit's,
 * a NULL pointer, an operand wider than the op takes, and any operand that is NaN or whose result would be NaN (0/0,
 * inf/inf). sqrt takes the operand's magnitude, as the probe's kernel does. */
int64_t gsb_sfu_model(uint32_t unit, uint32_t op, const uint64_t *a, const uint64_t *b, size_t n, uint64_t *out);
/* Pure: the MUFU vote over one launch's `ctas` CTAs for inputs of `seed`: folds[cta][op][thread],
 * raw[cta][op][thread][GSB_SFU_RAW] and smid[cta] as the kernel wrote them. Adds to out->unit[GSB_SFU_UNIT_MUFU]'s
 * words_checked, mismatch_words and mismatch_bits, to out->faulty, out->records and out->bound, and raises
 * out->max_err. Returns GSB_OK, or GSB_ERR_INVALID_ARGUMENT for a null pointer or ctas == 0. */
int gsb_sfu_vote(uint32_t seed, uint32_t ctas, const uint64_t *folds, const uint32_t *raw, const uint32_t *smid,
                 gsb_sfu_result *out);
/* Pure: GSB_SFU_* bits that hold for a result (see above). */
uint32_t gsb_sfu_conditions(const gsb_sfu_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_sfu_text(const gsb_sfu_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_sfu_probe of device idx, the CTA running on SM `smid` XORs xr into its fold `index`
 * (op * 256 + thread) of `unit` just before the compare (exact units) or the write (MUFU); once. Refused before any
 * device is touched: unit or smid out of range, or index past the unit's ops. */
int gsb_test_sfu_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
#define GSB_SFU_INPUTS_MAX (1u << 15) /* operand pairs of one gsb_test_sfu_inputs call */
/* test hook, synchronous: runs SFU instruction (unit, op) on the n operand pairs (a[i], b[i]; as gsb_sfu_model takes
 * them, b may be NULL) on every SM of device idx, through the same instruction code as the probe's kernels, and returns
 * every raw result: results[smid * n + i] (GSB_SM_MAX * n words; zero-extended) for each SM whose bit it sets in
 * covered (GSB_SM_MAX bits). One CTA per SM at the opt-in shared-memory maximum, repeated up to GSB_SFU_MAX_LAUNCHES
 * times until every SM is covered, in one transient buffer taken only while the keep-free margin holds. MUFU (every op)
 * is accepted; its 16-bit forms take two halves in a[i]. Refused with GSB_ERR_INVALID_ARGUMENT before any device is
 * touched: WARP, an out-of-range unit or op, n == 0 or above GSB_SFU_INPUTS_MAX, a NULL a, results or covered, and
 * operands gsb_sfu_model refuses (for MUFU: NaN, and negative nonzero operands of lg2, rsqrt and sqrt, infinite ones of
 * sin and cos). */
int gsb_test_sfu_inputs(uint32_t idx, uint32_t unit, uint32_t op, const uint64_t *a, const uint64_t *b, size_t n,
                        uint64_t *results, uint32_t *covered);

/* ---- L1 and constant-cache health (not in the reference; opt-in: GSB_OPT_L1_PROBE_EVERY_CYCLES) ---------------- */

/*
 * Bit-exact checks of every SM's L1 data cache, read-only and texture paths, constant bank and kernel parameters. Each
 * unit is one launch of sm_count CTAs of GSB_L1_THREADS; thread 0 of each CTA sets bit %smid of the launch's coverage
 * bitmap, and a launch that left an SM uncovered is repeated up to GSB_L1_MAX_LAUNCHES times. Every word a CTA reads is
 * a 16-byte HBM-probe pattern word (gsb_pattern.h) of its own address: the CTA computes the expected word in registers
 * and compares on the SM, so a wrong word classifies like an HBM fault (gsb_fault_classify: a missed update is STALE,
 * another address's line ALIASED). The buffer is sm_count regions of GSB_L1_REGION_WORDS words, CTA c owning region c,
 * filled by the HBM probe's FILL launch before every launch that reads it.
 *
 *   L1_LOAD   each CTA reads its region `passes` times with each of ld.global.ca, ld.global and
 *             ld.global.L1::evict_last; pass 0 in address order (cold), later passes in the orders of
 *             gsb_l1_schedule (sequential, reversed, lines 4, 16 and 64 KiB apart back to back)        forms 0..2
 *   L1_STORE  reads its region through L1 (form 0), then each thread stores generation 2 (seed ~seed) over bytes of
 *             words another warp owns with st.global.u8/u16/u32/v2/v4, then after bar.sync reads every word back
 *             through L1 (form 1): the byte merge of the two generations                                forms 0, 1
 *   NC        the passes of L1_LOAD through ld.global.nc                                                 form 0
 *   TEX       tex1Dfetch of its region (form 0); tex2D with point filtering and unnormalized coordinates over the
 *             buffer as one 64-word-wide pitch-2D texture, CTA c holding rows [128 c, 128 c + 128), x in [-32, 96)
 *             and y past the array's first and last rows, once with clamp addressing (form 1: the edge texel) and
 *             once with border addressing (form 2: 0 outside)
 *   CONST     a 64 KiB __constant__ bank holding the pattern, read by every thread with uniform indices (form 0) and
 *             once per CTA with per-thread indices (form 1)
 *   PARAM     a 32000-byte __grid_constant__ kernel parameter holding the pattern, read likewise
 *
 * Warm/cold ratio: each CTA times (clock64) its cold pass and its warm passes of every L1_LOAD and NC form; the result
 * reports the median over CTAs of (warm span / (passes - 1)) / cold span. It is logged, never judged.
 */
enum {
  GSB_L1_UNIT_L1_LOAD = 0,
  GSB_L1_UNIT_L1_STORE = 1,
  GSB_L1_UNIT_NC = 2,
  GSB_L1_UNIT_TEX = 3,
  GSB_L1_UNIT_CONST = 4,
  GSB_L1_UNIT_PARAM = 5
};
#define GSB_L1_UNITS 6
#define GSB_L1_THREADS 1024
#define GSB_L1_REGION_WORDS 8192   /* 128 KiB per CTA */
#define GSB_L1_STEPS 8             /* words per thread per pass: GSB_L1_REGION_WORDS / GSB_L1_THREADS */
#define GSB_L1_PASSES_DEFAULT 8
#define GSB_L1_PASSES_MAX 64
#define GSB_L1_TEX_WIDTH 64        /* words per row of the 2-D texture */
#define GSB_L1_TEX_ROWS 128        /* rows per CTA */
#define GSB_L1_TEX_2D_READS 16384  /* per CTA and addressing mode: x in [-32, 96) by 128 rows */
#define GSB_L1_CONST_WORDS 4096    /* 64 KiB */
#define GSB_L1_PARAM_WORDS 2000    /* 32000 bytes */
#define GSB_L1_RECORDS 64
#define GSB_L1_MAX_LAUNCHES 3
/* the load forms whose warm/cold ratio a result reports, in the order of gsb_l1_result.warm_cold */
enum { GSB_L1_FORM_CA = 0, GSB_L1_FORM_PLAIN = 1, GSB_L1_FORM_EVICT_LAST = 2, GSB_L1_FORM_NC = 3 };
#define GSB_L1_FORMS 4
/* gsb_l1_schedule's answer for a TEX border read outside the array: the texel reads as 0 */
#define GSB_L1_ZERO_TEXEL 0x7FFFFFFFFFFFFFFFll

typedef struct gsb_l1_cfg {
  uint32_t seed;        /* the pattern's seed; 0 = fresh per probe */
  uint32_t seed_expect; /* seed the kernels compare against; 0 = seed */
  uint32_t units;       /* mask of 1 << GSB_L1_UNIT_*; 0 = all */
  uint32_t passes;      /* L1_LOAD and NC passes per form, 1..GSB_L1_PASSES_MAX; 0 = GSB_L1_PASSES_DEFAULT */
} gsb_l1_cfg;

/* One wrong word. offset: byte offset of the expected word's address (buffer units: from the buffer's start; CONST and
 * PARAM: from the bank's or the parameter's start); cls .. flipped_bits: gsb_fault_classify's, filled by the host. */
typedef struct gsb_l1_record {
  uint32_t smid, unit, form, reserved0;
  uint64_t offset;
  uint32_t expected[4];
  uint32_t observed[4];
  uint32_t cls, alias_bit, seed_key, flipped_bits;
} gsb_l1_record;

typedef struct gsb_l1_unit_result {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = the unit did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t ctas_per_sm;    /* cudaOccupancyMaxActiveBlocksPerMultiprocessor of its kernel (logged only) */
  uint64_t words_checked;  /* 16-byte words compared, over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_l1_unit_result;

typedef struct gsb_l1_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units, passes;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t n_records;      /* records filled (the first GSB_L1_RECORDS mismatches) */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs with at least one wrong word */
  gsb_l1_unit_result unit[GSB_L1_UNITS];
  double warm_cold[GSB_L1_FORMS];     /* by GSB_L1_FORM_*: median warm/cold ratio; 0 = not measured */
  gsb_l1_record records[GSB_L1_RECORDS];
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_l1_result;

/* Conditions (gsb_l1_conditions), from the units that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_l1_stats.incomplete) and logged, never a condition. */
enum {
  GSB_L1_CORRUPT = 1u, /* a word read through L1, the read-only path, the texture path, the constant bank or the
                          kernel parameters differs from its pattern word on some SM */
  GSB_L1_FAILED = 2u   /* a launch failed or outlived the watchdog */
};

/* L1 probes of one device since gsb_health_start (counters restart with it; gsb_l1_probe calls count too). */
typedef struct gsb_l1_stats {
  uint64_t probes;     /* L1 probes run */
  uint64_t faults;     /* of which raised at least one GSB_L1_* condition */
  uint64_t skipped;    /* probes that ran no unit (buffer not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_l1_result last;
} gsb_l1_stats;

/* Holds the device while it runs; each launch under the completion watchdog. One transient buffer of sm_count x
 * 128 KiB plus the launch log, taken only while GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free; a probe that cannot take
 * it returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_l1_probe(uint32_t idx, const gsb_l1_cfg *cfg, gsb_l1_result *out);
int gsb_l1_stats_get(uint32_t idx, gsb_l1_stats *out);
/* Pure: the word read number `step` of thread `thread` reads in pass `pass` of form `form` of `unit`, in CTA `cta` of
 * `ctas`: the buffer word index (TEX: of the texel whose value the read returns; GSB_L1_ZERO_TEXEL for a border read
 * outside the array), or the bank's or parameter's word index for CONST and PARAM. Negative gsb_status for a tuple
 * the unit does not read (pass >= GSB_L1_PASSES_MAX, cta >= ctas, step past the form's reads, ...). */
int64_t gsb_l1_schedule(uint32_t unit, uint32_t form, uint32_t pass, uint32_t cta, uint32_t ctas, uint32_t thread,
                        uint32_t step);
/* Pure: GSB_L1_* bits that hold for a result (see above). */
uint32_t gsb_l1_conditions(const gsb_l1_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_l1_text(const gsb_l1_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_l1_probe of device idx, the CTA running on SM `smid` XORs xr into lanes 0-1 of its
 * observed word `index` of `unit` just before the compare, in the unit's first launch only. index: L1_LOAD and NC the
 * region word read in pass 0 of form 0, L1_STORE the region word read back, TEX [0, 8192) the 1-D read of that region
 * word and then the 2-D reads of forms 1 and 2 (GSB_L1_TEX_2D_READS each), CONST and PARAM the word of the per-thread
 * reads. Refused before any device is touched: unit or smid out of range, or index past the unit's words. */
int gsb_test_l1_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
/* test hook: in the next gsb_l1_probe of device idx, the CTA of the first L1_STORE launch on SM `smid` stores nothing,
 * so every word it owed reads back as generation 1 (STALE). Refused before any device is touched when smid is out of
 * range. */
int gsb_test_l1_skip(uint32_t idx, uint32_t smid);
/* gsb_test_l1_table: table sizes, the L1_STORE entry and flags, the TEX 1-D marker */
#define GSB_L1_TABLE_MAX (1u << 20)           /* uint32 table entries */
#define GSB_L1_TABLE_EXPECTED_MAX (1u << 24)  /* uint32 expected entries */
#define GSB_L1_TABLE_REGION_MAX 131072u       /* words of a buffer unit's region per CTA: 2 MiB */
#define GSB_L1_TABLE_ROUNDS_MAX 8u            /* L1_STORE rounds */
#define GSB_L1_STORE_WORD_BITS 17
/* one L1_STORE table entry: thread's store of generation gen (1..255) over bytes [lo, lo + (1 << width_log2)) of
 * region word `word`; 0 = no store */
#define GSB_L1_STORE_ENTRY(word, lo, width_log2, gen) \
  ((uint32_t)(word) | (uint32_t)(lo) << 17 | ((uint32_t)(width_log2) + 1u) << 21 | (uint32_t)(gen) << 24)
#define GSB_L1_TABLE_RESIDENT 1u /* L1_STORE: read the whole region through L1 before the first round */
#define GSB_L1_TABLE_READ_OWN 2u /* L1_STORE: each writer reads its word back right after its store, no barrier */
#define GSB_L1_TEX_1D 0x80000000u /* TEX: a read whose y is this is tex1Dfetch of region word x */
/* test hook: the next gsb_l1_probe of device idx that runs `unit` runs the unit's test-only twin on the chosen reads of
 * `table` (n uint32 entries) instead of the shipped schedule, in every launch of the unit; once. Every CTA c reads its
 * own region of `region_words` words (c * region_words onward), which the FILL launch fills with the seed's pattern:
 *   L1_LOAD, NC  table[p * region_words + k * GSB_L1_THREADS + t]: the region word thread t reads at step k of pass p
 *                (n / region_words passes, each timed as the shipped passes are; L1_LOAD runs the table once with each
 *                of its three load forms); the expected word is computed on the SM. region_words: a multiple of
 *                GSB_L1_THREADS up to GSB_L1_TABLE_REGION_MAX.
 *   L1_STORE     table[0]: GSB_L1_TABLE_* flags; table[1 + r * GSB_L1_THREADS + t]: thread t's store in round r
 *                (GSB_L1_STORE_ENTRY or 0), rounds separated by bar.sync; the value is generation gen's pattern word
 *                of the region word's index. After the last round every word is read back through L1 (form 1) and
 *                compared on the SM with expected[(c * region_words + w) * 4 + lane]; a read of the resident pass is
 *                form 0, a writer's own read-back form 2 (its stored bytes only). region_words as for L1_LOAD, at
 *                most 2^GSB_L1_STORE_WORD_BITS.
 *   TEX          (table[2 r], table[2 r + 1]) = (x, y) of read r = k * GSB_L1_THREADS + t: with y = GSB_L1_TEX_1D,
 *                tex1Dfetch of region word x (form 0); else the 2-D reads at texel (x, c * GSB_L1_TEX_ROWS + y) with
 *                clamp (form 1) and border addressing (form 2). expected[(c * n / 2 + r) * 2 + {0, 1}]: the buffer word
 *                each returns (form 0: slot 0), as int32, -1 for a border read that returns 0. region_words:
 *                GSB_L1_REGION_WORDS.
 *   CONST, PARAM table[k * GSB_L1_THREADS + t]: the bank's or the parameter's word thread t reads at step k (form 1).
 *                region_words: GSB_L1_CONST_WORDS or GSB_L1_PARAM_WORDS.
 * The table and the expected words take their share of the probe's transient buffer. gsb_test_l1_skip applies to an
 * L1_STORE twin too: the CTA on that SM stores nothing in the last round. table == NULL disarms the unit. Refused
 * before any device is touched: an unknown unit; n or n_expected past GSB_L1_TABLE_MAX or GSB_L1_TABLE_EXPECTED_MAX,
 * not a whole number of steps, passes or rounds, or n_expected not a whole number of CTAs; a region size the unit does
 * not take; an index outside the CTA's region, the bank or the parameter; unknown flags; a store that is misaligned,
 * wider than 16 bytes, past the word or of generation 0; two stores to the same byte in one round; a TEX coordinate
 * of magnitude 2^21 or more, a 1-D index outside the region, an expected texel below -1. n_expected other than the
 * device's sm_count CTAs is refused once the device is known. */
int gsb_test_l1_table(uint32_t idx, uint32_t unit, const uint32_t *table, size_t n, const uint32_t *expected,
                      size_t n_expected, uint32_t region_words);

/* ---- Memory-ordering health (not in the reference; opt-in: GSB_OPT_ORDER_PROBE_EVERY_CYCLES) ------------------- */

/*
 * Litmus tests of the PTX memory model at .gpu scope between SMs, through L2. Each unit runs at three distances d
 * (gsb_order_distance): one cooperative launch of sm_count CTAs of GSB_ORDER_THREADS, one per SM (the opt-in maximum
 * of dynamic shared memory), all co-resident. CTA rank r pairs with (r + d) mod n; thread 0 plays the litmus role and
 * warps 1-7 load and store (.cg) the CTA's own 64 KiB scratch region to perturb timing (not judged). Every shared
 * location is one aligned u64 (single-copy atomic): high 32 bits the iteration i, low 32 bits gsb_mix32(seed ^ key ^
 * i), key the location's gsb_order_key; a word whose low half is not that hash is CORRUPT. Every CTA writes its own
 * locations with i = 1..observations and observes its partners' once per iteration:
 *
 *   MP_RELACQ   4 data st.relaxed.gpu, st.release.gpu flag | ld.acquire.gpu flag, 4 data ld.relaxed.gpu
 *   MP_FENCE    relaxed data, fence.acq_rel.gpu, relaxed flag | relaxed flag, fence.acq_rel.gpu, relaxed data
 *               forbidden (both MP units): a data iteration below the flag's
 *   SB_SC       st x_r = i; fence.sc.gpu; ld x_(r+d); ld x_(r-d); fence.sc.gpu. Instance r is (r, r + d): forbidden in
 *               iteration i, both reads of the other's word < i, or both > i
 *   IRIW_SC     instance r: writers r (x) and r + e (y), readers r + 2e (a = ld x; fence.sc; b = ld y) and r + 3e
 *               (c = ld y; fence.sc; d = ld x), e = gsb_order_iriw_distance: forbidden for the k-th observations of
 *               both readers, a > d and c > b
 *   CORR        st.relaxed x = i | two ld.relaxed of x per observation: forbidden, a read older than the one before it
 *               (in the observation or the previous one)
 *   MP_RELAXED  relaxed data, relaxed flag, no fence, both sides: a data iteration below the flag's is counted (weak),
 *               never a condition; it shows whether the test can see reordering at all
 *
 * After the last observation every CTA meets at a grid barrier (release/acquire on a counter, bounded by
 * GSB_ORDER_WAIT_NS plus GSB_ORDER_WAIT_NS_PER_OBS per observation of %globaltimer, since the slowest CTA's loop may
 * trail the fastest's; one that runs out is TIMEOUT, as is the first barrier, before the loop, after GSB_ORDER_WAIT_NS);
 * then every consumer reads each location it
 * observed once more and must see iteration `observations` (older: LOST). Each CTA classifies its own observations
 * (gsb_order_classify) and records CORRUPT, FORBIDDEN and LOST ones; "overlap" counts observations that saw a partner
 * mid-stream (the race window was hit). Overlap and weak counts are logged, never judged.
 */
enum {
  GSB_ORDER_UNIT_MP_RELACQ = 0,
  GSB_ORDER_UNIT_MP_FENCE = 1,
  GSB_ORDER_UNIT_SB_SC = 2,
  GSB_ORDER_UNIT_IRIW_SC = 3,
  GSB_ORDER_UNIT_CORR = 4,
  GSB_ORDER_UNIT_MP_RELAXED = 5
};
#define GSB_ORDER_UNITS 6
#define GSB_ORDER_DISTANCES 3          /* launches per unit: d = 1, n / 2, 1 + seed mod (n - 1) */
#define GSB_ORDER_THREADS 256
#define GSB_ORDER_OBS_DEFAULT 1024
#define GSB_ORDER_OBS_MAX 65536
#define GSB_ORDER_WORDS 5              /* words of one observation (MP: the flag, then 4 data) */
#define GSB_ORDER_RECORDS 64
#define GSB_ORDER_WAIT_NS 100000000ull /* a grid barrier's %globaltimer bound */
#define GSB_ORDER_WAIT_NS_PER_OBS 5000ull /* the second barrier's bound grows by this per observation */
/* outcome classes of one observation (gsb_order_classify) */
enum {
  GSB_ORDER_CLS_ALLOWED = 0,   /* an outcome the model allows, no partner mid-stream */
  GSB_ORDER_CLS_OVERLAP = 1,   /* allowed, and a partner was seen mid-stream */
  GSB_ORDER_CLS_WEAK = 2,      /* MP_RELAXED: a data iteration below the flag's (allowed there) */
  GSB_ORDER_CLS_FORBIDDEN = 3, /* an outcome the model forbids */
  GSB_ORDER_CLS_CORRUPT = 4,   /* a word whose low half is not the hash of its high half */
  GSB_ORDER_CLS_LOST = 5       /* a final read older than the writer's last iteration */
};

typedef struct gsb_order_cfg {
  uint32_t seed;         /* the words' seed; 0 = fresh per probe */
  uint32_t seed_expect;  /* seed the kernels check hashes against; 0 = seed */
  uint32_t units;        /* mask of 1 << GSB_ORDER_UNIT_*; 0 = all */
  uint32_t observations; /* per CTA and launch, 1..GSB_ORDER_OBS_MAX; 0 = GSB_ORDER_OBS_DEFAULT */
} gsb_order_cfg;

/* One CORRUPT, FORBIDDEN or LOST observation. producer: the %smid of the CTAs whose stores or reads its words show,
 * GSB_SM_MAX where there are fewer: MP and CORR the producer r + d; SB the partner r + d (writer of the x_(r+d) this CTA
 * read) and this CTA r itself (writer of the x_r the partner read); IRIW the writers of x and y and the other reader
 * (gsb_order_pairing's order); LOST the writer of the location read. words: as gsb_order_classify takes them (LOST:
 * the final word). */
typedef struct gsb_order_record {
  uint32_t unit, distance;  /* distance: 0..GSB_ORDER_DISTANCES-1 */
  uint32_t cls;             /* GSB_ORDER_CLS_* */
  uint32_t smid;            /* the consumer's */
  uint32_t producer[3];
  uint32_t index;           /* observation (iteration - 1); LOST: the location's slot in gsb_order_pairing's order */
  uint64_t words[GSB_ORDER_WORDS];
} gsb_order_record;

typedef struct gsb_order_unit_result {
  int32_t status;           /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;        /* launches that ran (0 = the unit did not run) */
  uint32_t refused;         /* launches refused for co-residency: skipped, counted, not a condition */
  uint32_t sms_covered;     /* SMs covered, as producer and consumer, by every launch that ran */
  uint64_t words_checked;   /* u64 words read and checked, over every CTA of every launch */
  uint64_t mismatch_words;  /* observations and final reads classed CORRUPT, FORBIDDEN or LOST */
  uint64_t mismatch_bits;   /* bits of CORRUPT words' low halves that differ from the hash */
  uint64_t corrupt, forbidden, lost, timeout;
  uint64_t overlap;         /* observations that saw a partner mid-stream (logged only) */
  uint64_t weak;            /* MP_RELAXED: weak outcomes (logged only) */
  uint64_t kernel_ns;       /* CUDA-event time of its launches */
} gsb_order_unit_result;

typedef struct gsb_order_result {
  int32_t status;           /* GSB_OK iff every unit asked for ran or was refused (outcomes are a result) */
  uint32_t sm_count;        /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units, observations;
  uint32_t distance[GSB_ORDER_DISTANCES];
  uint32_t sms_covered;     /* SMs covered by every unit that ran */
  uint32_t n_records;       /* records filled (the first GSB_ORDER_RECORDS) */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* consumers' SMs with a CORRUPT, FORBIDDEN or LOST observation */
  gsb_order_unit_result unit[GSB_ORDER_UNITS];
  gsb_order_record records[GSB_ORDER_RECORDS];
  uint64_t wall_ns;         /* host time of the whole call */
} gsb_order_result;

/* Conditions (gsb_order_conditions), from the units that ran only. Overlap and weak counts and refused launches are
 * never conditions. */
enum {
  GSB_ORDER_CORRUPT = 1u,   /* a word read back is not a word any writer stored */
  GSB_ORDER_FORBIDDEN = 2u, /* an outcome the PTX memory model forbids at .gpu scope */
  GSB_ORDER_LOST = 4u,      /* a final read after the grid barrier older than the writer's last store */
  GSB_ORDER_TIMEOUT = 8u,   /* a grid barrier ran out: an SM stalled or a store never became visible */
  GSB_ORDER_FAILED = 16u    /* a launch failed or outlived the watchdog */
};

/* Memory-ordering probes of one device since gsb_health_start (counters restart with it; gsb_order_probe calls count
 * too). */
typedef struct gsb_order_stats {
  uint64_t probes;     /* probes run */
  uint64_t faults;     /* of which raised at least one GSB_ORDER_* condition */
  uint64_t skipped;    /* probes that ran no launch (buffer not allocatable, every launch refused): no condition */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs or had a launch refused */
  gsb_order_result last;
} gsb_order_stats;

/* Holds the device while it runs; each launch under the completion watchdog. One transient buffer of sm_count x
 * (80 KiB + 32 B per observation) plus the launch log, taken only while GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free; a
 * probe that cannot take it returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_order_probe(uint32_t idx, const gsb_order_cfg *cfg, gsb_order_result *out);
int gsb_order_stats_get(uint32_t idx, gsb_order_stats *out);
/* Pure: the distance of launch k (0..GSB_ORDER_DISTANCES-1) on n CTAs under seed; 0 when n < 2 or k is out of range. */
uint32_t gsb_order_distance(uint32_t k, uint32_t n, uint32_t seed);
/* Pure: IRIW's step e for distance d on n CTAs: the first of d, d + 1, ... (mod n, skipping 0) with e, 2e and 3e all
 * nonzero mod n; 0 when n < 4. */
uint32_t gsb_order_iriw_distance(uint32_t n, uint32_t d);
/* Pure: the ranks CTA `rank` of n reads in `unit` at distance d, in the order its observation's words take them
 * (MP: the producer; SB: r + d, then r - d whose read of x_r is the partner's half; IRIW: x, y, and the other reader
 * r + e of the instance r - 2e it classifies; CORR: the writer). Returns how many (0: a bad argument). */
int gsb_order_pairing(uint32_t unit, uint32_t n, uint32_t d, uint32_t rank, uint32_t ranks[3]);
/* Pure: the class of one observation. words as the consumer holds them (MP: flag, data 0-3; SB: its read of x_(r+d),
 * the partner's read of x_r; IRIW: a, b, c, d; CORR: the previous read, then the observation's two), keys each word's
 * location key, iteration the SB iteration (1..), seed the seed the hashes are checked against. GSB_ORDER_CLS_CORRUPT
 * for an unknown unit. */
uint32_t gsb_order_classify(uint32_t unit, uint32_t seed, const uint32_t keys[GSB_ORDER_WORDS],
                            const uint64_t words[GSB_ORDER_WORDS], uint32_t iteration);
/* Pure: GSB_ORDER_* bits that hold for a result (see above). */
uint32_t gsb_order_conditions(const gsb_order_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_order_text(const gsb_order_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_order_probe of device idx, the consumer on SM `smid` reports observation `index` of
 * `unit`'s first launch as a forbidden outcome with valid hashes. Refused before any device is touched: unit out of
 * range or MP_RELAXED (which forbids nothing), smid >= GSB_SM_MAX, index >= GSB_ORDER_OBS_MAX. The next probe takes
 * the hook whatever its observations; an index at or past them (known only then) injects nothing. */
int gsb_test_order_inject(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index);
/* test hook: in the next gsb_order_probe of device idx, the producer on SM `smid` writes nothing in the first
 * MP_RELACQ launch, so its consumer reads every location LOST. Refused before any device is touched when smid >=
 * GSB_SM_MAX. */
int gsb_test_order_skip(uint32_t idx, uint32_t smid);

/* ---- Sparse tensor-core health (not in the reference; opt-in: GSB_OPT_SPARSE_PROBE_EVERY_CYCLES) ---------------- */

/*
 * Known-answer checks of the 2:4-sparse tensor-core forms (1:2 for TF32), on every SM. Each unit is one launch as in the
 * tensor-core format check: one CTA per SM, each asking for the opt-in maximum of dynamic shared memory, thread 0
 * recording %smid, a launch that left an SM uncovered repeated up to GSB_SPARSE_MAX_LAUNCHES times. Each computes one
 * 64 x 128 D = A B, A 64 x K stored compressed (K / 2 values per row) with its metadata, and compares every word bit
 * for bit, on the SM, with answers computed exactly on the host (gsb_sparse_expected). K is the logical K:
 *
 *   F16_SP     wgmma.sp m64n128k32 .f32.f16.f16, K = 512
 *   BF16_SP    wgmma.sp m64n128k32 .f32.bf16.bf16, K = 512
 *   TF32_SP    wgmma.sp m64n128k16 .f32.tf32.tf32, K = 256 (1:2)
 *   E4M3_SP    wgmma.sp m64n128k64 .f32.e4m3.e4m3, K = 128
 *   E5M2_SP    wgmma.sp m64n128k64 .f32.e5m2.e5m2, K = 128
 *   S8_SP      wgmma.sp m64n128k64 .s32.s8.s8, K = 512
 *   HMMA_SP    mma.sp::ordered_metadata m16n8k32 .f32.f16.f16.f32, fragments loaded with ldmatrix, K = 512
 *
 * Every (row, group of four K) keeps one of the six increasing index pairs, drawn from the seed (TF32: one of each
 * pair of K). The 16-bit and TF32 units alternate sparsity selector 0 and 1 over their K steps, so both thread pairs'
 * metadata are read. HMMA_SP runs F16_SP's operands, so its answer is F16_SP's. The operands are generated on the
 * device from (unit, seed, row, col); only the expected answers are uploaded, into a transient buffer taken only when
 * GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free. A mismatch never touches the HBM fault log or reports.
 */
enum {
  GSB_SPARSE_UNIT_F16_SP = 0,
  GSB_SPARSE_UNIT_BF16_SP = 1,
  GSB_SPARSE_UNIT_TF32_SP = 2,
  GSB_SPARSE_UNIT_E4M3_SP = 3,
  GSB_SPARSE_UNIT_E5M2_SP = 4,
  GSB_SPARSE_UNIT_S8_SP = 5,
  GSB_SPARSE_UNIT_HMMA_SP = 6
};
#define GSB_SPARSE_UNITS 7
#define GSB_SPARSE_RECORDS 64
#define GSB_SPARSE_MAX_LAUNCHES 3
#define GSB_SPARSE_WORDS 8192 /* D words of one CTA: 64 x 128 */

typedef struct gsb_sparse_cfg {
  uint32_t seed;        /* operands' seed; 0 = fresh per probe */
  uint32_t seed_expect; /* seed of the expected answers; 0 = seed */
  uint32_t units;       /* mask of 1 << GSB_SPARSE_UNIT_*; 0 = all */
  uint32_t reserved0;
} gsb_sparse_cfg;

/* per unit: gsb_tensor_unit_result, its fields meaning the same */
typedef struct gsb_sparse_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs with at least one wrong word */
  gsb_tensor_unit_result unit[GSB_SPARSE_UNITS];
  uint32_t n_records;      /* records filled (the first GSB_SPARSE_RECORDS mismatches) */
  uint32_t reserved0;
  /* unit: GSB_SPARSE_UNIT_*; index: row * 128 + column of D; expected and observed: FP32 (S8_SP: S32) bits */
  gsb_sm_record records[GSB_SPARSE_RECORDS];
  uint64_t expected_ns;    /* host time spent computing the expected answers */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_sparse_result;

/* Conditions (gsb_sparse_conditions), from the units that ran only. Coverage short of sm_count after the relaunches is
 * counted (gsb_sparse_stats.incomplete) and logged, never a condition. */
enum {
  GSB_SPARSE_CORRUPT = 1u, /* a D word differs from its exact answer on some SM */
  GSB_SPARSE_FAILED = 2u   /* a launch failed or outlived the watchdog */
};

/* Sparse probes of one device since gsb_health_start (counters restart with it; gsb_sparse_probe calls count too). */
typedef struct gsb_sparse_stats {
  uint64_t probes;     /* sparse probes run */
  uint64_t faults;     /* of which raised at least one GSB_SPARSE_* condition */
  uint64_t skipped;    /* probes that ran no unit (buffers not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_sparse_result last;
} gsb_sparse_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_sparse_probe(uint32_t idx, const gsb_sparse_cfg *cfg, gsb_sparse_result *out);
int gsb_sparse_stats_get(uint32_t idx, gsb_sparse_stats *out);
/* Pure: the exact answers of `unit` for `seed`: the 8192 words of D in row-major order (FP32 bits, S8_SP's S32).
 * Returns the count, or with out == NULL the count required, or a negative status (GSB_ERR_BUFFER_TOO_SMALL when cap is
 * short, GSB_ERR_INVALID_ARGUMENT for an unknown unit). */
int64_t gsb_sparse_expected(uint32_t unit, uint32_t seed, uint32_t *out, size_t cap);
/* Pure: GSB_SPARSE_* bits that hold for a result (see above). */
uint32_t gsb_sparse_conditions(const gsb_sparse_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_sparse_text(const gsb_sparse_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_sparse_probe of device idx, the CTA running on SM `smid` XORs xr into its D word `index`
 * of `unit` just before the compare; once. Refused before any device is touched: unit, smid or index out of range, or
 * xr wider than 32 bits. */
int gsb_test_sparse_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
/* test hook: the next gsb_sparse_probe of device idx that runs `unit` runs it on chosen operands instead of the seed's:
 * every launch of the unit in that probe computes D = A B, A[i] being row i of the compressed
 * a[i * K / 2 + c] * 2^sa[i] spread by pattern[i * G + q] (G = K / 4 groups of four, pattern 0-5 the index pairs
 * (0,1) (0,2) (0,3) (1,2) (1,3) (2,3); TF32_SP: G = K / 2 groups of two, pattern 0 or 1 the element kept), and
 * B[k][j] = b[k * 128 + j] * 2^sb[j], through the same conversion, layout, metadata, instruction and compare, and
 * compares D with expected[row * 128 + col] (as gsb_sparse_expected gives them). Once. a == NULL disarms it. Refused
 * with GSB_ERR_INVALID_ARGUMENT before any device is touched: an unknown unit, an integer outside the unit's range, a
 * scale outside its range, a pattern outside the unit's set, or an expected word wider than 32 bits. */
int gsb_test_sparse_operands(uint32_t idx, uint32_t unit, const int32_t *a, const uint8_t *pattern, const int32_t *b,
                             const int32_t *sa, const int32_t *sb, const uint64_t *expected);

/* ---- Shared-memory atomic health (not in the reference; opt-in: GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES) ------- */

/*
 * Bit-exact checks of the atomic unit of every SM's shared memory (ATOMS), which histograms, radix sorts, block
 * reductions and work queues run on. Each unit is one launch of one CTA per SM (GSB_SHARED_ATOMIC_THREADS threads, the
 * opt-in maximum of dynamic shared memory, so no two CTAs share an SM; thread 0 records %smid); a launch that left an
 * SM uncovered is repeated up to GSB_SHARED_ATOMIC_MAX_LAUNCHES times. Each CTA writes the unit's starting words into
 * an area of its own shared memory (GSB_SHARED_ATOMIC_AREA_BYTES: a spread region of GSB_SHARED_ATOMIC_SPREAD_BYTES,
 * then GSB_SHARED_ATOMIC_HOT_WORDS hot slots GSB_SHARED_ATOMIC_HOT_STRIDE bytes apart), issues the unit's atomics, and
 * after a barrier compares every word of the area bit for bit, on the SM, with words computed on the host
 * (gsb_shared_atomic_expected) and uploaded into a transient buffer. Two phases:
 *
 *   spread  every thread issues one atomic in each of 2 x E rounds (E = spread bytes / 256 / unit bytes). Even rounds
 *           reach every word once, conflict-free, each lane's bank rotating by round and warp; in odd rounds the 32
 *           lanes of a warp hit 32 words of one bank at different addresses. Not for TICKET and CAS.
 *   hot     lane l of every warp hits hot slot l GSB_SHARED_ATOMIC_HOT_REPS times; the 32 slots lie in one bank, so the
 *           lanes of a warp never share an address and all warps contend on the same word.
 *
 * Every operand is a function of (unit, seed, thread, round or repetition), never of %smid or blockIdx, so every CTA's
 * area ends the same. Integer add, and/or/xor and min/max commute; inc and dec take one bound per word, so every order
 * gives the same word; float contributions are integers whose sum of magnitudes stays under the type's exact bound.
 * TICKET and CAS write their tickets, exchanged values and final exchange words to per-CTA slots of the buffer
 * (gsb_shared_atomic_slot in csrc/gsb_shared_atomic.h), checked on the host as permutations. Every CAS loop ends at a
 * GSB_SHARED_ATOMIC_CAS_WAIT_NS %globaltimer deadline. The log goes to the result only, never to the HBM fault log or
 * reports.
 *
 * DSMEM and REDAS run in thread-block clusters, first of 2 CTAs and then of the largest size the SM-to-SM check uses (16,
 * or 8 where 16 cannot be scheduled), as many clusters as fit at once. Every CTA writes its area's starting words; a
 * cluster barrier; then every thread sends its atomics to every OTHER rank's area (an address in the CTA's own rank would
 * take the local ATOMS path), each operand a function of (unit, seed, sender rank, thread, op). REDAS's receiver arms its
 * mbarrier with exactly the bytes its peers send before that barrier and waits for them with a
 * GSB_SHARED_ATOMIC_CAS_WAIT_NS %globaltimer deadline; a wait that runs out is counted as a timeout and the area is
 * checked anyway. DSMEM ends its sends with a cluster barrier. Each rank then compares its area with the words for its
 * rank and cluster size, and a last cluster barrier keeps every CTA alive until all of its cluster have compared, so no
 * peer can reach the shared memory of a CTA that has exited.
 */
enum {
  GSB_SHARED_ATOMIC_UNIT_INT32 = 0,  /* red.shared add.u32, and/or/xor.b32, min/max .s32 and .u32, inc/dec.u32, by word */
  GSB_SHARED_ATOMIC_UNIT_WIDE = 1,   /* red.shared add.u64, and/or/xor.b64, min.s64, max.u64, by word (8-byte words) */
  GSB_SHARED_ATOMIC_UNIT_FLOAT = 2,  /* red.shared add.f32, add.f64, add.noftz.f16x2, add.noftz.bf16x2, by word (8-byte
                                        words; the 32-bit forms on the low half) */
  GSB_SHARED_ATOMIC_UNIT_TICKET = 3, /* atom.shared add.u32 of 1, exch.b32, exch.b64, exch.b128 on the hot slots */
  GSB_SHARED_ATOMIC_UNIT_CAS = 4,    /* atom.shared cas.b32, cas.b64, cas.b128 increment loops on the hot slots */
  GSB_SHARED_ATOMIC_UNIT_DSMEM = 5,  /* red.shared::cluster add.u32, add.u64, add.f32 and an atom.shared::cluster
                                        cas.b32 increment loop into every other rank's area */
  GSB_SHARED_ATOMIC_UNIT_REDAS = 6   /* red.async ... mbarrier::complete_tx::bytes add.u32, add.u64, xor.b32, max.s32,
                                        inc.u32 into every other rank's area, completing on the receiver's mbarrier */
};
#define GSB_SHARED_ATOMIC_UNITS 7
#define GSB_SHARED_ATOMIC_RECORDS 64
#define GSB_SHARED_ATOMIC_MAX_LAUNCHES 3
#define GSB_SHARED_ATOMIC_THREADS 256
#define GSB_SHARED_ATOMIC_SPREAD_BYTES 8192u
#define GSB_SHARED_ATOMIC_HOT_WORDS 32u
#define GSB_SHARED_ATOMIC_HOT_STRIDE 128u
#define GSB_SHARED_ATOMIC_HOT_REPS 4u
#define GSB_SHARED_ATOMIC_AREA_BYTES (GSB_SHARED_ATOMIC_SPREAD_BYTES + GSB_SHARED_ATOMIC_HOT_WORDS * GSB_SHARED_ATOMIC_HOT_STRIDE)
#define GSB_SHARED_ATOMIC_AREA_WORDS (GSB_SHARED_ATOMIC_AREA_BYTES / 4u) /* the 4-byte words compared and recorded */
#define GSB_SHARED_ATOMIC_CAS_WAIT_NS 100000000u /* bound of every CAS loop: 100 ms */
#define GSB_SHARED_ATOMIC_NO_ID 0xFFFFFFFFu      /* what a slot starts as */
#define GSB_SHARED_ATOMIC_NO_SM 0xFFFFFFFFu
enum {
  GSB_SHARED_ATOMIC_REC_WORD = 0,   /* index: 4-byte word of the area (DSMEM, REDAS: rank x GSB_SHARED_ATOMIC_AREA_WORDS +
                                       word); expected and observed: that word */
  GSB_SHARED_ATOMIC_REC_SLOT = 1,   /* index: slot entry (gsb_shared_atomic_slot / 4); expected: the contributor count;
                                       observed: its first word, not a distinct valid id or exchanged value */
  GSB_SHARED_ATOMIC_REC_TICKET = 2, /* index: hot slot; expected: the count; observed: a ticket at or past it */
  GSB_SHARED_ATOMIC_REC_TORN = 3    /* index: hot slot; a CAS.b128 returned a pair whose halves do not belong together:
                                       expected the hash of observed's count, observed the returned upper half */
};

typedef struct gsb_shared_atomic_cfg {
  uint32_t units;       /* mask of 1 << GSB_SHARED_ATOMIC_UNIT_*; 0 = all */
  uint32_t seed;        /* 0 = fresh per probe */
  uint32_t seed_expect; /* seed the expected words are computed from; 0 = seed */
  uint32_t reserved0;
} gsb_shared_atomic_cfg;

/* One wrong word, slot, ticket or pair; smid is the SM that owns the area or slots (GSB_SHARED_ATOMIC_NO_SM: none). */
typedef struct gsb_shared_atomic_record {
  uint32_t smid;
  uint32_t unit;     /* GSB_SHARED_ATOMIC_UNIT_* */
  uint32_t kind;     /* GSB_SHARED_ATOMIC_REC_* */
  uint32_t index;
  uint64_t expected, observed;
} gsb_shared_atomic_record;

typedef struct gsb_shared_atomic_run {
  int32_t status;          /* GSB_OK, or the first failed launch's gsb_status (GSB_ERR_TIMEOUT: outlived the watchdog) */
  uint32_t launches;       /* 0 = the unit did not run */
  uint32_t sms_covered;    /* distinct %smid over its launches */
  uint32_t hook_cta;       /* the blockIdx that applied gsb_test_shared_atomic_skip; GSB_SHARED_ATOMIC_NO_SM: none */
  uint32_t cluster_launches[2]; /* DSMEM, REDAS: launches of each cluster size (gsb_shared_atomic_result.cluster_n) */
  uint32_t clusters[2];         /* and the clusters of each of those launches; 0 for the other units */
  uint64_t atomics_issued; /* atomic instructions issued (CAS: successful swaps) */
  uint64_t words_checked;  /* area words compared, over every CTA of every launch */
  uint64_t mismatch_words, mismatch_bits;
  uint64_t ticket_faults;  /* TICKET, CAS: slots without a distinct valid id or value, tickets out of range, torn pairs */
  uint64_t timeouts;       /* CAS loops and REDAS mbarrier waits that ran out of GSB_SHARED_ATOMIC_CAS_WAIT_NS */
  uint64_t cas_max_ns;     /* CAS: the longest loop of any thread, by %globaltimer */
  uint64_t kernel_ns;      /* CUDA-event time of its launches */
} gsb_shared_atomic_run;

typedef struct gsb_shared_atomic_result {
  int32_t status;          /* GSB_OK iff every unit asked for ran every launch (mismatches and faults are a result) */
  uint32_t sm_count;       /* the device's multiProcessorCount = the grid of every launch */
  uint32_t seed, seed_expect, units;
  uint32_t sms_covered;    /* SMs covered by every unit that ran */
  uint32_t covered[GSB_SM_MAX / 32];  /* their bitmap, bit smid */
  uint32_t faulty[GSB_SM_MAX / 32];   /* SMs a record names */
  uint32_t cluster_n[2];   /* DSMEM, REDAS: the cluster sizes run (2, then 16 or 8); 0 when no cluster unit ran */
  gsb_shared_atomic_run run[GSB_SHARED_ATOMIC_UNITS];
  uint32_t n_records;      /* records filled (the first GSB_SHARED_ATOMIC_RECORDS) */
  uint32_t reserved0;
  gsb_shared_atomic_record records[GSB_SHARED_ATOMIC_RECORDS];
  uint64_t expected_ns;    /* host time spent on the expected words */
  uint64_t wall_ns;        /* host time of the whole call */
} gsb_shared_atomic_result;

/* Conditions (gsb_shared_atomic_conditions), from the units that ran only. Coverage short of sm_count after the
 * relaunches is counted (gsb_shared_atomic_stats.incomplete) and logged, never a condition. */
enum {
  GSB_SHARED_ATOMIC_CORRUPT = 1u, /* a final word, a slot, a ticket or a CAS pair is wrong on some SM */
  GSB_SHARED_ATOMIC_FAILED = 2u   /* a launch failed or outlived the watchdog, or a CAS loop or REDAS wait ran out of
                                     its deadline */
};

/* Shared-memory atomic probes of one device since gsb_health_start (counters restart with it; gsb_shared_atomic_probe
 * calls count too). */
typedef struct gsb_shared_atomic_stats {
  uint64_t probes;
  uint64_t faults;     /* probes that raised at least one GSB_SHARED_ATOMIC_* condition */
  uint64_t skipped;    /* probes that ran no launch (the buffer was not allocatable): no condition, no event */
  uint64_t incomplete; /* probes in which some unit covered fewer than sm_count SMs */
  gsb_shared_atomic_result last;
} gsb_shared_atomic_stats;

/* Holds the device while it runs; each launch under the completion watchdog. A probe that cannot take its buffer
 * returns GSB_ERR_OUT_OF_MEMORY and counts as skipped. */
int gsb_shared_atomic_probe(uint32_t idx, const gsb_shared_atomic_cfg *cfg, gsb_shared_atomic_result *out);
int gsb_shared_atomic_stats_get(uint32_t idx, gsb_shared_atomic_stats *out);
/* Pure: the GSB_SHARED_ATOMIC_AREA_WORDS 4-byte words of one CTA's area after a clean run of `unit` under `seed`
 * (little-endian, as shared memory holds them; TICKET's exchange words, which the kernel does not compare, hold their
 * starting value): for DSMEM and REDAS the area of rank `rank` of a cluster of `cluster` CTAs (2, 4, 8 or 16), for the
 * other units cluster 1 and rank 0. The words do not depend on the SM count. Returns the count (with out == NULL too),
 * GSB_ERR_BUFFER_TOO_SMALL when cap is short, or GSB_ERR_INVALID_ARGUMENT for an unknown unit, a cluster size or rank
 * the unit does not take, or a float word whose sum of magnitudes would reach its exact bound. */
int64_t gsb_shared_atomic_expected(uint32_t unit, uint32_t seed, uint32_t cluster, uint32_t rank, uint32_t *out,
                                   size_t cap);
/* Pure: GSB_SHARED_ATOMIC_* bits that hold for a result (see above). */
uint32_t gsb_shared_atomic_conditions(const gsb_shared_atomic_result *r);
/* Pure: the one-line text both daemons log for a result. uuid may be NULL. Returns like gsb_sm_text. */
int64_t gsb_shared_atomic_text(const gsb_shared_atomic_result *r, const char *uuid, char *buf, size_t cap);
/* test hook: on the next gsb_shared_atomic_probe of device idx, in the first launch of `unit`, the CTA on SM `smid`
 * XORs xr into its observed area word `index` (4-byte words) just before the compare; once. Refused before any device
 * is touched: unit, smid or index out of range, or xr wider than 32 bits. */
int gsb_test_shared_atomic_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr);
/* test hook: on the next gsb_shared_atomic_probe of device idx, in the first launch of `unit` (DSMEM, REDAS: of clusters
 * of 2), the CTA on SM `smid` issues none of the unit's atomics (it still writes its starting words, takes part in every
 * cluster barrier and compares its area); once. Refused before any
 * device is touched: unit or smid out of range. */
int gsb_test_shared_atomic_skip(uint32_t idx, uint32_t smid, uint32_t unit);

/* ---- Allocate (a12, a13): wire bytes in, wire bytes out ---------------------------------- */

typedef struct gsb_pod {
  const char *name;
  const char *ns;
  const char *uid;
  uint64_t gpu_mem_limit;   /* Σ spec.containers[].resources.limits["aliyun.com/gpu-mem"] (podutils.go:122-131) */
  uint64_t assume_time;     /* ALIYUN_COM_GPU_MEM_ASSUME_TIME parsed as uint64, 0 on failure (podutils.go:64-75) */
  int32_t gpu_idx;          /* ALIYUN_COM_GPU_MEM_IDX via Atoi, -1 if absent/unparsable (podutils.go:37-61) */
  uint8_t has_assume_time;  /* annotation key present */
  uint8_t has_assigned;     /* ALIYUN_COM_GPU_MEM_ASSIGNED present */
  uint8_t assigned_is_false;/* value == "false" */
  uint8_t on_node;          /* spec.nodeName == $NODE_NAME (podmanager.go:187-193); others are skipped */
} gsb_pod;

typedef struct gsb_allocate_ctx {
  const char *const *uuids; /* per GPU, NVML order */
  const uint32_t *minors;   /* per GPU: devNameMap[uuid] */
  uint32_t n_gpus;
  uint32_t slices;          /* getGPUMemory() */
  int32_t unit_gib;         /* metric == GiBPrefix */
  int32_t disable_cgpu_isolation;
  int32_t pods_unique;      /* caller guarantees that no two on-node pods share a uid (a table keyed by uid):
                               getPendingPodsInNode's dedupe (podmanager.go:162-212) is then a no-op and is skipped.
                               0 = dedupe as the reference does */
} gsb_allocate_ctx;

enum {
  GSB_ALLOC_MATCHED = 1,     /* pod found; caller must PATCH pod `*pod_index` (allocate.go:130-149) */
  GSB_ALLOC_SINGLE_GPU = 2,  /* no pod matched, one GPU: shortcut response (allocate.go:151-177) */
  GSB_ALLOC_ERR_RESPONSE = 3 /* buildErrResponse (allocate.go:24-39) */
};

/*
 * Decode AllocateRequest wire bytes, run the reference's selection over `pods` (candidate filter
 * podutils.go:78-119, order podmanager.go:241-262, first pod whose limit == request
 * allocate.go:78-88), and encode the AllocateResponse wire bytes (env keys emitted in sorted key
 * order — gogo iterates a Go map, so any order is conformant; see DESIGN.md). Returns
 * GSB_ALLOC_* (>0) or a negative status. `*pod_index` = index into pods of the matched pod or -1.
 */
int gsb_allocate(const gsb_allocate_ctx *ctx, const gsb_pod *pods, uint32_t n_pods,
                 const uint8_t *req, size_t req_len, uint8_t *resp, size_t resp_cap,
                 size_t *resp_len, int32_t *pod_index, uint32_t *pod_req_gpu);
/* Re-encode the error response for a request (PATCH failed after a match: allocate.go:133-148). */
int gsb_allocate_err_response(const gsb_allocate_ctx *ctx, const uint8_t *req, size_t req_len,
                              uint8_t *resp, size_t resp_cap, size_t *resp_len);
/* {"metadata":{"annotations":{"ALIYUN_COM_GPU_MEM_ASSIGNED":"true","ALIYUN_COM_GPU_MEM_ASSUME_TIME":"<ns>"}}}
 * (podutils.go:27-35). Returns length or negative status. */
int gsb_patch_assigned_body(uint64_t now_unix_ns, char *buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* GPUSHARE_B200_H_ */
