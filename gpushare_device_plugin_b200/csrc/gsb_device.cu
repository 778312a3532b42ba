/*
 * gsb_device.cu — device layer of libgpushare_b200.so: lifecycle, inventory, arena, probe, cycle,
 * health events. Host code; the kernels live in hbm_probe_sm90a.cu.
 *
 * Replaces the reference's go-nvml use (vendor/github.com/NVIDIA/gpu-monitoring-tools/bindings/go/
 * nvml/{nvml.go,bindings.go,nvml_dl.c}) for the inventory+health path:
 *   - nvml.Init (nvml_dl.c:21-28: dlopen + nvmlInit_v2)             -> gsb_init
 *   - nvml.NewDevice's 11 getters + sysfs read (nvml.go:297-359)     -> 4 NVML calls per device
 *     (handle, UUID, minor, MemoryInfo v1) + 2 CUDA driver calls that cross-check identity; the
 *     eight getters whose values the plugin discards (name, power, PCI, BAR1, link gen/width,
 *     clocks, NUMA) are not made
 *   - total MiB = nvmlMemory_t.total / (1024*1024) (bindings.go:346-349): SAME call, SAME struct, so
 *     the slice count is bit-exact by construction. cuDeviceTotalMem is 503 316 480 B smaller on an
 *     H100 80GB (85 017 493 504 vs 85 520 809 984 B) and is reported only as information.
 *   - RegisterEventForDevice x fake devices (nvidia.go:104-117; O(S*N^2) NVML calls) -> one
 *     nvmlDeviceRegisterEvents per GPU
 *   - WaitForEvent (bindings.go:134-146) -> gsb_health_wait over a queue fed by the XID thread and
 *     by the active HBM prober
 *
 * libcuda.so.1 and libnvidia-ml.so.1 are dlopen'ed at gsb_init, never linked: the library loads on
 * a GPU-less builder (symbol check in tests/test_abi.py) and reports GSB_ERR_LIBRARY_NOT_FOUND there.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nvml.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <tuple>
#include <unordered_map>
#include <utility>
#include <vector>

#include "gsb_atomic.h"
#include "gsb_cluster.h"
#include "gsb_internal.h"
#include "gsb_sm_kat.h"
#include "gsb_tensor_kat.h"
#include "gsb_sfu_kat.h"
#include "gsb_l1.h"
#include "gsb_order.h"
#include "gsb_sparse_kat.h"
#include "gsb_shared_atomic.h"

namespace {

// ------------------------------------------------------------------ error text

thread_local char tl_error[512];

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tl_error, sizeof tl_error, fmt, ap);
  va_end(ap);
}

uint64_t now_ns() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}

// ------------------------------------------------------------------ dlopen'ed entry points

struct DriverApi {
  void *lib = nullptr;
  CUresult (*cuInit)(unsigned) = nullptr;
  CUresult (*cuDeviceGet)(CUdevice *, int) = nullptr;
  CUresult (*cuDeviceGetUuid)(CUuuid *, CUdevice) = nullptr;
  CUresult (*cuDeviceTotalMem)(size_t *, CUdevice) = nullptr;
  CUresult (*cuMemGetInfo)(size_t *, size_t *) = nullptr;
  CUresult (*cuMemGetAllocationGranularity)(size_t *, const CUmemAllocationProp *,
                                            CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*cuMemAddressReserve)(CUdeviceptr *, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*cuMemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*cuMemCreate)(CUmemGenericAllocationHandle *, size_t, const CUmemAllocationProp *,
                          unsigned long long) = nullptr;
  CUresult (*cuMemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*cuMemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*cuMemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*cuMemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc *, size_t) = nullptr;
  CUresult (*cuGetErrorString)(CUresult, const char **) = nullptr;
};

struct NvmlApi {
  void *lib = nullptr;
  nvmlReturn_t (*init)(void) = nullptr;
  nvmlReturn_t (*shutdown)(void) = nullptr;
  const char *(*errorString)(nvmlReturn_t) = nullptr;
  nvmlReturn_t (*getCount)(unsigned *) = nullptr;
  nvmlReturn_t (*handleByIndex)(unsigned, nvmlDevice_t *) = nullptr;
  nvmlReturn_t (*getUUID)(nvmlDevice_t, char *, unsigned) = nullptr;
  nvmlReturn_t (*getMinor)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getMemoryInfo)(nvmlDevice_t, nvmlMemory_t *) = nullptr;  // v1 struct: the reference's
  nvmlReturn_t (*getPciInfo)(nvmlDevice_t, nvmlPciInfo_t *) = nullptr;
  nvmlReturn_t (*eventSetCreate)(nvmlEventSet_t *) = nullptr;
  nvmlReturn_t (*registerEvents)(nvmlDevice_t, unsigned long long, nvmlEventSet_t) = nullptr;
  nvmlReturn_t (*eventSetWait)(nvmlEventSet_t, nvmlEventData_t *, unsigned) = nullptr;
  nvmlReturn_t (*eventSetFree)(nvmlEventSet_t) = nullptr;
  // ECC and row-remapper health (GSB_OPT_ECC_HEALTH, gsb_ecc_status_get)
  nvmlReturn_t (*getEccMode)(nvmlDevice_t, nvmlEnableState_t *, nvmlEnableState_t *) = nullptr;
  nvmlReturn_t (*getTotalEccErrors)(nvmlDevice_t, nvmlMemoryErrorType_t, nvmlEccCounterType_t,
                                    unsigned long long *) = nullptr;
  nvmlReturn_t (*getMemoryErrorCounter)(nvmlDevice_t, nvmlMemoryErrorType_t, nvmlEccCounterType_t, nvmlMemoryLocation_t,
                                        unsigned long long *) = nullptr;
  nvmlReturn_t (*getRemappedRows)(nvmlDevice_t, unsigned *, unsigned *, unsigned *, unsigned *) = nullptr;
  nvmlReturn_t (*getRowRemapperHistogram)(nvmlDevice_t, nvmlRowRemapperHistogramValues_t *) = nullptr;
  // PCIe link health (gsb_link_status_get, gsb_link_probe)
  nvmlReturn_t (*getCurrPcieLinkGeneration)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getCurrPcieLinkWidth)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getMaxPcieLinkGeneration)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getMaxPcieLinkWidth)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getGpuMaxPcieLinkGeneration)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getPcieReplayCounter)(nvmlDevice_t, unsigned *) = nullptr;
  // SM stress telemetry (gsb_sm_stress; read-only)
  nvmlReturn_t (*getTotalEnergyConsumption)(nvmlDevice_t, unsigned long long *) = nullptr;
  nvmlReturn_t (*getPowerUsage)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getEnforcedPowerLimit)(nvmlDevice_t, unsigned *) = nullptr;
  nvmlReturn_t (*getTemperature)(nvmlDevice_t, nvmlTemperatureSensors_t, unsigned *) = nullptr;
  nvmlReturn_t (*getClockInfo)(nvmlDevice_t, nvmlClockType_t, unsigned *) = nullptr;
  nvmlReturn_t (*getClocksEventReasons)(nvmlDevice_t, unsigned long long *) = nullptr;
};

template <typename F>
bool load_sym(void *lib, F &fn, const char *name, const char *alt = nullptr) {
  fn = reinterpret_cast<F>(dlsym(lib, name));
  if (!fn && alt) fn = reinterpret_cast<F>(dlsym(lib, alt));
  return fn != nullptr;
}

// ------------------------------------------------------------------ state

constexpr uint64_t kGranuleBytes = 64ull << 20;  // generation-table granularity
constexpr uint32_t kGranuleShiftWords = 22;      // log2(64 MiB / 16 B)

struct Chunk {
  CUmemGenericAllocationHandle handle;
  size_t size;
};

struct Snapshot {
  char uuid[GSB_UUID_BUFFER_SIZE] = {0};
  unsigned char uuid_bytes[16] = {0};  // the same UUID as the CUDA driver reports it (cuDeviceGetUuid)
  bool uuid_parsed = false;
  uint32_t minor = 0;
  uint64_t total = 0, free = 0;
  uint64_t taken_ns = 0;
  uint64_t refreshes = 0;
};

// what a device worker runs: plain data, no allocation per hand-off
struct Job {
  enum Kind { NONE, PROBE, CYCLE } kind = NONE;
  uint32_t idx = 0;
  const gsb_probe_cfg *cfg = nullptr;
  gsb_probe_result *probe_out = nullptr;
  uint64_t cycle_no = 0, window_bytes = 0;
  int unit_gib = 1;
  uint32_t variant = 0;
  gsb_cycle_result *cycle_out = nullptr;
  int rc = 0;
};

// What a device keeps for one periodic health check (kChecks). stats, raised and hooks are guarded by smu, seed by mu.
template <typename Stats, typename Hooks>
struct CheckState {
  Stats stats{};        // since gsb_health_start (the check's probe calls outside a session count too)
  uint32_t raised = 0;  // conditions already raised this health session
  uint32_t seed = 0;    // seeds handed out to the check's probes
  Hooks hooks{};        // gsb_test_* hooks: applied by the check's next probe, then dropped
};

struct Device {
  nvmlDevice_t nvml{};
  int ordinal = -1;
  CUdevice cudev = 0;
  char uuid[GSB_UUID_BUFFER_SIZE] = {0};
  char bus_id[GSB_BUSID_BUFFER_SIZE] = {0};
  uint32_t minor = 0;
  uint32_t sm_count = 0, cc_major = 0, cc_minor = 0;
  uint64_t cuda_total = 0;

  std::mutex mu;  // serialises arena + launches of this device
  bool ready = false;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  gsb_kernel_out *out_host = nullptr, *out_dev = nullptr;
  gsb_partial *partials = nullptr;
  unsigned int *ticket = nullptr;
  unsigned long long *tile_counter = nullptr;  // [2]: BULKD tile claims, verify tiles a refill has consumed
  uint32_t *seed_table = nullptr;  // generation that last wrote each granule (written only by the kernels' last CTA)
  uint32_t launch_seq = 0;
  gsb_fault_log *fault_log = nullptr;                                // device memory: the kernels' fault log
  gsb_fault_log *fault_host = nullptr, *fault_host_dev = nullptr;    // mapped host copy a faulted launch leaves

  CUdeviceptr va = 0;
  size_t va_size = 0;
  std::vector<Chunk> chunks;
  uint64_t arena_bytes = 0;
  std::map<uint64_t, gsb_launch_geom> geoms;  // (op, variant, grid request) -> resolved launch geometry
  uint32_t next_gen = 1;
  bool faulted = false;  // prober: sticky
  std::vector<uint8_t> bits_scratch;  // Unhealthy bit string of this device's own list (faulted devices only)
  bool transient_arena = false;  // the mapped arena is a transient window that could not be given back yet (wedged launch)
  bool wedged = false;   // a launch outlived the watchdog and is still on the stream: no new launches until it drains

  // inventory snapshot: what NVML said at the last (re)start-time query (server.go:39 -> nvidia.go:53-89 queries
  // once per plugin start, never per poll). The cycle serves identity/total from here and re-validates identity on
  // the CUDA side; gsb_device_info_get / gsb_inventory_refresh / the low-rate refresher rewrite it.
  std::mutex smu;
  Snapshot snap;
  gsb_health_stats hstats{};  // prober thread of this device; guarded by smu
  gsb_fault_report fault_first{}, fault_last{};  // evidence of the first / most recent faulted launch; guarded by smu
  // ECC health (GSB_OPT_ECC_HEALTH); guarded by smu
  gsb_ecc_status ecc_baseline{};  // the health session's gsb_health_start-time answer
  uint32_t ecc_raised = 0;        // GSB_ECC_* conditions already raised this session
  gsb_ecc_stats ecc_stats{};      // prober thread of this device
  bool ecc_override_set = false;  // gsb_test_ecc_override
  gsb_ecc_status ecc_override{};
  // PCIe link health
  struct LinkCorrupt {
    uint32_t phase;
    uint64_t offset;
    uint32_t xr[4];
  };
  CheckState<gsb_link_stats, std::vector<LinkCorrupt>> link;  // hooks: gsb_test_link_corrupt
  bool link_override_set = false;                             // gsb_test_link_override; guarded by smu
  gsb_link_status link_override{};
  void *link_kept[2] = {nullptr, nullptr};  // pinned buffers a wedged link launch still uses (guarded by mu)
  // copy-engine health
  struct CopyCorrupt {
    uint32_t dir;
    uint64_t offset;
    uint32_t xr[4];
  };
  struct CopyHooks {
    std::vector<CopyCorrupt> corrupt;  // gsb_test_copy_corrupt
    uint32_t skip = 0;                 // gsb_test_copy_skip: bit k = direction k's copy is not issued, once
  };
  CheckState<gsb_copy_stats, CopyHooks> copy;
  // the H2D and D2H copies' streams (the D2D copy runs on `stream`) and each copy's timing events, made by the first
  // copy probe (guarded by mu)
  cudaStream_t copy_streams[2] = {nullptr, nullptr};
  cudaEvent_t copy_ev[GSB_COPY_DIRECTIONS][2] = {};
  // buffers a wedged copy or verify still uses, given back once every stream has drained (guarded by mu)
  void *copy_kept_dev[3] = {nullptr, nullptr, nullptr};
  void *copy_kept_host[2] = {nullptr, nullptr};
  // SM compute health (the SM stress takes its seeds from the same counter)
  struct SmCorrupt {
    bool armed = false;
    uint32_t smid = 0, index = 0;
    uint64_t xr = 0;
  };
  struct SmHooks {
    std::array<SmCorrupt, GSB_SM_UNITS> corrupt;  // gsb_test_sm_corrupt
    // gsb_test_sm_operands: per tensor unit, the 8192 expected D words then the operand table (gsb_sm_table_*), taken
    // by the next gsb_sm_probe that runs the unit; empty = not armed
    std::vector<uint32_t> operands[GSB_SM_UNITS];
  };
  CheckState<gsb_sm_stats, SmHooks> sm;
  // buffer a wedged SM-check, SM-stress, SM-to-SM or L2 atomic launch still uses, and the texture objects over it a
  // wedged L1 launch may still read (guarded by mu)
  void *sm_kept = nullptr;
  std::vector<cudaTextureObject_t> sm_kept_tex;
  struct StressCorrupt {
    bool armed = false;
    uint32_t smid = 0, unit = 0, index = 0, xr = 0, slice = 0;
  };
  StressCorrupt stress_corrupt;  // gsb_test_stress_corrupt: applied by the next gsb_sm_stress, then dropped (smu)
  // SM-to-SM health
  struct ClusterHook {
    bool corrupt = false, skip = false;
    uint32_t corrupt_smid = 0, index = 0, skip_smid = 0;
    uint64_t xr = 0;
  };
  CheckState<gsb_cluster_stats, std::array<ClusterHook, GSB_CLUSTER_PATHS>> cluster;  // hooks: gsb_test_cluster_*
  // gsb_test_cluster_script, by path and size index (guarded by smu): taken by the next probe that runs the pair
  struct ClusterScript {
    bool armed = false;
    gsb_cluster_script script = {};
  };
  std::array<std::array<ClusterScript, GSB_CLUSTER_SIZES>, GSB_CLUSTER_PATHS> cluster_scripts;
  // L2 atomic health
  struct AtomicHook {
    bool corrupt = false, skip = false;
    uint32_t word = 0, skip_smid = 0;
    uint64_t xr = 0;
  };
  CheckState<gsb_atomic_stats, std::array<AtomicHook, GSB_ATOMIC_OPS>> atomic;  // hooks: gsb_test_atomic_*
  // gsb_test_atomic_values, by op (guarded by smu): the starting and expected words in the device's bytes, the table
  struct AtomicValues {
    bool armed = false;
    std::vector<unsigned char> init, expected;
    std::vector<uint64_t> table;
  };
  std::array<AtomicValues, GSB_ATOMIC_OPS> atomic_values;
  // tensor-core format health: the SM check's hooks, by GSB_TENSOR_UNIT_* (gsb_test_tensor_corrupt, and
  // gsb_test_tensor_operands' expected words, gsb_tensor_word_bytes each, then its operand table)
  static_assert(GSB_TENSOR_UNITS == GSB_SM_UNITS, "SmHooks has one slot per tensor unit");
  CheckState<gsb_tensor_stats, SmHooks> tensor;
  // SM special-function health: gsb_test_sfu_corrupt, by GSB_SFU_UNIT_*
  CheckState<gsb_sfu_stats, std::array<SmCorrupt, GSB_SFU_UNITS>> sfu;
  // L1 and constant-cache health: gsb_test_l1_corrupt by GSB_L1_UNIT_*, gsb_test_l1_skip
  struct L1Hooks {
    std::array<SmCorrupt, GSB_L1_UNITS> corrupt;
    bool skip_armed = false;
    uint32_t skip_smid = 0;
  };
  CheckState<gsb_l1_stats, L1Hooks> l1;
  // gsb_test_l1_table, by GSB_L1_UNIT_* (guarded by smu): a twin's table and expected words, taken by the next probe
  // that runs the unit
  struct L1Table {
    bool armed = false;
    uint32_t region_words = 0;
    std::vector<uint32_t> table, expected;
  };
  std::array<L1Table, GSB_L1_UNITS> l1_table;
  // what the L1 probe's CONST unit copies into its bank and its PARAM unit passes as its parameter: the copy is
  // asynchronous, so its source lives as long as the device
  std::vector<uint4> l1_const, l1_param;
  // memory-ordering health: gsb_test_order_inject by GSB_ORDER_UNIT_*, gsb_test_order_skip
  struct OrderInject {
    bool armed = false;
    uint32_t smid = 0, index = 0;
  };
  struct OrderHooks {
    std::array<OrderInject, GSB_ORDER_UNITS> inject;
    bool skip_armed = false;
    uint32_t skip_smid = 0;
  };
  CheckState<gsb_order_stats, OrderHooks> order;
  // sparse tensor-core health: gsb_test_sparse_corrupt, and gsb_test_sparse_operands' expected words then its operand
  // table (gsb_sparse_table_*), by GSB_SPARSE_UNIT_*; empty = not armed
  struct SparseHooks {
    std::array<SmCorrupt, GSB_SPARSE_UNITS> corrupt;
    std::vector<uint32_t> operands[GSB_SPARSE_UNITS];
  };
  CheckState<gsb_sparse_stats, SparseHooks> sparse;
  // shared-memory atomic health: gsb_test_shared_atomic_corrupt and _skip, by GSB_SHARED_ATOMIC_UNIT_*
  struct SharedAtomicHooks {
    std::array<SmCorrupt, GSB_SHARED_ATOMIC_UNITS> corrupt;
    std::array<SmCorrupt, GSB_SHARED_ATOMIC_UNITS> skip;  // smid only
  };
  CheckState<gsb_shared_atomic_stats, SharedAtomicHooks> shared_atomic;

  // persistent worker (gsb_cycle_all / gsb_probe_all): one host thread per device
  std::thread worker;
  std::mutex wmu;
  std::condition_variable wcv;
  Job job;
  bool job_ready = false, job_done = false, worker_quit = false;
  std::atomic<bool> job_flag{false}, done_flag{false}, quit_flag{false};  // lock-free mirrors for the spin phase
};

struct Global {
  // every device-touching entry point holds this shared; gsb_init/gsb_shutdown take it exclusively, so a
  // shutdown waits for calls still running on other threads (e.g. a start-up walk) instead of freeing
  // devices under them
  std::shared_mutex api_mu;
  std::mutex mu;
  bool inited = false;
  DriverApi cu;
  NvmlApi ml;
  std::vector<std::unique_ptr<Device>> devs;  // NVML index order

  // options (gsb_set_option)
  std::atomic<uint64_t> inventory_policy{GSB_INVENTORY_SNAPSHOT};
  std::atomic<uint64_t> wait_spin_us{2000};
  std::atomic<uint64_t> watchdog_ms{2000};
  std::atomic<uint64_t> inventory_refresh_ms{5000};
  std::atomic<uint64_t> transient_keep_free{1ull << 30};
  std::atomic<uint64_t> sweep_every{0};
  std::atomic<uint64_t> ecc_health{0};
  std::atomic<uint64_t> check_every[11] = {};  // GSB_OPT_*_PROBE_EVERY_CYCLES, by the check's place in Checks

  // one link or copy probe's pinned buffers at a time in the whole process (the DaemonSet's memory limit covers 8 GPUs)
  std::mutex link_mu;

  // node cycle (gsb_cycle_all / gsb_probe_all): one at a time; scratch of the join lives here, not on the heap per call
  std::mutex all_mu;
  std::vector<uint8_t> join_bits;

  // health
  // held through a whole gsb_health_stop (threads joined, event set freed, stop flag reset) and by gsb_health_start:
  // a second stop returns only once the threads the first one took are gone, so gsb_shutdown never frees a device
  // under a prober thread, and a start never re-arms the flag those threads are still to see
  std::mutex health_mu;
  std::mutex hmu;
  std::condition_variable hcv;
  std::deque<gsb_event> events;
  bool health_running = false;
  std::atomic<bool> health_stop{false};
  std::atomic<uint32_t> recovery_cycles{0};
  uint64_t stop_gen = 0;  // bumped by every gsb_health_stop: wakes all gsb_health_wait callers
  int shutting_down = 0;  // gsb_shutdown calls between their health stop and the device teardown; guarded by mu
  std::vector<std::thread> health_threads;
  nvmlEventSet_t event_set{};
  bool have_event_set = false;
};

Global G;

const char *cu_err(CUresult r) {
  const char *s = nullptr;
  if (G.cu.cuGetErrorString && G.cu.cuGetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
  return "unknown CUDA driver error";
}

#define CU_TRY(expr)                                                      \
  do {                                                                    \
    CUresult _r = (expr);                                                 \
    if (_r != CUDA_SUCCESS) {                                             \
      set_error("%s -> %d (%s)", #expr, (int)_r, cu_err(_r));             \
      return GSB_ERR_DRIVER;                                              \
    }                                                                     \
  } while (0)

#define RT_TRY(expr)                                                      \
  do {                                                                    \
    cudaError_t _r = (expr);                                              \
    if (_r != cudaSuccess) {                                              \
      set_error("%s -> %d (%s)", #expr, (int)_r, cudaGetErrorString(_r)); \
      return _r == cudaErrorMemoryAllocation ? GSB_ERR_OUT_OF_MEMORY : GSB_ERR_DRIVER; \
    }                                                                     \
  } while (0)

// "nvml: <nvmlErrorString>" is the reference's error text (bindings.go:52-58)
#define ML_TRY(expr)                                                      \
  do {                                                                    \
    nvmlReturn_t _r = (expr);                                             \
    if (_r != NVML_SUCCESS) {                                             \
      set_error("nvml: %s", G.ml.errorString ? G.ml.errorString(_r) : "?"); \
      return GSB_ERR_NVML;                                                \
    }                                                                     \
  } while (0)

void format_uuid(const CUuuid &u, char out[GSB_UUID_BUFFER_SIZE]) {
  const unsigned char *b = reinterpret_cast<const unsigned char *>(u.bytes);
  snprintf(out, GSB_UUID_BUFFER_SIZE,
           "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", b[0], b[1], b[2],
           b[3], b[4], b[5], b[6], b[7], b[8], b[9], b[10], b[11], b[12], b[13], b[14], b[15]);
}

int load_libraries() {
  if (!G.cu.lib) {
    G.cu.lib = dlopen("libcuda.so.1", RTLD_LAZY | RTLD_GLOBAL);
    if (!G.cu.lib) {
      set_error("could not load CUDA driver library: %s", dlerror());
      return GSB_ERR_LIBRARY_NOT_FOUND;
    }
    DriverApi &c = G.cu;
    bool ok = load_sym(c.lib, c.cuInit, "cuInit") && load_sym(c.lib, c.cuDeviceGet, "cuDeviceGet") &&
              load_sym(c.lib, c.cuDeviceGetUuid, "cuDeviceGetUuid_v2", "cuDeviceGetUuid") &&
              load_sym(c.lib, c.cuDeviceTotalMem, "cuDeviceTotalMem_v2") &&
              load_sym(c.lib, c.cuMemGetInfo, "cuMemGetInfo_v2") &&
              load_sym(c.lib, c.cuMemGetAllocationGranularity, "cuMemGetAllocationGranularity") &&
              load_sym(c.lib, c.cuMemAddressReserve, "cuMemAddressReserve") &&
              load_sym(c.lib, c.cuMemAddressFree, "cuMemAddressFree") &&
              load_sym(c.lib, c.cuMemCreate, "cuMemCreate") && load_sym(c.lib, c.cuMemRelease, "cuMemRelease") &&
              load_sym(c.lib, c.cuMemMap, "cuMemMap") && load_sym(c.lib, c.cuMemUnmap, "cuMemUnmap") &&
              load_sym(c.lib, c.cuMemSetAccess, "cuMemSetAccess") &&
              load_sym(c.lib, c.cuGetErrorString, "cuGetErrorString");
    if (!ok) {
      set_error("libcuda.so.1 lacks a required entry point");
      return GSB_ERR_LIBRARY_NOT_FOUND;
    }
  }
  if (!G.ml.lib) {
    // same library name and flags as the reference's shim (nvml_dl.c:23)
    G.ml.lib = dlopen("libnvidia-ml.so.1", RTLD_LAZY | RTLD_GLOBAL);
    if (!G.ml.lib) {
      set_error("could not load NVML library");  // bindings.go:63
      return GSB_ERR_LIBRARY_NOT_FOUND;
    }
    NvmlApi &m = G.ml;
    bool ok = load_sym(m.lib, m.init, "nvmlInit_v2") && load_sym(m.lib, m.shutdown, "nvmlShutdown") &&
              load_sym(m.lib, m.errorString, "nvmlErrorString") &&
              load_sym(m.lib, m.getCount, "nvmlDeviceGetCount_v2") &&
              load_sym(m.lib, m.handleByIndex, "nvmlDeviceGetHandleByIndex_v2") &&
              load_sym(m.lib, m.getUUID, "nvmlDeviceGetUUID") &&
              load_sym(m.lib, m.getMinor, "nvmlDeviceGetMinorNumber") &&
              load_sym(m.lib, m.getMemoryInfo, "nvmlDeviceGetMemoryInfo") &&
              load_sym(m.lib, m.getPciInfo, "nvmlDeviceGetPciInfo_v3");
    if (!ok) {
      set_error("libnvidia-ml.so.1 lacks a required entry point");
      return GSB_ERR_LIBRARY_NOT_FOUND;
    }
    // optional (health): absence only disables the XID half
    load_sym(m.lib, m.eventSetCreate, "nvmlEventSetCreate");
    load_sym(m.lib, m.registerEvents, "nvmlDeviceRegisterEvents");
    load_sym(m.lib, m.eventSetWait, "nvmlEventSetWait_v2", "nvmlEventSetWait");
    load_sym(m.lib, m.eventSetFree, "nvmlEventSetFree");
    // optional (ECC health): a missing one only leaves its fields unknown
    load_sym(m.lib, m.getEccMode, "nvmlDeviceGetEccMode");
    load_sym(m.lib, m.getTotalEccErrors, "nvmlDeviceGetTotalEccErrors");
    load_sym(m.lib, m.getMemoryErrorCounter, "nvmlDeviceGetMemoryErrorCounter");
    load_sym(m.lib, m.getRemappedRows, "nvmlDeviceGetRemappedRows");
    load_sym(m.lib, m.getRowRemapperHistogram, "nvmlDeviceGetRowRemapperHistogram");
    // optional (PCIe link health): likewise
    load_sym(m.lib, m.getCurrPcieLinkGeneration, "nvmlDeviceGetCurrPcieLinkGeneration");
    load_sym(m.lib, m.getCurrPcieLinkWidth, "nvmlDeviceGetCurrPcieLinkWidth");
    load_sym(m.lib, m.getMaxPcieLinkGeneration, "nvmlDeviceGetMaxPcieLinkGeneration");
    load_sym(m.lib, m.getMaxPcieLinkWidth, "nvmlDeviceGetMaxPcieLinkWidth");
    load_sym(m.lib, m.getGpuMaxPcieLinkGeneration, "nvmlDeviceGetGpuMaxPcieLinkGeneration");
    load_sym(m.lib, m.getPcieReplayCounter, "nvmlDeviceGetPcieReplayCounter");
    load_sym(m.lib, m.getTotalEnergyConsumption, "nvmlDeviceGetTotalEnergyConsumption");
    load_sym(m.lib, m.getPowerUsage, "nvmlDeviceGetPowerUsage");
    load_sym(m.lib, m.getEnforcedPowerLimit, "nvmlDeviceGetEnforcedPowerLimit");
    load_sym(m.lib, m.getTemperature, "nvmlDeviceGetTemperature");
    load_sym(m.lib, m.getClockInfo, "nvmlDeviceGetClockInfo");
    load_sym(m.lib, m.getClocksEventReasons, "nvmlDeviceGetCurrentClocksEventReasons",
             "nvmlDeviceGetCurrentClocksThrottleReasons");
  }
  return GSB_OK;
}

Device *device_at(uint32_t idx) {
  if (!G.inited) {
    set_error("gsb_init has not succeeded");
    return nullptr;
  }
  if (idx >= G.devs.size()) {
    set_error("nvml: device not found (index %u of %zu)", idx, G.devs.size());
    return nullptr;
  }
  return G.devs[idx].get();
}

// per-device CUDA resources, created on first probe/arena use (primary context via the runtime)
int ensure_ready(Device *d) {
  if (d->ordinal < 0) {
    set_error("device %s is not visible to the CUDA driver in this process", d->uuid);
    return GSB_ERR_NO_DEVICE;
  }
  if (d->cc_major != 9 || d->cc_minor != 0) {
    set_error("device %s is compute capability %u.%u; this library carries sm_90a code only", d->uuid,
              d->cc_major, d->cc_minor);
    return GSB_ERR_UNSUPPORTED_ARCH;
  }
  RT_TRY(cudaSetDevice(d->ordinal));
  if (d->ready) return GSB_OK;
  RT_TRY(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
  RT_TRY(cudaEventCreate(&d->ev0));
  RT_TRY(cudaEventCreate(&d->ev1));
  RT_TRY(cudaHostAlloc(reinterpret_cast<void **>(&d->out_host), sizeof(gsb_kernel_out),
                       cudaHostAllocMapped | cudaHostAllocPortable));
  memset(d->out_host, 0, sizeof(gsb_kernel_out));
  RT_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(&d->out_dev), d->out_host, 0));
  RT_TRY(cudaMalloc(reinterpret_cast<void **>(&d->partials),
                    sizeof(gsb_partial) * gsb_kernel_max_grid((int)d->sm_count)));
  // zeroed on the probe stream itself: it is non-blocking, so it would not wait for a memset on the legacy stream
  RT_TRY(cudaMalloc(reinterpret_cast<void **>(&d->ticket), sizeof(unsigned int)));
  RT_TRY(cudaMemsetAsync(d->ticket, 0, sizeof(unsigned int), d->stream));
  RT_TRY(cudaMalloc(reinterpret_cast<void **>(&d->tile_counter), 2 * sizeof(unsigned long long)));
  RT_TRY(cudaMemsetAsync(d->tile_counter, 0, 2 * sizeof(unsigned long long), d->stream));
  RT_TRY(cudaMalloc(reinterpret_cast<void **>(&d->fault_log), sizeof(gsb_fault_log)));
  RT_TRY(cudaMemsetAsync(d->fault_log, 0, sizeof(gsb_fault_log), d->stream));
  RT_TRY(cudaHostAlloc(reinterpret_cast<void **>(&d->fault_host), sizeof(gsb_fault_log),
                       cudaHostAllocMapped | cudaHostAllocPortable));
  memset(d->fault_host, 0, sizeof(gsb_fault_log));
  RT_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(&d->fault_host_dev), d->fault_host, 0));
  int smem_optin = 0;
  RT_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, d->ordinal));
  cudaError_t pe = (cudaError_t)gsb_kernel_preload();
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sm_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sm_operands_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_stress_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_cluster_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_cluster_script_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_atomic_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_atomic_values_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_tensor_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_tensor_operands_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sfu_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_l1_kernel_preload();
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sfu_operands_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_order_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sparse_kernel_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_sparse_operands_preload(smem_optin);
  if (pe == cudaSuccess) pe = (cudaError_t)gsb_shared_atomic_kernel_preload(smem_optin);
  if (pe != cudaSuccess) {
    set_error("loading the probe kernels on %s: %s", d->uuid, cudaGetErrorString(pe));
    return (pe == cudaErrorInvalidDeviceFunction || pe == cudaErrorNoKernelImageForDevice) ? GSB_ERR_UNSUPPORTED_ARCH
                                                                                            : GSB_ERR_DRIVER;
  }
  d->ready = true;
  return GSB_OK;
}

int arena_destroy_locked(Device *d) {
  if (!d->va) return GSB_OK;
  cudaSetDevice(d->ordinal);
  if (d->wedged && cudaStreamQuery(d->stream) == cudaErrorNotReady) {
    // unmapping under a kernel that may never end would block for ever: keep the mapping (the process is about to
    // report this GPU Unhealthy or exit; the driver reclaims the memory with the context)
    set_error("%s: arena kept, a wedged launch still uses it", d->uuid);
    return GSB_ERR_TIMEOUT;
  }
  cudaStreamSynchronize(d->stream);
  size_t off = 0;
  for (const Chunk &c : d->chunks) {
    G.cu.cuMemUnmap(d->va + off, c.size);
    G.cu.cuMemRelease(c.handle);
    off += c.size;
  }
  d->chunks.clear();
  G.cu.cuMemAddressFree(d->va, d->va_size);
  d->va = 0;
  d->va_size = 0;
  d->arena_bytes = 0;
  d->transient_arena = false;
  if (d->seed_table) cudaFree(d->seed_table);
  d->seed_table = nullptr;
  return GSB_OK;
}

int run_probe_locked(Device *d, const gsb_probe_cfg *cfg, gsb_probe_result *out);

int arena_create_locked(Device *d, uint64_t max_bytes, uint64_t keep_free, uint64_t *arena_bytes,
                        gsb_probe_result *fill_res = nullptr) {
  int rc = ensure_ready(d);
  if (rc) return rc;
  if ((rc = arena_destroy_locked(d)) != GSB_OK) return rc;

  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof prop);
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = d->ordinal;
  size_t gran = 0;
  CU_TRY(G.cu.cuMemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
  size_t free_b = 0, total_b = 0;
  CU_TRY(G.cu.cuMemGetInfo(&free_b, &total_b));
  uint64_t target = free_b > keep_free ? free_b - keep_free : 0;
  if (max_bytes && max_bytes < target) target = max_bytes;
  target = target / gran * gran;
  if (target == 0) {
    set_error("nothing allocatable on %s (free %zu, keep_free %llu)", d->uuid, free_b,
              (unsigned long long)keep_free);
    return GSB_ERR_OUT_OF_MEMORY;
  }
  CU_TRY(G.cu.cuMemAddressReserve(&d->va, target, 0, 0, 0));
  d->va_size = target;

  // Map physical chunks, largest first, until the driver refuses: what got mapped IS the
  // "actually allocatable" figure.
  const size_t ladder[] = {8ull << 30, 1ull << 30, 128ull << 20, 16ull << 20, 2ull << 20};
  uint64_t mapped = 0;
  for (size_t want : ladder) {
    size_t sz = want / gran * gran;
    if (sz == 0) sz = gran;
    while (mapped + sz <= target) {
      CUmemGenericAllocationHandle h;
      CUresult r = G.cu.cuMemCreate(&h, sz, &prop, 0);
      if (r != CUDA_SUCCESS) break;  // try the next smaller rung
      r = G.cu.cuMemMap(d->va + mapped, sz, 0, h, 0);
      if (r != CUDA_SUCCESS) {
        G.cu.cuMemRelease(h);
        set_error("cuMemMap -> %d (%s)", (int)r, cu_err(r));
        arena_destroy_locked(d);
        return GSB_ERR_DRIVER;
      }
      d->chunks.push_back({h, sz});
      mapped += sz;
    }
  }
  if (mapped == 0) {
    arena_destroy_locked(d);
    set_error("driver refused every allocation on %s", d->uuid);
    return GSB_ERR_OUT_OF_MEMORY;
  }
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof acc);
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  CUresult r = G.cu.cuMemSetAccess(d->va, mapped, &acc, 1);
  if (r != CUDA_SUCCESS) {
    set_error("cuMemSetAccess -> %d (%s)", (int)r, cu_err(r));
    arena_destroy_locked(d);
    return GSB_ERR_DRIVER;
  }
  d->arena_bytes = mapped;
  const size_t n_gran = (size_t)((mapped + kGranuleBytes - 1) / kGranuleBytes);
  if (cudaMalloc(reinterpret_cast<void **>(&d->seed_table), n_gran * sizeof(uint32_t)) != cudaSuccess) {
    arena_destroy_locked(d);
    set_error("cudaMalloc(seed table) failed");
    return GSB_ERR_OUT_OF_MEMORY;
  }
  // on the probe stream, ahead of the FILL whose last CTA writes the table
  if (cudaMemsetAsync(d->seed_table, 0, n_gran * sizeof(uint32_t), d->stream) != cudaSuccess) {
    arena_destroy_locked(d);
    set_error("cudaMemsetAsync(seed table) failed");
    return GSB_ERR_DRIVER;
  }

  // First generation: write every word once (proves every mapped byte is writable) so that all
  // later cycles are VERIFY_REFILL.
  gsb_probe_cfg fill;
  memset(&fill, 0, sizeof fill);
  fill.op = GSB_OP_FILL;
  fill.variant = GSB_VARIANT_AUTO;
  fill.seed_write = d->next_gen;
  fill.flags = GSB_PROBE_SEED_TABLE;
  fill.flags = GSB_PROBE_SEED_TABLE | (fill_res ? GSB_PROBE_TIMED : 0u);
  gsb_probe_result res;
  rc = run_probe_locked(d, &fill, &res);
  if (fill_res) *fill_res = res;
  if (rc) {
    arena_destroy_locked(d);
    return rc;
  }
  d->next_gen++;
  if (d->next_gen == 0) d->next_gen = 1;
  if (arena_bytes) *arena_bytes = mapped;
  return GSB_OK;
}

struct ProbeFlight {
  gsb_probe_cfg cfg;
  gsb_launch_geom geom;
  gsb_kernel_args args;
  uint64_t bytes = 0;
  uint64_t t_begin = 0;
  bool timed = false;
  bool launched = false;
  bool transient = false;  // the window is a transient allocation (the cycle sets it)
  uint64_t extra_ns = 0;   // watchdog budget beyond GSB_OPT_WATCHDOG_MS (probe_begin_locked: 1 ns per 10 window bytes)
  uint64_t words = 0;      // words the launch must report done
};

// validate + enqueue (does not wait)
int probe_begin_locked(Device *d, const gsb_probe_cfg *cfg, gsb_probe_result *out, ProbeFlight *fl) {
  fl->t_begin = now_ns();
  fl->cfg = *cfg;
  memset(out, 0, sizeof *out);
  out->first_bad_offset = UINT64_MAX;
  int rc = ensure_ready(d);
  if (rc) return out->status = rc;
  if (!d->va) {
    set_error("no arena on %s: call gsb_arena_create first", d->uuid);
    return out->status = GSB_ERR_NO_ARENA;
  }
  if (d->wedged) {  // a launch that outlived the watchdog: queue nothing behind it until it has drained
    if (cudaStreamQuery(d->stream) == cudaErrorNotReady) {
      set_error("%s: an earlier probe launch is still running (wedged)", d->uuid);
      return out->status = GSB_ERR_TIMEOUT;
    }
    d->wedged = false;
  }
  if (cfg->op < GSB_OP_FILL || cfg->op > GSB_OP_MARCH_RW_DOWN || (cfg->window_offset & 15) ||
      (cfg->window_bytes & 15) || cfg->window_offset > d->arena_bytes) {
    set_error("invalid probe window/op (op %u, offset %llu, bytes %llu)", cfg->op,
              (unsigned long long)cfg->window_offset, (unsigned long long)cfg->window_bytes);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  const uint64_t bytes = cfg->window_bytes ? cfg->window_bytes : d->arena_bytes - cfg->window_offset;
  if (cfg->window_offset + bytes > d->arena_bytes) {
    set_error("probe window [%llu, +%llu) exceeds arena of %llu bytes", (unsigned long long)cfg->window_offset,
              (unsigned long long)bytes, (unsigned long long)d->arena_bytes);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  const bool table = (cfg->flags & GSB_PROBE_SEED_TABLE) != 0;
  if (table && (cfg->window_offset & 0xFFFF)) {
    set_error("seed-table probes need a 64 KiB aligned window offset");
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  // occupancy + function attributes are queried once per (op, variant, grid) and device, not per launch
  const uint64_t gkey = ((uint64_t)cfg->op << 48) | ((uint64_t)cfg->variant << 32) | cfg->grid_ctas;
  int e = 0;
  auto git = d->geoms.find(gkey);
  if (git != d->geoms.end()) {
    fl->geom = git->second;
  } else {
    e = gsb_kernel_geometry(cfg->op, cfg->variant, cfg->grid_ctas, (int)d->sm_count, &fl->geom);
    if (!e) d->geoms.emplace(gkey, fl->geom);
  }
  if (e) {
    set_error("kernel geometry: %s", cudaGetErrorString((cudaError_t)e));
    return out->status = (e == (int)cudaErrorInvalidDeviceFunction || e == (int)cudaErrorNoKernelImageForDevice)
                             ? GSB_ERR_UNSUPPORTED_ARCH
                             : GSB_ERR_DRIVER;
  }
  gsb_kernel_args &a = fl->args;
  memset(&a, 0, sizeof a);
  a.base = reinterpret_cast<uint4 *>(d->va);
  a.first_word = cfg->window_offset >> 4;
  a.n_words = bytes >> 4;
  a.seed_expect = cfg->seed_expect;
  a.seed_write = cfg->seed_write;
  a.seed_table = table ? d->seed_table : nullptr;
  a.table_update = (table && cfg->op != GSB_OP_VERIFY) ? d->seed_table : nullptr;
  a.arena_words = d->arena_bytes >> 4;
  a.granule_shift = kGranuleShiftWords;
  a.launch_seq = ++d->launch_seq;
  a.partials = d->partials;
  a.ticket = d->ticket;
  a.tile_counter = d->tile_counter;
  a.out = d->out_dev;
  a.fault = d->fault_log;
  a.fault_out = d->fault_host_dev;
  if (cfg->op >= GSB_OP_MARCH_FILL) {  // March C- (gsb_memtest): the seeds are the solid backgrounds' lane values
    a.solid_expect = cfg->seed_expect;
    a.solid_write = cfg->seed_write;
  }
  fl->bytes = bytes;
  fl->extra_ns = bytes / 10;
  fl->words = a.n_words;
  fl->timed = (cfg->flags & GSB_PROBE_TIMED) != 0;
  if (bytes > 0) {
    if (fl->timed) RT_TRY(cudaEventRecord(d->ev0, d->stream));
    e = gsb_kernel_launch(cfg->op, &fl->geom, &a, d->stream);
    if (e) {
      set_error("kernel launch: %s", cudaGetErrorString((cudaError_t)e));
      return out->status = GSB_ERR_DRIVER;
    }
    if (fl->timed) RT_TRY(cudaEventRecord(d->ev1, d->stream));
    fl->launched = true;
  }
  return GSB_OK;
}

// wait for the launch and collect what the last CTA wrote into pinned host memory
//
// Three phases, none of which can park the thread for ever:
//   1. spin on the sequence word the last CTA stores into pinned host memory (option GSB_OPT_WAIT_SPIN_US, default
//      2000; a prober thread with a period >= 10 ms passes 0): a sleeping wait costs 10-30 us of wake-up latency, a
//      tenth of a 1 GiB-window cycle, which matters to a caller cycling back to back and not at all to a 1 Hz prober
//      inside a 1-CPU pod (device-plugin-ds.yaml:34-40);
//   2. sleep-poll the same word (50 us naps, the stream queried every ~1 ms so a faulted launch is noticed) against
//      the completion watchdog: GSB_OPT_WATCHDOG_MS (default 2000) + 1 ns per 10 window bytes (10 GB/s is "wedged").
//      The reference's WaitForEvent returns every 5 s whatever the GPU does (nvidia.go:126); a kernel that never
//      finishes must not keep this thread — and the GPU's Healthy flag — for ever;
//   3. cudaStreamSynchronize, which by then returns at once and orders the events.
thread_local bool tl_wait_blocking = false;  // set by prober threads that have milliseconds to spare

// A faulted launch: what its last CTA copied into the mapped fault log (checked to be this launch's), with the
// launch's window and counts, becomes the device's LAST report, and its FIRST when there is none yet.
void store_fault_report(Device *d, const ProbeFlight *fl, const gsb_probe_result *out) {
  const gsb_fault_log &h = *d->fault_host;  // the stream sync before the caller read gsb_kernel_out orders it
  if (h.launch_seq != fl->args.launch_seq) return;
  gsb_fault_report r;
  memset(&r, 0, sizeof r);
  r.valid = 1;
  r.op = fl->cfg.op;
  r.transient = fl->transient ? 1u : 0u;
  r.n_records = h.count < GSB_FAULT_RECORDS ? h.count : GSB_FAULT_RECORDS;
  struct timespec ts;
  clock_gettime(CLOCK_REALTIME, &ts);
  r.unix_ns = (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
  r.window_offset = fl->cfg.window_offset;
  r.window_bytes = fl->bytes;
  r.mismatch_words = out->mismatch_words;
  r.mismatch_bits = out->mismatch_bits;
  r.first_bad_offset = out->first_bad_offset;
  for (int b = 0; b < 128; b++) {
    r.flips_0to1[b] = h.flips[0][b];
    r.flips_1to0[b] = h.flips[1][b];
  }
  for (uint32_t i = 0; i < r.n_records; i++) {
    gsb_fault_record &rec = r.records[i];
    rec.offset = h.rec[i].word << 4;
    memcpy(rec.expected, h.rec[i].expected, sizeof rec.expected);
    memcpy(rec.observed, h.rec[i].observed, sizeof rec.observed);
    gsb_fault_classify(&rec);
  }
  std::sort(r.records, r.records + r.n_records,
            [](const gsb_fault_record &x, const gsb_fault_record &y) { return x.offset < y.offset; });
  std::lock_guard<std::mutex> lk(d->smu);
  d->fault_last = r;
  // FIRST is the first HBM fault, which both daemons log with a PROBE mismatch verdict; a link phase's report (op
  // GSB_OP_LINK_*, host memory) and a copy verify's (GSB_OP_COPY_*, what a copy engine left) only ever become LAST
  const bool last_only = (r.op >= GSB_OP_LINK_UP && r.op <= GSB_OP_LINK_DUPLEX) ||
                         (r.op >= GSB_OP_COPY_H2D && r.op <= GSB_OP_COPY_D2D);
  if (!d->fault_first.valid && !last_only) d->fault_first = r;
}

int probe_end_locked(Device *d, ProbeFlight *fl, gsb_probe_result *out) {
  const gsb_probe_cfg *cfg = &fl->cfg;
  const gsb_kernel_args &a = fl->args;
  if (fl->launched) {
    const volatile uint32_t *flag = &d->out_host->done_flag;
    const uint64_t spin_ns = tl_wait_blocking ? 0 : G.wait_spin_us.load(std::memory_order_relaxed) * 1000ull;
    if (spin_ns) {
      const uint64_t deadline = now_ns() + spin_ns;
      while (*flag != a.launch_seq) {
        for (int i = 0; i < 8; i++) __builtin_ia32_pause();
        if (now_ns() > deadline) break;
      }
    }
    const uint64_t wd_ms = G.watchdog_ms.load(std::memory_order_relaxed);
    if (wd_ms && *flag != a.launch_seq) {
      const uint64_t budget = wd_ms * 1000000ull + fl->extra_ns;
      const uint64_t deadline = fl->t_begin + budget;
      unsigned naps = 0;
      while (*flag != a.launch_seq) {
        if ((++naps & 15u) == 0 && cudaStreamQuery(d->stream) != cudaErrorNotReady) break;  // finished or faulted
        if (now_ns() > deadline) {
          d->wedged = true;  // the launch is still on the stream: nothing new is queued behind it
          set_error("probe kernel on %s did not finish within %llu ms: device wedged?", d->uuid,
                    (unsigned long long)(budget / 1000000ull));
          out->wall_ns = now_ns() - fl->t_begin;
          return out->status = GSB_ERR_TIMEOUT;
        }
        struct timespec ts = {0, 50000};
        nanosleep(&ts, nullptr);
      }
    }
    cudaError_t se = cudaStreamSynchronize(d->stream);
    if (se != cudaSuccess) {
      set_error("probe kernel failed: %s", cudaGetErrorString(se));
      return out->status = GSB_ERR_DRIVER;
    }
    gsb_kernel_out ko;
    memcpy(&ko, d->out_host, sizeof ko);  // written by the last CTA; the stream sync above orders it
    if (ko.done_flag != a.launch_seq || ko.words_done != fl->words) {
      set_error("probe kernel did not complete the window (seq %u/%u, words %llu/%llu)", ko.done_flag,
                a.launch_seq, ko.words_done, (unsigned long long)fl->words);
      return out->status = GSB_ERR_DRIVER;
    }
    out->mismatch_words = ko.mismatch_words;
    out->mismatch_bits = ko.mismatch_bits;
    out->first_bad_offset = ko.first_bad_word == ~0ull ? UINT64_MAX : ko.first_bad_word << 4;
    out->checksum_xor = ko.checksum_xor;
    out->checksum_sum = ko.checksum_sum;
    if (fl->timed) {
      float ms = 0.f;
      RT_TRY(cudaEventElapsedTime(&ms, d->ev0, d->ev1));
      out->kernel_ns = (uint64_t)((double)ms * 1e6);
    }
    if (ko.mismatch_words) store_fault_report(d, fl, out);
  }
  out->variant = fl->geom.variant;
  out->grid_ctas = fl->geom.grid;
  out->block_threads = fl->geom.block;
  out->bytes_walked = fl->bytes;
  out->bytes_read = cfg->op == GSB_OP_FILL || cfg->op == GSB_OP_MARCH_FILL ? 0 : fl->bytes;
  out->bytes_written = cfg->op == GSB_OP_VERIFY || cfg->op == GSB_OP_MARCH_VERIFY ? 0 : fl->bytes;
  out->wall_ns = now_ns() - fl->t_begin;
  return out->status = GSB_OK;
}

int run_probe_locked(Device *d, const gsb_probe_cfg *cfg, gsb_probe_result *out) {
  ProbeFlight fl;
  int rc = probe_begin_locked(d, cfg, out, &fl);
  if (rc) return rc;
  return probe_end_locked(d, &fl, out);
}

// gsb_arena_read / gsb_arena_write: one copy on the probe stream, complete when this returns. The probe stream is
// non-blocking, so a plain cudaMemcpy (legacy stream) would be ordered with neither the launches before it nor the
// ones after it, and a pageable host-to-device cudaMemcpy may return before its DMA has landed.
int arena_copy_locked(Device *d, void *dst, const void *src, uint64_t bytes, cudaMemcpyKind kind) {
  if (d->wedged && cudaStreamQuery(d->stream) == cudaErrorNotReady) {  // the copy would wait behind that launch
    set_error("%s: an earlier probe launch is still running (wedged)", d->uuid);
    return GSB_ERR_TIMEOUT;
  }
  RT_TRY(cudaSetDevice(d->ordinal));
  RT_TRY(cudaMemcpyAsync(dst, src, bytes, kind, d->stream));
  RT_TRY(cudaStreamSynchronize(d->stream));
  return GSB_OK;
}

// diagnostic knob GSB_NVML_SERIAL=1: one NVML/driver query at a time across this process's device threads
// (GSB_INVENTORY_LIVE only)
std::mutex g_nvml_serial_mu;
const bool kNvmlSerial = [] {
  const char *e = getenv("GSB_NVML_SERIAL");
  return e && atoi(e) != 0;
}();

// "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx" -> the 16 bytes cuDeviceGetUuid reports for the same device
bool parse_uuid(const char *s, unsigned char out[16]) {
  if (strncmp(s, "GPU-", 4) != 0) return false;
  s += 4;
  int n = 0;
  auto hex = [](char c) -> int {
    if (c >= '0' && c <= '9') return c - '0';
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    if (c >= 'A' && c <= 'F') return c - 'A' + 10;
    return -1;
  };
  while (*s && n < 16) {
    if (*s == '-') {
      s++;
      continue;
    }
    const int hi = hex(s[0]), lo = hi < 0 ? -1 : hex(s[1]);
    if (lo < 0) return false;
    out[n++] = (unsigned char)(hi << 4 | lo);
    s += 2;
  }
  return n == 16 && *s == 0;
}

void fill_static_info(const Device *d, gsb_device_info *out) {
  snprintf(out->bus_id, sizeof out->bus_id, "%s", d->bus_id);
  out->cuda_ordinal = d->ordinal;
  out->sm_count = d->sm_count;
  out->cc_major = d->cc_major;
  out->cc_minor = d->cc_minor;
  out->cuda_total_bytes = d->cuda_total;
}

// LIVE inventory of one device: the reference's source (NVML UUID, minor, MemoryInfo v1) re-read and the identity
// cross-checked against the CUDA driver. This is what nvml.NewDevice does at every plugin (re)start
// (server.go:39 -> nvidia.go:60); it also rewrites the device's snapshot.
int query_info(Device *d, gsb_device_info *out) {
  memset(out, 0, sizeof *out);
  std::unique_lock<std::mutex> serial(g_nvml_serial_mu, std::defer_lock);
  if (kNvmlSerial) serial.lock();
  char uuid[GSB_UUID_BUFFER_SIZE] = {0};
  ML_TRY(G.ml.getUUID(d->nvml, uuid, GSB_UUID_BUFFER_SIZE));
  unsigned minor = 0;
  ML_TRY(G.ml.getMinor(d->nvml, &minor));
  nvmlMemory_t mem;
  memset(&mem, 0, sizeof mem);
  ML_TRY(G.ml.getMemoryInfo(d->nvml, &mem));
  if (d->ordinal >= 0) {
    CUuuid cu;
    CU_TRY(G.cu.cuDeviceGetUuid(&cu, d->cudev));
    char cuda_uuid[GSB_UUID_BUFFER_SIZE];
    format_uuid(cu, cuda_uuid);
    if (strcmp(cuda_uuid, uuid) != 0) {
      set_error("identity mismatch on minor %u: CUDA %s vs NVML %s", d->minor, cuda_uuid, uuid);
      return GSB_ERR_IDENTITY_MISMATCH;
    }
  }
  snprintf(out->uuid, sizeof out->uuid, "%s", uuid);
  fill_static_info(d, out);
  out->minor = minor;
  out->total_bytes = mem.total;
  out->total_mib = mem.total / (1024ull * 1024ull);  // bindings.go:346-349
  out->free_bytes = mem.free;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    Snapshot &sn = d->snap;
    snprintf(sn.uuid, sizeof sn.uuid, "%s", uuid);
    sn.uuid_parsed = parse_uuid(uuid, sn.uuid_bytes);
    sn.minor = minor;
    sn.total = mem.total;
    sn.free = mem.free;
    sn.taken_ns = now_ns();
    sn.refreshes++;
  }
  return GSB_OK;
}

// SNAPSHOT inventory: identity/total as NVML reported them at the last live query, with the identity re-validated
// against the CUDA driver on every call (cuDeviceGetUuid is answered by the user-mode driver: no ioctl, no
// driver-wide lock — unlike nvmlDeviceGetMemoryInfo, which serialises with every other NVML client of the box, an
// nvidia-smi or dcgm-exporter poller included).
int snapshot_info(Device *d, gsb_device_info *out, uint64_t *age_ns) {
  memset(out, 0, sizeof *out);
  Snapshot sn;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    sn = d->snap;
  }
  if (sn.refreshes == 0) return query_info(d, out);  // never queried: take the live path once
  if (d->ordinal >= 0 && sn.uuid_parsed) {
    CUuuid cu;
    CU_TRY(G.cu.cuDeviceGetUuid(&cu, d->cudev));
    if (memcmp(cu.bytes, sn.uuid_bytes, 16) != 0) {
      char cuda_uuid[GSB_UUID_BUFFER_SIZE];
      format_uuid(cu, cuda_uuid);
      set_error("identity mismatch on minor %u: CUDA %s vs NVML snapshot %s", sn.minor, cuda_uuid, sn.uuid);
      return GSB_ERR_IDENTITY_MISMATCH;
    }
  }
  memcpy(out->uuid, sn.uuid, sizeof out->uuid);
  fill_static_info(d, out);
  out->minor = sn.minor;
  out->total_bytes = sn.total;
  out->total_mib = sn.total / (1024ull * 1024ull);
  out->free_bytes = sn.free;
  if (age_ns) *age_ns = now_ns() - sn.taken_ns;
  return GSB_OK;
}

// Run a Job on the device's own persistent thread (created on first use). Hand-off is spin-then-block in both
// directions: a node cycle every few hundred microseconds never pays a futex wake-up (tens of us per hop, a tenth
// of a 1 GiB-window cycle), an idle daemon's workers park after ~200 us. The job is plain data (no std::function,
// no allocation per hand-off).
// knob GSB_WORKER_SPIN_US (default 200; 0 = pure condition-variable hand-off)
const uint64_t kSpinNs = [] {
  const char *e = getenv("GSB_WORKER_SPIN_US");
  return (uint64_t)(e ? atoi(e) : 200) * 1000ull;
}();

int cycle_impl(Device *d, uint32_t idx, uint64_t cycle_no, uint64_t window_bytes, int unit_gib, uint32_t variant,
               uint8_t *lw_buf, size_t lw_cap, bool encode_lw, gsb_cycle_result *out);

void run_job(Device *d, Job *j) {  // on the worker thread; the submitting call holds G.api_mu (shared) throughout
  switch (j->kind) {
    case Job::PROBE: {
      std::lock_guard<std::mutex> lk(d->mu);
      j->rc = run_probe_locked(d, j->cfg, j->probe_out);
      break;
    }
    case Job::CYCLE:
      // the node cycle's join re-encodes the whole node's list: the per-device list is not built here
      j->rc = cycle_impl(d, j->idx, j->cycle_no, j->window_bytes, j->unit_gib, j->variant, nullptr, 0, false,
                         j->cycle_out);
      break;
    default:
      j->rc = GSB_ERR_INVALID_ARGUMENT;
  }
}

void worker_submit(Device *d, const Job &job) {
  std::unique_lock<std::mutex> lk(d->wmu);
  if (!d->worker.joinable()) {
    d->worker = std::thread([d] {
      for (;;) {
        // spin for a job first
        const uint64_t until = now_ns() + kSpinNs;
        while (!d->job_flag.load(std::memory_order_acquire) && !d->quit_flag.load(std::memory_order_acquire) &&
               now_ns() < until)
          __builtin_ia32_pause();
        std::unique_lock<std::mutex> wl(d->wmu);
        d->wcv.wait(wl, [d] { return d->job_ready || d->worker_quit; });
        if (d->worker_quit) return;
        d->job_ready = false;
        d->job_flag.store(false, std::memory_order_relaxed);
        wl.unlock();
        run_job(d, &d->job);  // the submitter does not touch d->job until job_done
        wl.lock();
        d->job_done = true;
        d->done_flag.store(true, std::memory_order_release);
        d->wcv.notify_all();
      }
    });
  }
  d->job = job;
  d->job_done = false;
  d->done_flag.store(false, std::memory_order_relaxed);
  d->job_ready = true;
  d->job_flag.store(true, std::memory_order_release);
  d->wcv.notify_all();
}

int worker_wait(Device *d) {
  const uint64_t until = now_ns() + 5 * kSpinNs;
  while (!d->done_flag.load(std::memory_order_acquire) && now_ns() < until) __builtin_ia32_pause();
  std::unique_lock<std::mutex> lk(d->wmu);
  d->wcv.wait(lk, [d] { return d->job_done; });
  return d->job.rc;
}

void worker_stop(Device *d) {
  {
    std::lock_guard<std::mutex> lk(d->wmu);
    d->worker_quit = true;
    d->quit_flag.store(true, std::memory_order_release);
  }
  d->wcv.notify_all();
  if (d->worker.joinable()) d->worker.join();
}

void push_event(const gsb_event &ev) {
  {
    std::lock_guard<std::mutex> lk(G.hmu);
    G.events.push_back(ev);
  }
  G.hcv.notify_all();
}

// ------------------------------------------------------------------ what every health check does the same way

// Raise every condition of `conditions()` (evaluated under smu) that this device has not raised yet: one event of
// `etype` per condition per device per health session.
template <typename Conditions>
void raise_conditions(Device *d, uint64_t etype, uint32_t *raised, Conditions conditions) {
  uint32_t fresh;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    fresh = conditions() & ~*raised;
    *raised |= fresh;
  }
  for (uint32_t bit = 1; fresh; bit <<= 1) {
    if (!(fresh & bit)) continue;
    fresh &= ~bit;
    gsb_event ev;
    memset(&ev, 0, sizeof ev);
    snprintf(ev.uuid, sizeof ev.uuid, "%s", d->uuid);
    ev.etype = etype;
    ev.edata = bit;
    push_event(ev);
  }
}

// The statistics of one finished probe. A probe that ran nothing learnt nothing and counts as skipped; `incomplete`
// is the check's counter of probes that covered less than they should have, or null when this one covered it all (the
// link and copy checks have no such counter).
template <typename Stats, typename Result>
void count_probe(Device *d, Stats *st, const Result &r, bool ran, uint32_t conditions, uint64_t *incomplete = nullptr) {
  std::lock_guard<std::mutex> lk(d->smu);
  st->probes++;
  if (!ran) st->skipped++;
  if (incomplete) ++*incomplete;
  if (conditions) st->faults++;
  st->last = r;
}

// The armed test hooks, disarmed: a hook applies to the next probe only.
template <typename Hooks>
Hooks take_hooks(Device *d, Hooks *armed) {
  std::lock_guard<std::mutex> lk(d->smu);
  return std::exchange(*armed, Hooks{});
}

// The seed the caller gave or, for 0, a fresh one: old data then reads as stale, and no two probes share operands.
uint32_t seed_or_fresh(uint32_t given, uint32_t base, uint32_t *handed_out, uint32_t stride = 1) {
  return given ? given : base + stride * ++*handed_out;
}

// A launch that outlived the watchdog is still on the device's stream: nothing is queued behind it until it drained.
int wedged_drain_locked(Device *d) {
  if (cudaStreamQuery(d->stream) == cudaErrorNotReady) {
    set_error("%s: an earlier launch is still running (wedged)", d->uuid);
    return GSB_ERR_TIMEOUT;
  }
  d->wedged = false;
  return GSB_OK;
}

// ------------------------------------------------------------------ ECC health

uint64_t realtime_ns() {
  struct timespec ts;
  clock_gettime(CLOCK_REALTIME, &ts);
  return (uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec;
}

// One ECC / row-remapper status of a device: the test override when one is set, else NVML. A call that is missing or
// does not answer SUCCESS (NOT_SUPPORTED, NO_PERMISSION, ...) leaves its group's valid bit clear and its fields 0.
void query_ecc(Device *d, gsb_ecc_status *out) {
  memset(out, 0, sizeof *out);
  bool overridden;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    overridden = d->ecc_override_set;
    if (overridden) *out = d->ecc_override;
  }
  if (!overridden) {
    const NvmlApi &m = G.ml;
    const nvmlDevice_t h = d->nvml;
    nvmlEnableState_t cur = NVML_FEATURE_DISABLED, pend = NVML_FEATURE_DISABLED;
    if (m.getEccMode && m.getEccMode(h, &cur, &pend) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_MODE;
      out->mode_current = cur == NVML_FEATURE_ENABLED;
      out->mode_pending = pend == NVML_FEATURE_ENABLED;
    }
    unsigned long long c = 0, u = 0;
    if (m.getTotalEccErrors && m.getTotalEccErrors(h, NVML_MEMORY_ERROR_TYPE_CORRECTED, NVML_VOLATILE_ECC, &c) == NVML_SUCCESS &&
        m.getTotalEccErrors(h, NVML_MEMORY_ERROR_TYPE_UNCORRECTED, NVML_VOLATILE_ECC, &u) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_VOLATILE;
      out->corrected_volatile = c;
      out->uncorrected_volatile = u;
    }
    if (m.getTotalEccErrors && m.getTotalEccErrors(h, NVML_MEMORY_ERROR_TYPE_CORRECTED, NVML_AGGREGATE_ECC, &c) == NVML_SUCCESS &&
        m.getTotalEccErrors(h, NVML_MEMORY_ERROR_TYPE_UNCORRECTED, NVML_AGGREGATE_ECC, &u) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_AGGREGATE;
      out->corrected_aggregate = c;
      out->uncorrected_aggregate = u;
    }
    if (m.getMemoryErrorCounter &&
        m.getMemoryErrorCounter(h, NVML_MEMORY_ERROR_TYPE_CORRECTED, NVML_VOLATILE_ECC, NVML_MEMORY_LOCATION_DRAM, &c) == NVML_SUCCESS &&
        m.getMemoryErrorCounter(h, NVML_MEMORY_ERROR_TYPE_UNCORRECTED, NVML_VOLATILE_ECC, NVML_MEMORY_LOCATION_DRAM, &u) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_DRAM;
      out->dram_corrected_volatile = c;
      out->dram_uncorrected_volatile = u;
    }
    unsigned corr = 0, unc = 0, pending = 0, failure = 0;
    if (m.getRemappedRows && m.getRemappedRows(h, &corr, &unc, &pending, &failure) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_REMAP;
      out->remapped_correctable = corr;
      out->remapped_uncorrectable = unc;
      out->remap_pending = pending != 0;
      out->remap_failure = failure != 0;
    }
    nvmlRowRemapperHistogramValues_t hv;
    memset(&hv, 0, sizeof hv);
    if (m.getRowRemapperHistogram && m.getRowRemapperHistogram(h, &hv) == NVML_SUCCESS) {
      out->valid |= GSB_ECC_VALID_HISTOGRAM;
      out->hist_max = hv.max;
      out->hist_high = hv.high;
      out->hist_partial = hv.partial;
      out->hist_low = hv.low;
      out->hist_none = hv.none;
    }
  }
  out->unix_ns = realtime_ns();
}

// The prober's bracket read: the volatile corrected / uncorrected totals only (two NVML calls), override honoured.
// false = unknown.
bool read_ecc_totals(Device *d, uint64_t *corrected, uint64_t *uncorrected) {
  {
    std::lock_guard<std::mutex> lk(d->smu);
    if (d->ecc_override_set) {
      *corrected = d->ecc_override.corrected_volatile;
      *uncorrected = d->ecc_override.uncorrected_volatile;
      return (d->ecc_override.valid & GSB_ECC_VALID_VOLATILE) != 0;
    }
  }
  unsigned long long c = 0, u = 0;
  if (!G.ml.getTotalEccErrors ||
      G.ml.getTotalEccErrors(d->nvml, NVML_MEMORY_ERROR_TYPE_CORRECTED, NVML_VOLATILE_ECC, &c) != NVML_SUCCESS ||
      G.ml.getTotalEccErrors(d->nvml, NVML_MEMORY_ERROR_TYPE_UNCORRECTED, NVML_VOLATILE_ECC, &u) != NVML_SUCCESS)
    return false;
  *corrected = c;
  *uncorrected = u;
  return true;
}

// Raise every condition of `now` against the session's baseline that this device has not raised yet (one event per
// condition per device per health session).
void raise_ecc_conditions(Device *d, const gsb_ecc_status &now) {
  raise_conditions(d, GSB_EVENT_ECC, &d->ecc_raised, [&] { return gsb_ecc_conditions(&d->ecc_baseline, &now); });
}

struct EccPrev {  // a prober thread's last valid post-cycle read
  bool valid = false;
  uint64_t corrected = 0;
};

// Attribution of one prober cycle: what the volatile totals did across it (the walk's) and since the previous
// cycle's post read (everyone else's). A cycle with an unknown read is counted, not attributed: the next valid
// bracket's between-walk figure absorbs it, so in + between = latest - first still holds.
void ecc_account(Device *d, bool pre_ok, uint64_t c0, uint64_t u0, bool post_ok, uint64_t c1, uint64_t u1,
                 uint64_t cycle_no, uint64_t window_bytes, const gsb_cycle_result &cr, EccPrev *prev) {
  const uint64_t dc = c1 > c0 ? c1 - c0 : 0, du = u1 > u0 ? u1 - u0 : 0;
  uint64_t offset = 0;
  if (pre_ok && post_ok && dc && !cr.transient) {  // the window gsb_cycle rotated to (cycle_impl's rule)
    std::lock_guard<std::mutex> dl(d->mu);
    if (window_bytes && window_bytes < d->arena_bytes) offset = (cycle_no % (d->arena_bytes / window_bytes)) * window_bytes;
  }
  std::lock_guard<std::mutex> lk(d->smu);
  gsb_ecc_stats &es = d->ecc_stats;
  es.cycles++;
  es.queries += 2;
  if (!(pre_ok && post_ok)) return;
  if (prev->valid) es.corrected_between_walks += c0 > prev->corrected ? c0 - prev->corrected : 0;
  else es.first_corrected_volatile = c0;
  es.corrected_in_walks += dc;
  es.uncorrected_in_walks += du;
  es.bytes_walked += cr.probe.bytes_walked;
  if (dc) {
    es.last_corrected = dc;
    es.last_window_offset = offset;
    es.last_window_bytes = cr.probe.bytes_walked;
  }
  es.latest_corrected_volatile = c1;
  prev->valid = true;
  prev->corrected = c1;
}


// ------------------------------------------------------------------ March C- (gsb_memtest)

struct MarchElement {
  uint32_t op;
  uint32_t expect, write;  // lane values of the backgrounds read and written
};
// ⇕(w0); ⇑(r0,w1); ⇑(r1,w0); ⇓(r0,w1); ⇓(r1,w0); ⇕(r0)
constexpr MarchElement kMarch[GSB_MEMTEST_ELEMENTS] = {
    {GSB_OP_MARCH_FILL, 0u, 0u},          {GSB_OP_MARCH_RW_UP, 0u, ~0u},   {GSB_OP_MARCH_RW_UP, ~0u, 0u},
    {GSB_OP_MARCH_RW_DOWN, 0u, ~0u},      {GSB_OP_MARCH_RW_DOWN, ~0u, 0u}, {GSB_OP_MARCH_VERIFY, 0u, 0u}};

// The steady-state pattern back into [off, off + bytes) of the standing arena after a March C- run, so the next cycle
// over it is clean and no byte outside it changes. The granules the window covers completely (the arena's ragged tail
// granule counts when the window reaches the end, as in the kernels' table update) get a new generation, recorded by
// the FILL's last CTA; the words of a granule it covers in part get the generation the table already holds for it.
int march_refill_locked(Device *d, uint64_t off, uint64_t bytes) {
  const uint64_t end = off + bytes;
  const uint64_t mid_lo = (off + kGranuleBytes - 1) / kGranuleBytes * kGranuleBytes;
  const uint64_t mid_hi = end == d->arena_bytes ? end : end / kGranuleBytes * kGranuleBytes;
  gsb_probe_cfg fill;
  gsb_probe_result res;
  auto partial = [&](uint64_t lo, uint64_t hi) -> int {
    while (lo < hi) {
      const uint64_t g = lo / kGranuleBytes, next = std::min(hi, (g + 1) * kGranuleBytes);
      uint32_t gen = 0;
      RT_TRY(cudaMemcpy(&gen, d->seed_table + g, sizeof gen, cudaMemcpyDeviceToHost));
      memset(&fill, 0, sizeof fill);
      fill.op = GSB_OP_FILL;
      fill.window_offset = lo;
      fill.window_bytes = next - lo;
      fill.seed_write = gen;
      if (int rc = run_probe_locked(d, &fill, &res)) return rc;
      lo = next;
    }
    return GSB_OK;
  };
  if (mid_lo >= mid_hi) return partial(off, end);
  if (int rc = partial(off, mid_lo)) return rc;
  memset(&fill, 0, sizeof fill);
  fill.op = GSB_OP_FILL;
  fill.window_offset = mid_lo;
  fill.window_bytes = mid_hi - mid_lo;
  fill.seed_write = d->next_gen++;
  if (d->next_gen == 0) d->next_gen = 1;
  fill.flags = GSB_PROBE_SEED_TABLE;
  if (int rc = run_probe_locked(d, &fill, &res)) return rc;
  return partial(mid_hi, end);
}

int memtest_locked(Device *d, const gsb_memtest_cfg *cfg, gsb_memtest_result *out) {
  const uint64_t t0 = now_ns();
  const uint32_t first = cfg->first_element;
  const uint32_t n = cfg->n_elements ? cfg->n_elements : GSB_MEMTEST_ELEMENTS - std::min<uint32_t>(first, GSB_MEMTEST_ELEMENTS);
  if (first >= GSB_MEMTEST_ELEMENTS || n == 0 || n > GSB_MEMTEST_ELEMENTS - first || (cfg->window_offset & 15) ||
      (cfg->window_bytes & 15)) {
    set_error("invalid memtest elements or window (first %u, n %u, offset %llu, bytes %llu)", first, cfg->n_elements,
              (unsigned long long)cfg->window_offset, (unsigned long long)cfg->window_bytes);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  int rc = ensure_ready(d);
  if (rc) return out->status = rc;
  if (d->va && d->transient_arena) {  // a transient window a wedged launch kept: give it back if the stream has drained
    if (d->wedged && cudaStreamQuery(d->stream) != cudaErrorNotReady) d->wedged = false;
    if (arena_destroy_locked(d) != GSB_OK) return out->status = GSB_ERR_TIMEOUT;
  }
  const bool transient = !d->va;
  uint64_t off = cfg->window_offset, bytes = cfg->window_bytes;
  if (transient) {
    if (off) {
      set_error("a transient memtest window starts at 0 (offset %llu)", (unsigned long long)off);
      return out->status = GSB_ERR_INVALID_ARGUMENT;
    }
    rc = arena_create_locked(d, bytes, G.transient_keep_free.load(), &bytes);
    if (rc) {
      if (d->va) d->transient_arena = true;  // could not be unmapped under a wedged launch: given back later
      out->wall_ns = now_ns() - t0;
      return out->status = rc;
    }
  } else {
    if (off > d->arena_bytes || (bytes && bytes > d->arena_bytes - off)) {
      set_error("memtest window [%llu, +%llu) exceeds arena of %llu bytes", (unsigned long long)off,
                (unsigned long long)bytes, (unsigned long long)d->arena_bytes);
      return out->status = GSB_ERR_INVALID_ARGUMENT;
    }
    if (!bytes) bytes = d->arena_bytes - off;
  }
  out->transient = transient ? 1u : 0u;
  out->window_offset = off;
  out->window_bytes = bytes;
  const bool ecc = G.ecc_health.load() != 0;  // off: no ECC query at all
  bool bad = false;
  for (uint32_t k = first; k < first + n; k++) {
    const MarchElement &m = kMarch[k];
    const bool reads = m.op != GSB_OP_MARCH_FILL, writes = m.op != GSB_OP_MARCH_VERIFY;
    gsb_memtest_element &e = out->elements[out->n_elements++];
    e.element = k;
    e.op = m.op;
    e.descending = m.op == GSB_OP_MARCH_RW_DOWN;
    e.expected = reads ? m.expect : 0u;
    e.written = writes ? m.write : 0u;
    gsb_probe_cfg pc;
    memset(&pc, 0, sizeof pc);
    pc.op = m.op;
    pc.window_offset = off;
    pc.window_bytes = bytes;
    pc.seed_expect = m.expect;
    pc.seed_write = m.write;
    pc.flags = GSB_PROBE_TIMED;
    uint64_t c0 = 0, u0 = 0, c1 = 0, u1 = 0;
    const bool pre_ok = ecc && read_ecc_totals(d, &c0, &u0);
    ProbeFlight fl;
    fl.transient = transient;
    gsb_probe_result pr;
    int prc = probe_begin_locked(d, &pc, &pr, &fl);
    if (prc == GSB_OK) prc = probe_end_locked(d, &fl, &pr);
    const bool post_ok = ecc && read_ecc_totals(d, &c1, &u1);
    e.status = prc;
    e.bytes_read = pr.bytes_read;
    e.bytes_written = pr.bytes_written;
    e.mismatch_words = pr.mismatch_words;
    e.mismatch_bits = pr.mismatch_bits;
    e.first_bad_offset = pr.first_bad_offset;
    e.kernel_ns = pr.kernel_ns;
    if (pre_ok && post_ok) {
      e.ecc_valid = 1;
      e.ecc_corrected = c1 > c0 ? c1 - c0 : 0;
      e.ecc_uncorrected = u1 > u0 ? u1 - u0 : 0;
    }
    if (prc != GSB_OK || pr.mismatch_words) bad = true;
    if (prc != GSB_OK) {  // a failed or wedged element ends the run
      rc = prc;
      break;
    }
  }
  if (bad) d->faulted = true;  // sticky, as a faulted cycle
  if (rc == GSB_OK && !transient && first + n == GSB_MEMTEST_ELEMENTS) {
    rc = march_refill_locked(d, off, bytes);
    out->refilled = rc == GSB_OK ? 1u : 0u;
    if (rc != GSB_OK) d->faulted = true;
  }
  if (transient && arena_destroy_locked(d) != GSB_OK) d->transient_arena = true;  // wedged: kept, given back later
  out->wall_ns = now_ns() - t0;
  return out->status = rc;
}

// ------------------------------------------------------------------ PCIe link health (gsb_link_probe)

constexpr uint64_t kLinkDefaultBytes = 32ull << 20;
constexpr uint32_t kLinkDefaultPasses = 8;
constexpr uint64_t kLinkNsPerByte = 4;  // watchdog: a link trained at Gen1 x1 (250 MB/s) is slow, not wedged

// One link status of a device: the test override when one is set, else NVML, limited to the GSB_LINK_VALID_* bits of
// `what`. A call that is missing or does not answer SUCCESS leaves its bit clear and its field 0. Under the override the
// replay counter advances by one at every query that reads it, so each probe sees a rise (of one) across it.
void query_link(Device *d, gsb_link_status *out, uint32_t what = ~0u) {
  memset(out, 0, sizeof *out);
  bool overridden;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    d->link.stats.queries++;
    overridden = d->link_override_set;
    if (overridden) {
      *out = d->link_override;
      out->valid &= what;
      if (what & GSB_LINK_VALID_REPLAY) d->link_override.replay_counter++;
    }
  }
  if (!overridden) {
    const NvmlApi &m = G.ml;
    auto ask = [&](nvmlReturn_t (*fn)(nvmlDevice_t, unsigned *), uint32_t bit) -> unsigned {
      unsigned v = 0;
      if (!(what & bit) || !fn || fn(d->nvml, &v) != NVML_SUCCESS) return 0;
      out->valid |= bit;
      return v;
    };
    out->cur_gen = ask(m.getCurrPcieLinkGeneration, GSB_LINK_VALID_CUR_GEN);
    out->cur_width = ask(m.getCurrPcieLinkWidth, GSB_LINK_VALID_CUR_WIDTH);
    out->max_gen = ask(m.getMaxPcieLinkGeneration, GSB_LINK_VALID_MAX_GEN);
    out->max_width = ask(m.getMaxPcieLinkWidth, GSB_LINK_VALID_MAX_WIDTH);
    out->gpu_max_gen = ask(m.getGpuMaxPcieLinkGeneration, GSB_LINK_VALID_GPU_MAX_GEN);
    out->replay_counter = ask(m.getPcieReplayCounter, GSB_LINK_VALID_REPLAY);
  }
  out->unix_ns = realtime_ns();
}

// the highest current generation / width of `st` into the result's under-load reading
void note_load(gsb_link_result *out, const gsb_link_status &st) {
  out->polls++;
  if (st.valid & GSB_LINK_VALID_CUR_GEN) {
    out->load_gen = (out->load_valid & GSB_LINK_VALID_CUR_GEN) ? std::max(out->load_gen, st.cur_gen) : st.cur_gen;
    out->load_valid |= GSB_LINK_VALID_CUR_GEN;
  }
  if (st.valid & GSB_LINK_VALID_CUR_WIDTH) {
    out->load_width = (out->load_valid & GSB_LINK_VALID_CUR_WIDTH) ? std::max(out->load_width, st.cur_width) : st.cur_width;
    out->load_valid |= GSB_LINK_VALID_CUR_WIDTH;
  }
}

struct LinkPhase {
  uint32_t op;
  int down, up;  // buffer (0 = A, 1 = B) the phase reads / writes, -1 = none
  bool repeated; // runs cfg passes times (the duplex phase)
};
// up A; down A ‖ up B (passes times); down B: every word written up is read back down
constexpr LinkPhase kLinkPhases[GSB_LINK_PHASES] = {
    {GSB_OP_LINK_UP, -1, 0, false}, {GSB_OP_LINK_DUPLEX, 0, 1, true}, {GSB_OP_LINK_DOWN, 1, -1, false}};

int link_probe_locked(Device *d, const gsb_link_cfg *cfg, gsb_link_result *out) {
  const uint64_t t0 = now_ns();
  const uint64_t L = cfg->buffer_bytes ? cfg->buffer_bytes : kLinkDefaultBytes;
  const uint32_t passes = cfg->passes ? cfg->passes : kLinkDefaultPasses;
  if ((L & 15) || L == 0) {
    set_error("link buffer bytes must be a non-zero multiple of 16 (%llu)", (unsigned long long)L);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  int rc = ensure_ready(d);
  if (!rc && d->wedged) rc = wedged_drain_locked(d);
  if (rc) return out->status = rc;
  for (void *&p : d->link_kept) {  // buffers a wedged link launch kept: the stream has drained, give them back
    if (p) cudaFreeHost(p);
    p = nullptr;
  }
  out->passes = passes;
  out->buffer_bytes = L;
  if (!cfg->seed_a || !cfg->seed_b) d->link.seed += 2;
  out->seed_a = cfg->seed_a ? cfg->seed_a : 0x4C4E0000u + d->link.seed;  // fresh per probe: old data reads as STALE
  out->seed_b = cfg->seed_b ? cfg->seed_b : 0x4C4E0001u + d->link.seed;
  const std::vector<Device::LinkCorrupt> corrupt = take_hooks(d, &d->link.hooks);
  query_link(d, &out->idle);  // at idle, before any probe traffic: current, maximum, replay counter

  std::lock_guard<std::mutex> one(G.link_mu);
  void *host[2] = {nullptr, nullptr};
  uint4 *dev[2] = {nullptr, nullptr};
  for (int i = 0; i < 2 && rc == GSB_OK; i++) {
    // one device uses the buffer: mapped, not portable
    cudaError_t e = cudaHostAlloc(&host[i], L, cudaHostAllocMapped);
    if (e != cudaSuccess) {
      host[i] = nullptr;
      set_error("pinning %llu bytes of host memory for the link probe: %s", (unsigned long long)L, cudaGetErrorString(e));
      rc = GSB_ERR_OUT_OF_MEMORY;
    } else if ((e = cudaHostGetDevicePointer(reinterpret_cast<void **>(&dev[i]), host[i], 0)) != cudaSuccess) {
      set_error("mapping the link probe's host buffer into %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  const uint32_t side_ctas = gsb_kernel_link_ctas((int)d->sm_count);
  const uint64_t words = L >> 4;
  bool wedged = false;
  for (int k = 0; k < GSB_LINK_PHASES && rc == GSB_OK; k++) {
    const LinkPhase &ph = kLinkPhases[k];
    const uint32_t reps = ph.repeated ? passes : 1u;
    gsb_link_phase &po = out->phases[k];
    po.op = ph.op;
    po.first_bad_offset = UINT64_MAX;
    for (const Device::LinkCorrupt &c : corrupt) {  // test hook: host memory only, right before the phase reads it
      if (c.phase != (uint32_t)k + 1 || ph.down < 0 || c.offset + 16 > L) continue;
      uint32_t *w = reinterpret_cast<uint32_t *>(static_cast<char *>(host[ph.down]) + c.offset);
      for (int l = 0; l < 4; l++) w[l] ^= c.xr[l];
    }
    ProbeFlight fl;
    memset(&fl.cfg, 0, sizeof fl.cfg);
    fl.cfg.op = ph.op;
    fl.cfg.window_bytes = L;
    fl.transient = true;
    fl.bytes = L;
    fl.t_begin = now_ns();
    fl.geom.variant = GSB_VARIANT_AUTO;
    fl.geom.grid = (ph.down >= 0 ? side_ctas : 0u) + (ph.up >= 0 ? side_ctas : 0u);
    fl.geom.block = 256;
    fl.geom.smem_bytes = 0;
    gsb_kernel_args &a = fl.args;
    memset(&a, 0, sizeof a);
    a.base = ph.down >= 0 ? dev[ph.down] : nullptr;
    a.n_words = ph.down >= 0 ? words : 0;
    a.link_up = ph.up >= 0 ? reinterpret_cast<unsigned long long>(dev[ph.up]) : 0ull;
    a.link_up_words = ph.up >= 0 ? words : 0;
    a.seed_expect = ph.down == 0 ? out->seed_a : out->seed_b;
    a.seed_write = ph.up == 0 ? out->seed_a : out->seed_b;
    a.link_down_ctas = ph.down >= 0 ? side_ctas : 0u;
    a.link_passes = reps;
    a.launch_seq = ++d->launch_seq;
    a.partials = d->partials;
    a.ticket = d->ticket;
    a.out = d->out_dev;
    a.fault = d->fault_log;
    a.fault_out = d->fault_host_dev;
    fl.words = (a.n_words + a.link_up_words) * reps;
    fl.extra_ns = kLinkNsPerByte * 16 * fl.words;
    fl.timed = true;
    gsb_probe_result pr;
    memset(&pr, 0, sizeof pr);
    pr.first_bad_offset = UINT64_MAX;
    int prc = (int)cudaEventRecord(d->ev0, d->stream);
    if (prc == cudaSuccess) prc = gsb_kernel_launch(ph.op, &fl.geom, &a, d->stream);
    if (prc == cudaSuccess) prc = (int)cudaEventRecord(d->ev1, d->stream);
    if (prc != cudaSuccess) {
      set_error("link kernel launch: %s", cudaGetErrorString((cudaError_t)prc));
      prc = GSB_ERR_DRIVER;
    } else {
      fl.launched = true;
      if (ph.down >= 0 && ph.up >= 0) {
        // the duplex phase: poll the current generation and width while the link carries traffic both ways (at least
        // once, right after the launch), until the launch completes or the watchdog's budget is spent
        const volatile uint32_t *flag = &d->out_host->done_flag;
        const uint64_t wd_ms = G.watchdog_ms.load(std::memory_order_relaxed);
        const uint64_t deadline = fl.t_begin + wd_ms * 1000000ull + fl.extra_ns;
        do {
          gsb_link_status st;
          query_link(d, &st, GSB_LINK_VALID_CUR_GEN | GSB_LINK_VALID_CUR_WIDTH);
          note_load(out, st);
          if (*flag == a.launch_seq || cudaStreamQuery(d->stream) != cudaErrorNotReady) break;
          struct timespec ts = {0, 200000};
          nanosleep(&ts, nullptr);
        } while (!(wd_ms && now_ns() > deadline));
      }
      prc = probe_end_locked(d, &fl, &pr);
    }
    po.status = prc;
    po.bytes_read = ph.down >= 0 ? L * reps : 0;
    po.bytes_written = ph.up >= 0 ? L * reps : 0;
    po.mismatch_words = pr.mismatch_words;
    po.mismatch_bits = pr.mismatch_bits;
    po.first_bad_offset = pr.first_bad_offset;
    po.checksum_xor = pr.checksum_xor;
    po.checksum_sum = pr.checksum_sum;
    po.kernel_ns = pr.kernel_ns;
    if (prc != GSB_OK) {
      wedged = prc == GSB_ERR_TIMEOUT;
      rc = prc;
    }
  }
  gsb_link_status after;
  query_link(d, &after, GSB_LINK_VALID_REPLAY);
  if ((out->idle.valid & GSB_LINK_VALID_REPLAY) && (after.valid & GSB_LINK_VALID_REPLAY)) {
    out->replay_valid = 1;
    out->replays = after.replay_counter > out->idle.replay_counter ? after.replay_counter - out->idle.replay_counter : 0;
  }
  for (int i = 0; i < 2; i++) {
    if (wedged) d->link_kept[i] = host[i];  // still in use by a launch on the stream: freed once it has drained
    else if (host[i]) cudaFreeHost(host[i]);
  }
  auto gbps = [](uint64_t bytes, uint64_t ns) { return ns ? (double)bytes / (double)ns : 0.0; };
  out->up_gbps = gbps(out->phases[0].bytes_written, out->phases[0].kernel_ns);
  out->duplex_down_gbps = gbps(out->phases[1].bytes_read, out->phases[1].kernel_ns);
  out->duplex_up_gbps = gbps(out->phases[1].bytes_written, out->phases[1].kernel_ns);
  out->down_gbps = gbps(out->phases[2].bytes_read, out->phases[2].kernel_ns);
  const uint32_t both = GSB_LINK_VALID_CUR_GEN | GSB_LINK_VALID_CUR_WIDTH;
  out->link_gbps = (out->load_valid & both) == both ? gsb_link_rate_gbps(out->load_gen, out->load_width) : 0.0;
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  if (out->replay_valid) {
    std::lock_guard<std::mutex> lk(d->smu);
    d->link.stats.replays += out->replays;
  }
  count_probe(d, &d->link.stats, *out, out->phases[0].op != 0, gsb_link_conditions(out));
  return rc;
}

// ------------------------------------------------------------------ copy-engine health (gsb_copy_probe)

constexpr uint64_t kCopyDefaultBytes = 32ull << 20;
constexpr uint64_t kCopyDefaultGuard = 64;  // bytes left untouched at each end of a default copy
constexpr uint64_t kCopyNsPerByte = 4;      // watchdog of the copies and of the host verify: the link probe's budget
constexpr uint32_t kCopyOps[GSB_COPY_DIRECTIONS] = {GSB_OP_COPY_H2D, GSB_OP_COPY_D2H, GSB_OP_COPY_D2D};
const char *const kCopyDirName[GSB_COPY_DIRECTIONS] = {"H2D", "D2H", "D2D"};

// launch geometry of (op, AUTO), queried once per device like probe_begin_locked's
int copy_geom_locked(Device *d, uint32_t op, gsb_launch_geom *geom) {
  const uint64_t gkey = ((uint64_t)op << 48) | ((uint64_t)GSB_VARIANT_AUTO << 32);
  auto it = d->geoms.find(gkey);
  if (it != d->geoms.end()) {
    *geom = it->second;
    return GSB_OK;
  }
  const int e = gsb_kernel_geometry(op, GSB_VARIANT_AUTO, 0, (int)d->sm_count, geom);
  if (e) {
    set_error("kernel geometry: %s", cudaGetErrorString((cudaError_t)e));
    return GSB_ERR_DRIVER;
  }
  d->geoms.emplace(gkey, *geom);
  return GSB_OK;
}

// One launch of a copy probe on the device's stream, waited for like every probe launch (probe_end_locked: watchdog,
// words-done check, fault report). `a` carries the launch's own fields; the device's are filled in here.
int copy_launch_locked(Device *d, uint32_t op, const gsb_launch_geom &geom, const gsb_kernel_args &args, uint64_t bytes,
                       uint64_t words, uint64_t extra_ns, gsb_probe_result *pr) {
  ProbeFlight fl;
  memset(&fl.cfg, 0, sizeof fl.cfg);
  fl.cfg.op = op;
  fl.cfg.window_bytes = bytes;
  fl.transient = true;
  fl.bytes = bytes;
  fl.t_begin = now_ns();
  fl.geom = geom;
  fl.args = args;
  gsb_kernel_args &a = fl.args;
  a.launch_seq = ++d->launch_seq;
  a.partials = d->partials;
  a.ticket = d->ticket;
  a.out = d->out_dev;
  a.fault = d->fault_log;
  a.fault_out = d->fault_host_dev;
  fl.words = words;
  fl.extra_ns = extra_ns;
  fl.timed = true;
  memset(pr, 0, sizeof *pr);
  pr->first_bad_offset = UINT64_MAX;
  int e = (int)cudaEventRecord(d->ev0, d->stream);
  if (e == cudaSuccess) e = gsb_kernel_launch(op, &fl.geom, &a, d->stream);
  if (e == cudaSuccess) e = (int)cudaEventRecord(d->ev1, d->stream);
  if (e != cudaSuccess) {
    set_error("copy probe launch: %s", cudaGetErrorString((cudaError_t)e));
    return pr->status = GSB_ERR_DRIVER;
  }
  fl.launched = true;
  return probe_end_locked(d, &fl, pr);
}

// Every stream a copy probe uses has drained (nothing of an earlier, wedged probe still runs on it).
bool copy_streams_idle(Device *d) {
  if (cudaStreamQuery(d->stream) == cudaErrorNotReady) return false;
  for (cudaStream_t s : d->copy_streams)
    if (s && cudaStreamQuery(s) == cudaErrorNotReady) return false;
  return true;
}

void copy_free_buffers(void *dev[3], void *host[2]) {
  for (int i = 0; i < 3; i++) {
    if (dev[i]) cudaFree(dev[i]);
    dev[i] = nullptr;
  }
  for (int i = 0; i < 2; i++) {
    if (host[i]) cudaFreeHost(host[i]);
    host[i] = nullptr;
  }
}

int copy_probe_locked(Device *d, const gsb_copy_cfg *cfg, gsb_copy_result *out) {
  const uint64_t t0 = now_ns();
  const uint64_t B = cfg->buffer_bytes ? cfg->buffer_bytes : kCopyDefaultBytes;
  const bool given = (cfg->flags & GSB_COPY_GEOMETRY) != 0;
  const uint64_t so = given ? cfg->src_offset : kCopyDefaultGuard, dof = given ? cfg->dst_offset : kCopyDefaultGuard;
  const uint64_t n = given ? cfg->copy_bytes : (B >= 2 * kCopyDefaultGuard ? B - 2 * kCopyDefaultGuard : 0);
  if ((B & 15) || B >= (1ull << 32) || (!given && B < 2 * kCopyDefaultGuard) || so > B || n > B - so || dof > B ||
      n > B - dof) {
    set_error("invalid copy probe geometry (buffers %llu, %llu bytes from +%llu to +%llu)", (unsigned long long)B,
              (unsigned long long)n, (unsigned long long)so, (unsigned long long)dof);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->buffer_bytes = B;
  out->src_offset = so;
  out->dst_offset = dof;
  out->copy_bytes = n;
  int rc = ensure_ready(d);
  if (rc) return out->status = rc;
  const bool kept = d->copy_kept_host[0] || d->copy_kept_dev[0];
  if (d->wedged || kept) {  // an earlier launch or copy outlived the watchdog: queue nothing behind it until it drained
    if (!copy_streams_idle(d)) {
      set_error("%s: an earlier launch or copy is still running (wedged)", d->uuid);
      return out->status = GSB_ERR_TIMEOUT;
    }
    d->wedged = false;
    copy_free_buffers(d->copy_kept_dev, d->copy_kept_host);
  }
  if (!d->copy_ev[GSB_COPY_DIRECTIONS - 1][1]) {  // the first copy probe of this device: its streams and events
    cudaError_t e = cudaSuccess;
    for (cudaStream_t &st : d->copy_streams)
      if (e == cudaSuccess && !st) e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    for (auto &pair : d->copy_ev)
      for (cudaEvent_t &ev : pair)
        if (e == cudaSuccess && !ev) e = cudaEventCreate(&ev);
    if (e != cudaSuccess) {  // what was made is kept; the next probe makes the rest
      set_error("copy probe streams and events on %s: %s", d->uuid, cudaGetErrorString(e));
      return out->status = GSB_ERR_DRIVER;
    }
  }
  int engines = 0;
  if (cudaDeviceGetAttribute(&engines, cudaDevAttrAsyncEngineCount, d->ordinal) == cudaSuccess)
    out->async_engines = (uint32_t)engines;
  if (!cfg->seed_src || !cfg->seed_host || !cfg->seed_bg) d->copy.seed += 3;
  out->seed_src = cfg->seed_src ? cfg->seed_src : 0x43500000u + d->copy.seed;  // fresh per probe: old data reads STALE
  out->seed_host = cfg->seed_host ? cfg->seed_host : 0x43500001u + d->copy.seed;
  out->seed_bg = cfg->seed_bg ? cfg->seed_bg : 0x43500002u + d->copy.seed;
  const Device::CopyHooks hooks = take_hooks(d, &d->copy.hooks);
  const std::vector<Device::CopyCorrupt> &corrupt = hooks.corrupt;
  const uint32_t skip = hooks.skip;

  std::lock_guard<std::mutex> one(G.link_mu);
  void *dev[3] = {nullptr, nullptr, nullptr};  // S, D_h2d, D_d2d
  void *host[2] = {nullptr, nullptr};          // H_s, H_d
  uint4 *host_dev[2] = {nullptr, nullptr};     // their device mappings
  {
    // transient HBM, under the keep-free margin of every transient probe window: a busy GPU skips the probe
    size_t free_b = 0, total_b = 0;
    const uint64_t keep_free = G.transient_keep_free.load();
    if (G.cu.cuMemGetInfo(&free_b, &total_b) != CUDA_SUCCESS || free_b < keep_free || free_b - keep_free < 3 * B) {
      set_error("copy probe: %llu bytes of HBM are not allocatable on %s (free %zu, keep_free %llu)",
                (unsigned long long)(3 * B), d->uuid, free_b, (unsigned long long)keep_free);
      rc = GSB_ERR_OUT_OF_MEMORY;
    }
    for (int i = 0; i < 3 && rc == GSB_OK; i++) {
      if (cudaMalloc(&dev[i], B) != cudaSuccess) {
        dev[i] = nullptr;
        cudaGetLastError();
        set_error("allocating %llu bytes of HBM for the copy probe on %s", (unsigned long long)B, d->uuid);
        rc = GSB_ERR_OUT_OF_MEMORY;
      }
    }
    for (int i = 0; i < 2 && rc == GSB_OK; i++) {
      cudaError_t e = cudaHostAlloc(&host[i], B, cudaHostAllocMapped);
      if (e != cudaSuccess) {
        host[i] = nullptr;
        set_error("pinning %llu bytes of host memory for the copy probe: %s", (unsigned long long)B, cudaGetErrorString(e));
        rc = GSB_ERR_OUT_OF_MEMORY;
      } else if ((e = cudaHostGetDevicePointer(reinterpret_cast<void **>(&host_dev[i]), host[i], 0)) != cudaSuccess) {
        set_error("mapping the copy probe's host buffer into %s: %s", d->uuid, cudaGetErrorString(e));
        rc = GSB_ERR_DRIVER;
      }
    }
  }
  const uint64_t words = B >> 4;
  bool wedged = false;
  auto failed = [&](int prc) {
    if (rc == GSB_OK) rc = prc;
    if (prc == GSB_ERR_TIMEOUT) wedged = true;
  };
  // 1. prepare: the sources' patterns and every destination's background
  if (rc == GSB_OK) {
    gsb_launch_geom fill_geom, up_geom;
    up_geom.variant = GSB_VARIANT_AUTO;
    up_geom.grid = gsb_kernel_link_ctas((int)d->sm_count);
    up_geom.block = 256;
    up_geom.smem_bytes = 0;
    rc = copy_geom_locked(d, GSB_OP_FILL, &fill_geom);
    const struct {
      bool in_hbm;
      int buf;
      uint32_t seed;
    } prep[5] = {{true, 0, out->seed_src}, {true, 1, out->seed_bg}, {true, 2, out->seed_bg},
                 {false, 0, out->seed_host}, {false, 1, out->seed_bg}};
    for (int i = 0; i < 5 && rc == GSB_OK; i++) {
      gsb_kernel_args a;
      memset(&a, 0, sizeof a);
      a.seed_write = prep[i].seed;
      gsb_probe_result pr;
      int prc;
      if (prep[i].in_hbm) {
        a.base = static_cast<uint4 *>(dev[prep[i].buf]);
        a.n_words = words;
        a.tile_counter = d->tile_counter;
        prc = copy_launch_locked(d, GSB_OP_FILL, fill_geom, a, B, words, B / 10, &pr);
      } else {
        a.link_up = reinterpret_cast<unsigned long long>(host_dev[prep[i].buf]);
        a.link_up_words = words;
        a.link_passes = 1;
        prc = copy_launch_locked(d, GSB_OP_LINK_UP, up_geom, a, B, words, kCopyNsPerByte * B, &pr);
      }
      if (prc != GSB_OK) failed(prc);
    }
  }
  // 2. the three copies at once, each on its own stream (the device's stream is idle: every launch above was waited for)
  if (rc == GSB_OK) {
    cudaStream_t streams[GSB_COPY_DIRECTIONS] = {d->copy_streams[0], d->copy_streams[1], d->stream};
    void *dst[GSB_COPY_DIRECTIONS] = {static_cast<char *>(dev[1]) + dof, static_cast<char *>(host[1]) + dof,
                                      static_cast<char *>(dev[2]) + dof};
    const void *src[GSB_COPY_DIRECTIONS] = {static_cast<char *>(host[0]) + so, static_cast<char *>(dev[0]) + so,
                                            static_cast<char *>(dev[0]) + so};
    const cudaMemcpyKind kinds[GSB_COPY_DIRECTIONS] = {cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost,
                                                        cudaMemcpyDeviceToDevice};
    bool issued[GSB_COPY_DIRECTIONS] = {false, false, false};
    const uint64_t t_copy = now_ns();
    for (int k = 0; k < GSB_COPY_DIRECTIONS; k++) {
      gsb_copy_direction &o = out->dirs[k];
      o.op = kCopyOps[k];
      o.first_bad_offset = UINT64_MAX;
      if (skip & (1u << k)) continue;  // test hook: the copy that never happened
      cudaError_t e = cudaEventRecord(d->copy_ev[k][0], streams[k]);
      if (e == cudaSuccess) e = cudaMemcpyAsync(dst[k], src[k], n, kinds[k], streams[k]);
      if (e == cudaSuccess) e = cudaEventRecord(d->copy_ev[k][1], streams[k]);
      if (e != cudaSuccess) {
        set_error("copy probe: cudaMemcpyAsync %s: %s", kCopyDirName[k], cudaGetErrorString(e));
        o.copy_status = GSB_ERR_DRIVER;
        failed(GSB_ERR_DRIVER);
        continue;
      }
      o.copied = 1;
      o.bytes = n;
      issued[k] = true;
    }
    // completion watchdog over the three: GSB_OPT_WATCHDOG_MS + 4 ns per byte copied
    const uint64_t wd_ms = G.watchdog_ms.load(std::memory_order_relaxed);
    const uint64_t deadline = t_copy + wd_ms * 1000000ull + kCopyNsPerByte * 3 * n;
    for (;;) {
      bool pending = false;
      for (int k = 0; k < GSB_COPY_DIRECTIONS; k++)
        if (issued[k] && cudaEventQuery(d->copy_ev[k][1]) == cudaErrorNotReady) pending = true;
      if (!pending) break;
      if (wd_ms && now_ns() > deadline) break;
      struct timespec ts = {0, 50000};
      nanosleep(&ts, nullptr);
    }
    for (int k = 0; k < GSB_COPY_DIRECTIONS; k++) {
      if (!issued[k]) continue;
      gsb_copy_direction &o = out->dirs[k];
      const cudaError_t e = cudaEventQuery(d->copy_ev[k][1]);
      if (e == cudaErrorNotReady) {
        set_error("copy probe: the %s copy on %s did not finish within the watchdog", kCopyDirName[k], d->uuid);
        o.copy_status = GSB_ERR_TIMEOUT;
        if (k == 2) d->wedged = true;  // still on the device's stream: nothing new is queued behind it
        failed(GSB_ERR_TIMEOUT);
        continue;
      }
      float ms = 0.f;
      if (e != cudaSuccess || cudaEventElapsedTime(&ms, d->copy_ev[k][0], d->copy_ev[k][1]) != cudaSuccess) {
        set_error("copy probe: the %s copy failed: %s", kCopyDirName[k], cudaGetErrorString(e));
        o.copy_status = GSB_ERR_DRIVER;
        failed(GSB_ERR_DRIVER);
        continue;
      }
      o.copy_ns = (uint64_t)((double)ms * 1e6);
      o.gbps = o.copy_ns ? (double)n / (double)o.copy_ns : 0.0;
    }
  }
  // 3. verify every destination on the GPU, each against the copy's geometry
  if (out->dirs[0].op) {
    uint4 *vbase[GSB_COPY_DIRECTIONS] = {static_cast<uint4 *>(dev[1]), host_dev[1], static_cast<uint4 *>(dev[2])};
    for (int k = 0; k < GSB_COPY_DIRECTIONS; k++) {
      gsb_copy_direction &o = out->dirs[k];
      if (o.copy_status != GSB_OK) {  // the destination is not what a finished copy left: nothing to check
        o.verify_status = o.copy_status;
        continue;
      }
      if (wedged) {  // a copy or launch outlived the watchdog: the probe checks nothing more
        o.verify_status = GSB_ERR_TIMEOUT;
        continue;
      }
      for (const Device::CopyCorrupt &c : corrupt) {  // test hook: after the copy, before the verify
        if (c.dir != (uint32_t)k || c.offset + 16 > B) continue;
        if (k == 1) {
          uint32_t *w = reinterpret_cast<uint32_t *>(static_cast<char *>(host[1]) + c.offset);
          for (int l = 0; l < 4; l++) w[l] ^= c.xr[l];
        } else {
          gsb_kernel_xor_word(vbase[k] + (c.offset >> 4), make_uint4(c.xr[0], c.xr[1], c.xr[2], c.xr[3]), d->stream);
        }
      }
      gsb_launch_geom geom;
      int prc = copy_geom_locked(d, o.op, &geom);
      gsb_probe_result pr;
      memset(&pr, 0, sizeof pr);
      if (prc == GSB_OK) {
        gsb_kernel_args a;
        memset(&a, 0, sizeof a);
        a.base = vbase[k];
        a.n_words = words;
        a.copy_begin = dof;
        a.copy_end = dof + n;
        a.copy_delta = (uint32_t)(so - dof);
        a.seed_expect = out->seed_bg;
        a.seed_write = k == 0 ? out->seed_host : out->seed_src;
        prc = copy_launch_locked(d, o.op, geom, a, B, words, k == 1 ? kCopyNsPerByte * B : B / 10, &pr);
      }
      o.verify_status = prc;
      o.mismatch_words = pr.mismatch_words;
      o.mismatch_bits = pr.mismatch_bits;
      o.first_bad_offset = pr.first_bad_offset;
      o.checksum_xor = pr.checksum_xor;
      o.checksum_sum = pr.checksum_sum;
      o.kernel_ns = pr.kernel_ns;
      if (prc != GSB_OK) failed(prc);
    }
  }
  if (wedged) {  // still in use by a copy or a launch: given back once every stream has drained
    for (int i = 0; i < 3; i++) d->copy_kept_dev[i] = dev[i];
    for (int i = 0; i < 2; i++) d->copy_kept_host[i] = host[i];
  } else {
    copy_free_buffers(dev, host);
  }
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  count_probe(d, &d->copy.stats, *out, out->dirs[0].op != 0, gsb_copy_conditions(out));
  return rc;
}

// ------------------------------------------------------------------ SM compute health (gsb_sm_probe)

constexpr uint32_t kSmAllUnits = (1u << GSB_SM_UNITS) - 1;

// Expected answers of every unit in one device buffer, after a head of `head` bytes (the launch log): chains as
// uint64, D words as uint32; `sets` tables per unit, one after the other, `set_bytes[u]` each.
struct SmLayout {
  size_t offset[GSB_SM_UNITS] = {};
  size_t set_bytes[GSB_SM_UNITS] = {};
  size_t bytes = 0;
  explicit SmLayout(size_t head = sizeof(gsb_sm_log), uint32_t sets = 1) {
    bytes = (head + 255) / 256 * 256;
    for (uint32_t u = 0; u < GSB_SM_UNITS; u++) {
      offset[u] = bytes;
      const int64_t n = gsb_sm_expected(u, 0, nullptr, 0);
      set_bytes[u] = (size_t)n * (u <= GSB_SM_UNIT_FP64 ? sizeof(uint64_t) : sizeof(uint32_t));
      bytes += set_bytes[u] * sets;
    }
  }
};

uint32_t popcount_bitmap(const uint32_t *b) {
  uint32_t n = 0;
  for (int i = 0; i < GSB_SM_MAX / 32; i++) n += (uint32_t)__builtin_popcount(b[i]);
  return n;
}

// One launch on the device's stream under the completion watchdog, whose budget is GSB_OPT_WATCHDOG_MS plus
// `extra_ms`: the launch's log (log_bytes at dev_log) is zeroed before it and copied into *log after it, and `poll`
// (if any) is called every few tens of microseconds while the host waits.
int sm_launch_locked(Device *d, const char *what, const std::function<int()> &launch, void *dev_log, void *log,
                     size_t log_bytes, uint64_t extra_ms, const std::function<void()> &poll, uint64_t *kernel_ns) {
  const uint64_t t0 = now_ns();
  cudaError_t e = cudaMemsetAsync(dev_log, 0, log_bytes, d->stream);
  if (e == cudaSuccess) e = cudaEventRecord(d->ev0, d->stream);
  if (e == cudaSuccess) e = (cudaError_t)launch();
  if (e == cudaSuccess) e = cudaEventRecord(d->ev1, d->stream);
  if (e != cudaSuccess) {
    set_error("%s launch on %s: %s", what, d->uuid, cudaGetErrorString(e));
    return GSB_ERR_DRIVER;
  }
  const uint64_t wd_ms = G.watchdog_ms.load(std::memory_order_relaxed);
  while ((e = cudaEventQuery(d->ev1)) == cudaErrorNotReady) {
    if (wd_ms && now_ns() > t0 + (wd_ms + extra_ms) * 1000000ull) {
      d->wedged = true;  // still on the stream: nothing new is queued behind it
      set_error("%s kernel on %s did not finish within %llu ms: device wedged?", what, d->uuid,
                (unsigned long long)(wd_ms + extra_ms));
      return GSB_ERR_TIMEOUT;
    }
    if (poll) poll();
    struct timespec ts = {0, 20000};
    nanosleep(&ts, nullptr);
  }
  float ms = 0.f;
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, d->ev0, d->ev1);
  if (e == cudaSuccess) e = cudaMemcpyAsync(log, dev_log, log_bytes, cudaMemcpyDeviceToHost, d->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
  if (e != cudaSuccess) {
    set_error("%s kernel failed on %s: %s", what, d->uuid, cudaGetErrorString(e));
    return GSB_ERR_DRIVER;
  }
  *kernel_ns += (uint64_t)((double)ms * 1e6);
  return GSB_OK;
}

// One SM-check launch of `unit` (from_table: the test-only kernel on chosen operands).
int sm_launch_locked(Device *d, uint32_t unit, const gsb_sm_args &args, gsb_sm_log *log, uint64_t *kernel_ns,
                     bool from_table) {
  return sm_launch_locked(
      d, "SM check",
      [&] {
        return from_table ? gsb_sm_operands_launch(unit, d->sm_count, &args, d->stream)
                          : gsb_sm_kernel_launch(unit, d->sm_count, &args, d->stream);
      },
      args.log, log, sizeof *log, 0, nullptr, kernel_ns);
}

// Before a new SM check or stress: a launch that outlived the watchdog must have drained (its buffer is given back).
int sm_drain_kept_locked(Device *d) {
  if (!d->wedged && !d->sm_kept) return GSB_OK;
  const int rc = wedged_drain_locked(d);
  if (rc) return rc;
  for (cudaTextureObject_t t : d->sm_kept_tex) cudaDestroyTextureObject(t);  // before the memory they describe
  d->sm_kept_tex.clear();
  if (d->sm_kept) cudaFree(d->sm_kept);
  d->sm_kept = nullptr;
  return GSB_OK;
}

// A transient buffer of `bytes` for an SM check or stress, only while GSB_OPT_TRANSIENT_KEEP_FREE_BYTES stays free.
int sm_alloc_locked(Device *d, const char *what, size_t bytes, void **buf) {
  *buf = nullptr;
  size_t free_b = 0, total_b = 0;
  const uint64_t keep_free = G.transient_keep_free.load();
  if (G.cu.cuMemGetInfo(&free_b, &total_b) != CUDA_SUCCESS || free_b < keep_free || free_b - keep_free < bytes) {
    set_error("%s: %zu bytes of HBM are not allocatable on %s (free %zu, keep_free %llu)", what, bytes, d->uuid, free_b,
              (unsigned long long)keep_free);
    return GSB_ERR_OUT_OF_MEMORY;
  }
  if (cudaMalloc(buf, bytes) != cudaSuccess) {
    *buf = nullptr;
    cudaGetLastError();
    set_error("allocating %zu bytes of HBM for the %s on %s", bytes, what, d->uuid);
    return GSB_ERR_OUT_OF_MEMORY;
  }
  return GSB_OK;
}

// Owns the transient buffer of one SM-side run whose status is `rc`, and the texture objects created over it (`tex`).
// On release (at the latest when the run returns) the objects are destroyed and then the buffer freed, unless the run
// ended in GSB_ERR_TIMEOUT: then a launch still on the stream uses them, and they go to sm_kept and sm_kept_tex, which
// sm_drain_kept_locked gives back once the stream has drained.
struct SmBuffer {
  Device *d;
  const int &rc;
  void *p = nullptr;
  std::vector<cudaTextureObject_t> tex;
  SmBuffer(Device *d, const int &rc) : d(d), rc(rc) {}
  SmBuffer(const SmBuffer &) = delete;
  ~SmBuffer() { release(); }
  int alloc(const char *what, size_t bytes) { return sm_alloc_locked(d, what, bytes, &p); }
  void release() {
    if (!p) return;
    if (rc == GSB_ERR_TIMEOUT) {
      d->sm_kept = p;
      d->sm_kept_tex = std::move(tex);
    } else {
      for (cudaTextureObject_t t : tex) cudaDestroyTextureObject(t);
      cudaFree(p);
    }
    tex.clear();
    p = nullptr;
  }
};

// The most dynamic shared memory a CTA of this device can opt in to.
int smem_optin_locked(Device *d, int *smem) {
  if (cudaDeviceGetAttribute(smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, d->ordinal) == cudaSuccess) return GSB_OK;
  set_error("querying the shared-memory opt-in maximum of %s", d->uuid);
  return GSB_ERR_DRIVER;
}

// Folds one launch's log into its run (or unit) and into the probe's result: the words compared and found wrong, the
// SMs the launch ran on into `covered`, the SMs with a wrong word, and its records while the result has room.
template <typename Log, typename Run, typename Result>
void fold_log(const Log &log, Run *run, Result *out, uint32_t *covered) {
  run->words_checked += log.words;
  run->mismatch_words += log.mismatch_words;
  run->mismatch_bits += log.mismatch_bits;
  for (size_t i = 0; i < std::size(log.covered); i++) {
    covered[i] |= log.covered[i];
    out->faulty[i] |= log.faulty[i];
  }
  const uint32_t got = std::min<uint32_t>(log.count, std::size(log.rec));
  for (uint32_t i = 0; i < got && out->n_records < std::size(out->records); i++)
    out->records[out->n_records++] = log.rec[i];
}

int sm_probe_locked(Device *d, const gsb_sm_cfg *cfg, gsb_sm_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kSmAllUnits) {
    set_error("invalid SM unit mask 0x%x", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kSmAllUnits;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x534D0000u, &d->sm.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const auto hooks = take_hooks(d, &d->sm.hooks.corrupt);
  std::vector<uint32_t> chosen[GSB_SM_UNITS];  // gsb_test_sm_operands of the units this probe runs
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t u = 0; u < GSB_SM_UNITS; u++)
      if (out->units >> u & 1u) chosen[u].swap(d->sm.hooks.operands[u]);
  }
  static const SmLayout layout;
  // chosen operands and their expected words go after the tables, one 256-byte aligned block per unit
  size_t chosen_off[GSB_SM_UNITS] = {}, bytes = layout.bytes;
  for (uint32_t u = 0; u < GSB_SM_UNITS; u++) {
    if (chosen[u].empty()) continue;
    chosen_off[u] = bytes;
    bytes += (chosen[u].size() * sizeof(uint32_t) + 255) / 256 * 256;
  }
  // the exact answers, computed on the host
  const uint64_t t_exp = now_ns();
  std::vector<uint64_t> answers[GSB_SM_UNITS];
  std::string tables(layout.bytes, '\0');
  for (uint32_t u = 0; u < GSB_SM_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    answers[u].resize((size_t)gsb_sm_expected(u, 0, nullptr, 0));
    gsb_sm_expected(u, out->seed_expect, answers[u].data(), answers[u].size());
    for (size_t w = 0; w < answers[u].size(); w++) {
      char *p = &tables[layout.offset[u]];
      if (u <= GSB_SM_UNIT_FP64) memcpy(p + 8 * w, &answers[u][w], 8);
      else {
        const uint32_t v = (uint32_t)answers[u][w];
        memcpy(p + 4 * w, &v, 4);
      }
    }
  }
  out->expected_ns = now_ns() - t_exp;
  // one transient buffer: the launch log and the tables, under the keep-free margin of every transient probe
  SmBuffer buf(d, rc);
  rc = buf.alloc("SM probe", bytes);
  char *const base = static_cast<char *>(buf.p);
  if (rc == GSB_OK) {
    cudaError_t e = cudaMemcpyAsync(base + layout.offset[0], &tables[layout.offset[0]],
                                    layout.bytes - layout.offset[0], cudaMemcpyHostToDevice, d->stream);
    for (uint32_t u = 0; u < GSB_SM_UNITS && e == cudaSuccess; u++)
      if (!chosen[u].empty())
        e = cudaMemcpyAsync(base + chosen_off[u], chosen[u].data(), chosen[u].size() * sizeof(uint32_t),
                            cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || cudaStreamSynchronize(d->stream) != cudaSuccess) {
      set_error("uploading the SM probe's expected answers to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  bool first = true;
  for (uint32_t u = 0; u < GSB_SM_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_sm_unit_result &ur = out->unit[u];
    gsb_sm_args a;
    memset(&a, 0, sizeof a);
    a.log = reinterpret_cast<gsb_sm_log *>(base);
    a.expected = base + (chosen[u].empty() ? layout.offset[u] : chosen_off[u]);
    a.seed = out->seed;
    a.smem_bytes = (uint32_t)smem;
    a.hook_smid = GSB_SM_MAX;
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    // one CTA per SM: a launch that left an SM uncovered (another context held it) is repeated
    while (ur.launches < GSB_SM_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count) {
      if (ur.launches == 0 && hooks[u].armed) {  // test hook: the unit's first launch only
        a.hook_smid = hooks[u].smid;
        a.hook_index = hooks[u].index;
        a.hook_xr = hooks[u].xr;
      } else {
        a.hook_smid = GSB_SM_MAX;
      }
      ur.launches++;
      gsb_sm_log log;
      const int lrc = sm_launch_locked(d, u, a, &log, &ur.kernel_ns, !chosen[u].empty());
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      fold_log(log, &ur, out, covered);
    }
    ur.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_sm_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < out->sm_count);
  }
  count_probe(d, &d->sm.stats, *out, ran, gsb_sm_conditions(out), short_cover ? &d->sm.stats.incomplete : nullptr);
  return rc;
}


// ------------------------------------------------------------------ SM stress (gsb_sm_stress)

// Read-only NVML telemetry while a stress runs: a clear valid bit means no sample of that query was answered.
struct StressSampler {
  Device *d;
  gsb_stress_telemetry *t;
  uint64_t energy0 = 0, energy_t0 = 0, last = 0;
  bool have_energy0 = false;

  void begin() {
    unsigned limit = 0;
    if (G.ml.getEnforcedPowerLimit && G.ml.getEnforcedPowerLimit(d->nvml, &limit) == NVML_SUCCESS) {
      t->valid |= GSB_STRESS_VALID_POWER_LIMIT;
      t->power_limit_w = limit / 1000.0;
    }
    unsigned long long mj = 0;
    if (G.ml.getTotalEnergyConsumption && G.ml.getTotalEnergyConsumption(d->nvml, &mj) == NVML_SUCCESS) {
      have_energy0 = true;
      energy0 = mj;
      energy_t0 = now_ns();
    }
    sample();
  }
  void sample() {
    last = now_ns();
    t->samples++;
    unsigned v = 0;
    if (G.ml.getPowerUsage && G.ml.getPowerUsage(d->nvml, &v) == NVML_SUCCESS) {
      t->power_peak_w = std::max(t->power_peak_w, v / 1000.0);
      t->valid |= GSB_STRESS_VALID_POWER;
    }
    if (G.ml.getTemperature && G.ml.getTemperature(d->nvml, NVML_TEMPERATURE_GPU, &v) == NVML_SUCCESS) {
      t->temp_peak_c = std::max(t->temp_peak_c, v);
      t->valid |= GSB_STRESS_VALID_TEMP;
    }
    if (G.ml.getClockInfo && G.ml.getClockInfo(d->nvml, NVML_CLOCK_SM, &v) == NVML_SUCCESS) {
      const bool first = !(t->valid & GSB_STRESS_VALID_SM_CLOCK);
      t->sm_clock_min_mhz = first ? v : std::min(t->sm_clock_min_mhz, v);
      t->sm_clock_max_mhz = first ? v : std::max(t->sm_clock_max_mhz, v);
      t->valid |= GSB_STRESS_VALID_SM_CLOCK;
    }
    unsigned long long reasons = 0;
    if (G.ml.getClocksEventReasons && G.ml.getClocksEventReasons(d->nvml, &reasons) == NVML_SUCCESS) {
      t->reasons |= reasons;
      if (reasons & GSB_STRESS_SLOWDOWN_REASONS) t->slowdown_samples++;
      t->valid |= GSB_STRESS_VALID_REASONS;
    }
  }
  void poll() {
    if (now_ns() - last >= GSB_STRESS_SAMPLE_MS * 1000000ull) sample();
  }
  void end() {
    unsigned long long mj = 0;
    if (have_energy0 && G.ml.getTotalEnergyConsumption(d->nvml, &mj) == NVML_SUCCESS && mj >= energy0) {
      const uint64_t ns = now_ns() - energy_t0;
      t->power_mean_w = ns ? (double)(mj - energy0) * 1e6 / (double)ns : 0.0;  // mJ / ns * 1e6 = W
      t->valid |= GSB_STRESS_VALID_ENERGY;
    }
  }
};

int stress_locked(Device *d, const gsb_stress_cfg *cfg, gsb_stress_result *out) {
  const uint64_t t0 = now_ns();
  out->first_mismatch_slice = UINT32_MAX;
  if (cfg->units & ~GSB_STRESS_UNIT_MASK) {
    set_error("invalid SM stress unit mask 0x%x (tensor units only)", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  if (cfg->duration_ms == 0 || cfg->duration_ms > GSB_STRESS_DURATION_MAX_MS || cfg->slice_ms > GSB_STRESS_SLICE_MAX_MS) {
    set_error("invalid SM stress duration %u ms or slice %u ms", cfg->duration_ms, cfg->slice_ms);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : GSB_STRESS_UNIT_MASK;
  out->duration_ms = cfg->duration_ms;
  out->slice_ms = cfg->slice_ms ? cfg->slice_ms : GSB_STRESS_SLICE_DEFAULT_MS;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  // no two runs share an operand set (set s uses seed + s)
  out->seed = seed_or_fresh(cfg->seed, 0x53540000u, &d->sm.seed, GSB_STRESS_SETS_MAX);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const Device::StressCorrupt hook = take_hooks(d, &d->stress_corrupt);
  // the buffer: the slice log, every unit's expected folds, then SmLayout's answers, one table per operand set
  const size_t folds_at = (sizeof(gsb_stress_log) + 255) / 256 * 256;
  const size_t fold_set_bytes = GSB_STRESS_FOLD_THREADS * sizeof(uint32_t);
  static const SmLayout layout(folds_at + GSB_STRESS_UNITS * GSB_STRESS_SETS_MAX * fold_set_bytes,
                               GSB_STRESS_SETS_MAX);
  const uint64_t t_exp = now_ns();
  std::string tables(layout.bytes, '\0');
  std::vector<uint64_t> answer(GSB_SM_TENSOR_WORDS);
  for (uint32_t u = GSB_SM_UNIT_F16; u <= GSB_SM_UNIT_S8; u++) {
    if (!(out->units >> u & 1u)) continue;
    for (uint32_t set = 0; set < gsb_stress_sets(u); set++) {
      gsb_sm_expected(u, out->seed_expect + set, answer.data(), answer.size());
      uint32_t *words = reinterpret_cast<uint32_t *>(&tables[layout.offset[u] + set * layout.set_bytes[u]]);
      for (size_t w = 0; w < answer.size(); w++) words[w] = (uint32_t)answer[w];
      gsb_stress_fold(u, out->seed_expect + set,
                      reinterpret_cast<uint32_t *>(&tables[folds_at + ((u - GSB_SM_UNIT_F16) * GSB_STRESS_SETS_MAX + set) *
                                                                          fold_set_bytes]),
                      GSB_STRESS_FOLD_THREADS);
    }
  }
  out->expected_ns = now_ns() - t_exp;
  SmBuffer buf(d, rc);
  rc = buf.alloc("SM stress", layout.bytes);
  char *const base = static_cast<char *>(buf.p);
  if (rc == GSB_OK) {
    const cudaError_t e = cudaMemcpyAsync(base + folds_at, &tables[folds_at], layout.bytes - folds_at,
                                          cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || cudaStreamSynchronize(d->stream) != cudaSuccess) {
      set_error("uploading the SM stress's expected answers to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  uint32_t sel[GSB_STRESS_UNITS], nsel = 0;
  for (uint32_t u = GSB_SM_UNIT_F16; u <= GSB_SM_UNIT_S8; u++)
    if (out->units >> u & 1u) sel[nsel++] = u;
  StressSampler sampler{d, &out->telemetry};
  if (rc == GSB_OK) sampler.begin();
  const std::function<void()> poll = [&] { sampler.poll(); };
  uint64_t sm_iters[GSB_SM_MAX] = {};
  const uint32_t n_slices = (out->duration_ms + out->slice_ms - 1) / out->slice_ms;
  for (uint32_t i = 0; i < n_slices && rc == GSB_OK; i++) {
    const uint32_t u = sel[i % nsel], k = u - GSB_SM_UNIT_F16;
    const uint32_t len_ms = std::min(out->slice_ms, out->duration_ms - i * out->slice_ms);
    gsb_stress_unit_result &ur = out->unit[k];
    gsb_stress_args a;
    memset(&a, 0, sizeof a);
    a.log = reinterpret_cast<gsb_stress_log *>(base);
    a.expected = reinterpret_cast<const uint32_t *>(base + layout.offset[u]);
    a.folds = reinterpret_cast<const uint32_t *>(base + folds_at + k * GSB_STRESS_SETS_MAX * fold_set_bytes);
    a.slice_ns = len_ms * 1000000ull;
    a.max_iters = (uint64_t)len_ms * 1000 * gsb_stress_iters_per_us(u);
    a.seed = out->seed;
    a.slice = i;
    a.smem_bytes = (uint32_t)smem;
    a.hook_smid = GSB_SM_MAX;
    if (hook.armed && hook.slice == i && hook.unit == u) {
      a.hook_smid = hook.smid;
      a.hook_index = hook.index;
      a.hook_xr = hook.xr;
    }
    ur.slices++;
    ur.sets = gsb_stress_sets(u);
    out->slices++;
    gsb_stress_log log;
    const uint64_t ts = now_ns(), kernel_before = ur.kernel_ns;
    const int lrc = sm_launch_locked(
        d, "SM stress", [&] { return gsb_stress_kernel_launch(u, d->sm_count, &a, d->stream); }, a.log, &log,
        sizeof log, len_ms, poll, &ur.kernel_ns);
    out->gap_ns += (now_ns() - ts) - (ur.kernel_ns - kernel_before);
    if (lrc != GSB_OK) {
      ur.status = rc = lrc;
      break;
    }
    for (uint32_t s = 0; s < GSB_STRESS_SETS_MAX; s++) {
      ur.set_iterations[s] += log.set_iterations[s];
      ur.iterations += log.set_iterations[s];
    }
    if (log.mismatch_words && out->first_mismatch_slice == UINT32_MAX) {
      out->first_mismatch_slice = i;
      out->first_mismatch_ms = (now_ns() - t0) / 1000000ull;
    }
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    fold_log(log, &ur, out, covered);
    for (int w = 0; w < GSB_SM_MAX / 32; w++) out->covered[w] = i == 0 ? covered[w] : out->covered[w] & covered[w];
    for (uint32_t sm = 0; sm < GSB_SM_MAX; sm++) sm_iters[sm] += log.sm_iterations[sm];
  }
  if (out->slices) sampler.end();
  for (gsb_stress_unit_result &ur : out->unit) {
    const uint32_t u = (uint32_t)(&ur - out->unit) + GSB_SM_UNIT_F16;
    const double ops = 2.0 * GSB_SM_M * GSB_SM_N * gsb_sm_shape(u).k * (double)ur.iterations;
    ur.tera_ops = ur.kernel_ns ? ops / (double)ur.kernel_ns / 1e3 : 0.0;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  bool first = true;
  for (uint32_t sm = 0; sm < GSB_SM_MAX; sm++) {
    if (!(out->covered[sm >> 5] >> (sm & 31u) & 1u)) continue;
    if (first || sm_iters[sm] < out->sm_iterations_min) {
      out->sm_iterations_min = sm_iters[sm];
      out->sm_iterations_min_smid = sm;
    }
    if (first || sm_iters[sm] > out->sm_iterations_max) out->sm_iterations_max = sm_iters[sm];
    first = false;
  }
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  return rc;
}

// ------------------------------------------------------------------ SM-to-SM health (gsb_cluster_probe)

constexpr uint32_t kClusterAllPaths = (1u << GSB_CLUSTER_PATHS) - 1;
constexpr uint32_t kClusterAllSizes = (1u << GSB_CLUSTER_SIZES) - 1;
// a launch whose waits all run out takes two of them (ST_ASYNC: the free wait, then the receive waits)
constexpr uint64_t kClusterWaitsMs = 2ull * GSB_CLUSTER_WAIT_NS / 1000000ull;

// One SM-to-SM launch of `path`: `clusters` clusters of n CTAs; with `script` (device memory), the path's test-only twin.
int cluster_launch_locked(Device *d, uint32_t path, uint32_t n, uint32_t clusters, const gsb_cluster_args &args,
                          const gsb_cluster_script *script, gsb_cluster_log *log, uint64_t *kernel_ns) {
  return sm_launch_locked(
      d, "SM-to-SM check",
      [&] {
        return script ? gsb_cluster_script_launch(path, n, clusters, &args, script, d->stream)
                      : gsb_cluster_kernel_launch(path, n, clusters, &args, d->stream);
      },
      args.log, log, sizeof *log, kClusterWaitsMs, nullptr, kernel_ns);
}

int cluster_probe_locked(Device *d, const gsb_cluster_cfg *cfg, gsb_cluster_result *out) {
  const uint64_t t0 = now_ns();
  if ((cfg->paths & ~kClusterAllPaths) || (cfg->sizes & ~kClusterAllSizes)) {
    set_error("invalid SM-to-SM path mask 0x%x or size mask 0x%x", cfg->paths, cfg->sizes);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->paths = cfg->paths ? cfg->paths : kClusterAllPaths;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  int smem = 0;
  if (!rc) rc = smem_optin_locked(d, &smem);
  if (rc) return out->status = rc;
  out->smem_bytes = (uint32_t)smem;
  for (uint32_t k = 0; k < GSB_CLUSTER_SIZES; k++) {
    const uint32_t n = 2u << k;
    int m = 0;
    if (gsb_cluster_max_active(n, smem, &m) != cudaSuccess) {
      cudaGetLastError();
      m = 0;
    }
    out->max_clusters[k] = m > 0 ? (uint32_t)m : 0u;
    const uint64_t reach = (uint64_t)out->max_clusters[k] * n;
    out->expect_covered[k] = (uint32_t)(reach < d->sm_count ? reach : d->sm_count);
  }
  // the defaults: n = 2 (most likely the two SMs of a TPC) and the largest of 16 and 8 that can be scheduled (a GPC)
  out->sizes = cfg->sizes ? cfg->sizes : 1u | (out->max_clusters[3] ? 8u : out->max_clusters[2] ? 4u : 0u);
  out->seed = seed_or_fresh(cfg->seed, 0x434C0000u, &d->cluster.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  auto hooks = take_hooks(d, &d->cluster.hooks);
  // gsb_test_cluster_script: taken by the first probe that runs its (path, size)
  std::array<std::array<Device::ClusterScript, GSB_CLUSTER_SIZES>, GSB_CLUSTER_PATHS> scripts;
  bool any_script = false;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t p = 0; p < GSB_CLUSTER_PATHS; p++)
      for (uint32_t k = 0; k < GSB_CLUSTER_SIZES; k++)
        if (out->paths >> p & 1u && out->sizes >> k & 1u && d->cluster_scripts[p][k].armed) {
          scripts[p][k] = std::exchange(d->cluster_scripts[p][k], Device::ClusterScript{});
          any_script = true;
        }
  }
  // one transient buffer: the launch log, then the multicast source (n segments; at most the area of one CTA), then
  // with a script, the script and its own multicast source
  const size_t log_bytes = (sizeof(gsb_cluster_log) + 255) / 256 * 256;
  const size_t src_bytes = 16ull * gsb_cluster_area_words((uint32_t)smem);
  const size_t script_bytes = (sizeof(gsb_cluster_script) + 255) / 256 * 256;
  SmBuffer buf(d, rc);
  rc = buf.alloc("SM-to-SM probe", log_bytes + src_bytes + (any_script ? script_bytes + src_bytes : 0));
  gsb_cluster_script *script_dev = reinterpret_cast<gsb_cluster_script *>(static_cast<char *>(buf.p) + log_bytes + src_bytes);
  const void *script_src = static_cast<char *>(buf.p) + log_bytes + src_bytes + script_bytes;
  std::vector<uint32_t> src_words;
  for (uint32_t k = 0; k < GSB_CLUSTER_SIZES && rc == GSB_OK; k++) {
    if (!(out->sizes >> k & 1u)) continue;
    const uint32_t n = 2u << k;
    if (!out->max_clusters[k]) {  // asked for explicitly, and no cluster of n fits: nothing to launch
      set_error("clusters of %u CTAs with %d bytes of shared memory each cannot be scheduled on %s", n, smem, d->uuid);
      rc = GSB_ERR_INVALID_ARGUMENT;
      break;
    }
    for (uint32_t p = 0; p < GSB_CLUSTER_PATHS && rc == GSB_OK; p++) {
      if (!(out->paths >> p & 1u)) continue;
      gsb_cluster_run &run = out->run[p][k];
      gsb_cluster_args a;
      memset(&a, 0, sizeof a);
      a.log = static_cast<gsb_cluster_log *>(buf.p);
      a.mc_src = static_cast<char *>(buf.p) + log_bytes;
      a.seed = out->seed;
      a.seed_expect = out->seed_expect;
      a.smem_bytes = (uint32_t)smem;
      const Device::ClusterScript &sc = scripts[p][k];
      if (sc.armed && sc.script.region_words > gsb_cluster_region_words(p, n, (uint32_t)smem)) {
        set_error("an SM-to-SM script of %u words per region does not fit %d bytes of shared memory on %s",
                  sc.script.region_words, smem, d->uuid);
        run.status = rc = GSB_ERR_INVALID_ARGUMENT;
        break;
      }
      // segment s: what rank s multicasts to every rank, at the probe's region size and at the script's
      const auto upload = [&](const void *dst, uint32_t rw) {
        const uint32_t key = gsb_seed_key(out->seed);
        src_words.resize(4ull * n * rw);
        for (uint32_t s = 0; s < n; s++)
          for (uint32_t i = 0; i < rw; i++)
            gsb_pattern_word(gsb_cluster_word_addr(p, n, s, GSB_CLUSTER_EVERY_RANK, i), key,
                             &src_words[4ull * (s * rw + i)]);
        return cudaMemcpyAsync(const_cast<void *>(dst), src_words.data(), 4 * src_words.size(), cudaMemcpyHostToDevice,
                               d->stream);
      };
      cudaError_t e = cudaSuccess;
      if (p == GSB_CLUSTER_PATH_MULTICAST) e = upload(a.mc_src, gsb_cluster_region_words(p, n, (uint32_t)smem));
      if (e == cudaSuccess && sc.armed && p == GSB_CLUSTER_PATH_MULTICAST) e = upload(script_src, sc.script.region_words);
      if (e == cudaSuccess && sc.armed)
        e = cudaMemcpyAsync(script_dev, &sc.script, sizeof sc.script, cudaMemcpyHostToDevice, d->stream);
      if (e != cudaSuccess || (e = cudaStreamSynchronize(d->stream)) != cudaSuccess) {
        set_error("uploading the SM-to-SM probe's multicast source or script to %s: %s", d->uuid,
                  cudaGetErrorString(e));
        run.status = rc = GSB_ERR_DRIVER;
        break;
      }
      uint32_t covered[GSB_CLUSTER_SM_MAX / 32] = {0};
      // a launch that left an SM it could reach uncovered (another context held it) is repeated
      while (run.launches < GSB_CLUSTER_MAX_LAUNCHES && popcount_bitmap(covered) < out->expect_covered[k]) {
        a.hook_smid = a.skip_smid = GSB_CLUSTER_SM_MAX;
        if (hooks[p].corrupt) {  // test hooks: the path's first launch only
          a.hook_smid = hooks[p].corrupt_smid;
          a.hook_index = hooks[p].index;
          a.hook_xr = hooks[p].xr;
        }
        if (hooks[p].skip) a.skip_smid = hooks[p].skip_smid;
        hooks[p] = Device::ClusterHook{};
        // a script runs in the pair's first launch only; a relaunch for coverage is the probe's own
        const bool scripted = sc.armed && run.launches == 0;
        gsb_cluster_args la = a;
        if (scripted && p == GSB_CLUSTER_PATH_MULTICAST) la.mc_src = script_src;
        run.launches++;
        gsb_cluster_log log;
        const int lrc = cluster_launch_locked(d, p, n, out->max_clusters[k], la, scripted ? script_dev : nullptr, &log,
                                              &run.kernel_ns);
        if (lrc != GSB_OK) {
          run.status = rc = lrc;
          break;
        }
        run.timeouts += log.timeouts;
        fold_log(log, &run, out, covered);
      }
      run.sms_covered = popcount_bitmap(covered);
      for (int i = 0; i < GSB_CLUSTER_SM_MAX / 32; i++) out->covered[i] |= covered[i];
    }
  }
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (uint32_t p = 0; p < GSB_CLUSTER_PATHS; p++)
    for (uint32_t k = 0; k < GSB_CLUSTER_SIZES; k++) {
      const gsb_cluster_run &run = out->run[p][k];
      ran = ran || run.launches != 0;
      short_cover = short_cover || (run.launches != 0 && run.status == GSB_OK && run.sms_covered < out->expect_covered[k]);
    }
  count_probe(d, &d->cluster.stats, *out, ran, gsb_cluster_conditions(out),
              short_cover ? &d->cluster.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ L2 atomic health (gsb_atomic_probe)

constexpr uint32_t kAtomicAllOps = (1u << GSB_ATOMIC_OPS) - 1;
constexpr size_t kAtomicLogBytes = (sizeof(gsb_atomic_log) + 255) / 256 * 256;

// Adds one record to the result, and the SM it names to the faulty bitmap.
void atomic_add_record(gsb_atomic_result *out, const gsb_atomic_record &rec) {
  if (rec.smid < GSB_ATOMIC_SM_MAX) out->faulty[rec.smid >> 5] |= 1u << (rec.smid & 31u);
  if (out->n_records < GSB_ATOMIC_RECORDS) out->records[out->n_records++] = rec;
}

// TICKET and CAS: every slot of hot word l must hold a distinct id below its contributor count. Returns the slots that
// do not; each is recorded, naming the SM of the CTA whose id it holds twice (GSB_ATOMIC_NO_SM for an empty slot).
uint64_t atomic_check_slots(uint32_t op, uint32_t ctas, const std::vector<uint32_t> &slots, const gsb_atomic_log &log,
                            gsb_atomic_result *out) {
  const uint32_t count = gsb_atomic_hot_count(op, ctas), per_cta = count / ctas;
  uint64_t bad = 0;
  std::vector<char> seen(count);
  for (uint32_t l = 0; l < GSB_ATOMIC_HOT_WORDS; l++) {
    std::fill(seen.begin(), seen.end(), 0);
    for (uint32_t t = 0; t < count; t++) {
      const uint32_t id = slots[(size_t)l * count + t];
      if (id < count && !seen[id]) {
        seen[id] = 1;
        continue;
      }
      bad++;
      gsb_atomic_record rec{op, GSB_ATOMIC_PHASE_SLOT, l * count + t, GSB_ATOMIC_NO_SM, count, id};
      if (id < count) rec.smid = log.cta_smid[id / per_cta];
      atomic_add_record(out, rec);
    }
  }
  return bad;
}

int atomic_probe_locked(Device *d, const gsb_atomic_cfg *cfg, gsb_atomic_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->ops & ~kAtomicAllOps) {
    set_error("invalid L2 atomic op mask 0x%x", cfg->ops);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->ops = cfg->ops ? cfg->ops : kAtomicAllOps;
  out->sm_count = d->sm_count;
  for (gsb_atomic_run &run : out->run) run.hook_cta = GSB_ATOMIC_NO_SM;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  if (d->sm_count > GSB_ATOMIC_SM_MAX) {
    set_error("%s has %u SMs, more than the L2 atomic probe's %d", d->uuid, d->sm_count, GSB_ATOMIC_SM_MAX);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  int smem = 0;
  if ((rc = smem_optin_locked(d, &smem))) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x41540000u, &d->atomic.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const auto hooks = take_hooks(d, &d->atomic.hooks);
  // gsb_test_atomic_values: taken by the first probe that runs its op
  std::array<Device::AtomicValues, GSB_ATOMIC_OPS> chosen;
  bool any_chosen = false;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t op = 0; op < GSB_ATOMIC_OPS; op++)
      if (out->ops >> op & 1u && d->atomic_values[op].armed) {
        chosen[op] = std::exchange(d->atomic_values[op], Device::AtomicValues{});
        any_chosen = true;
      }
  }
  // one transient buffer: the run and check logs, the words, the expected words, the ticket slots, a chosen table
  const uint32_t ctas = d->sm_count;
  const size_t slot_words = (size_t)GSB_ATOMIC_HOT_WORDS * gsb_atomic_hot_count(GSB_ATOMIC_OP_TICKET, ctas);
  const size_t off_words = 2 * kAtomicLogBytes, off_expect = off_words + GSB_ATOMIC_BYTES;
  const size_t off_slots = off_expect + GSB_ATOMIC_BYTES, off_values = off_slots + 4 * slot_words;
  const size_t bytes = off_values + (any_chosen ? 8 * gsb_atomic_value_count(ctas) : 0);
  SmBuffer buf(d, rc);
  rc = buf.alloc("L2 atomic probe", bytes);
  char *base = static_cast<char *>(buf.p);
  bool first = true;
  std::vector<unsigned char> expect(GSB_ATOMIC_BYTES);
  std::vector<uint32_t> slots;
  for (uint32_t op = 0; op < GSB_ATOMIC_OPS && rc == GSB_OK; op++) {
    if (!(out->ops >> op & 1u)) continue;
    gsb_atomic_run &run = out->run[op];
    const Device::AtomicValues &cv = chosen[op];
    const uint64_t *values = reinterpret_cast<const uint64_t *>(base + off_values);
    if (!cv.armed) {
      const uint64_t t_exp = now_ns();
      const int64_t n = gsb_atomic_expected(op, out->seed_expect, ctas, expect.data(), expect.size());
      out->expected_ns += now_ns() - t_exp;
      if (n != (int64_t)GSB_ATOMIC_BYTES) {
        set_error("computing the L2 atomic probe's expected words of op %u on %s", op, d->uuid);
        run.status = rc = GSB_ERR_INVALID_ARGUMENT;
        break;
      }
    }
    const std::vector<unsigned char> &want = cv.armed ? cv.expected : expect;
    cudaError_t e = cudaMemcpyAsync(base + off_expect, want.data(), want.size(), cudaMemcpyHostToDevice, d->stream);
    if (e == cudaSuccess && cv.armed)
      e = cudaMemcpyAsync(base + off_values, cv.table.data(), 8 * cv.table.size(), cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || (e = cudaStreamSynchronize(d->stream)) != cudaSuccess) {
      set_error("uploading the L2 atomic probe's expected words to %s: %s", d->uuid, cudaGetErrorString(e));
      run.status = rc = GSB_ERR_DRIVER;
      break;
    }
    gsb_atomic_args a;
    memset(&a, 0, sizeof a);
    gsb_atomic_log *run_log = reinterpret_cast<gsb_atomic_log *>(base);
    gsb_atomic_log *check_log = reinterpret_cast<gsb_atomic_log *>(base + kAtomicLogBytes);
    a.buf = base + off_words;
    a.expected = base + off_expect;
    a.slots = reinterpret_cast<uint32_t *>(base + off_slots);
    a.op = op;
    a.seed = out->seed;
    a.ctas = ctas;
    a.smem_bytes = (uint32_t)smem;
    const bool tickets = op == GSB_ATOMIC_OP_TICKET || op == GSB_ATOMIC_OP_CAS;
    // a CAS loop may run to its deadline
    const uint64_t extra_ms = op == GSB_ATOMIC_OP_CAS ? GSB_ATOMIC_CAS_WAIT_NS / 1000000u : 0u;
    uint32_t covered[GSB_ATOMIC_SM_MAX / 32] = {0};
    // one CTA per SM: a run that left an SM uncovered (another context held it) is repeated from its init
    while (run.launches < GSB_ATOMIC_MAX_LAUNCHES && popcount_bitmap(covered) < ctas) {
      a.hook_word = 0xFFFFFFFFu;
      a.hook_xr = 0;
      a.skip_smid = GSB_ATOMIC_SM_MAX;
      if (run.launches == 0) {  // test hooks: the op's first launches only
        if (hooks[op].corrupt) a.hook_word = hooks[op].word, a.hook_xr = hooks[op].xr;
        if (hooks[op].skip) a.skip_smid = hooks[op].skip_smid;
      }
      run.launches++;
      gsb_atomic_log rl, cl;
      const auto stage = [&](uint32_t s) { return [&a, d, s] { return gsb_atomic_kernel_launch(s, &a, d->stream); }; };
      // chosen values: the starting words are uploaded (again on a relaunch) and the twin runs on the table
      const auto upload_init = [&] {
        return (int)cudaMemcpyAsync(a.buf, cv.init.data(), cv.init.size(), cudaMemcpyHostToDevice, d->stream);
      };
      const auto run_table = [&] { return gsb_atomic_values_launch(&a, values, d->stream); };
      a.log = check_log;
      int lrc = cv.armed ? sm_launch_locked(d, "L2 atomic init", upload_init, check_log, &cl, sizeof cl, 0, nullptr,
                                            &run.kernel_ns)
                         : sm_launch_locked(d, "L2 atomic init", stage(GSB_ATOMIC_STAGE_INIT), check_log, &cl,
                                            sizeof cl, 0, nullptr, &run.kernel_ns);
      a.log = run_log;
      if (lrc == GSB_OK)
        lrc = cv.armed ? sm_launch_locked(d, "L2 atomic run", run_table, run_log, &rl, sizeof rl, extra_ms, nullptr,
                                          &run.kernel_ns)
                       : sm_launch_locked(d, "L2 atomic run", stage(GSB_ATOMIC_STAGE_RUN), run_log, &rl, sizeof rl,
                                          extra_ms, nullptr, &run.kernel_ns);
      a.log = check_log;
      if (lrc == GSB_OK)
        lrc = sm_launch_locked(d, "L2 atomic verify", stage(GSB_ATOMIC_STAGE_CHECK), check_log, &cl, sizeof cl, 0,
                               nullptr, &run.kernel_ns);
      if (lrc == GSB_OK && tickets) {
        slots.resize((size_t)GSB_ATOMIC_HOT_WORDS * gsb_atomic_hot_count(op, ctas));
        e = cudaMemcpy(slots.data(), a.slots, 4 * slots.size(), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) {
          set_error("reading the L2 atomic probe's ticket slots on %s: %s", d->uuid, cudaGetErrorString(e));
          lrc = GSB_ERR_DRIVER;
        }
      }
      if (lrc != GSB_OK) {
        run.status = rc = lrc;
        break;
      }
      if (rl.skipped_cta) run.hook_cta = rl.skipped_cta - 1u;
      run.atomics_issued += rl.issued;
      run.cas_timeouts += rl.timeouts;
      run.cas_max_ns = std::max<uint64_t>(run.cas_max_ns, rl.cas_max_ns);
      run.ticket_faults += rl.out_of_range;
      run.words_checked += cl.words;
      run.mismatch_words += cl.mismatch_words;
      run.mismatch_bits += cl.mismatch_bits;
      for (int i = 0; i < GSB_ATOMIC_SM_MAX / 32; i++) covered[i] |= rl.covered[i];
      // records: out-of-range tickets first, then wrong words, then slots
      for (uint32_t i = 0; i < std::min<uint32_t>(rl.count, GSB_ATOMIC_RECORDS); i++) atomic_add_record(out, rl.rec[i]);
      for (uint32_t i = 0; i < std::min<uint32_t>(cl.count, GSB_ATOMIC_RECORDS); i++) atomic_add_record(out, cl.rec[i]);
      if (tickets) run.ticket_faults += atomic_check_slots(op, ctas, slots, rl, out);
    }
    run.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_ATOMIC_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_atomic_run &run : out->run) {
    ran = ran || run.launches != 0;
    short_cover = short_cover || (run.launches != 0 && run.status == GSB_OK && run.sms_covered < out->sm_count);
  }
  count_probe(d, &d->atomic.stats, *out, ran, gsb_atomic_conditions(out),
              short_cover ? &d->atomic.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ tensor-core format health

constexpr uint32_t kTensorAllUnits = (1u << GSB_TENSOR_UNITS) - 1;

int tensor_probe_locked(Device *d, const gsb_tensor_cfg *cfg, gsb_tensor_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kTensorAllUnits) {
    set_error("invalid tensor unit mask 0x%x", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kTensorAllUnits;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x54430000u, &d->tensor.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const auto hooks = take_hooks(d, &d->tensor.hooks.corrupt);
  std::vector<uint32_t> chosen[GSB_TENSOR_UNITS];  // gsb_test_tensor_operands of the units this probe runs
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t u = 0; u < GSB_TENSOR_UNITS; u++)
      if (out->units >> u & 1u) chosen[u].swap(d->tensor.hooks.operands[u]);
  }
  // the buffer: the launch log, then per unit its 8192 expected words or its chosen operands' block, 256-byte aligned
  size_t offset[GSB_TENSOR_UNITS] = {}, bytes = (sizeof(gsb_sm_log) + 255) / 256 * 256;
  for (uint32_t u = 0; u < GSB_TENSOR_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    offset[u] = bytes;
    const size_t n = chosen[u].empty() ? (size_t)GSB_TENSOR_WORDS * gsb_tensor_word_bytes(u)
                                       : chosen[u].size() * sizeof(uint32_t);
    bytes += (n + 255) / 256 * 256;
  }
  // the exact answers, computed on the host; HMMA and F16_RS share one (the SM check's F16 GEMM)
  const uint64_t t_exp = now_ns();
  std::string tables(bytes, '\0');
  std::vector<uint64_t> words(GSB_TENSOR_WORDS), f16;
  for (uint32_t u = 0; u < GSB_TENSOR_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    char *p = &tables[offset[u]];
    if (!chosen[u].empty()) {
      memcpy(p, chosen[u].data(), chosen[u].size() * sizeof(uint32_t));
      continue;
    }
    const bool f16_gemm = u == GSB_TENSOR_UNIT_HMMA || u == GSB_TENSOR_UNIT_F16_RS;
    if (f16_gemm && !f16.empty()) {
      words = f16;
    } else {
      gsb_tensor_expected(u, out->seed_expect, words.data(), words.size());
      if (f16_gemm) f16 = words;
    }
    for (size_t w = 0; w < words.size(); w++) {
      if (u == GSB_TENSOR_UNIT_DMMA) memcpy(p + 8 * w, &words[w], 8);
      else {
        const uint32_t v = (uint32_t)words[w];
        memcpy(p + 4 * w, &v, 4);
      }
    }
  }
  out->expected_ns = now_ns() - t_exp;
  // one transient buffer: the launch log and the tables, under the keep-free margin of every transient probe
  SmBuffer buf(d, rc);
  rc = buf.alloc("tensor probe", bytes);
  char *const base = static_cast<char *>(buf.p);
  if (rc == GSB_OK) {
    const size_t head = (sizeof(gsb_sm_log) + 255) / 256 * 256;
    const cudaError_t e = cudaMemcpyAsync(base + head, &tables[head], bytes - head, cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || cudaStreamSynchronize(d->stream) != cudaSuccess) {
      set_error("uploading the tensor probe's expected answers to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  bool first = true;
  for (uint32_t u = 0; u < GSB_TENSOR_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_tensor_unit_result &ur = out->unit[u];
    gsb_sm_args a;
    memset(&a, 0, sizeof a);
    a.log = reinterpret_cast<gsb_sm_log *>(base);
    a.expected = base + offset[u];
    a.seed = out->seed;
    a.smem_bytes = (uint32_t)smem;
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    // one CTA per SM: a launch that left an SM uncovered (another context held it) is repeated
    while (ur.launches < GSB_TENSOR_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count) {
      const bool hook = ur.launches == 0 && hooks[u].armed;  // test hook: the unit's first launch only
      a.hook_smid = hook ? hooks[u].smid : GSB_SM_MAX;
      a.hook_index = hooks[u].index;
      a.hook_xr = hooks[u].xr;
      ur.launches++;
      gsb_sm_log log;
      const int lrc = sm_launch_locked(
          d, "tensor check",
          [&] {
            return chosen[u].empty() ? gsb_tensor_kernel_launch(u, d->sm_count, &a, d->stream)
                                     : gsb_tensor_operands_launch(u, d->sm_count, &a, d->stream);
          },
          a.log, &log, sizeof log, 0, nullptr, &ur.kernel_ns);
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      fold_log(log, &ur, out, covered);
    }
    ur.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_tensor_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < out->sm_count);
  }
  count_probe(d, &d->tensor.stats, *out, ran, gsb_tensor_conditions(out),
              short_cover ? &d->tensor.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ SM special-function health

constexpr uint32_t kSfuAllUnits = (1u << GSB_SFU_UNITS) - 1;

int sfu_probe_locked(Device *d, const gsb_sfu_cfg *cfg, gsb_sfu_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kSfuAllUnits) {
    set_error("invalid SFU unit mask 0x%x", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kSfuAllUnits;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x53460000u, &d->sfu.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const auto hooks = take_hooks(d, &d->sfu.hooks);
  // the buffer: the launch log, then per exact unit its folds, then MUFU's folds, raw results and %smid per CTA, each
  // 256-byte aligned
  const auto align = [](size_t n) { return (n + 255) / 256 * 256; };
  const bool mufu = out->units >> GSB_SFU_UNIT_MUFU & 1u;
  const size_t ctas = (size_t)d->sm_count;
  const size_t fold_bytes = mufu ? ctas * GSB_SFU_MUFU_FOLDS * sizeof(uint64_t) : 0;
  const size_t raw_bytes = mufu ? ctas * GSB_SFU_MUFU_FOLDS * GSB_SFU_RAW * sizeof(uint32_t) : 0;
  const size_t smid_bytes = mufu ? ctas * sizeof(uint32_t) : 0;
  size_t offset[GSB_SFU_UNITS] = {}, bytes = align(sizeof(gsb_sm_log));
  for (uint32_t u = 0; u < GSB_SFU_UNIT_MUFU; u++) {
    if (!(out->units >> u & 1u)) continue;
    offset[u] = bytes;
    bytes += align((size_t)gsb_sfu_ops(u) * GSB_SFU_THREADS * sizeof(uint64_t));
  }
  const size_t fold_off = bytes, raw_off = fold_off + align(fold_bytes), smid_off = raw_off + align(raw_bytes);
  bytes = smid_off + align(smid_bytes);
  // the exact units' folds, computed on the host, one thread per unit
  const uint64_t t_exp = now_ns();
  std::string tables(fold_off, '\0');
  {
    std::vector<std::thread> units;
    for (uint32_t u = 0; u < GSB_SFU_UNIT_MUFU; u++)
      if (out->units >> u & 1u)
        units.emplace_back(gsb_sfu_expected, u, out->seed_expect, reinterpret_cast<uint64_t *>(&tables[offset[u]]),
                           (size_t)gsb_sfu_ops(u) * GSB_SFU_THREADS);
    for (std::thread &t : units) t.join();
  }
  out->expected_ns = now_ns() - t_exp;
  // one transient buffer: the launch log, the folds and MUFU's output, under the keep-free margin of every transient
  // probe
  SmBuffer buf(d, rc);
  rc = buf.alloc("SFU probe", bytes);
  char *const base = static_cast<char *>(buf.p);
  const size_t head = align(sizeof(gsb_sm_log));
  if (rc == GSB_OK && fold_off > head) {
    const cudaError_t e = cudaMemcpyAsync(base + head, &tables[head], fold_off - head, cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || cudaStreamSynchronize(d->stream) != cudaSuccess) {
      set_error("uploading the SFU probe's expected folds to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  std::vector<uint64_t> folds(mufu ? ctas * GSB_SFU_MUFU_FOLDS : 0);
  std::vector<uint32_t> raw(mufu ? ctas * GSB_SFU_MUFU_FOLDS * GSB_SFU_RAW : 0), smids(mufu ? ctas : 0);
  bool first = true;
  for (uint32_t u = 0; u < GSB_SFU_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_sfu_unit_result &ur = out->unit[u];
    gsb_sfu_args a;
    memset(&a, 0, sizeof a);
    a.sm.log = reinterpret_cast<gsb_sm_log *>(base);
    a.sm.expected = base + offset[u];
    a.sm.seed = out->seed;
    a.sm.smem_bytes = (uint32_t)smem;
    a.folds = reinterpret_cast<unsigned long long *>(base + fold_off);
    a.raw = reinterpret_cast<uint32_t *>(base + raw_off);
    a.smid = reinterpret_cast<uint32_t *>(base + smid_off);
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    // one CTA per SM: a launch that left an SM uncovered (another context held it) is repeated
    while (ur.launches < GSB_SFU_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count) {
      const bool hook = ur.launches == 0 && hooks[u].armed;  // test hook: the unit's first launch only
      a.sm.hook_smid = hook ? hooks[u].smid : GSB_SM_MAX;
      a.sm.hook_index = hooks[u].index;
      a.sm.hook_xr = hooks[u].xr;
      ur.launches++;
      gsb_sm_log log;
      const int lrc = sm_launch_locked(
          d, "SFU check", [&] { return gsb_sfu_kernel_launch(u, d->sm_count, &a, d->stream); }, a.sm.log, &log,
          sizeof log, 0, nullptr, &ur.kernel_ns);
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      fold_log(log, &ur, out, covered);
      if (u != GSB_SFU_UNIT_MUFU) continue;
      // MUFU: every CTA's folds and raw results to the host, then the vote
      cudaError_t e = cudaMemcpyAsync(folds.data(), a.folds, fold_bytes, cudaMemcpyDeviceToHost, d->stream);
      if (e == cudaSuccess) e = cudaMemcpyAsync(raw.data(), a.raw, raw_bytes, cudaMemcpyDeviceToHost, d->stream);
      if (e == cudaSuccess) e = cudaMemcpyAsync(smids.data(), a.smid, smid_bytes, cudaMemcpyDeviceToHost, d->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
      if (e != cudaSuccess) {
        set_error("reading the SFU probe's MUFU results from %s: %s", d->uuid, cudaGetErrorString(e));
        ur.status = rc = GSB_ERR_DRIVER;
        break;
      }
      const uint64_t t_vote = now_ns();
      gsb_sfu_vote(out->seed, d->sm_count, folds.data(), raw.data(), smids.data(), out);
      out->vote_ns += now_ns() - t_vote;
    }
    ur.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_sfu_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < out->sm_count);
  }
  count_probe(d, &d->sfu.stats, *out, ran, gsb_sfu_conditions(out), short_cover ? &d->sfu.stats.incomplete : nullptr);
  return rc;
}

// gsb_test_sfu_inputs on a device: the chosen operands to the device, one CTA of the unit's twin per SM until every SM
// ran (or GSB_SFU_MAX_LAUNCHES), then each SM's raw results to results[smid * n + i].
int sfu_inputs_locked(Device *d, uint32_t unit, uint32_t op, const uint64_t *a, const uint64_t *b, size_t n,
                      uint64_t *results, uint32_t *covered) {
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return rc;
  const auto align = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t ctas = (size_t)d->sm_count, words = n * sizeof(uint64_t);
  const size_t a_off = align(sizeof(gsb_sm_log)), b_off = a_off + align(words), out_off = b_off + align(words);
  const size_t smid_off = out_off + align(ctas * words), bytes = smid_off + align(ctas * sizeof(uint32_t));
  SmBuffer buf(d, rc);
  rc = buf.alloc("SFU chosen inputs", bytes);
  char *const base = static_cast<char *>(buf.p);
  std::vector<uint64_t> zeros(b ? 0 : n, 0);
  if (rc == GSB_OK) {
    cudaError_t e = cudaMemcpyAsync(base + a_off, a, words, cudaMemcpyHostToDevice, d->stream);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(base + b_off, b ? b : zeros.data(), words, cudaMemcpyHostToDevice, d->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
    if (e != cudaSuccess) {
      set_error("uploading the SFU chosen inputs to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  gsb_sfu_table_args args;
  memset(&args, 0, sizeof args);
  args.log = reinterpret_cast<gsb_sm_log *>(base);
  args.a = reinterpret_cast<const unsigned long long *>(base + a_off);
  args.b = reinterpret_cast<const unsigned long long *>(base + b_off);
  args.out = reinterpret_cast<unsigned long long *>(base + out_off);
  args.smid = reinterpret_cast<uint32_t *>(base + smid_off);
  args.n = (uint32_t)n;
  args.op = op;
  args.smem_bytes = (uint32_t)smem;
  memset(covered, 0, GSB_SM_MAX / 8);
  std::vector<uint64_t> got(rc == GSB_OK ? ctas * n : 0);
  std::vector<uint32_t> smids(ctas);
  uint64_t kernel_ns = 0;
  for (uint32_t launch = 0; rc == GSB_OK && launch < GSB_SFU_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count;
       launch++) {
    gsb_sm_log log;
    rc = sm_launch_locked(
        d, "SFU chosen inputs", [&] { return gsb_sfu_operands_launch(unit, d->sm_count, &args, d->stream); }, args.log,
        &log, sizeof log, 0, nullptr, &kernel_ns);
    if (rc != GSB_OK) break;
    cudaError_t e = cudaMemcpyAsync(got.data(), args.out, ctas * words, cudaMemcpyDeviceToHost, d->stream);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(smids.data(), args.smid, ctas * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
    if (e != cudaSuccess) {
      set_error("reading the SFU chosen inputs' results from %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
      break;
    }
    for (size_t c = 0; c < ctas; c++) {  // an SM already covered keeps its first launch's results
      const uint32_t sm = smids[c];
      if (sm >= GSB_SM_MAX || covered[sm >> 5] >> (sm & 31u) & 1u) continue;
      covered[sm >> 5] |= 1u << (sm & 31u);
      memcpy(results + (size_t)sm * n, got.data() + c * n, words);
    }
  }
  buf.release();
  return rc;
}

// ------------------------------------------------------------------ L1 and constant-cache health

constexpr uint32_t kL1AllUnits = (1u << GSB_L1_UNITS) - 1;

// The TEX unit's texture objects over the L1 probe's regions (`rows` rows of GSB_L1_TEX_WIDTH words at buf), added to
// buf.tex as they are made: one linear resource, then the pitch-2D resource with clamp and with border addressing.
int l1_textures_locked(Device *d, SmBuffer *buf, uint32_t rows, gsb_l1_args *a) {
  unsigned long long *const slot[3] = {&a->tex_linear, &a->tex_clamp, &a->tex_border};
  for (int i = 0; i < 3; i++) {
    cudaResourceDesc res;
    memset(&res, 0, sizeof res);
    if (i == 0) {
      res.resType = cudaResourceTypeLinear;
      res.res.linear.devPtr = buf->p;
      res.res.linear.desc = cudaCreateChannelDesc<uint4>();
      res.res.linear.sizeInBytes = (size_t)rows * GSB_L1_TEX_WIDTH * 16;
    } else {
      res.resType = cudaResourceTypePitch2D;
      res.res.pitch2D.devPtr = buf->p;
      res.res.pitch2D.desc = cudaCreateChannelDesc<uint4>();
      res.res.pitch2D.width = GSB_L1_TEX_WIDTH;
      res.res.pitch2D.height = rows;
      res.res.pitch2D.pitchInBytes = GSB_L1_TEX_WIDTH * 16;
    }
    cudaTextureDesc td;
    memset(&td, 0, sizeof td);
    td.addressMode[0] = td.addressMode[1] = i == 2 ? cudaAddressModeBorder : cudaAddressModeClamp;
    td.filterMode = cudaFilterModePoint;
    td.readMode = cudaReadModeElementType;
    td.normalizedCoords = 0;
    cudaTextureObject_t t = 0;
    const cudaError_t e = cudaCreateTextureObject(&t, &res, &td, nullptr);
    if (e != cudaSuccess) {
      set_error("creating the L1 probe's texture objects on %s: %s", d->uuid, cudaGetErrorString(e));
      return GSB_ERR_DRIVER;
    }
    buf->tex.push_back(t);
    *slot[i] = t;
  }
  return GSB_OK;
}

// The median over CTAs of (warm span / (passes - 1)) / cold span of one load form, from spans[cta][form][2].
double l1_warm_cold(const std::vector<unsigned long long> &spans, uint32_t ctas, uint32_t form, uint32_t passes) {
  std::vector<double> r;
  for (uint32_t c = 0; c < ctas && passes > 1; c++) {
    const unsigned long long cold = spans[((size_t)c * GSB_L1_FORMS + form) * 2];
    const unsigned long long warm = spans[((size_t)c * GSB_L1_FORMS + form) * 2 + 1];
    if (cold) r.push_back((double)warm / (passes - 1) / (double)cold);
  }
  if (r.empty()) return 0.0;
  std::sort(r.begin(), r.end());
  return r.size() % 2 ? r[r.size() / 2] : (r[r.size() / 2 - 1] + r[r.size() / 2]) / 2;
}

int l1_probe_locked(Device *d, const gsb_l1_cfg *cfg, gsb_l1_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kL1AllUnits || cfg->passes > GSB_L1_PASSES_MAX) {
    set_error("invalid L1 probe configuration (units 0x%x, passes %u)", cfg->units, cfg->passes);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kL1AllUnits;
  out->passes = cfg->passes ? cfg->passes : GSB_L1_PASSES_DEFAULT;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x4C310000u, &d->l1.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const Device::L1Hooks hooks = take_hooks(d, &d->l1.hooks);
  // gsb_test_l1_table: taken by the first probe that runs its unit
  std::array<Device::L1Table, GSB_L1_UNITS> chosen;
  uint32_t region_max = GSB_L1_REGION_WORDS;
  size_t table_bytes = 0, expected_bytes = 0;
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t u = 0; u < GSB_L1_UNITS; u++) {
      if (!(out->units >> u & 1u) || !d->l1_table[u].armed) continue;
      chosen[u] = std::exchange(d->l1_table[u], Device::L1Table{});
      region_max = std::max(region_max, chosen[u].region_words);
      table_bytes = std::max(table_bytes, (4 * chosen[u].table.size() + 255) / 256 * 256);
      expected_bytes = std::max(expected_bytes, 4 * chosen[u].expected.size());
    }
  }
  const uint32_t ctas = d->sm_count, rows = ctas * GSB_L1_TEX_ROWS;
  // one transient buffer: the regions (first, so the texture resources start aligned), the launch log, the spans, a
  // chosen table and its expected words
  const size_t log_off = ctas * (size_t)region_max * 16, span_off = log_off + (sizeof(gsb_l1_log) + 255) / 256 * 256;
  const size_t span_bytes = (size_t)ctas * GSB_L1_FORMS * 2 * sizeof(unsigned long long);
  const size_t table_off = span_off + (span_bytes + 255) / 256 * 256, expected_off = table_off + table_bytes;
  SmBuffer buf(d, rc);
  rc = buf.alloc("L1 probe", expected_off + expected_bytes);
  char *const base = static_cast<char *>(buf.p);
  gsb_l1_args a;
  memset(&a, 0, sizeof a);
  a.log = reinterpret_cast<gsb_l1_log *>(base + log_off);
  a.buf = reinterpret_cast<uint4 *>(base);
  a.spans = reinterpret_cast<unsigned long long *>(base + span_off);
  a.seed = out->seed;
  a.seed_expect = out->seed_expect;
  a.passes = out->passes;
  a.rows = rows;
  if (rc == GSB_OK && (out->units >> GSB_L1_UNIT_TEX & 1u)) rc = l1_textures_locked(d, &buf, rows, &a);
  gsb_launch_geom fill_geom;
  if (rc == GSB_OK) rc = copy_geom_locked(d, GSB_OP_FILL, &fill_geom);
  // the bank's and the parameter's pattern words
  const uint32_t key = gsb_seed_key(out->seed);
  d->l1_const.resize(GSB_L1_CONST_WORDS);
  d->l1_param.resize(GSB_L1_PARAM_WORDS);
  for (uint32_t w = 0; w < GSB_L1_CONST_WORDS; w++) {
    uint32_t l[4];
    gsb_pattern_word(w, key, l);
    d->l1_const[w] = make_uint4(l[0], l[1], l[2], l[3]);
    if (w < GSB_L1_PARAM_WORDS) d->l1_param[w] = d->l1_const[w];
  }
  std::vector<unsigned long long> spans(span_bytes / sizeof(unsigned long long));
  bool first = true;
  for (uint32_t u = 0; u < GSB_L1_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_l1_unit_result &ur = out->unit[u];
    const Device::L1Table &tb = chosen[u];
    gsb_l1_table_args ta;
    memset(&ta, 0, sizeof ta);
    if (tb.armed) {
      ta.table = reinterpret_cast<const uint32_t *>(base + table_off);
      ta.expected = reinterpret_cast<const uint32_t *>(base + expected_off);
      ta.n = (uint32_t)tb.table.size();
      ta.region_words = tb.region_words;
      cudaError_t e = cudaMemcpyAsync(base + table_off, tb.table.data(), 4 * tb.table.size(), cudaMemcpyHostToDevice,
                                      d->stream);
      if (e == cudaSuccess && !tb.expected.empty())
        e = cudaMemcpyAsync(base + expected_off, tb.expected.data(), 4 * tb.expected.size(), cudaMemcpyHostToDevice,
                            d->stream);
      if (e != cudaSuccess) {
        set_error("uploading the L1 probe's chosen table to %s: %s", d->uuid, cudaGetErrorString(e));
        ur.status = rc = GSB_ERR_DRIVER;
        break;
      }
    }
    // a chosen table of a buffer unit sets the region size
    const uint64_t words = (uint64_t)ctas * (tb.armed && u < GSB_L1_UNIT_TEX ? tb.region_words : GSB_L1_REGION_WORDS);
    int per_sm = 0;
    if (gsb_l1_occupancy(u, &per_sm) == cudaSuccess) ur.ctas_per_sm = (uint32_t)per_sm;
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    while (ur.launches < GSB_L1_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count) {
      const bool hook = ur.launches == 0;  // test hooks: the unit's first launch only
      a.hook_smid = hook && hooks.corrupt[u].armed ? hooks.corrupt[u].smid : GSB_SM_MAX;
      a.hook_index = hooks.corrupt[u].index;
      a.hook_xr = hooks.corrupt[u].xr;
      a.skip_smid = hook && u == GSB_L1_UNIT_L1_STORE && hooks.skip_armed ? hooks.skip_smid : GSB_SM_MAX;
      ur.launches++;
      int lrc = GSB_OK;
      if (u <= GSB_L1_UNIT_TEX) {  // the regions hold generation 1 before every launch that reads them
        gsb_kernel_args fa;
        memset(&fa, 0, sizeof fa);
        fa.base = a.buf;
        fa.n_words = words;
        fa.seed_write = out->seed;
        fa.tile_counter = d->tile_counter;
        gsb_probe_result pr;
        lrc = copy_launch_locked(d, GSB_OP_FILL, fill_geom, fa, words * 16, words, words * 16 / 10, &pr);
      } else if (u == GSB_L1_UNIT_CONST) {
        const cudaError_t e = (cudaError_t)gsb_l1_const_upload(d->l1_const.data(), d->stream);
        if (e != cudaSuccess) {
          set_error("copying the L1 probe's constant bank to %s: %s", d->uuid, cudaGetErrorString(e));
          lrc = GSB_ERR_DRIVER;
        }
      }
      gsb_l1_log log;
      if (lrc == GSB_OK)
        lrc = sm_launch_locked(
            d, "L1 check",
            [&] {
              return tb.armed ? gsb_l1_table_launch(u, ctas, &a, &ta, d->l1_const.data(), d->l1_param.data(), d->stream)
                              : gsb_l1_kernel_launch(u, ctas, &a, d->l1_param.data(), d->stream);
            },
            a.log, &log,
            sizeof log, 0, nullptr, &ur.kernel_ns);
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      fold_log(log, &ur, out, covered);
      if (u != GSB_L1_UNIT_L1_LOAD && u != GSB_L1_UNIT_NC) continue;
      cudaError_t e = cudaMemcpyAsync(spans.data(), a.spans, span_bytes, cudaMemcpyDeviceToHost, d->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
      if (e != cudaSuccess) {
        set_error("reading the L1 probe's pass times from %s: %s", d->uuid, cudaGetErrorString(e));
        ur.status = rc = GSB_ERR_DRIVER;
        break;
      }
      for (uint32_t f = 0; f < GSB_L1_FORMS; f++)
        if ((u == GSB_L1_UNIT_NC) == (f == GSB_L1_FORM_NC))
          out->warm_cold[f] = l1_warm_cold(spans, ctas, f, tb.armed ? ta.n / ta.region_words : out->passes);
    }
    ur.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  // every record classified as an HBM fault record of the same word would be
  for (uint32_t i = 0; i < out->n_records; i++) {
    gsb_l1_record &r = out->records[i];
    gsb_fault_record f;
    memset(&f, 0, sizeof f);
    f.offset = r.offset;
    memcpy(f.expected, r.expected, sizeof f.expected);
    memcpy(f.observed, r.observed, sizeof f.observed);
    gsb_fault_classify(&f);
    r.cls = f.cls;
    r.alias_bit = f.alias_bit;
    r.seed_key = f.seed_key;
    r.flipped_bits = f.flipped_bits;
  }
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_l1_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < out->sm_count);
  }
  count_probe(d, &d->l1.stats, *out, ran, gsb_l1_conditions(out), short_cover ? &d->l1.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ memory-ordering health

constexpr uint32_t kOrderAllUnits = (1u << GSB_ORDER_UNITS) - 1;

int order_probe_locked(Device *d, const gsb_order_cfg *cfg, gsb_order_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kOrderAllUnits || cfg->observations > GSB_ORDER_OBS_MAX) {
    set_error("invalid memory-ordering probe configuration (units 0x%x, observations %u)", cfg->units,
              cfg->observations);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kOrderAllUnits;
  out->observations = cfg->observations ? cfg->observations : GSB_ORDER_OBS_DEFAULT;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x4F520000u, &d->order.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const Device::OrderHooks hooks = take_hooks(d, &d->order.hooks);
  const uint32_t n = d->sm_count, m = out->observations;
  for (uint32_t k = 0; k < GSB_ORDER_DISTANCES; k++) out->distance[k] = gsb_order_distance_of(k, n, out->seed);
  // one transient buffer: the launch log, every CTA's locations and scratch region, the published observations and
  // the ranks' %smid, each 256-byte aligned
  const auto align = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t locs_off = align(sizeof(gsb_order_log)), scratch_off = locs_off + (size_t)n * GSB_ORDER_LOC_WORDS * 8;
  const size_t obs_off = scratch_off + (size_t)n * GSB_ORDER_SCRATCH_WORDS * 16;
  const size_t smid_off = obs_off + align((size_t)n * m * GSB_ORDER_OBS_WORDS * 8);
  SmBuffer buf(d, rc);
  rc = buf.alloc("memory-ordering probe", smid_off + align((size_t)n * sizeof(uint32_t)));
  char *const base = static_cast<char *>(buf.p);
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  gsb_order_args a;
  memset(&a, 0, sizeof a);
  a.log = reinterpret_cast<gsb_order_log *>(base);
  a.locs = reinterpret_cast<unsigned long long *>(base + locs_off);
  a.scratch = reinterpret_cast<uint4 *>(base + scratch_off);
  a.obs = reinterpret_cast<unsigned long long *>(base + obs_off);
  a.smids = reinterpret_cast<uint32_t *>(base + smid_off);
  a.seed = out->seed;
  a.seed_expect = out->seed_expect;
  a.observations = m;
  a.smem_bytes = (uint32_t)smem;
  bool first = true;
  for (uint32_t u = 0; u < GSB_ORDER_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_order_unit_result &ur = out->unit[u];
    uint32_t unit_cov[GSB_SM_MAX / 32] = {0};
    for (uint32_t k = 0; k < GSB_ORDER_DISTANCES; k++) {
      a.unit = u;
      a.distance = out->distance[k];
      a.dist_index = k;
      // test hooks: the unit's first launch only
      a.inject_smid = k == 0 && hooks.inject[u].armed ? hooks.inject[u].smid : GSB_SM_MAX;
      a.inject_index = hooks.inject[u].index;
      a.skip_smid = k == 0 && u == GSB_ORDER_UNIT_MP_RELACQ && hooks.skip_armed ? hooks.skip_smid : GSB_SM_MAX;
      bool refused = false;
      gsb_order_log log;
      const int lrc = sm_launch_locked(
          d, "memory-ordering check",
          [&] {
            const int e = gsb_order_kernel_launch(n, &a, d->stream);
            if (e != (int)cudaErrorCooperativeLaunchTooLarge) return e;
            refused = true;  // the CTAs cannot all be resident at once: the launch is skipped, not failed
            return (int)cudaSuccess;
          },
          a.log, &log, sizeof log, (GSB_ORDER_WAIT_NS + gsb_order_wait_ns(m)) / 1000000ull, nullptr, &ur.kernel_ns);
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      if (refused) {
        ur.refused++;
        continue;
      }
      uint32_t covered[GSB_SM_MAX / 32] = {0};
      fold_log(log, &ur, out, covered);
      ur.corrupt += log.corrupt;
      ur.forbidden += log.forbidden;
      ur.lost += log.lost;
      ur.timeout += log.timeout;
      ur.overlap += log.overlap;
      ur.weak += log.weak;
      for (int i = 0; i < GSB_SM_MAX / 32; i++) unit_cov[i] = ur.launches ? unit_cov[i] & covered[i] : covered[i];
      ur.launches++;
    }
    if (!ur.launches) continue;
    ur.sms_covered = popcount_bitmap(unit_cov);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? unit_cov[i] : out->covered[i] & unit_cov[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_order_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || ur.refused != 0 || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < n);
  }
  count_probe(d, &d->order.stats, *out, ran, gsb_order_conditions(out),
              short_cover ? &d->order.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ sparse tensor-core health

constexpr uint32_t kSparseAllUnits = (1u << GSB_SPARSE_UNITS) - 1;

int sparse_probe_locked(Device *d, const gsb_sparse_cfg *cfg, gsb_sparse_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kSparseAllUnits) {
    set_error("invalid sparse unit mask 0x%x", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kSparseAllUnits;
  out->sm_count = d->sm_count;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x53500000u, &d->sparse.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const auto corrupt = take_hooks(d, &d->sparse.hooks.corrupt);
  std::vector<uint32_t> chosen[GSB_SPARSE_UNITS];  // gsb_test_sparse_operands of the units this probe runs
  {
    std::lock_guard<std::mutex> lk(d->smu);
    for (uint32_t u = 0; u < GSB_SPARSE_UNITS; u++)
      if (out->units >> u & 1u) chosen[u].swap(d->sparse.hooks.operands[u]);
  }
  // the buffer: the launch log, then per unit its 8192 expected words or its chosen operands' block, 256-byte aligned
  size_t offset[GSB_SPARSE_UNITS] = {}, bytes = (sizeof(gsb_sm_log) + 255) / 256 * 256;
  for (uint32_t u = 0; u < GSB_SPARSE_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    offset[u] = bytes;
    const size_t n = chosen[u].empty() ? (size_t)GSB_SPARSE_WORDS : chosen[u].size();
    bytes += (n * sizeof(uint32_t) + 255) / 256 * 256;
  }
  // the exact answers, computed on the host; HMMA_SP's is F16_SP's
  const uint64_t t_exp = now_ns();
  std::string tables(bytes, '\0');
  std::vector<uint32_t> f16;
  for (uint32_t u = 0; u < GSB_SPARSE_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    uint32_t *p = reinterpret_cast<uint32_t *>(&tables[offset[u]]);
    if (!chosen[u].empty()) {
      memcpy(p, chosen[u].data(), chosen[u].size() * sizeof(uint32_t));
      continue;
    }
    const bool f16_gemm = u == GSB_SPARSE_UNIT_F16_SP || u == GSB_SPARSE_UNIT_HMMA_SP;
    if (f16_gemm && !f16.empty()) {
      memcpy(p, f16.data(), GSB_SPARSE_WORDS * sizeof(uint32_t));
    } else {
      gsb_sparse_expected(u, out->seed_expect, p, GSB_SPARSE_WORDS);
      if (f16_gemm) f16.assign(p, p + GSB_SPARSE_WORDS);
    }
  }
  out->expected_ns = now_ns() - t_exp;
  // one transient buffer: the launch log and the tables, under the keep-free margin of every transient probe
  SmBuffer buf(d, rc);
  rc = buf.alloc("sparse probe", bytes);
  char *const base = static_cast<char *>(buf.p);
  if (rc == GSB_OK) {
    const size_t head = (sizeof(gsb_sm_log) + 255) / 256 * 256;
    const cudaError_t e = cudaMemcpyAsync(base + head, &tables[head], bytes - head, cudaMemcpyHostToDevice, d->stream);
    if (e != cudaSuccess || cudaStreamSynchronize(d->stream) != cudaSuccess) {
      set_error("uploading the sparse probe's expected answers to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  int smem = 0;
  if (rc == GSB_OK) rc = smem_optin_locked(d, &smem);
  bool first = true;
  for (uint32_t u = 0; u < GSB_SPARSE_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_tensor_unit_result &ur = out->unit[u];
    gsb_sm_args a;
    memset(&a, 0, sizeof a);
    a.log = reinterpret_cast<gsb_sm_log *>(base);
    a.expected = base + offset[u];
    a.seed = out->seed;
    a.smem_bytes = (uint32_t)smem;
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    // one CTA per SM: a launch that left an SM uncovered (another context held it) is repeated
    while (ur.launches < GSB_SPARSE_MAX_LAUNCHES && popcount_bitmap(covered) < d->sm_count) {
      const bool hook = ur.launches == 0 && corrupt[u].armed;  // test hook: the unit's first launch only
      a.hook_smid = hook ? corrupt[u].smid : GSB_SM_MAX;
      a.hook_index = corrupt[u].index;
      a.hook_xr = corrupt[u].xr;
      ur.launches++;
      gsb_sm_log log;
      const int lrc = sm_launch_locked(
          d, "sparse check",
          [&] {
            return chosen[u].empty() ? gsb_sparse_kernel_launch(u, d->sm_count, &a, d->stream)
                                             : gsb_sparse_operands_launch(u, d->sm_count, &a, d->stream);
          },
          a.log, &log, sizeof log, 0, nullptr, &ur.kernel_ns);
      if (lrc != GSB_OK) {
        ur.status = rc = lrc;
        break;
      }
      fold_log(log, &ur, out, covered);
    }
    ur.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_tensor_unit_result &ur : out->unit) {
    ran = ran || ur.launches != 0;
    short_cover = short_cover || (ur.launches != 0 && ur.status == GSB_OK && ur.sms_covered < out->sm_count);
  }
  count_probe(d, &d->sparse.stats, *out, ran, gsb_sparse_conditions(out),
              short_cover ? &d->sparse.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ shared-memory atomic health

constexpr uint32_t kSharedAtomicAllUnits = (1u << GSB_SHARED_ATOMIC_UNITS) - 1;
constexpr size_t kSharedAtomicLogBytes = (sizeof(gsb_shared_atomic_log) + 255) / 256 * 256;

void shared_atomic_add_record(gsb_shared_atomic_result *out, const gsb_shared_atomic_record &rec) {
  if (rec.smid < GSB_SM_MAX) out->faulty[rec.smid >> 5] |= 1u << (rec.smid & 31u);
  if (out->n_records < GSB_SHARED_ATOMIC_RECORDS) out->records[out->n_records++] = rec;
}

// TICKET and CAS: per CTA, form and hot slot, the entries must name every contributor once. Add and CAS forms: entry t
// holds the id that drew ticket t (the final counter is compared on the SM). Exchange forms: the values returned to the
// contributors plus the final word (entry COUNT) must be the values of ids 0 .. COUNT (COUNT's is the starting word),
// each once. Returns the entries that do not; each is recorded, naming the SM that owns the slots.
uint64_t shared_atomic_check_slots(uint32_t unit, uint32_t seed, uint32_t ctas, const std::vector<uint32_t> &slots,
                                   const gsb_shared_atomic_log &log, gsb_shared_atomic_result *out) {
  constexpr uint32_t kCount = GSB_SHARED_ATOMIC_COUNT;
  const uint32_t forms = unit == GSB_SHARED_ATOMIC_UNIT_TICKET ? 4u : 3u;
  uint64_t bad = 0;
  std::vector<char> seen(kCount + 1);
  // TICKET: the id of each exchanged value, by form and hot slot, found by its first word
  std::vector<std::unordered_map<uint32_t, uint32_t>> id_of(unit == GSB_SHARED_ATOMIC_UNIT_TICKET ? 4u * 32u : 0u);
  for (uint32_t f = 1; f < id_of.size() / 32u; f++)
    for (uint32_t l = 0; l < GSB_SHARED_ATOMIC_HOT_WORDS; l++)
      for (uint32_t id = 0; id <= kCount; id++) id_of[f * 32u + l][gsb_shared_atomic_exch(seed, f, l, id, 0u)] = id;
  for (uint32_t b = 0; b < ctas; b++)
    for (uint32_t f = 0; f < forms; f++)
      for (uint32_t l = 0; l < GSB_SHARED_ATOMIC_HOT_WORDS; l++) {
        std::fill(seen.begin(), seen.end(), 0);
        const bool exch = unit == GSB_SHARED_ATOMIC_UNIT_TICKET && f > 0;
        const uint32_t comps = exch ? (f == 1u ? 1u : f == 2u ? 2u : 4u) : 1u;
        for (uint32_t i = 0; i < (exch ? kCount + 1u : kCount); i++) {
          const uint32_t *e = &slots[gsb_shared_atomic_slot(b, f, l, i)];
          uint32_t id = e[0];
          if (exch) {  // the id whose value this is, every component of it
            const auto it = id_of[f * 32u + l].find(e[0]);
            id = it == id_of[f * 32u + l].end() ? GSB_SHARED_ATOMIC_NO_ID : it->second;
            for (uint32_t c = 1; c < comps && id != GSB_SHARED_ATOMIC_NO_ID; c++)
              if (e[c] != gsb_shared_atomic_exch(seed, f, l, id, c)) id = GSB_SHARED_ATOMIC_NO_ID;
          }
          if (id <= (exch ? kCount : kCount - 1u) && !seen[id]) {
            seen[id] = 1;
            continue;
          }
          bad++;
          const uint32_t sm = b < GSB_SM_MAX ? log.cta_smid[b] : GSB_SHARED_ATOMIC_NO_SM;
          shared_atomic_add_record(out, {sm, unit, GSB_SHARED_ATOMIC_REC_SLOT,
                                         (uint32_t)(gsb_shared_atomic_slot(b, f, l, i) / 4u), kCount, e[0]});
        }
      }
  return bad;
}

int shared_atomic_probe_locked(Device *d, const gsb_shared_atomic_cfg *cfg, gsb_shared_atomic_result *out) {
  const uint64_t t0 = now_ns();
  if (cfg->units & ~kSharedAtomicAllUnits) {
    set_error("invalid shared-memory atomic unit mask 0x%x", cfg->units);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  out->units = cfg->units ? cfg->units : kSharedAtomicAllUnits;
  out->sm_count = d->sm_count;
  for (gsb_shared_atomic_run &run : out->run) run.hook_cta = GSB_SHARED_ATOMIC_NO_SM;
  int rc = ensure_ready(d);
  if (!rc) rc = sm_drain_kept_locked(d);
  if (rc) return out->status = rc;
  if (d->sm_count > GSB_SM_MAX) {
    set_error("%s has %u SMs, more than the shared-memory atomic probe's %d", d->uuid, d->sm_count, GSB_SM_MAX);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  int smem = 0;
  if ((rc = smem_optin_locked(d, &smem))) return out->status = rc;
  out->seed = seed_or_fresh(cfg->seed, 0x53410000u, &d->shared_atomic.seed);
  out->seed_expect = cfg->seed_expect ? cfg->seed_expect : out->seed;
  const Device::SharedAtomicHooks hooks = take_hooks(d, &d->shared_atomic.hooks);
  // DSMEM and REDAS: clusters of 2, then the largest of 16 and 8 that can be scheduled, as many as fit at once
  const bool any_cluster = out->units >> GSB_SHARED_ATOMIC_UNIT_DSMEM & 1u || out->units >> GSB_SHARED_ATOMIC_UNIT_REDAS & 1u;
  uint32_t max_clusters[2][2] = {};  // [DSMEM, REDAS][size]
  if (any_cluster) {
    const auto fit = [&](uint32_t u, uint32_t n) {
      int m = 0;
      if (gsb_shared_atomic_max_clusters(u, n, smem, &m) != cudaSuccess) {
        cudaGetLastError();
        m = 0;
      }
      return (uint32_t)std::max(0, std::min(m, (int)(GSB_SM_MAX / n)));
    };
    const uint32_t big = fit(GSB_SHARED_ATOMIC_UNIT_DSMEM, 16u) ? 16u : fit(GSB_SHARED_ATOMIC_UNIT_DSMEM, 8u) ? 8u : 0u;
    out->cluster_n[0] = 2u;
    out->cluster_n[1] = big;
    for (uint32_t c = 0; c < 2; c++)
      for (uint32_t k = 0; k < 2; k++)
        max_clusters[c][k] = out->cluster_n[k] ? fit(GSB_SHARED_ATOMIC_UNIT_DSMEM + c, out->cluster_n[k]) : 0u;
  }
  // one transient buffer: the launch log, every local unit's expected area, DSMEM's and REDAS's areas by cluster size
  // and rank (16 each), the TICKET and CAS slots
  const uint32_t ctas = d->sm_count;
  const size_t area = (size_t)GSB_SHARED_ATOMIC_AREA_WORDS * 4u;
  constexpr uint32_t kLocal = GSB_SHARED_ATOMIC_UNIT_DSMEM;  // units 0 .. kLocal - 1 run one CTA per SM
  const auto area_index = [&](uint32_t u, uint32_t k, uint32_t rank) {
    return u < kLocal ? (size_t)u : kLocal + ((size_t)(u - kLocal) * 2u + k) * 16u + rank;
  };
  const size_t n_areas = kLocal + 2u * 2u * 16u;
  const size_t off_expect = kSharedAtomicLogBytes, off_slots = off_expect + n_areas * area;
  const bool any_slots = out->units >> GSB_SHARED_ATOMIC_UNIT_TICKET & 1u || out->units >> GSB_SHARED_ATOMIC_UNIT_CAS & 1u;
  const size_t slot_words = any_slots ? (size_t)ctas * GSB_SHARED_ATOMIC_SLOT_WORDS : 0u;
  const size_t bytes = off_slots + 4u * slot_words;
  std::vector<uint32_t> expect(n_areas * GSB_SHARED_ATOMIC_AREA_WORDS);
  const uint64_t t_exp = now_ns();
  for (uint32_t u = 0; u < GSB_SHARED_ATOMIC_UNITS; u++) {
    if (!(out->units >> u & 1u)) continue;
    for (uint32_t k = 0; k < (u < kLocal ? 1u : 2u); k++) {
      const uint32_t n = u < kLocal ? 1u : out->cluster_n[k];
      for (uint32_t rank = 0; rank < n; rank++)
        if (gsb_shared_atomic_expected(u, out->seed_expect, n, rank,
                                       &expect[area_index(u, k, rank) * GSB_SHARED_ATOMIC_AREA_WORDS],
                                       GSB_SHARED_ATOMIC_AREA_WORDS) != GSB_SHARED_ATOMIC_AREA_WORDS) {
          set_error("computing the shared-memory atomic probe's expected words of unit %u on %s", u, d->uuid);
          return out->status = GSB_ERR_INVALID_ARGUMENT;
        }
    }
  }
  out->expected_ns = now_ns() - t_exp;
  SmBuffer buf(d, rc);
  rc = buf.alloc("shared-memory atomic probe", bytes);
  char *const base = static_cast<char *>(buf.p);
  if (rc == GSB_OK) {
    cudaError_t e = cudaMemcpyAsync(base + off_expect, expect.data(), 4u * expect.size(), cudaMemcpyHostToDevice, d->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(d->stream);
    if (e != cudaSuccess) {
      set_error("uploading the shared-memory atomic probe's expected words to %s: %s", d->uuid, cudaGetErrorString(e));
      rc = GSB_ERR_DRIVER;
    }
  }
  bool first = true;
  std::vector<uint32_t> slots;
  for (uint32_t u = 0; u < GSB_SHARED_ATOMIC_UNITS && rc == GSB_OK; u++) {
    if (!(out->units >> u & 1u)) continue;
    gsb_shared_atomic_run &run = out->run[u];
    const bool tickets = u == GSB_SHARED_ATOMIC_UNIT_TICKET || u == GSB_SHARED_ATOMIC_UNIT_CAS;
    const bool cluster = u >= kLocal;
    gsb_shared_atomic_args a;
    memset(&a, 0, sizeof a);
    a.log = reinterpret_cast<gsb_shared_atomic_log *>(base);
    a.slots = tickets ? reinterpret_cast<uint32_t *>(base + off_slots) : nullptr;
    a.seed = out->seed;
    a.smem_bytes = (uint32_t)smem;
    // a CAS loop or a REDAS wait may run to its deadline (one per thread, one per CTA)
    const uint64_t extra_ms =
        u == GSB_SHARED_ATOMIC_UNIT_CAS || cluster ? GSB_SHARED_ATOMIC_CAS_WAIT_NS / 1000000u : 0u;
    uint32_t covered[GSB_SM_MAX / 32] = {0};
    for (uint32_t k = 0; k < (cluster ? 2u : 1u) && rc == GSB_OK; k++) {
      const uint32_t n = cluster ? out->cluster_n[k] : 1u;
      const uint32_t clusters = cluster ? max_clusters[u - kLocal][k] : ctas;
      if (cluster && !clusters) {
        if (k == 0) {  // not even clusters of 2 can be scheduled: nothing of the unit can run
          set_error("clusters of 2 CTAs with %d bytes of shared memory each cannot be scheduled on %s", smem, d->uuid);
          run.status = rc = GSB_ERR_UNSUPPORTED_ARCH;
        }
        continue;
      }
      a.expected = reinterpret_cast<const uint32_t *>(base + off_expect + area_index(u, k, 0) * area);
      const uint32_t reach = std::min(clusters * n, ctas);
      uint32_t size_covered[GSB_SM_MAX / 32] = {0}, launches = 0;
      if (cluster) run.clusters[k] = clusters;
      // a launch that left an SM it could reach uncovered (another context held it) is repeated
      while (launches < GSB_SHARED_ATOMIC_MAX_LAUNCHES && popcount_bitmap(size_covered) < reach) {
        const bool first_launch = run.launches == 0;  // test hooks: the unit's first launch only
        a.hook_smid = first_launch && hooks.corrupt[u].armed ? hooks.corrupt[u].smid : GSB_SM_MAX;
        a.hook_index = hooks.corrupt[u].index;
        a.hook_xr = hooks.corrupt[u].xr;
        a.skip_smid = first_launch && hooks.skip[u].armed ? hooks.skip[u].smid : GSB_SM_MAX;
        run.launches++;
        launches++;
        if (cluster) run.cluster_launches[k]++;
        gsb_shared_atomic_log log;
        int lrc = sm_launch_locked(
            d, "shared-memory atomic check",
            [&] {
              return cluster ? gsb_shared_atomic_cluster_launch(u, n, clusters, &a, d->stream)
                             : gsb_shared_atomic_kernel_launch(u, ctas, &a, d->stream);
            },
            a.log, &log, sizeof log, extra_ms, nullptr, &run.kernel_ns);
        if (lrc == GSB_OK && tickets) {
          slots.resize(slot_words);
          const cudaError_t e = cudaMemcpy(slots.data(), a.slots, 4u * slots.size(), cudaMemcpyDeviceToHost);
          if (e != cudaSuccess) {
            set_error("reading the shared-memory atomic probe's slots on %s: %s", d->uuid, cudaGetErrorString(e));
            lrc = GSB_ERR_DRIVER;
          }
        }
        if (lrc != GSB_OK) {
          run.status = rc = lrc;
          break;
        }
        if (log.skipped_cta) run.hook_cta = log.skipped_cta - 1u;
        run.atomics_issued += log.issued;
        run.timeouts += log.timeouts;
        run.cas_max_ns = std::max<uint64_t>(run.cas_max_ns, log.cas_max_ns);
        run.ticket_faults += log.faults;
        // records: the kernel's (out-of-range tickets, torn pairs, wrong words), then slots
        fold_log(log, &run, out, size_covered);
        if (tickets) run.ticket_faults += shared_atomic_check_slots(u, out->seed_expect, ctas, slots, log, out);
      }
      for (int i = 0; i < GSB_SM_MAX / 32; i++) covered[i] |= size_covered[i];
    }
    run.sms_covered = popcount_bitmap(covered);
    for (int i = 0; i < GSB_SM_MAX / 32; i++) out->covered[i] = first ? covered[i] : out->covered[i] & covered[i];
    first = false;
  }
  out->sms_covered = popcount_bitmap(out->covered);
  buf.release();
  out->wall_ns = now_ns() - t0;
  out->status = rc;
  bool ran = false, short_cover = false;
  for (const gsb_shared_atomic_run &run : out->run) {
    ran = ran || run.launches != 0;
    short_cover = short_cover || (run.launches != 0 && run.status == GSB_OK && run.sms_covered < out->sm_count);
  }
  count_probe(d, &d->shared_atomic.stats, *out, ran, gsb_shared_atomic_conditions(out),
              short_cover ? &d->shared_atomic.stats.incomplete : nullptr);
  return rc;
}

// ------------------------------------------------------------------ the periodic checks, described once

template <typename Run>
struct RunTypes;
template <typename C, typename R>
struct RunTypes<int (*)(Device *, const C *, R *)> {
  using Cfg = C;
  using Result = R;
};

// One check the prober runs every Nth cycle: its cadence option, the event its conditions raise, where a device keeps
// its state, its run under d->mu and the conditions of a result.
template <uint32_t kOption, uint64_t kEvent, auto kState, auto kRun, auto kConditions>
struct Check {
  static constexpr uint32_t option = kOption;
  static constexpr uint64_t event = kEvent;
  using Cfg = typename RunTypes<decltype(kRun)>::Cfg;
  using Result = typename RunTypes<decltype(kRun)>::Result;
  static auto &state(Device *d) { return d->*kState; }
  static int run(Device *d, const Cfg *cfg, Result *out) { return kRun(d, cfg, out); }
  static uint32_t conditions(const Result *r) { return kConditions(r); }
};
using LinkCheck = Check<GSB_OPT_LINK_PROBE_EVERY_CYCLES, GSB_EVENT_LINK, &Device::link, &link_probe_locked, &gsb_link_conditions>;
using CopyCheck = Check<GSB_OPT_COPY_PROBE_EVERY_CYCLES, GSB_EVENT_COPY, &Device::copy, &copy_probe_locked, &gsb_copy_conditions>;
using SmCheck = Check<GSB_OPT_SM_PROBE_EVERY_CYCLES, GSB_EVENT_SM, &Device::sm, &sm_probe_locked, &gsb_sm_conditions>;
using ClusterCheck = Check<GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, GSB_EVENT_CLUSTER, &Device::cluster,
                           &cluster_probe_locked, &gsb_cluster_conditions>;
using AtomicCheck = Check<GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_ATOMIC, &Device::atomic, &atomic_probe_locked,
                          &gsb_atomic_conditions>;
using TensorCheck = Check<GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, GSB_EVENT_TENSOR, &Device::tensor, &tensor_probe_locked,
                          &gsb_tensor_conditions>;
using SfuCheck = Check<GSB_OPT_SFU_PROBE_EVERY_CYCLES, GSB_EVENT_SFU, &Device::sfu, &sfu_probe_locked, &gsb_sfu_conditions>;
using L1Check = Check<GSB_OPT_L1_PROBE_EVERY_CYCLES, GSB_EVENT_L1, &Device::l1, &l1_probe_locked, &gsb_l1_conditions>;
using OrderCheck = Check<GSB_OPT_ORDER_PROBE_EVERY_CYCLES, GSB_EVENT_ORDER, &Device::order, &order_probe_locked,
                         &gsb_order_conditions>;
using SparseCheck = Check<GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, GSB_EVENT_SPARSE, &Device::sparse, &sparse_probe_locked,
                          &gsb_sparse_conditions>;
using SharedAtomicCheck = Check<GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_SHARED_ATOMIC, &Device::shared_atomic,
                                &shared_atomic_probe_locked, &gsb_shared_atomic_conditions>;
// in the order the prober runs them when several are due after the same cycle; G.check_every follows it
using Checks =
    std::tuple<LinkCheck, CopyCheck, SmCheck, ClusterCheck, AtomicCheck, TensorCheck, SfuCheck, L1Check, OrderCheck,
               SparseCheck, SharedAtomicCheck>;
static_assert(std::tuple_size<Checks>::value == std::extent<decltype(G.check_every)>::value, "one cadence per check");

// f(check, its place in Checks) for every periodic check, in order
template <typename F, size_t... I>
void for_each_check(F &&f, std::index_sequence<I...>) {
  (f(std::tuple_element_t<I, Checks>{}, I), ...);
}
template <typename F>
void for_each_check(F &&f) {
  for_each_check(f, std::make_index_sequence<std::tuple_size<Checks>::value>{});
}

// The cadence a GSB_OPT_*_PROBE_EVERY_CYCLES key sets, or null for any other key.
std::atomic<uint64_t> *check_every_of(uint32_t key) {
  std::atomic<uint64_t> *every = nullptr;
  for_each_check([&](auto check, size_t i) {
    if (decltype(check)::option == key) every = &G.check_every[i];
  });
  return every;
}

// The body of a probe entry point: `pre` (if any) may refuse the arguments before any device is touched; the run then
// holds d->mu from start to end, so a prober cycle waits for it.
template <typename Cfg, typename Result, typename Pre>
int probe_entry(uint32_t idx, const Cfg *cfg, Result *out, int (*run)(Device *, const Cfg *, Result *), Pre pre) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!cfg || !out) return GSB_ERR_INVALID_ARGUMENT;
  memset(out, 0, sizeof *out);
  const int refused = pre(cfg, out);
  if (refused) return out->status = refused;
  Device *d = device_at(idx);
  if (!d) return out->status = G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  return run(d, cfg, out);
}
template <typename Cfg, typename Result>
int probe_entry(uint32_t idx, const Cfg *cfg, Result *out, int (*run)(Device *, const Cfg *, Result *)) {
  return probe_entry(idx, cfg, out, run, [](const Cfg *, Result *) { return GSB_OK; });
}

// The body of a gsb_*_stats_get: a copy, under smu, of the statistics `stats` finds in the device.
template <typename Stats, typename Find>
int stats_entry(uint32_t idx, Stats *out, Find stats) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  *out = *stats(d);
  return GSB_OK;
}

// One periodic check of device idx on default settings, and an event for every condition it finds for the first time
// this health session.
template <typename C>
void run_check(uint32_t idx) {
  typename C::Cfg cfg;
  memset(&cfg, 0, sizeof cfg);
  typename C::Result r;
  probe_entry(idx, &cfg, &r, &C::run);
  Device *d = G.devs[idx].get();
  raise_conditions(d, C::event, &C::state(d).raised, [&] { return C::conditions(&r); });
}

}  // namespace

// ====================================================================== C ABI

extern "C" {

int gsb_abi_version(void) { return (int)GSB_ABI_VERSION; }

const char *gsb_strerror(int status) {
  switch (status) {
    case GSB_OK: return "ok";
    case GSB_ERR_NOT_INITIALIZED: return "not initialized";
    case GSB_ERR_INVALID_ARGUMENT: return "invalid argument";
    case GSB_ERR_LIBRARY_NOT_FOUND: return "could not load NVML library";
    case GSB_ERR_DRIVER: return "CUDA driver error";
    case GSB_ERR_NVML: return "NVML error";
    case GSB_ERR_NO_DEVICE: return "nvml: device not found";
    case GSB_ERR_IDENTITY_MISMATCH: return "CUDA/NVML device identity mismatch";
    case GSB_ERR_BUFFER_TOO_SMALL: return "buffer too small";
    case GSB_ERR_OUT_OF_MEMORY: return "out of device memory";
    case GSB_ERR_UNSUPPORTED_ARCH: return "device is not sm_90: no kernel image, no fallback";
    case GSB_ERR_TIMEOUT: return "timeout";
    case GSB_ERR_NO_ARENA: return "no probe arena";
    case GSB_ERR_MALFORMED: return "malformed protobuf";
    case GSB_ERR_STOPPED: return "health queue stopped";
    default: return "unknown gsb status";
  }
}

int gsb_last_error(char *buf, size_t cap) {
  if (!buf || cap == 0) return GSB_ERR_INVALID_ARGUMENT;
  snprintf(buf, cap, "%s", tl_error);
  return GSB_OK;
}

int gsb_init(void) {
  std::unique_lock<std::shared_mutex> api_lk(G.api_mu);
  std::lock_guard<std::mutex> lk(G.mu);
  if (G.inited) return GSB_OK;
  int rc = load_libraries();
  if (rc) return rc;
  ML_TRY(G.ml.init());
  CU_TRY(G.cu.cuInit(0));

  unsigned n_ml = 0;
  ML_TRY(G.ml.getCount(&n_ml));
  int n_cu = 0;
  RT_TRY(cudaGetDeviceCount(&n_cu));
  struct CudaDev {
    CUdevice dev;
    char uuid[GSB_UUID_BUFFER_SIZE];
  };
  std::vector<CudaDev> cds((size_t)n_cu);
  for (int i = 0; i < n_cu; i++) {
    CU_TRY(G.cu.cuDeviceGet(&cds[i].dev, i));
    CUuuid u;
    CU_TRY(G.cu.cuDeviceGetUuid(&u, cds[i].dev));
    format_uuid(u, cds[i].uuid);
  }
  G.devs.clear();
  for (unsigned i = 0; i < n_ml; i++) {  // NVML index order = the reference's order (nvidia.go:59)
    auto d = std::make_unique<Device>();
    ML_TRY(G.ml.handleByIndex(i, &d->nvml));
    ML_TRY(G.ml.getUUID(d->nvml, d->uuid, GSB_UUID_BUFFER_SIZE));
    unsigned minor = 0;
    ML_TRY(G.ml.getMinor(d->nvml, &minor));
    d->minor = minor;
    nvmlPciInfo_t pci;
    memset(&pci, 0, sizeof pci);
    // the bus id is reported for information only; some virtualised hosts answer NOT_SUPPORTED, which leaves it empty
    const nvmlReturn_t pr = G.ml.getPciInfo(d->nvml, &pci);
    if (pr != NVML_SUCCESS && pr != NVML_ERROR_NOT_SUPPORTED) ML_TRY(pr);
    snprintf(d->bus_id, sizeof d->bus_id, "%s", pr == NVML_SUCCESS ? pci.busId : "");
    for (int c = 0; c < n_cu; c++) {
      if (strcmp(cds[c].uuid, d->uuid) == 0) {
        d->ordinal = c;
        d->cudev = cds[c].dev;
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, c);
        d->sm_count = (uint32_t)v;
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, c);
        d->cc_major = (uint32_t)v;
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, c);
        d->cc_minor = (uint32_t)v;
        size_t tot = 0;
        G.cu.cuDeviceTotalMem(&tot, d->cudev);
        d->cuda_total = tot;
        break;
      }
    }
    G.devs.push_back(std::move(d));
  }
  // the (re)start-time inventory: every device's identity + memory read from NVML once, as getDevices does
  for (auto &d : G.devs) {
    gsb_device_info info;
    int qrc = query_info(d.get(), &info);
    if (qrc) {
      G.devs.clear();
      return qrc;
    }
  }
  if (const char *e = getenv("GSB_PROBE_WATCHDOG_MS")) G.watchdog_ms = (uint64_t)atoll(e);
  if (const char *e = getenv("GSB_INVENTORY_POLICY")) G.inventory_policy = strcmp(e, "live") == 0 ? GSB_INVENTORY_LIVE : GSB_INVENTORY_SNAPSHOT;
  G.inited = true;
  return GSB_OK;
}

int gsb_shutdown(void) {
  {
    // no gsb_health_start from here on: the prober threads it would start use the devices freed below
    std::lock_guard<std::mutex> lk(G.mu);
    G.shutting_down++;
  }
  gsb_health_stop();
  std::unique_lock<std::shared_mutex> api_lk(G.api_mu);  // waits for in-flight calls of other threads
  std::lock_guard<std::mutex> lk(G.mu);
  G.shutting_down--;
  if (!G.inited) return GSB_OK;
  for (auto &d : G.devs) {
    worker_stop(d.get());
    std::lock_guard<std::mutex> dl(d->mu);
    bool still_wedged = false;
    if (d->ready && d->wedged) {
      cudaSetDevice(d->ordinal);
      still_wedged = cudaStreamQuery(d->stream) == cudaErrorNotReady;
    }
    if (d->ready && !still_wedged) {  // a copy of a wedged copy probe still on its stream
      cudaSetDevice(d->ordinal);
      for (cudaStream_t s : d->copy_streams)
        if (s && cudaStreamQuery(s) == cudaErrorNotReady) still_wedged = true;
    }
    if (!still_wedged) arena_destroy_locked(d.get());
    if (d->ready && still_wedged) {
      // cudaFree and cudaStreamDestroy wait for the device: under a launch that never ends they would hang the
      // shutdown for ever. The resources go with the process / the context instead.
      d->ready = false;
    }
    if (d->ready) {
      cudaSetDevice(d->ordinal);
      cudaStreamDestroy(d->stream);
      cudaEventDestroy(d->ev0);
      cudaEventDestroy(d->ev1);
      cudaFreeHost(d->out_host);
      cudaFree(d->partials);
      cudaFree(d->ticket);
      cudaFree(d->tile_counter);
      cudaFree(d->fault_log);
      cudaFreeHost(d->fault_host);
      for (void *p : d->link_kept)
        if (p) cudaFreeHost(p);
      copy_free_buffers(d->copy_kept_dev, d->copy_kept_host);
      if (d->sm_kept) cudaFree(d->sm_kept);
      d->sm_kept = nullptr;
      for (cudaStream_t s : d->copy_streams)
        if (s) cudaStreamDestroy(s);
      for (auto &pair : d->copy_ev)
        for (cudaEvent_t ev : pair)
          if (ev) cudaEventDestroy(ev);
      d->ready = false;
    }
  }
  G.devs.clear();
  G.inited = false;
  nvmlReturn_t r = G.ml.shutdown();  // library handles stay open: re-init is cheap and safe
  if (r != NVML_SUCCESS) {
    set_error("nvml: %s", G.ml.errorString(r));
    return GSB_ERR_NVML;
  }
  return GSB_OK;
}

int gsb_device_count(uint32_t *n) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!n) return GSB_ERR_INVALID_ARGUMENT;
  if (!G.inited) {
    set_error("gsb_init has not succeeded");
    return GSB_ERR_NOT_INITIALIZED;
  }
  unsigned c = 0;
  ML_TRY(G.ml.getCount(&c));  // live query, like nvml.GetDeviceCount
  *n = c < G.devs.size() ? c : (uint32_t)G.devs.size();
  return GSB_OK;
}

int gsb_device_info_get(uint32_t idx, gsb_device_info *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  int rc = query_info(d, out);
  out->index = idx;
  return rc;
}

int gsb_arena_create(uint32_t idx, uint64_t max_bytes, uint64_t keep_free_bytes, uint64_t *arena_bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  return arena_create_locked(d, max_bytes, keep_free_bytes, arena_bytes);
}

int gsb_arena_destroy(uint32_t idx) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  return arena_destroy_locked(d);
}

int gsb_arena_bytes(uint32_t idx, uint64_t *arena_bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d || !arena_bytes) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  *arena_bytes = d->arena_bytes;
  return d->va ? GSB_OK : GSB_ERR_NO_ARENA;
}

int gsb_probe(uint32_t idx, const gsb_probe_cfg *cfg, gsb_probe_result *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!cfg || !out) return GSB_ERR_INVALID_ARGUMENT;
  if (cfg->op > GSB_OP_VERIFY_REFILL) {  // the March C- ops run only inside gsb_memtest
    memset(out, 0, sizeof *out);
    set_error("op %u is a March C- element: run it through gsb_memtest", cfg->op);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  Device *d = device_at(idx);
  if (!d) {
    memset(out, 0, sizeof *out);
    return out->status = G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  }
  std::lock_guard<std::mutex> lk(d->mu);
  return run_probe_locked(d, cfg, out);
}

int gsb_test_march_probe(uint32_t idx, const gsb_probe_cfg *cfg, gsb_probe_result *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!cfg || !out) return GSB_ERR_INVALID_ARGUMENT;
  if (cfg->op < GSB_OP_MARCH_FILL || cfg->op > GSB_OP_MARCH_RW_DOWN || (cfg->flags & GSB_PROBE_SEED_TABLE)) {
    memset(out, 0, sizeof *out);
    set_error("gsb_test_march_probe: op %u flags 0x%x: a GSB_OP_MARCH_* op without the seed table", cfg->op,
              cfg->flags);
    return out->status = GSB_ERR_INVALID_ARGUMENT;
  }
  Device *d = device_at(idx);
  if (!d) {
    memset(out, 0, sizeof *out);
    return out->status = G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  }
  std::lock_guard<std::mutex> lk(d->mu);
  return run_probe_locked(d, cfg, out);
}

int gsb_probe_all(uint32_t n, const uint32_t *idxs, const gsb_probe_cfg *cfg, gsb_probe_result *results) {
  if (!idxs || !cfg || !results || n > GSB_MAX_DEVICES || cfg->op > GSB_OP_VERIFY_REFILL) return GSB_ERR_INVALID_ARGUMENT;
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);  // held across the fan-out: a shutdown waits for it
  std::lock_guard<std::mutex> one(G.all_mu);             // each device worker has one job slot
  Device *ds[GSB_MAX_DEVICES];
  for (uint32_t i = 0; i < n; i++) {
    ds[i] = device_at(idxs[i]);
    for (uint32_t k = 0; k < i && ds[i]; k++)
      if (ds[k] == ds[i]) ds[i] = nullptr;  // a device listed twice runs once; the second slot reports the error
    if (!ds[i]) {
      memset(&results[i], 0, sizeof results[i]);
      results[i].status = !G.inited ? GSB_ERR_NOT_INITIALIZED : idxs[i] < G.devs.size() ? GSB_ERR_INVALID_ARGUMENT : GSB_ERR_NO_DEVICE;
      continue;
    }
    Job j;
    j.kind = Job::PROBE;
    j.idx = idxs[i];
    j.cfg = cfg;
    j.probe_out = &results[i];
    worker_submit(ds[i], j);
  }
  int rc = GSB_OK;
  for (uint32_t i = 0; i < n; i++) {
    if (ds[i]) worker_wait(ds[i]);
    if (results[i].status != GSB_OK) rc = results[i].status;
  }
  return rc;
}

int64_t gsb_cycle_all(uint32_t n, const uint32_t *idxs, uint64_t cycle_no, uint64_t window_bytes, int unit_gib,
                      uint32_t variant, uint8_t *lw_buf, size_t lw_cap, gsb_cycle_result *results) {
  if (!idxs || !results || n == 0 || n > GSB_MAX_DEVICES) return GSB_ERR_INVALID_ARGUMENT;
  if (window_bytes % kGranuleBytes) {
    set_error("cycle window must be a multiple of 64 MiB (or 0 = whole arena)");
    return GSB_ERR_INVALID_ARGUMENT;
  }
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  std::lock_guard<std::mutex> one(G.all_mu);
  Device *ds[GSB_MAX_DEVICES];
  int rcs[GSB_MAX_DEVICES];
  for (uint32_t i = 0; i < n; i++) {
    ds[i] = device_at(idxs[i]);
    if (!ds[i]) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
    for (uint32_t k = 0; k < i; k++)
      if (ds[k] == ds[i]) {
        set_error("device %u listed twice", idxs[i]);
        return GSB_ERR_INVALID_ARGUMENT;
      }
  }
  for (uint32_t i = 0; i < n; i++) {  // fan out: every device runs its own cycle on its own thread
    Job j;
    j.kind = Job::CYCLE;
    j.idx = idxs[i];
    j.cycle_no = cycle_no;
    j.window_bytes = window_bytes;
    j.unit_gib = unit_gib;
    j.variant = variant;
    j.cycle_out = &results[i];
    worker_submit(ds[i], j);
  }
  for (uint32_t i = 0; i < n; i++) rcs[i] = worker_wait(ds[i]);
  // the one join: concatenate in index order, slices from the first device, health from each verdict
  const uint32_t slices = results[0].slices;
  const char *uuids[GSB_MAX_DEVICES];
  bool any_bad = false;
  int rc_all = GSB_OK;
  for (uint32_t i = 0; i < n; i++) {
    // a failed or timed-out launch is a verdict (healthy = 0), not an API error
    if (rcs[i] < 0 && rcs[i] != GSB_ERR_DRIVER && rcs[i] != GSB_ERR_TIMEOUT) rc_all = rcs[i];
    uuids[i] = results[i].info.uuid;
    if (!results[i].healthy) any_bad = true;
  }
  if (rc_all) return rc_all;
  if (any_bad) {
    G.join_bits.assign(((size_t)n * slices + 7) / 8, 0);
    for (uint32_t i = 0; i < n; i++)
      if (!results[i].healthy)
        for (uint32_t j = 0; j < slices; j++) {  // every fake device of that GPU (nvidia.go:146-150)
          const size_t b = (size_t)i * slices + j;
          G.join_bits[b >> 3] |= (uint8_t)(1u << (b & 7));
        }
  }
  const int64_t len = gsb_encode_list_and_watch(uuids, n, slices, any_bad ? G.join_bits.data() : nullptr, lw_buf, lw_cap);
  if (len >= 0)
    for (uint32_t i = 0; i < n; i++) results[i].lw_len = i == 0 ? len : 0;  // the node's list is reported once
  return len;
}

int gsb_arena_read(uint32_t idx, uint64_t offset, void *dst, uint64_t bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d || !dst) return GSB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(d->mu);
  if (!d->va) return GSB_ERR_NO_ARENA;
  if (offset + bytes > d->arena_bytes) return GSB_ERR_INVALID_ARGUMENT;
  return arena_copy_locked(d, dst, reinterpret_cast<const void *>(d->va + offset), bytes, cudaMemcpyDeviceToHost);
}

int gsb_arena_write(uint32_t idx, uint64_t offset, const void *src, uint64_t bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d || !src) return GSB_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lk(d->mu);
  if (!d->va) return GSB_ERR_NO_ARENA;
  if (offset + bytes > d->arena_bytes) return GSB_ERR_INVALID_ARGUMENT;
  return arena_copy_locked(d, reinterpret_cast<void *>(d->va + offset), src, bytes, cudaMemcpyHostToDevice);
}

int gsb_cycle(uint32_t idx, uint64_t cycle_no, uint64_t window_bytes, int unit_gib, uint32_t variant,
              uint8_t *lw_buf, size_t lw_cap, gsb_cycle_result *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  memset(out, 0, sizeof *out);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  return cycle_impl(d, idx, cycle_no, window_bytes, unit_gib, variant, lw_buf, lw_cap, true, out);
}

int gsb_set_option(uint32_t key, uint64_t value) {
  switch (key) {
    case GSB_OPT_INVENTORY_POLICY:
      if (value != GSB_INVENTORY_SNAPSHOT && value != GSB_INVENTORY_LIVE) return GSB_ERR_INVALID_ARGUMENT;
      G.inventory_policy = value;
      return GSB_OK;
    case GSB_OPT_WAIT_SPIN_US: G.wait_spin_us = value; return GSB_OK;
    case GSB_OPT_WATCHDOG_MS: G.watchdog_ms = value; return GSB_OK;
    case GSB_OPT_INVENTORY_REFRESH_MS: G.inventory_refresh_ms = value; return GSB_OK;
    case GSB_OPT_TRANSIENT_KEEP_FREE_BYTES: G.transient_keep_free = value; return GSB_OK;
    case GSB_OPT_SWEEP_EVERY_CYCLES: G.sweep_every = value; return GSB_OK;
    case GSB_OPT_ECC_HEALTH:
      if (value > 1) return GSB_ERR_INVALID_ARGUMENT;
      G.ecc_health = value;
      return GSB_OK;
    default:
      if (std::atomic<uint64_t> *every = check_every_of(key)) {
        *every = value;
        return GSB_OK;
      }
      set_error("unknown option %u", key);
      return GSB_ERR_INVALID_ARGUMENT;
  }
}

int gsb_get_option(uint32_t key, uint64_t *value) {
  if (!value) return GSB_ERR_INVALID_ARGUMENT;
  switch (key) {
    case GSB_OPT_INVENTORY_POLICY: *value = G.inventory_policy; return GSB_OK;
    case GSB_OPT_WAIT_SPIN_US: *value = G.wait_spin_us; return GSB_OK;
    case GSB_OPT_WATCHDOG_MS: *value = G.watchdog_ms; return GSB_OK;
    case GSB_OPT_INVENTORY_REFRESH_MS: *value = G.inventory_refresh_ms; return GSB_OK;
    case GSB_OPT_TRANSIENT_KEEP_FREE_BYTES: *value = G.transient_keep_free; return GSB_OK;
    case GSB_OPT_SWEEP_EVERY_CYCLES: *value = G.sweep_every; return GSB_OK;
    case GSB_OPT_ECC_HEALTH: *value = G.ecc_health; return GSB_OK;
    default:
      if (const std::atomic<uint64_t> *every = check_every_of(key)) {
        *value = *every;
        return GSB_OK;
      }
      set_error("unknown option %u", key);
      return GSB_ERR_INVALID_ARGUMENT;
  }
}

int gsb_health_stats_get(uint32_t idx, gsb_health_stats *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  *out = d->hstats;
  return GSB_OK;
}

int gsb_inventory_refresh(uint32_t idx) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!G.inited) return GSB_ERR_NOT_INITIALIZED;
  gsb_device_info info;
  if (idx == GSB_ALL_DEVICES) {
    for (auto &d : G.devs) {
      int rc = query_info(d.get(), &info);
      if (rc) return rc;
    }
    return GSB_OK;
  }
  Device *d = device_at(idx);
  if (!d) return GSB_ERR_NO_DEVICE;
  return query_info(d, &info);
}

int gsb_inventory_snapshot(uint32_t idx, gsb_device_info *out, uint64_t *age_ns) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  int rc = snapshot_info(d, out, age_ns);
  out->index = idx;
  return rc;
}

int gsb_fault_report_get(uint32_t idx, uint32_t which, gsb_fault_report *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out || (which != GSB_FAULT_REPORT_FIRST && which != GSB_FAULT_REPORT_LAST)) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  *out = which == GSB_FAULT_REPORT_FIRST ? d->fault_first : d->fault_last;
  return GSB_OK;
}

int gsb_test_stall(uint32_t idx, uint32_t ms) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  int rc = ensure_ready(d);
  if (rc) return rc;
  const int e = gsb_kernel_stall((unsigned long long)ms * 1000000ull, d->stream);
  if (e) {
    set_error("stall kernel: %s", cudaGetErrorString((cudaError_t)e));
    return GSB_ERR_DRIVER;
  }
  return GSB_OK;
}

int gsb_test_skew_snapshot(uint32_t idx, uint64_t total_bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->snap.total = total_bytes;
  return GSB_OK;
}

int gsb_ecc_status_get(uint32_t idx, gsb_ecc_status *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  query_ecc(d, out);
  return GSB_OK;
}

int gsb_ecc_stats_get(uint32_t idx, gsb_ecc_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->ecc_stats; });
}

int gsb_memtest(uint32_t idx, const gsb_memtest_cfg *cfg, gsb_memtest_result *out) {
  return probe_entry(idx, cfg, out, &memtest_locked);
}

int gsb_test_ecc_override(uint32_t idx, const gsb_ecc_status *st) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->ecc_override_set = st != nullptr;
  d->ecc_override = st ? *st : gsb_ecc_status{};
  return GSB_OK;
}

int gsb_link_probe(uint32_t idx, const gsb_link_cfg *cfg, gsb_link_result *out) {
  return probe_entry(idx, cfg, out, &LinkCheck::run);
}

int gsb_link_status_get(uint32_t idx, gsb_link_status *out) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!out) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  query_link(d, out);
  return GSB_OK;
}

int gsb_link_stats_get(uint32_t idx, gsb_link_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->link.stats; });
}

int gsb_test_link_override(uint32_t idx, const gsb_link_status *st) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->link_override_set = st != nullptr;
  d->link_override = st ? *st : gsb_link_status{};
  return GSB_OK;
}

int gsb_test_link_corrupt(uint32_t idx, uint32_t phase, uint64_t offset, const uint32_t xr[4]) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!xr || (phase != 2 && phase != 3) || (offset & 15)) return GSB_ERR_INVALID_ARGUMENT;  // phases 2 and 3 read
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::LinkCorrupt c;
  c.phase = phase;
  c.offset = offset;
  memcpy(c.xr, xr, sizeof c.xr);
  d->link.hooks.push_back(c);
  return GSB_OK;
}

int gsb_copy_probe(uint32_t idx, const gsb_copy_cfg *cfg, gsb_copy_result *out) {
  return probe_entry(idx, cfg, out, &CopyCheck::run);
}

int gsb_copy_stats_get(uint32_t idx, gsb_copy_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->copy.stats; });
}

int gsb_test_copy_corrupt(uint32_t idx, uint32_t op, uint64_t offset, const uint32_t xr[4]) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!xr || op < GSB_OP_COPY_H2D || op > GSB_OP_COPY_D2D || (offset & 15)) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::CopyCorrupt c;
  c.dir = op - GSB_OP_COPY_H2D;
  c.offset = offset;
  memcpy(c.xr, xr, sizeof c.xr);
  d->copy.hooks.corrupt.push_back(c);
  return GSB_OK;
}

int gsb_test_copy_skip(uint32_t idx, uint32_t op) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (op < GSB_OP_COPY_H2D || op > GSB_OP_COPY_D2D) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->copy.hooks.skip |= 1u << (op - GSB_OP_COPY_H2D);
  return GSB_OK;
}

int gsb_sm_probe(uint32_t idx, const gsb_sm_cfg *cfg, gsb_sm_result *out) {
  return probe_entry(idx, cfg, out, &SmCheck::run);
}

int gsb_sm_stats_get(uint32_t idx, gsb_sm_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->sm.stats; });
}

int gsb_test_sm_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SM_UNITS || smid >= GSB_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  const int64_t words = unit == GSB_SM_UNIT_SMEM ? GSB_SM_SMEM_WORDS_MAX : gsb_sm_expected(unit, 0, nullptr, 0);
  if ((int64_t)index >= words) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->sm.hooks.corrupt[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_test_sm_operands(uint32_t idx, uint32_t unit, const int32_t *a, const int32_t *b, const int32_t *sa,
                         const int32_t *sb, const uint32_t *expected) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit < GSB_SM_UNIT_F16 || unit > GSB_SM_UNIT_S8) return GSB_ERR_INVALID_ARGUMENT;
  const gsb_sm_tensor_shape s = gsb_sm_shape(unit);
  const uint32_t K = s.k;
  std::vector<uint32_t> t;
  if (a) {
    if (!b || !sa || !sb || !expected) return GSB_ERR_INVALID_ARGUMENT;
    // the integers the generator can make ([-amp, amp]; S8 [-128, 127]) and the scales of gsb_sm_shape
    const int32_t a_lo = unit == GSB_SM_UNIT_S8 ? -128 : -s.amp_a, a_hi = unit == GSB_SM_UNIT_S8 ? 127 : s.amp_a;
    const int32_t b_lo = unit == GSB_SM_UNIT_S8 ? -128 : -s.amp_b, b_hi = unit == GSB_SM_UNIT_S8 ? 127 : s.amp_b;
    for (uint32_t n = 0; n < GSB_SM_M * K; n++)
      if (a[n] < a_lo || a[n] > a_hi) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t n = 0; n < K * GSB_SM_N; n++)
      if (b[n] < b_lo || b[n] > b_hi) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < GSB_SM_M; i++)
      if (sa[i] < s.sa_min || sa[i] > s.sa_max) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t j = 0; j < GSB_SM_N; j++)
      if (sb[j] < s.sb_min || sb[j] > s.sb_max) return GSB_ERR_INVALID_ARGUMENT;
    t.resize(GSB_SM_TENSOR_WORDS + gsb_sm_table_words(K));
    memcpy(t.data(), expected, GSB_SM_TENSOR_WORDS * sizeof(uint32_t));
    uint32_t *tab = t.data() + GSB_SM_TENSOR_WORDS;
    memcpy(tab + gsb_sm_table_a(K, 0, 0), a, GSB_SM_M * K * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_b(K, 0, 0), b, K * GSB_SM_N * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_sa(K, 0), sa, GSB_SM_M * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_sb(K, 0), sb, GSB_SM_N * sizeof(int32_t));
  }
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->sm.hooks.operands[unit].swap(t);
  return GSB_OK;
}

int gsb_sm_stress(uint32_t idx, const gsb_stress_cfg *cfg, gsb_stress_result *out) {
  return probe_entry(idx, cfg, out, &stress_locked, [](const gsb_stress_cfg *cfg, gsb_stress_result *out) {
    out->first_mismatch_slice = UINT32_MAX;
    // refused here, before any device is touched
    const bool bad = (cfg->units & ~GSB_STRESS_UNIT_MASK) || cfg->duration_ms == 0 ||
                     cfg->duration_ms > GSB_STRESS_DURATION_MAX_MS || cfg->slice_ms > GSB_STRESS_SLICE_MAX_MS;
    return bad ? GSB_ERR_INVALID_ARGUMENT : GSB_OK;
  });
}

int gsb_test_stress_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint32_t xr, uint32_t slice) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SM_UNITS || !(GSB_STRESS_UNIT_MASK >> unit & 1u) || smid >= GSB_SM_MAX ||
      index >= GSB_SM_TENSOR_WORDS)
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->stress_corrupt = Device::StressCorrupt{true, smid, unit, index, xr, slice};
  return GSB_OK;
}

int gsb_cluster_probe(uint32_t idx, const gsb_cluster_cfg *cfg, gsb_cluster_result *out) {
  return probe_entry(idx, cfg, out, &ClusterCheck::run);
}

int gsb_cluster_stats_get(uint32_t idx, gsb_cluster_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->cluster.stats; });
}

int gsb_test_cluster_corrupt(uint32_t idx, uint32_t smid, uint32_t path, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (path >= GSB_CLUSTER_PATHS || smid >= GSB_CLUSTER_SM_MAX || index >= GSB_CLUSTER_HOOK_INDEX_MAX)
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::ClusterHook &h = d->cluster.hooks[path];
  h.corrupt = true;
  h.corrupt_smid = smid;
  h.index = index;
  h.xr = xr;
  return GSB_OK;
}

int gsb_test_cluster_skip(uint32_t idx, uint32_t smid, uint32_t path) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (path >= GSB_CLUSTER_PATHS || smid >= GSB_CLUSTER_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::ClusterHook &h = d->cluster.hooks[path];
  h.skip = true;
  h.skip_smid = smid;
  return GSB_OK;
}

int gsb_test_cluster_script(uint32_t idx, uint32_t path, uint32_t n, uint32_t region_words, const uint8_t *route) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!gsb_cluster_script_valid(path, n, region_words, route)) return GSB_ERR_INVALID_ARGUMENT;  // before any device
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  Device::ClusterScript sc;
  if (route) {
    sc.armed = true;
    sc.script.region_words = region_words;
    memset(sc.script.route, GSB_CLUSTER_UNROUTED, sizeof sc.script.route);
    memcpy(sc.script.route, route, (size_t)n * n);
  }
  std::lock_guard<std::mutex> lk(d->smu);
  d->cluster_scripts[path][__builtin_ctz(n) - 1] = sc;
  return GSB_OK;
}

int gsb_atomic_probe(uint32_t idx, const gsb_atomic_cfg *cfg, gsb_atomic_result *out) {
  return probe_entry(idx, cfg, out, &AtomicCheck::run);
}

int gsb_atomic_stats_get(uint32_t idx, gsb_atomic_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->atomic.stats; });
}

int gsb_test_atomic_corrupt(uint32_t idx, uint32_t op, uint32_t word, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (op >= GSB_ATOMIC_OPS || word >= gsb_atomic_units(op) || (gsb_atomic_unit_bytes(op) == 4u && xr >> 32))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::AtomicHook &h = d->atomic.hooks[op];
  h.corrupt = true;
  h.word = word;
  h.xr = xr;
  return GSB_OK;
}

int gsb_test_atomic_skip(uint32_t idx, uint32_t smid, uint32_t op) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (op >= GSB_ATOMIC_OPS || smid >= GSB_ATOMIC_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::AtomicHook &h = d->atomic.hooks[op];
  h.skip = true;
  h.skip_smid = smid;
  return GSB_OK;
}

int gsb_test_atomic_values(uint32_t idx, uint32_t op, uint32_t ctas, const uint64_t *init, const uint64_t *values,
                           size_t n_values, const uint64_t *expected) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  // refused here, before any device is touched
  if (op >= GSB_ATOMIC_OPS || op == GSB_ATOMIC_OP_TICKET || op == GSB_ATOMIC_OP_CAS) return GSB_ERR_INVALID_ARGUMENT;
  if (init && !gsb_atomic_values_valid(op, ctas, init, values, n_values, expected)) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  if (init && ctas != d->sm_count) return GSB_ERR_INVALID_ARGUMENT;
  Device::AtomicValues v;
  if (init) {
    const uint32_t ub = gsb_atomic_unit_bytes(op), n = gsb_atomic_units(op);
    v.armed = true;
    v.init.resize(GSB_ATOMIC_BYTES);
    v.expected.resize(GSB_ATOMIC_BYTES);
    for (uint32_t u = 0; u < n; u++) {  // little-endian words, as the device holds them
      memcpy(&v.init[(size_t)u * ub], &init[u], ub);
      memcpy(&v.expected[(size_t)u * ub], &expected[u], ub);
    }
    v.table.assign(values, values + n_values);
  }
  std::lock_guard<std::mutex> lk(d->smu);
  d->atomic_values[op] = std::move(v);
  return GSB_OK;
}

int gsb_tensor_probe(uint32_t idx, const gsb_tensor_cfg *cfg, gsb_tensor_result *out) {
  return probe_entry(idx, cfg, out, &TensorCheck::run);
}

int gsb_tensor_stats_get(uint32_t idx, gsb_tensor_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->tensor.stats; });
}

int gsb_sfu_probe(uint32_t idx, const gsb_sfu_cfg *cfg, gsb_sfu_result *out) {
  return probe_entry(idx, cfg, out, &SfuCheck::run);
}

int gsb_sfu_stats_get(uint32_t idx, gsb_sfu_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->sfu.stats; });
}

int gsb_test_sfu_inputs(uint32_t idx, uint32_t unit, uint32_t op, const uint64_t *a, const uint64_t *b, size_t n,
                        uint64_t *results, uint32_t *covered) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  // refused here, before any device is touched
  if (n == 0 || n > GSB_SFU_INPUTS_MAX || !results || !covered || !gsb_sfu_operands_valid(unit, op, a, b, n))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->mu);
  return sfu_inputs_locked(d, unit, op, a, b, n, results, covered);
}

int gsb_test_sfu_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SFU_UNITS || smid >= GSB_SM_MAX || index >= gsb_sfu_ops(unit) * GSB_SFU_THREADS)
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->sfu.hooks[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_l1_probe(uint32_t idx, const gsb_l1_cfg *cfg, gsb_l1_result *out) {
  return probe_entry(idx, cfg, out, &L1Check::run);
}

int gsb_l1_stats_get(uint32_t idx, gsb_l1_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->l1.stats; });
}

int gsb_test_l1_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_L1_UNITS || smid >= GSB_SM_MAX || index >= gsb_l1_hook_words(unit)) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->l1.hooks.corrupt[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_test_l1_table(uint32_t idx, uint32_t unit, const uint32_t *table, size_t n, const uint32_t *expected,
                      size_t n_expected, uint32_t region_words) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  // refused here, before any device is touched
  if (unit >= GSB_L1_UNITS || (table && !gsb_l1_table_valid(unit, table, n, expected, n_expected, region_words)))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  Device::L1Table tb;
  if (table) {
    if (n_expected != gsb_l1_table_expected_per_cta(unit, n, region_words) * d->sm_count) return GSB_ERR_INVALID_ARGUMENT;
    tb.armed = true;
    tb.region_words = region_words;
    tb.table.assign(table, table + n);
    if (n_expected) tb.expected.assign(expected, expected + n_expected);
  }
  std::lock_guard<std::mutex> lk(d->smu);
  d->l1_table[unit] = std::move(tb);
  return GSB_OK;
}

int gsb_test_l1_skip(uint32_t idx, uint32_t smid) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (smid >= GSB_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->l1.hooks.skip_armed = true;
  d->l1.hooks.skip_smid = smid;
  return GSB_OK;
}

int gsb_order_probe(uint32_t idx, const gsb_order_cfg *cfg, gsb_order_result *out) {
  // a bad configuration is refused before any device is touched
  return probe_entry(idx, cfg, out, &OrderCheck::run, [](const gsb_order_cfg *c, gsb_order_result *) {
    return c->units & ~kOrderAllUnits || c->observations > GSB_ORDER_OBS_MAX ? GSB_ERR_INVALID_ARGUMENT : GSB_OK;
  });
}

int gsb_order_stats_get(uint32_t idx, gsb_order_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->order.stats; });
}

int gsb_test_order_inject(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_ORDER_UNITS || unit == GSB_ORDER_UNIT_MP_RELAXED || smid >= GSB_SM_MAX || index >= GSB_ORDER_OBS_MAX)
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::OrderInject &h = d->order.hooks.inject[unit];
  h.armed = true;
  h.smid = smid;
  h.index = index;
  return GSB_OK;
}

int gsb_test_order_skip(uint32_t idx, uint32_t smid) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (smid >= GSB_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->order.hooks.skip_armed = true;
  d->order.hooks.skip_smid = smid;
  return GSB_OK;
}

}  // extern "C"

namespace {

// The bits a D word of tensor unit `unit` has: FP64, FP16 (F16_ACC) or FP32.
uint64_t tensor_word_mask(uint32_t unit) {
  return unit == GSB_TENSOR_UNIT_DMMA ? ~0ull : unit == GSB_TENSOR_UNIT_F16_ACC ? 0xFFFFull : 0xFFFFFFFFull;
}

}  // namespace

extern "C" {

int gsb_shared_atomic_probe(uint32_t idx, const gsb_shared_atomic_cfg *cfg, gsb_shared_atomic_result *out) {
  return probe_entry(idx, cfg, out, &SharedAtomicCheck::run);
}

int gsb_shared_atomic_stats_get(uint32_t idx, gsb_shared_atomic_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->shared_atomic.stats; });
}

int gsb_test_shared_atomic_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SHARED_ATOMIC_UNITS || smid >= GSB_SM_MAX || index >= GSB_SHARED_ATOMIC_AREA_WORDS || (xr >> 32))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->shared_atomic.hooks.corrupt[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_test_shared_atomic_skip(uint32_t idx, uint32_t smid, uint32_t unit) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SHARED_ATOMIC_UNITS || smid >= GSB_SM_MAX) return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->shared_atomic.hooks.skip[unit];
  c.armed = true;
  c.smid = smid;
  return GSB_OK;
}

int gsb_sparse_probe(uint32_t idx, const gsb_sparse_cfg *cfg, gsb_sparse_result *out) {
  return probe_entry(idx, cfg, out, &SparseCheck::run);
}

int gsb_sparse_stats_get(uint32_t idx, gsb_sparse_stats *out) {
  return stats_entry(idx, out, [](Device *d) { return &d->sparse.stats; });
}

int gsb_test_sparse_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SPARSE_UNITS || smid >= GSB_SM_MAX || index >= GSB_SPARSE_WORDS || (xr >> 32))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->sparse.hooks.corrupt[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_test_sparse_operands(uint32_t idx, uint32_t unit, const int32_t *a, const uint8_t *pattern, const int32_t *b,
                             const int32_t *sa, const int32_t *sb, const uint64_t *expected) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_SPARSE_UNITS) return GSB_ERR_INVALID_ARGUMENT;
  const gsb_sm_tensor_shape s = gsb_sparse_shape(unit);
  const uint32_t K = s.k, groups = gsb_sparse_groups(unit);
  // S8: the full int8 range; otherwise [-amp, amp], as the generator makes them
  const int32_t a_lo = unit == GSB_SPARSE_UNIT_S8_SP ? -128 : -s.amp_a, a_hi = unit == GSB_SPARSE_UNIT_S8_SP ? 127 : s.amp_a;
  const int32_t b_lo = unit == GSB_SPARSE_UNIT_S8_SP ? -128 : -s.amp_b, b_hi = unit == GSB_SPARSE_UNIT_S8_SP ? 127 : s.amp_b;
  std::vector<uint32_t> t;
  if (a) {
    if (!pattern || !b || !sa || !sb || !expected) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t n = 0; n < GSB_SM_M * K / 2; n++)
      if (a[n] < a_lo || a[n] > a_hi) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t n = 0; n < GSB_SM_M * groups; n++)
      if (pattern[n] >= gsb_sparse_patterns(unit)) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t n = 0; n < K * GSB_SM_N; n++)
      if (b[n] < b_lo || b[n] > b_hi) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < GSB_SM_M; i++)
      if (sa[i] < s.sa_min || sa[i] > s.sa_max) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t j = 0; j < GSB_SM_N; j++)
      if (sb[j] < s.sb_min || sb[j] > s.sb_max) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t w = 0; w < GSB_SPARSE_WORDS; w++)
      if (expected[w] >> 32) return GSB_ERR_INVALID_ARGUMENT;
    t.resize(GSB_SPARSE_WORDS + gsb_sparse_table_words(unit));
    for (uint32_t w = 0; w < GSB_SPARSE_WORDS; w++) t[w] = (uint32_t)expected[w];
    uint32_t *tab = t.data() + GSB_SPARSE_WORDS;
    memcpy(tab + gsb_sparse_table_a(unit, 0, 0), a, GSB_SM_M * K / 2 * sizeof(int32_t));
    for (uint32_t n = 0; n < GSB_SM_M * groups; n++) tab[gsb_sparse_table_p(unit, 0, 0) + n] = pattern[n];
    memcpy(tab + gsb_sparse_table_b(unit, 0, 0), b, K * GSB_SM_N * sizeof(int32_t));
    memcpy(tab + gsb_sparse_table_sa(unit, 0), sa, GSB_SM_M * sizeof(int32_t));
    memcpy(tab + gsb_sparse_table_sb(unit, 0), sb, GSB_SM_N * sizeof(int32_t));
  }
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->sparse.hooks.operands[unit].swap(t);
  return GSB_OK;
}

int gsb_test_tensor_corrupt(uint32_t idx, uint32_t smid, uint32_t unit, uint32_t index, uint64_t xr) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_TENSOR_UNITS || smid >= GSB_SM_MAX || index >= GSB_TENSOR_WORDS || (xr & ~tensor_word_mask(unit)))
    return GSB_ERR_INVALID_ARGUMENT;
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  Device::SmCorrupt &c = d->tensor.hooks.corrupt[unit];
  c.armed = true;
  c.smid = smid;
  c.index = index;
  c.xr = xr;
  return GSB_OK;
}

int gsb_test_tensor_operands(uint32_t idx, uint32_t unit, const int32_t *a, const int32_t *b, const int32_t *sa,
                             const int32_t *sb, const uint64_t *expected) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (unit >= GSB_TENSOR_UNITS) return GSB_ERR_INVALID_ARGUMENT;
  const gsb_sm_tensor_shape s = gsb_tensor_shape(unit);
  const uint32_t K = s.k, wb = gsb_tensor_word_bytes(unit);
  std::vector<uint32_t> t;
  if (a) {
    if (!b || !sa || !sb || !expected) return GSB_ERR_INVALID_ARGUMENT;
    // the integers ([-amp, amp]) and scales the generator can make, and words the unit's D can hold
    for (uint32_t n = 0; n < GSB_SM_M * K; n++)
      if (a[n] < -s.amp_a || a[n] > s.amp_a) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t n = 0; n < K * GSB_SM_N; n++)
      if (b[n] < -s.amp_b || b[n] > s.amp_b) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t i = 0; i < GSB_SM_M; i++)
      if (sa[i] < s.sa_min || sa[i] > s.sa_max) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t j = 0; j < GSB_SM_N; j++)
      if (sb[j] < s.sb_min || sb[j] > s.sb_max) return GSB_ERR_INVALID_ARGUMENT;
    for (uint32_t w = 0; w < GSB_TENSOR_WORDS; w++)
      if (expected[w] & ~tensor_word_mask(unit)) return GSB_ERR_INVALID_ARGUMENT;
    const uint32_t head = GSB_TENSOR_WORDS * wb / sizeof(uint32_t);  // the expected words, as uint32
    t.resize(head + gsb_sm_table_words(K));
    for (uint32_t w = 0; w < GSB_TENSOR_WORDS; w++) memcpy(reinterpret_cast<char *>(t.data()) + w * wb, &expected[w], wb);
    uint32_t *tab = t.data() + head;
    memcpy(tab + gsb_sm_table_a(K, 0, 0), a, GSB_SM_M * K * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_b(K, 0, 0), b, K * GSB_SM_N * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_sa(K, 0), sa, GSB_SM_M * sizeof(int32_t));
    memcpy(tab + gsb_sm_table_sb(K, 0), sb, GSB_SM_N * sizeof(int32_t));
  }
  Device *d = device_at(idx);
  if (!d) return G.inited ? GSB_ERR_NO_DEVICE : GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> lk(d->smu);
  d->tensor.hooks.operands[unit].swap(t);
  return GSB_OK;
}

}  // extern "C"

namespace {

// One inventory + health-probe cycle of one device. The caller holds G.api_mu (shared).
int cycle_impl(Device *d, uint32_t idx, uint64_t cycle_no, uint64_t window_bytes, int unit_gib, uint32_t variant,
               uint8_t *lw_buf, size_t lw_cap, bool encode_lw, gsb_cycle_result *out) {
  memset(out, 0, sizeof *out);
  if (window_bytes % kGranuleBytes) {
    set_error("cycle window must be a multiple of 64 MiB (or 0 = whole arena)");
    return GSB_ERR_INVALID_ARGUMENT;
  }
  std::lock_guard<std::mutex> lk(d->mu);
  // Transient window (SURVEY §7 hard-part 2, the tenant-safe steady state): with no standing arena the cycle
  // allocates the window, fills it, verifies it and gives it back, so between cycles the plugin holds no HBM beyond
  // its CUDA context and the advertised slices are not oversold. "Nothing free to probe" (tenants hold the
  // HBM) is not a GPU fault.
  if (d->va && d->transient_arena) {
    // a transient window that a wedged launch kept mapped: give it back now if the stream has drained, otherwise this
    // cycle's verdict is the same wedge (nothing new is queued, nothing more is allocated)
    if (d->wedged && cudaStreamQuery(d->stream) != cudaErrorNotReady) d->wedged = false;
    if (arena_destroy_locked(d) == GSB_OK) d->transient_arena = false;
  }
  const bool leftover = d->va && d->transient_arena;
  const bool transient = !d->va || leftover;
  gsb_probe_result fill_res;
  memset(&fill_res, 0, sizeof fill_res);
  int prc = GSB_OK;
  bool skip_probe = false;
  if (transient) {
    if (window_bytes == 0) {
      set_error("no arena on %s: call gsb_arena_create first (or pass a window for a transient probe)", d->uuid);
      return GSB_ERR_NO_ARENA;
    }
    out->transient = 1;
    uint64_t got = 0;
    if (leftover) {
      set_error("%s: the previous transient window is still held by a wedged launch", d->uuid);
      prc = GSB_ERR_TIMEOUT;
    } else {
      prc = arena_create_locked(d, window_bytes, G.transient_keep_free.load(), &got, &fill_res);
      if (prc != GSB_OK && d->va) d->transient_arena = true;  // could not be unmapped under a wedged launch: retried next cycle
    }
    if (prc == GSB_ERR_OUT_OF_MEMORY) {
      out->probe.status = GSB_ERR_OUT_OF_MEMORY;
      prc = GSB_OK;
      skip_probe = true;
    } else if (prc) {
      out->probe = fill_res;
      out->probe.status = prc;
      skip_probe = true;
    }
  }
  // 1. health: enqueue this cycle's walk (asynchronous). Standing arena: VERIFY_REFILL of the cycle's window.
  //    Transient window: the FILL above wrote generation g, VERIFY reads it back.
  gsb_probe_cfg cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.op = transient ? GSB_OP_VERIFY : GSB_OP_VERIFY_REFILL;
  cfg.variant = variant;
  cfg.flags = GSB_PROBE_TIMED | GSB_PROBE_SEED_TABLE;
  if (!transient) {
    if (window_bytes && window_bytes < d->arena_bytes) {
      const uint64_t n_win = d->arena_bytes / window_bytes;
      cfg.window_offset = (cycle_no % n_win) * window_bytes;
      cfg.window_bytes = window_bytes;
    }
    cfg.seed_write = d->next_gen++;
    if (d->next_gen == 0) d->next_gen = 1;
  }
  // diagnostic knob GSB_CYCLE_ORDER (tools/cycle_breakdown.py): 0 = launch, then inventory while the kernel
  // runs (shipped); 1 = inventory first, then launch
  static const int order = [] {
    const char *e = getenv("GSB_CYCLE_ORDER");
    return e ? atoi(e) : 0;
  }();
  ProbeFlight fl;
  fl.transient = transient;
  if (!skip_probe && order != 1) prc = probe_begin_locked(d, &cfg, &out->probe, &fl);

  // 2. inventory while the kernel walks HBM: identity + total (policy SNAPSHOT: NVML's (re)start-time answer,
  //    identity re-validated on the CUDA side; policy LIVE: a fresh NVML query), slices, S fake devices, wire bytes
  //    (optimistically with the health this device had going into the cycle)
  const uint64_t t0 = now_ns();
  int rc;
  if (G.inventory_policy.load(std::memory_order_relaxed) == GSB_INVENTORY_LIVE) {
    rc = query_info(d, &out->info);
    out->inventory_live = 1;
  } else {
    rc = snapshot_info(d, &out->info, &out->snapshot_age_ns);
  }
  if (rc == GSB_OK) {
    out->info.index = idx;
    out->slices = gsb_slices(out->info.total_mib, unit_gib);
  }
  const char *uuids[1] = {out->info.uuid};
  auto encode = [&](bool unhealthy) -> int64_t {
    if (!encode_lw) return 0;
    const uint8_t *bits = nullptr;
    if (unhealthy) {  // every fake device of a faulted GPU (nvidia.go:146-150)
      d->bits_scratch.assign((out->slices + 7) / 8, 0xFF);
      bits = d->bits_scratch.data();
    }
    return gsb_encode_list_and_watch(uuids, 1, out->slices, bits, lw_buf, lw_cap);
  };
  if (rc == GSB_OK) out->lw_len = encode(d->faulted);
  out->inventory_ns = now_ns() - t0;
  if (!skip_probe && order == 1) prc = probe_begin_locked(d, &cfg, &out->probe, &fl);

  // 3. verdict
  if (!skip_probe && prc == GSB_OK) prc = probe_end_locked(d, &fl, &out->probe);
  if (transient) {
    if (!skip_probe && prc == GSB_OK) {  // one figure for the window: FILL wrote it, VERIFY read it
      out->probe.kernel_ns += fill_res.kernel_ns;
      out->probe.bytes_written = fill_res.bytes_written;
    }
    if (!leftover && d->va && arena_destroy_locked(d) != GSB_OK) d->transient_arena = true;  // wedged: kept, retried next cycle
  }
  if (rc) return rc;
  if (out->lw_len < 0) return (int)out->lw_len;
  out->healthy = (prc == GSB_OK && out->probe.mismatch_words == 0 && !d->faulted) ? 1u : 0u;
  if (!(prc == GSB_OK && out->probe.mismatch_words == 0) && !d->faulted) {
    d->faulted = true;  // sticky (server.go:180 FIXME): the list this cycle reports already carries it
    out->lw_len = encode(true);
    if (out->lw_len < 0) return (int)out->lw_len;
  }
  return prc;
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------------- health

int gsb_xid_is_benign(uint64_t xid) { return xid == 31 || xid == 43 || xid == 45; }

int gsb_health_set_recovery(uint32_t clean_cycles) {
  G.recovery_cycles = clean_cycles;
  return GSB_OK;
}

int gsb_health_inject(const gsb_event *ev) {
  if (!ev) return GSB_ERR_INVALID_ARGUMENT;
  push_event(*ev);
  return GSB_OK;
}

int gsb_health_wait(uint32_t timeout_ms, gsb_event *ev) {
  if (!ev) return GSB_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lk(G.hmu);
  const uint64_t gen = G.stop_gen;
  G.hcv.wait_for(lk, std::chrono::milliseconds(timeout_ms), [&] { return !G.events.empty() || G.stop_gen != gen; });
  if (!G.events.empty()) {
    *ev = G.events.front();
    G.events.pop_front();
    return GSB_OK;
  }
  return G.stop_gen != gen ? GSB_ERR_STOPPED : GSB_ERR_TIMEOUT;
}

int gsb_health_start(uint32_t probe_period_ms, uint64_t window_bytes) {
  std::shared_lock<std::shared_mutex> api_lk(G.api_mu);
  if (!G.inited) return GSB_ERR_NOT_INITIALIZED;
  std::lock_guard<std::mutex> hl(G.health_mu);
  std::lock_guard<std::mutex> lk(G.mu);
  if (G.shutting_down) {
    set_error("gsb_shutdown is in progress");
    return GSB_ERR_NOT_INITIALIZED;
  }
  if (G.health_running) return GSB_OK;
  G.health_stop = false;
  // ECC half (opt-in): every device's status now is the session's baseline. A pending remap or a remap failure is
  // level-triggered — it outlives a plugin restart that an XID event does not — so it is raised at once.
  const bool ecc = G.ecc_health.load() != 0;
  for (auto &d : G.devs) {
    gsb_ecc_status base;
    if (ecc) query_ecc(d.get(), &base);
    {
      std::lock_guard<std::mutex> sl(d->smu);
      d->ecc_stats = gsb_ecc_stats{};
      d->ecc_raised = 0;
      d->ecc_baseline = ecc ? base : gsb_ecc_status{};
      if (ecc) d->ecc_stats.queries = 1;
      for_each_check([&](auto check, size_t) {
        auto &state = decltype(check)::state(d.get());
        state.stats = {};
        state.raised = 0;
      });
    }
    if (ecc) raise_ecc_conditions(d.get(), base);
  }
  // XID half: one registration per GPU (the reference registers the same GPU once per fake device)
  if (G.ml.eventSetCreate && G.ml.registerEvents && G.ml.eventSetWait && G.ml.eventSetFree) {
    nvmlReturn_t cr = G.ml.eventSetCreate(&G.event_set);
    if (cr != NVML_SUCCESS) {
      set_error("nvml: %s (nvmlEventSetCreate)", G.ml.errorString(cr));
      return GSB_ERR_NVML;
    }
    G.have_event_set = true;
    for (auto &d : G.devs) {
      nvmlReturn_t r = G.ml.registerEvents(d->nvml, nvmlEventTypeXidCriticalError, G.event_set);
      if (r == NVML_ERROR_NOT_SUPPORTED) {
        // nvidia.go:107-112: too old to support health checking -> marked unhealthy
        gsb_event ev;
        memset(&ev, 0, sizeof ev);
        snprintf(ev.uuid, sizeof ev.uuid, "%s", d->uuid);
        ev.etype = GSB_EVENT_XID;
        ev.edata = ~0ull;
        push_event(ev);
      } else if (r != NVML_SUCCESS) {
        // nvidia.go:114-116: any other registration error is fatal (log.Fatalf) — a GPU without XID coverage must
        // not stay silently Healthy. The caller decides what fatal means; nothing is left half started.
        set_error("nvml: %s (nvmlDeviceRegisterEvents on %s)", G.ml.errorString(r), d->uuid);
        G.ml.eventSetFree(G.event_set);
        G.have_event_set = false;
        std::lock_guard<std::mutex> hl(G.hmu);
        G.events.clear();
        return GSB_ERR_NVML;
      }
    }
    G.health_threads.emplace_back([] {
      uint64_t last_refresh = now_ns();
      while (!G.health_stop.load()) {
        // low-rate inventory refresh (GSB_OPT_INVENTORY_REFRESH_MS, default 5000 = the reference's WaitForEvent
        // period; 0 = never): NVML is re-asked off the cycle's path, and an answer that differs from the snapshot
        // (a different GPU behind the handle, a different total) is reported as an event, not papered over
        const uint64_t period = G.inventory_refresh_ms.load() * 1000000ull;
        if (period && now_ns() - last_refresh >= period) {
          last_refresh = now_ns();
          for (auto &d : G.devs) {
            Snapshot before;
            {
              std::lock_guard<std::mutex> sl(d->smu);
              before = d->snap;
            }
            gsb_device_info info;
            const int qrc = query_info(d.get(), &info);
            uint64_t what = 0;
            if (qrc == GSB_ERR_IDENTITY_MISMATCH || (qrc == GSB_OK && strcmp(before.uuid, info.uuid) != 0))
              what = GSB_INVENTORY_IDENTITY_CHANGED;
            else if (qrc == GSB_OK && before.total != info.total_bytes)
              what = GSB_INVENTORY_TOTAL_CHANGED;
            if (what) {
              gsb_event ev;
              memset(&ev, 0, sizeof ev);
              snprintf(ev.uuid, sizeof ev.uuid, "%s", before.uuid);
              ev.etype = GSB_EVENT_INVENTORY;
              ev.edata = what;
              push_event(ev);
            }
            if (G.ecc_health.load()) {  // ECC health: the status again, against the session's baseline
              gsb_ecc_status now;
              query_ecc(d.get(), &now);
              {
                std::lock_guard<std::mutex> sl(d->smu);
                d->ecc_stats.queries++;
              }
              raise_ecc_conditions(d.get(), now);
            }
          }
        }
        // with ECC health on, a refresh period under the 200 ms wait is kept: a condition is raised within one period
        const uint64_t refresh_ms = G.inventory_refresh_ms.load();
        const unsigned wait_ms = G.ecc_health.load() && refresh_ms && refresh_ms < 200 ? (unsigned)refresh_ms : 200u;
        nvmlEventData_t data;
        memset(&data, 0, sizeof data);
        nvmlReturn_t r = G.ml.eventSetWait(G.event_set, &data, wait_ms);
        if (r != NVML_SUCCESS) {
          if (r != NVML_ERROR_TIMEOUT) std::this_thread::sleep_for(std::chrono::milliseconds(200));
          continue;
        }
        if (data.eventType != nvmlEventTypeXidCriticalError) continue;  // nvidia.go:127-129
        gsb_event ev;
        memset(&ev, 0, sizeof ev);
        if (data.device) G.ml.getUUID(data.device, ev.uuid, GSB_UUID_BUFFER_SIZE);
        ev.etype = data.eventType;
        ev.edata = data.eventData;
        push_event(ev);
      }
    });
  }
  // active half: rotate a window probe over each device's arena
  if (probe_period_ms > 0) {
    for (uint32_t i = 0; i < G.devs.size(); i++) {
      G.health_threads.emplace_back([i, probe_period_ms, window_bytes] {
        // a prober with milliseconds between cycles sleeps through the kernel instead of spinning a core: the
        // DaemonSet gives the whole plugin one CPU (device-plugin-ds.yaml:34-40)
        tl_wait_blocking = probe_period_ms >= 10;
        std::vector<uint8_t> buf(1 << 16);
        uint64_t cycle = 0;
        bool reported = false;
        uint32_t clean = 0;
        EccPrev ecc_prev;
        {
          std::lock_guard<std::mutex> sl(G.devs[i]->smu);
          G.devs[i]->hstats = gsb_health_stats{};
        }
        while (!G.health_stop.load()) {
          gsb_cycle_result cr;
          // every Nth cycle of a device WITHOUT a standing arena is a sweep: a transient window as large as whatever is
          // allocatable right now (minus the keep-free margin) — all free HBM walked, then given back (SURVEY §7
          // hard-part 2: "full walk only at start-up / idle"). With a standing arena the request is just a whole-arena cycle.
          const uint64_t every = G.sweep_every.load(std::memory_order_relaxed);
          const bool sweep = every > 0 && window_bytes > 0 && (cycle + 1) % every == 0;
          const uint64_t cycle_window = sweep ? (1ull << 46) : window_bytes;
          // ECC health: the volatile totals right before and right after the cycle, read here and not inside gsb_cycle
          // (the cycle's own cost stays NVML-free). The difference across a cycle is its walk's.
          const bool ecc = G.ecc_health.load(std::memory_order_relaxed) != 0;
          uint64_t c0 = 0, u0 = 0, c1 = 0, u1 = 0;
          const bool pre_ok = ecc && read_ecc_totals(G.devs[i].get(), &c0, &u0);
          const uint64_t this_cycle = cycle;
          const uint64_t t_cycle = now_ns();
          int rc = gsb_cycle(i, cycle++, cycle_window, 1, GSB_VARIANT_AUTO, buf.data(), buf.size(), &cr);
          if (ecc) {
            const bool post_ok = read_ecc_totals(G.devs[i].get(), &c1, &u1);
            ecc_account(G.devs[i].get(), pre_ok, c0, u0, post_ok, c1, u1, this_cycle, cycle_window, cr, &ecc_prev);
          }
          {
            std::lock_guard<std::mutex> sl(G.devs[i]->smu);
            gsb_health_stats &st = G.devs[i]->hstats;
            st.cycles++;
            st.last_bytes_walked = cr.probe.bytes_walked;
            st.last_kernel_ns = cr.probe.kernel_ns;
            if (cr.probe.status == GSB_ERR_OUT_OF_MEMORY) st.skipped++;
            if (!(rc == GSB_OK && cr.probe.mismatch_words == 0) && rc != GSB_ERR_NO_ARENA) st.faults++;
            if (sweep && cr.transient) {
              st.sweeps++;
              st.last_sweep_bytes = cr.probe.bytes_walked;
              st.last_sweep_ns = now_ns() - t_cycle;
            }
          }
          // with no standing arena the cycle probes a transient window (allocate -> fill -> verify -> free); a
          // window that could not be allocated (tenants hold the HBM) is silence, not a fault
          const bool this_cycle_clean = rc == GSB_OK && cr.probe.mismatch_words == 0;
          if (rc != GSB_ERR_NO_ARENA && !this_cycle_clean && !reported) {
            gsb_event ev;
            memset(&ev, 0, sizeof ev);
            snprintf(ev.uuid, sizeof ev.uuid, "%s", G.devs[i]->uuid);
            ev.etype = GSB_EVENT_PROBE;
            ev.edata = rc == GSB_OK ? GSB_PROBE_FAULT_MISMATCH : rc == GSB_ERR_TIMEOUT ? GSB_PROBE_FAULT_WEDGED : GSB_PROBE_FAULT_LAUNCH;
            push_event(ev);
            reported = true;
            clean = 0;
          } else if (reported) {
            clean = this_cycle_clean ? clean + 1 : 0;
            const uint32_t need = G.recovery_cycles.load();
            if (need > 0 && clean >= need) {  // optional recovery: the refills since the fault all verified
              {
                std::lock_guard<std::mutex> dl(G.devs[i]->mu);
                G.devs[i]->faulted = false;
              }
              {
                std::lock_guard<std::mutex> sl(G.devs[i]->smu);  // the next fault is latched as FIRST again
                G.devs[i]->fault_first = gsb_fault_report{};
              }
              gsb_event ev;
              memset(&ev, 0, sizeof ev);
              snprintf(ev.uuid, sizeof ev.uuid, "%s", G.devs[i]->uuid);
              ev.etype = GSB_EVENT_PROBE;
              ev.edata = GSB_PROBE_RECOVERED;
              push_event(ev);
              reported = false;
              clean = 0;
            }
          }
          // the periodic checks (each opt-in): after the session's first cycle and every Nth one, outside gsb_cycle, in
          // the order of Checks when several are due
          for_each_check([&](auto check, size_t k) {
            const uint64_t n = G.check_every[k].load(std::memory_order_relaxed);
            if (n && this_cycle % n == 0 && !G.health_stop.load()) run_check<decltype(check)>(i);
          });
          for (uint32_t slept = 0; slept < probe_period_ms && !G.health_stop.load(); slept += 10)
            std::this_thread::sleep_for(std::chrono::milliseconds(10));
        }
      });
    }
  }
  G.health_running = true;
  return GSB_OK;
}

int gsb_health_stop(void) {
  {  // wake every waiter, whether or not the internal threads are running
    std::lock_guard<std::mutex> lk(G.hmu);
    G.stop_gen++;
  }
  G.hcv.notify_all();
  std::lock_guard<std::mutex> hl(G.health_mu);
  std::vector<std::thread> ts;
  {
    std::lock_guard<std::mutex> lk(G.mu);
    if (!G.health_running) return GSB_OK;
    G.health_stop = true;
    ts.swap(G.health_threads);
    G.health_running = false;
  }
  for (auto &t : ts) t.join();
  if (G.have_event_set) {
    G.ml.eventSetFree(G.event_set);
    G.have_event_set = false;
  }
  std::lock_guard<std::mutex> lk(G.hmu);
  G.events.clear();
  G.health_stop = false;
  return GSB_OK;
}

}  // extern "C"
