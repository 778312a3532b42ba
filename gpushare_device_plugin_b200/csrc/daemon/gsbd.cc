// gsbd — native (C++) gpushare device-plugin daemon over libgpushare_b200.so.
//
// The same process the reference builds from cmd/nvidia/main.go + pkg/gpu/nvidia/*.go, with the same
// flags, wire surface, side effects and exit codes, and no interpreter on any RPC path:
//   main / flags                cmd/nvidia/main.go:15-78
//   manager loop, watchers      pkg/gpu/nvidia/gpumanager.go:33-111, watchers.go:10-32
//   plugin server               pkg/gpu/nvidia/server.go (Start/Stop/Register/ListAndWatch/healthcheck/Serve)
//   Allocate                    pkg/gpu/nvidia/allocate.go:42-198 -> gsb_allocate (C ABI) + LIST/PATCH here
//   pod / node helpers          pkg/gpu/nvidia/podmanager.go, podutils.go
//   kubelet /pods/ client       pkg/kubelet/client/client.go:75-134
// gRPC framing is csrc/daemon/h2.hpp; every message byte comes from the C ABI encoders.
// Pieces private to this translation unit: gsbd_log.hpp (constants, logging), gsbd_flags.hpp (command line),
// gsbd_kube.hpp (apiserver client configuration and calls), gsbd_pods.hpp (pod JSON -> gsb_pod table); this file is
// the plugin (server.go + allocate.go) and the manager loop.
#include <fcntl.h>
#include <poll.h>
#include <signal.h>
#include <stdarg.h>
#include <stdio.h>
#include <sys/resource.h>
#include <stdlib.h>
#include <string.h>
#include <sys/inotify.h>
#include <sys/signalfd.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <time.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <fstream>
#include <memory>
#include <mutex>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../../include/gpushare_b200.h"
#include "h2.hpp"
#include "http_client.hpp"
#include "json.hpp"

#include "gsbd_flags.hpp"
#include "gsbd_kube.hpp"
#include "gsbd_log.hpp"
#include "gsbd_pods.hpp"

namespace {

// ---------------------------------------------------------------- the periodic health checks (not in the reference)

// What a gsb_*_text function writes: asked for its length, then for the text. Empty when it has nothing to say.
template <typename Text>
std::string text_of(Text text) {
  const int64_t need = text(nullptr, 0);
  if (need <= 0) return "";
  std::string s((size_t)need, '\0');
  const int64_t n = text(&s[0], s.size());
  s.resize(n > 0 ? (size_t)n : 0);
  return s;
}

// One GPU's statistics of one check: zero, and the line of a probe that did not run, when they cannot be read
// (--fake-inventory, or no such GPU).
struct Probed {
  uint64_t probes;
  std::string counters;  // as dump() prints them
  std::string line;      // gsb_*_text of the most recent probe
};

template <typename Stats, typename Result>
Probed probed(uint32_t idx, const std::string &uuid, int (*get)(uint32_t, Stats *),
              int64_t (*text)(const Result *, const char *, char *, size_t), uint64_t Stats::*replays,
              uint64_t Stats::*incomplete) {
  Stats st;
  if (get(idx, &st) != GSB_OK) memset(&st, 0, sizeof st);
  std::ostringstream o;
  o << " probes " << st.probes << " faults " << st.faults;
  if (replays) o << " replays " << st.*replays;
  o << " skipped " << st.skipped;
  if (incomplete) o << " incomplete " << st.*incomplete;
  return {st.probes, o.str(), text_of([&](char *buf, size_t cap) { return text(&st.last, uuid.c_str(), buf, cap); })};
}

struct Check {
  int Flags::*every;    // --probe-*-every: N > 0 turns the check on
  uint32_t option;      // the library's cadence option the flag sets
  uint64_t event;       // the event type of its conditions
  const char *label;    // in the warning
  const char *keyword;  // in dump()
  Probed (*probed)(uint32_t idx, const std::string &uuid);
  std::vector<std::pair<uint64_t, const char *>> conditions;
  const char *unknown_condition;

  const char *condition_name(uint64_t c) const {
    for (const auto &k : conditions)
      if (k.first == c) return k.second;
    return unknown_condition;
  }
};

// in the order the library runs them, which is the order they are logged and dumped in
const Check kChecks[] = {
    {&Flags::probe_link_every, GSB_OPT_LINK_PROBE_EVERY_CYCLES, GSB_EVENT_LINK, "PCIe link health", "link",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_link_stats>(i, u, gsb_link_stats_get, gsb_link_text, &gsb_link_stats::replays, nullptr);
     },
     {{GSB_LINK_CORRUPT, "corrupted data across the link"},
      {GSB_LINK_FAILED, "link probe failed"},
      {GSB_LINK_WIDTH_DEGRADED, "link width degraded"},
      {GSB_LINK_SPEED_DEGRADED, "link speed degraded"}},
     "link condition ?"},
    {&Flags::probe_copy_every, GSB_OPT_COPY_PROBE_EVERY_CYCLES, GSB_EVENT_COPY, "copy-engine health", "copy",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_copy_stats>(i, u, gsb_copy_stats_get, gsb_copy_text, nullptr, nullptr);
     },
     {{GSB_COPY_CORRUPT, "corrupted data after a DMA copy"}, {GSB_COPY_FAILED, "copy probe failed"}},
     "copy condition ?"},
    {&Flags::probe_sm_every, GSB_OPT_SM_PROBE_EVERY_CYCLES, GSB_EVENT_SM, "SM compute health", "sm",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_sm_stats>(i, u, gsb_sm_stats_get, gsb_sm_text, nullptr, &gsb_sm_stats::incomplete);
     },
     {{GSB_SM_CORRUPT, "wrong result on an SM"}, {GSB_SM_FAILED, "SM probe failed"}},
     "SM condition ?"},
    {&Flags::probe_cluster_every, GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, GSB_EVENT_CLUSTER, "SM-to-SM health", "cluster",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_cluster_stats>(i, u, gsb_cluster_stats_get, gsb_cluster_text, nullptr,
                                        &gsb_cluster_stats::incomplete);
     },
     {{GSB_CLUSTER_CORRUPT, "wrong word across the SM-to-SM network"}, {GSB_CLUSTER_FAILED, "SM-to-SM probe failed"}},
     "SM-to-SM condition ?"},
    {&Flags::probe_atomic_every, GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_ATOMIC, "L2 atomic health", "atomic",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_atomic_stats>(i, u, gsb_atomic_stats_get, gsb_atomic_text, nullptr,
                                       &gsb_atomic_stats::incomplete);
     },
     {{GSB_ATOMIC_CORRUPT, "wrong result of an L2 atomic"}, {GSB_ATOMIC_FAILED, "L2 atomic probe failed"}},
     "L2 atomic condition ?"},
    {&Flags::probe_tensor_every, GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, GSB_EVENT_TENSOR, "tensor-core format health",
     "tensor",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_tensor_stats>(i, u, gsb_tensor_stats_get, gsb_tensor_text, nullptr,
                                       &gsb_tensor_stats::incomplete);
     },
     {{GSB_TENSOR_CORRUPT, "wrong tensor-core result"}, {GSB_TENSOR_FAILED, "tensor probe failed"}},
     "tensor condition ?"},
    {&Flags::probe_sfu_every, GSB_OPT_SFU_PROBE_EVERY_CYCLES, GSB_EVENT_SFU, "SM special-function health", "sfu",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_sfu_stats>(i, u, gsb_sfu_stats_get, gsb_sfu_text, nullptr, &gsb_sfu_stats::incomplete);
     },
     {{GSB_SFU_CORRUPT, "wrong special-function result"},
      {GSB_SFU_BOUND, "MUFU result outside its envelope"},
      {GSB_SFU_FAILED, "SFU probe failed"}},
     "SFU condition ?"},
    {&Flags::probe_l1_every, GSB_OPT_L1_PROBE_EVERY_CYCLES, GSB_EVENT_L1, "L1 and constant-cache health", "l1",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_l1_stats>(i, u, gsb_l1_stats_get, gsb_l1_text, nullptr, &gsb_l1_stats::incomplete);
     },
     {{GSB_L1_CORRUPT, "wrong word through L1, texture or constant cache"}, {GSB_L1_FAILED, "L1 probe failed"}},
     "L1 condition ?"},
    {&Flags::probe_order_every, GSB_OPT_ORDER_PROBE_EVERY_CYCLES, GSB_EVENT_ORDER, "memory-ordering health", "order",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_order_stats>(i, u, gsb_order_stats_get, gsb_order_text, nullptr, &gsb_order_stats::incomplete);
     },
     {{GSB_ORDER_CORRUPT, "word read back that no writer stored"},
      {GSB_ORDER_FORBIDDEN, "outcome the memory model forbids"},
      {GSB_ORDER_LOST, "store lost after the grid barrier"},
      {GSB_ORDER_TIMEOUT, "grid barrier ran out"},
      {GSB_ORDER_FAILED, "memory-ordering probe failed"}},
     "memory-ordering condition ?"},
    {&Flags::probe_sparse_every, GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, GSB_EVENT_SPARSE, "sparse tensor-core health",
     "sparse",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_sparse_stats>(i, u, gsb_sparse_stats_get, gsb_sparse_text, nullptr,
                                       &gsb_sparse_stats::incomplete);
     },
     {{GSB_SPARSE_CORRUPT, "wrong sparse tensor-core result"}, {GSB_SPARSE_FAILED, "sparse probe failed"}},
     "sparse condition ?"},
    {&Flags::probe_shared_atomic_every, GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_SHARED_ATOMIC,
     "shared-memory atomic health", "shared-atomic",
     [](uint32_t i, const std::string &u) {
       return probed<gsb_shared_atomic_stats>(i, u, gsb_shared_atomic_stats_get, gsb_shared_atomic_text, nullptr,
                                              &gsb_shared_atomic_stats::incomplete);
     },
     {{GSB_SHARED_ATOMIC_CORRUPT, "wrong shared-memory atomic result"},
      {GSB_SHARED_ATOMIC_FAILED, "shared-memory atomic probe failed"}},
     "shared-memory atomic condition ?"},
};
constexpr size_t kNumChecks = sizeof kChecks / sizeof kChecks[0];

// ---------------------------------------------------------------- the plugin (server.go)
class Plugin {
 public:
  Plugin(const Flags &f, Kube *kube, const std::string &socket) : f_(f), kube_(kube), socket_(socket) {}
  ~Plugin() { stop(); }

  // NewNvidiaDevicePlugin (server.go:38-70): getDevices + patchGPUCount + disableCGPUIsolationOrNot
  bool build(std::string *err) {
    const bool gib = f_.memory_unit == "GiB";
    if (f_.fake_inventory > 0) {  // test hook: synthetic node, no driver needed
      static const unsigned minors[16] = {2, 3, 0, 1, 6, 7, 4, 5, 8, 9, 10, 11, 12, 13, 14, 15};
      for (int i = 0; i < f_.fake_inventory && i < 16; i++) {
        char u[64];
        snprintf(u, sizeof u, "GPU-%08x-4820-abfc-e83e-9431819757%02x", 0xfef80890u + i, i);
        uuids_.push_back(u);
        minors_.push_back(minors[i]);
      }
      slices_ = gsb_slices(183359, gib);
    } else {
      uint32_t n = 0;
      if (gsb_device_count(&n) != GSB_OK) {
        *err = last_error();
        return false;
      }
      for (uint32_t i = 0; i < n; i++) {  // getDevices (nvidia.go:53-89)
        gsb_device_info info;
        if (gsb_device_info_get(i, &info) != GSB_OK) {
          *err = last_error();  // check(err): fatal
          return false;
        }
        INFO("Deivce %s's Path is /dev/nvidia%u", info.uuid, info.minor);
        INFO("# device Memory: %llu", (unsigned long long)info.total_mib);
        uuids_.push_back(info.uuid);
        minors_.push_back(info.minor);
        if (slices_ == 0) {  // process-global gpuMemory: first GPU only (nvidia.go:70-72)
          slices_ = gsb_slices(info.total_mib, gib);
          INFO("set gpu memory: %u", slices_);
        }
      }
    }
    for (auto &u : uuids_) uuid_ptrs_.push_back(u.c_str());
    bits_.assign(((size_t)uuids_.size() * slices_ + 7) / 8, 0);
    if (!patch_gpu_count((int)uuids_.size(), err)) return false;
    if (!cgpu_disabled(&disable_cgpu_, err)) return false;
    actx_.uuids = uuid_ptrs_.data();
    actx_.minors = minors_.data();
    actx_.n_gpus = (uint32_t)uuids_.size();
    actx_.slices = slices_;
    actx_.unit_gib = gib;
    actx_.disable_cgpu_isolation = disable_cgpu_;
    return true;
  }

  // Start (server.go:106-134)
  bool start(std::string *err) {
    ::unlink(socket_.c_str());  // cleanup()
    stopping_ = false;
    if (f_.startup_memtest && f_.fake_inventory == 0) startup_memtest();
    if (f_.startup_stress_ms > 0 && f_.fake_inventory == 0) startup_stress();
    srv_.reset(new h2::Server());
    srv_->handle("/v1beta1.DevicePlugin/GetDevicePluginOptions", [](h2::Call &c, const std::string &) {
      c.send_message("", 0);
      return 0;
    });
    srv_->handle("/v1beta1.DevicePlugin/PreStartContainer", [](h2::Call &c, const std::string &) {
      c.send_message("", 0);
      return 0;
    });
    srv_->handle("/v1beta1.DevicePlugin/ListAndWatch", [this](h2::Call &c, const std::string &) { return list_and_watch(c); });
    srv_->handle("/v1beta1.DevicePlugin/Allocate", [this](h2::Call &c, const std::string &req) {
      // grpc-go decodes the request before the handler runs: bytes gogo's Unmarshal refuses never reach Allocate and
      // the call fails with INTERNAL (vendor/google.golang.org/grpc: "grpc: error unmarshalling request: ...")
      size_t ignored = 0;
      if (gsb_allocate_err_response(&actx_, (const uint8_t *)req.data(), req.size(), nullptr, 0, &ignored) == GSB_ERR_MALFORMED) {
        c.set_status_message("grpc: error unmarshalling request");
        return 13;
      }
      const std::string resp = allocate(req);
      c.send_message(resp.data(), resp.size());
      return 0;  // Allocate itself never returns a gRPC error (allocate.go: every failure is in the envs)
    });
    if (f_.fake_inventory > 0) {
      // test hook (synthetic-inventory mode only): "<uuid|-> <etype> <edata>" -> gsb_health_inject, i.e. an
      // event as the driver would deliver it
      srv_->handle("/gsbd.Test/InjectEvent", [](h2::Call &c, const std::string &req) {
        char uuid[GSB_UUID_BUFFER_SIZE] = {0};
        unsigned long long etype = 0, edata = 0;
        if (sscanf(req.c_str(), "%79s %llu %llu", uuid, &etype, &edata) != 3) return 3;
        gsb_event ev;
        memset(&ev, 0, sizeof ev);
        if (strcmp(uuid, "-") != 0) snprintf(ev.uuid, sizeof ev.uuid, "%s", uuid);
        ev.etype = etype;
        ev.edata = edata;
        gsb_health_inject(&ev);
        c.send_message("", 0);
        return 0;
      });
    }
    if (!srv_->start(socket_, err)) return false;
    health_thread_ = std::thread([this] { healthcheck(); });
    if (f_.pod_informer && !f_.query_kubelet) informer_thread_ = std::thread([this] { informer(); });
    return true;
  }

  void stop() {  // Stop (server.go:137-147)
    if (!srv_) return;
    stopping_ = true;
    if (f_.health_check) gsb_health_stop();
    {
      std::lock_guard<std::mutex> lk(hmu_);
      hcv_.notify_all();
    }
    {
      std::lock_guard<std::mutex> lk(wmu_);
      if (watch_conn_) watch_conn_->abort();
    }
    srv_->stop();
    srv_.reset();
    if (health_thread_.joinable()) health_thread_.join();
    if (informer_thread_.joinable()) informer_thread_.join();
    ::unlink(socket_.c_str());
  }

  // Register (server.go:150-169)
  bool register_with(const std::string &kubelet_sock, std::string *err) {
    uint8_t buf[512];
    const int64_t n = gsb_encode_register_request("v1beta1", kServerSockName, kResourceName, buf, sizeof buf);
    std::string resp;
    const int st = h2::unary_call(kubelet_sock, "/v1beta1.Registration/Register", std::string((char *)buf, (size_t)n),
                                  &resp, 5, err);
    if (st != 0) {
      if (err->empty()) *err = "Register returned grpc-status " + std::to_string(st);
      return false;
    }
    return true;
  }

 private:
  // ---- node helpers (podmanager.go:59-99)
  bool patch_gpu_count(int count, std::string *err) {
    json::Value node;
    if (!kube_->call("GET", "/api/v1/nodes/" + kube_->node_name, "", "", &node, err)) return false;
    if (const json::Value *cap = node.path({"status", "capacity", kResourceCount}))
      if (quantity_value(*cap) == (uint64_t)count) {
        INFO("No need to update Capacity %s", kResourceCount);
        return true;
      }
    char body[256];
    snprintf(body, sizeof body, "{\"status\":{\"allocatable\":{\"%s\":\"%d\"},\"capacity\":{\"%s\":\"%d\"}}}",
             kResourceCount, count, kResourceCount, count);
    if (!kube_->call("PATCH", "/api/v1/nodes/" + kube_->node_name + "/status", body,
                     "application/strategic-merge-patch+json", nullptr, err)) {
      INFO("Failed to update Capacity %s.", kResourceCount);
      return false;
    }
    INFO("Updated Capacity %s successfully.", kResourceCount);
    return true;
  }
  bool cgpu_disabled(int *out, std::string *err) {
    json::Value node;
    if (!kube_->call("GET", "/api/v1/nodes/" + kube_->node_name, "", "", &node, err)) return false;
    const json::Value *l = node.path({"metadata", "labels", kEnvNodeLabelForDisableCGPU});
    *out = l && l->str() == "true";
    return true;
  }

  std::string list_bytes(const std::vector<uint8_t> &bits) {
    bool any = false;
    for (uint8_t b : bits) any = any || b;
    const int64_t need = gsb_encode_list_and_watch(uuid_ptrs_.data(), (uint32_t)uuids_.size(), slices_,
                                                   any ? bits.data() : nullptr, nullptr, 0);
    std::string out((size_t)(need > 0 ? need : 0), '\0');
    if (need > 0)
      gsb_encode_list_and_watch(uuid_ptrs_.data(), (uint32_t)uuids_.size(), slices_, any ? bits.data() : nullptr,
                                (uint8_t *)&out[0], out.size());
    return out;
  }

  // ListAndWatch (server.go:172-185). The node's health state (bits_) is written by the PRODUCER of an event
  // (mark), never by a stream: an event raised while no stream is attached — a start-up walk fault, a NOT_SUPPORTED
  // registration, a probe fault during a kubelet reconnect — is in the first frame of the next stream. (The
  // reference's unbuffered channel gets the same result by blocking the producer until a stream takes the event.)
  // Each stream replays the events it has not yet sent onto its own copy, which is what makes the reference-exact
  // mode (one resend per fake device, each frame the state after that event) independent of how far a stream lags.
  int list_and_watch(h2::Call &c) {
    std::string frame;
    size_t cursor;
    std::vector<uint8_t> mine;
    {
      std::lock_guard<std::mutex> lk(hmu_);
      mine = bits_;
      frame = list_bytes(mine);
      cursor = pending_.size();
    }
    if (!c.send_message(frame.data(), frame.size())) return 1;
    for (;;) {
      std::vector<std::string> frames;
      {
        std::unique_lock<std::mutex> lk(hmu_);
        while (cursor >= pending_.size() && !stopping_ && !c.cancelled()) hcv_.wait_for(lk, std::chrono::milliseconds(250));
        if (stopping_ || c.cancelled()) return 0;  // `case <-m.stop: return nil`
        for (; cursor < pending_.size(); cursor++) {
          apply(&mine, pending_[cursor]);  // d.Health = Unhealthy (server.go:181)
          if (!f_.coalesce_health) frames.push_back(list_bytes(mine));  // the reference's stream: one resend per event
        }
        if (f_.coalesce_health) frames.push_back(list_bytes(mine));
      }
      for (auto &fr : frames)
        if (!c.send_message(fr.data(), fr.size())) return 1;
    }
  }

  static void apply(std::vector<uint8_t> *bits, long long e) {
    if (e >= 0) {
      (*bits)[(size_t)e >> 3] |= (uint8_t)(1u << (e & 7));
    } else {  // optional recovery (not in the reference): ~e is the device index
      const size_t i = (size_t)~e;
      (*bits)[i >> 3] &= (uint8_t)~(1u << (i & 7));
    }
  }

  void mark(const std::string &uuid, bool healthy) {  // watchXIDs' fan-out (nvidia.go:138-150) + m.unhealthy
    std::lock_guard<std::mutex> lk(hmu_);
    for (size_t g = 0; g < uuids_.size(); g++)
      if (uuid.empty() || uuids_[g] == uuid)
        for (uint32_t j = 0; j < slices_; j++) {
          const long long i = (long long)(g * slices_ + j);
          const long long e = healthy ? ~i : i;
          apply(&bits_, e);
          pending_.push_back(e);
        }
    hcv_.notify_all();
  }
  void mark_unhealthy(const std::string &uuid) { mark(uuid, false); }

  // Probe memory. Default (--probe-arena-mib 0): none is held — every probe cycle allocates its window, walks it and
  // frees it (transient window), so the slices the node advertises are not oversold by the plugin itself. A standing
  // arena (--probe-arena-mib N) rotates the window over N MiB the plugin keeps for its lifetime: wider coverage, but
  // that HBM is then NOT available to tenants although ListAndWatch still advertises it (the reference's count is
  // kept bit-exact, nvidia.go:73-85) — the log line below says how much. Neither takes the last
  // --probe-keep-free-mib of free HBM, the start-up walk included.
  void setup_probe_arenas() {
    const uint64_t keep_free = (uint64_t)f_.probe_keep_free_mib << 20;
    gsb_set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, keep_free);
    for (uint32_t i = 0; i < uuids_.size(); i++) {
      uint64_t nbytes = 0;
      if (f_.startup_full_walk) {
        if (gsb_arena_create(i, 0, keep_free, &nbytes) == GSB_OK) {
          gsb_probe_cfg cfg;
          memset(&cfg, 0, sizeof cfg);
          cfg.op = GSB_OP_VERIFY;
          cfg.flags = GSB_PROBE_TIMED | GSB_PROBE_SEED_TABLE;
          gsb_probe_result r;
          gsb_probe(i, &cfg, &r);
          INFO("start-up walk of %s: %llu bytes actually allocatable (%llu MiB left free for tenants), %llu mismatching words, %.1f ms",
               uuids_[i].c_str(), (unsigned long long)nbytes, (unsigned long long)f_.probe_keep_free_mib,
               (unsigned long long)r.mismatch_words, r.kernel_ns / 1e6);
          if (r.status != GSB_OK || r.mismatch_words) mark_unhealthy(uuids_[i]);
          gsb_arena_destroy(i);
        } else {
          WARN("start-up walk of %s skipped: %s", uuids_[i].c_str(), last_error().c_str());
        }
      }
      if (f_.probe_arena_mib > 0) {
        // the start-up memtest's standing arena, refilled, serves as it is (unless the full walk replaced it)
        if ((f_.startup_memtest && !f_.startup_full_walk && gsb_arena_bytes(i, &nbytes) == GSB_OK) ||
            gsb_arena_create(i, (uint64_t)f_.probe_arena_mib << 20, keep_free, &nbytes) == GSB_OK)
          WARN("standing probe arena on %s: %llu bytes held by the plugin and NOT available to tenants "
               "(aliyun.com/gpu-mem still advertises %u slices)", uuids_[i].c_str(), (unsigned long long)nbytes, slices_);
        else
          WARN("no probe arena on %s: %s (falling back to transient windows)", uuids_[i].c_str(), last_error().c_str());
      } else {
        INFO("probe of %s: transient %d MiB window per cycle, nothing held between cycles", uuids_[i].c_str(),
             f_.probe_window_mib);
      }
    }
  }

  // --startup-memtest (not in the reference): a March C- run on every GPU before the plugin serves or registers, so a
  // GPU it faults is Unhealthy in the first ListAndWatch frame. With --probe-arena-mib it tests the standing arena and
  // leaves it, refilled, to the prober; otherwise all allocatable HBM but the last --probe-keep-free-mib, given back.
  void startup_memtest() {
    const uint64_t keep_free = (uint64_t)f_.probe_keep_free_mib << 20;
    gsb_set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, keep_free);
    gsb_set_option(GSB_OPT_ECC_HEALTH, f_.health_ecc ? 1 : 0);
    const bool prober_keeps_arena = f_.health_check && f_.probe_period_ms > 0;
    for (uint32_t i = 0; i < uuids_.size(); i++) {
      uint64_t nbytes = 0;
      const bool standing = f_.probe_arena_mib > 0 &&
                            gsb_arena_create(i, (uint64_t)f_.probe_arena_mib << 20, keep_free, &nbytes) == GSB_OK;
      if (f_.probe_arena_mib > 0 && !standing)
        WARN("memtest of %s: no standing arena (%s): testing a transient window", uuids_[i].c_str(), last_error().c_str());
      gsb_memtest_cfg cfg;
      memset(&cfg, 0, sizeof cfg);
      gsb_memtest_result r;
      const int rc = gsb_memtest(i, &cfg, &r);
      if (standing && !prober_keeps_arena) gsb_arena_destroy(i);
      if (r.n_elements == 0) {  // nothing was tested (no memory to allocate, no usable device)
        WARN("memtest of %s skipped: %s", uuids_[i].c_str(), last_error().c_str());
        continue;
      }
      bool bad = rc != GSB_OK;
      for (uint32_t k = 0; k < r.n_elements; k++) bad = bad || r.elements[k].mismatch_words != 0;
      const int64_t need = gsb_memtest_text(&r, uuids_[i].c_str(), nullptr, 0);
      std::string line((size_t)(need > 0 ? need : 0), '\0');
      const int64_t n = need > 0 ? gsb_memtest_text(&r, uuids_[i].c_str(), &line[0], line.size()) : 0;
      line.resize(n > 0 ? (size_t)n : 0);
      if (!bad) {
        INFO("%s", line.c_str());
        continue;
      }
      WARN("%s: marking it unhealthy", line.c_str());
      const std::string first = fault_report_line(i, GSB_FAULT_REPORT_FIRST);
      if (!first.empty()) WARN("%s", first.c_str());
      mark_unhealthy(uuids_[i]);
    }
  }

  // --startup-stress-ms N (not in the reference): N ms of full-rate, bit-checked tensor-core load on every SM of every
  // GPU before the plugin serves or registers (after --startup-memtest), so a GPU that computes a wrong product under
  // load is Unhealthy in the first ListAndWatch frame. The GPUs run at once, one thread each.
  void startup_stress() {
    gsb_set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, (uint64_t)f_.probe_keep_free_mib << 20);
    std::vector<gsb_stress_result> rs(uuids_.size());
    std::vector<int> rcs(uuids_.size(), GSB_OK);
    std::vector<std::thread> ts;
    for (uint32_t i = 0; i < uuids_.size(); i++)
      ts.emplace_back([this, i, &rs, &rcs] {
        gsb_stress_cfg cfg;
        memset(&cfg, 0, sizeof cfg);
        cfg.duration_ms = (uint32_t)f_.startup_stress_ms;
        rcs[i] = gsb_sm_stress(i, &cfg, &rs[i]);
      });
    for (std::thread &t : ts) t.join();
    for (uint32_t i = 0; i < uuids_.size(); i++) {
      const gsb_stress_result &r = rs[i];
      if (r.slices == 0) {  // nothing ran (no memory to allocate, no usable device, a bad duration)
        WARN("SM stress of %s skipped: %s", uuids_[i].c_str(), gsb_strerror(rcs[i]));
        continue;
      }
      const int64_t need = gsb_stress_text(&r, uuids_[i].c_str(), nullptr, 0);
      std::string line((size_t)(need > 0 ? need : 0), '\0');
      const int64_t n = need > 0 ? gsb_stress_text(&r, uuids_[i].c_str(), &line[0], line.size()) : 0;
      line.resize(n > 0 ? (size_t)n : 0);
      if (gsb_stress_conditions(&r) == 0) {
        INFO("%s", line.c_str());
        continue;
      }
      WARN("%s: marking it unhealthy", line.c_str());
      mark_unhealthy(uuids_[i]);
    }
  }

  // healthcheck + watchXIDs (server.go:203-221, nvidia.go:100-152) over gsb_health_wait
  void healthcheck() {
    if (!f_.health_check) return;
    if (f_.fake_inventory == 0) {
      if (f_.probe_period_ms > 0) setup_probe_arenas();
      gsb_health_set_recovery((uint32_t)f_.health_recovery_cycles);
      gsb_set_option(GSB_OPT_WATCHDOG_MS, (uint64_t)f_.probe_watchdog_ms);
      gsb_set_option(GSB_OPT_INVENTORY_REFRESH_MS, (uint64_t)f_.inventory_refresh_ms);
      gsb_set_option(GSB_OPT_SWEEP_EVERY_CYCLES, (uint64_t)(f_.probe_sweep_every > 0 ? f_.probe_sweep_every : 0));
      gsb_set_option(GSB_OPT_ECC_HEALTH, f_.health_ecc ? 1 : 0);
      for (const Check &c : kChecks) gsb_set_option(c.option, (uint64_t)(f_.*c.every > 0 ? f_.*c.every : 0));
      if (gsb_health_start((uint32_t)f_.probe_period_ms, (uint64_t)f_.probe_window_mib << 20) != GSB_OK) {
        // nvidia.go:114-116: a registration error other than "Not Supported" is log.Fatalf
        logf('F', "Fatal error: %s", last_error().c_str());
        log_flush();
        _exit(255);
      }
    }
    std::vector<uint64_t> sweeps_seen(uuids_.size(), 0);
    std::vector<uint64_t> probes_seen[kNumChecks];
    for (auto &seen : probes_seen) seen.assign(uuids_.size(), 0);
    while (!stopping_) {
      gsb_event ev;
      const int rc = gsb_health_wait(5000, &ev);  // nvidia.go:126
      if (f_.fake_inventory == 0 && f_.probe_sweep_every > 0) {  // what each sweep found actually allocatable
        for (uint32_t i = 0; i < uuids_.size(); i++) {
          gsb_health_stats st;
          if (gsb_health_stats_get(i, &st) == GSB_OK && st.sweeps > sweeps_seen[i]) {
            sweeps_seen[i] = st.sweeps;
            INFO("sweep %llu of %s: %llu bytes actually allocatable walked clean-or-not in %.1f ms (%llu faults so far)",
                 (unsigned long long)st.sweeps, uuids_[i].c_str(), (unsigned long long)st.last_sweep_bytes,
                 st.last_sweep_ns / 1e6, (unsigned long long)st.faults);
          }
        }
      }
      for (size_t k = 0; k < kNumChecks; k++) {  // each GPU's most recent probe of every check that is on, once
        if (f_.fake_inventory != 0 || f_.*kChecks[k].every <= 0) continue;
        for (uint32_t i = 0; i < uuids_.size(); i++) {
          const Probed p = kChecks[k].probed(i, uuids_[i]);
          if (p.probes > probes_seen[k][i]) {
            probes_seen[k][i] = p.probes;
            INFO("%s", p.line.c_str());
          }
        }
      }
      if (rc != GSB_OK) continue;                 // timeout / stopped
      if (ev.etype == GSB_EVENT_INVENTORY) {  // the low-rate NVML refresh no longer agrees with what is advertised
        WARN("inventory of %s changed under the plugin (%s): marking it unhealthy; SIGHUP re-reads it", ev.uuid,
             ev.edata == GSB_INVENTORY_IDENTITY_CHANGED ? "identity" : "total memory");
        mark_unhealthy(ev.uuid);
        continue;
      }
      if (ev.etype == GSB_EVENT_ECC && f_.health_ecc) {  // not in the reference: what the GPU records about its HBM
        WARN("ECC health of %s: %s: marking it unhealthy", ev.uuid, ecc_condition_name(ev.edata));
        WARN("%s", ecc_status_line(ev.uuid).c_str());
        mark_unhealthy(ev.uuid);
        continue;
      }
      const Check *check = nullptr;
      for (const Check &c : kChecks)
        if (ev.etype == c.event && f_.*c.every > 0) check = &c;
      if (check) {
        WARN("%s of %s: %s: marking it unhealthy", check->label, ev.uuid, check->condition_name(ev.edata));
        WARN("%s", check->probed(gpu_index(ev.uuid), ev.uuid).line.c_str());
        mark_unhealthy(ev.uuid);
        continue;
      }
      if (ev.etype != GSB_EVENT_XID && ev.etype != GSB_EVENT_PROBE) continue;   // nvidia.go:127-129
      if (ev.etype == GSB_EVENT_XID && gsb_xid_is_benign(ev.edata)) continue;  // nvidia.go:134-136
      if (ev.etype == GSB_EVENT_PROBE && ev.edata == GSB_PROBE_RECOVERED) {  // not in the reference: flag-gated
        if (f_.health_recovery_cycles > 0 && ev.uuid[0]) mark(ev.uuid, true);
        continue;
      }
      if (ev.etype == GSB_EVENT_PROBE && ev.edata == GSB_PROBE_FAULT_MISMATCH) {  // not in the reference: the evidence
        for (uint32_t i = 0; i < uuids_.size(); i++) {
          if (uuids_[i] != ev.uuid) continue;
          const std::string line = fault_report_line(i, GSB_FAULT_REPORT_FIRST);
          if (!line.empty()) WARN("%s", line.c_str());
        }
      }
      mark_unhealthy(ev.uuid);
    }
    if (f_.fake_inventory == 0) gsb_health_stop();
  }

  // ---- pending-pod informer (SURVEY.md §8(f) row 2, second step): LIST once, then follow the apiserver's watch
  // stream so the table is current without a LIST per call or per TTL. Optimistic like the TTL cache: a request
  // that finds no candidate still re-LISTs, a failed PATCH forces a resync. Falls back to the TTL cache whenever
  // the watch cannot be established (synced_ == false).
  // 1 s, 2 s, 4 s ... 64 s between attempts while the apiserver refuses the LIST or the watch (the TTL path serves
  // meanwhile); a stream that delivered anything resets it
  void backoff(int *failures) {
    const int ticks = 20 << std::min(*failures, 6);
    if (*failures < 6) (*failures)++;
    const bool resync_at_entry = resync_;  // a resync requested DURING the wait cuts it short, a pending one does not
    for (int i = 0; i < ticks && !stopping_ && (resync_at_entry || !resync_); i++)
      std::this_thread::sleep_for(std::chrono::milliseconds(50));
  }
  void informer() {
    int failures = 0;
    const std::string sel = "fieldSelector=spec.nodeName%3D" + kube_->node_name + "%2Cstatus.phase%3DPending";
    while (!stopping_) {
      std::string err, rv;
      json::Value list;
      const auto list_started = std::chrono::steady_clock::now();
      if (!kube_->call("GET", "/api/v1/pods?" + sel, "", "", &list, &err)) {
        backoff(&failures);
        continue;
      }
      if (const json::Value *v = list.path({"metadata", "resourceVersion"})) rv = v->str();
      {
        std::lock_guard<std::mutex> lk(amu_);
        uint64_t rv_num = 0;
        parse_uint64(rv, &rv_num);
        if (!(table_.valid && rv_num && rv_num < table_.list_rv)) {  // an Allocate's own LIST may already be newer
          build_table(list, kube_->node_name, false, &table_);
          reconcile_claims(list_started);
          table_.stamp = std::chrono::steady_clock::now();
          table_.valid = true;
        }
        resync_ = false;
      }
      // the server ends the stream itself (timeoutSeconds) before our read timeout would: a quiet node re-lists every
      // 4.5 min, a dead peer is noticed after 5; bookmarks keep resourceVersion fresh on quiet streams
      std::unique_ptr<http::Conn> conn = kube_->api.open_stream(
          "/api/v1/pods?watch=true&allowWatchBookmarks=true&timeoutSeconds=270&" + sel + "&resourceVersion=" + rv, 300, &err);
      if (!conn) {
        synced_ = false;
        backoff(&failures);
        continue;
      }
      {
        std::lock_guard<std::mutex> lk(wmu_);
        watch_conn_ = conn.get();
        // a stop or a resync request that arrived while the stream was being opened found nothing to abort
        if (stopping_ || resync_) conn->abort();
      }
      int status = 0;
      size_t events = 0;
      const auto opened = std::chrono::steady_clock::now();
      conn->read_stream(&status, [&](int st) { synced_ = st == 200; },  // stream is up: table kept current from here on
                        [&](const std::string &line) -> bool {
        if (status >= 400) return false;
        json::Value ev;
        if (!json::parse(line, &ev)) return true;
        const json::Value *type = ev.get("type"), *obj = ev.get("object");
        if (!type || !obj) return true;
        if (type->str() == "ERROR") return false;  // e.g. 410 Gone (resourceVersion too old): start over from a LIST
        apply_event(type->str(), *obj);
        events++;
        return !stopping_ && !resync_;
      });
      {
        std::lock_guard<std::mutex> lk(wmu_);
        watch_conn_ = nullptr;
      }
      synced_ = false;  // until the next LIST + watch are in place the TTL path answers
      // a stream that was refused (4xx), never answered, or was closed at once without delivering anything counts as
      // a failure; one that worked resets the backoff
      const bool worked = status == 200 && (events > 0 || std::chrono::steady_clock::now() - opened > std::chrono::seconds(5));
      if (worked || resync_) failures = 0;
      else backoff(&failures);
    }
    synced_ = false;
  }

  void apply_event(const std::string &type, const json::Value &obj) {
    PodRec r;
    gsb_pod g;
    pod_row(obj, kube_->node_name, &r, &g);
    std::lock_guard<std::mutex> lk(amu_);
    // the stream is ordered, but the table can be NEWER than the stream (an Allocate that found no candidate
    // rebuilt it from its own LIST): an event at or below that LIST's resourceVersion, or older than the row it
    // touches, would move the table back in time
    if (r.rv && r.rv <= table_.list_rv) return;
    auto row = table_.by_uid.find(r.uid);
    if (row != table_.by_uid.end() && r.rv && table_.recs[row->second]->rv > r.rv) return;
    if (type == "DELETED") {
      claimed_.erase(r.uid);
      table_.remove(r.uid);
    } else if (type == "ADDED" || type == "MODIFIED") {
      if (claimed_.count(r.uid)) g.assigned_is_false = 0;  // handed out by this daemon: never a candidate again
      table_.upsert(std::move(r), g);
    } else {
      return;  // BOOKMARK: nothing to apply
    }
    table_.stamp = std::chrono::steady_clock::now();
  }

  // ---- Allocate
  bool load_pods(std::string *err) {
    const auto list_started = std::chrono::steady_clock::now();
    json::Value list;
    bool pending_only = false;
    bool ok = false;
    if (f_.query_kubelet) {  // podmanager.go:125-140: 1 try + 8 retries of the kubelet, then the apiserver
      for (int attempt = 0; attempt <= 8 && !ok; attempt++) {
        http::Response r;
        std::string e;
        if (kubelet_.request("GET", "/pods/", "", "", &r, &e) && r.status == 200 && json::parse(r.body, &list)) {
          PodTable probe;
          build_table(list, kube_->node_name, true, &probe);
          if (!probe.pods.empty()) {
            ok = true;
            pending_only = true;
            break;
          }
        }
        if (attempt < 8) {
          WARN("failed to get pending pod list, retry");
          std::this_thread::sleep_for(std::chrono::milliseconds(100));
        }
      }
      if (!ok) WARN("not found from kubelet /pods api, start to list apiserver");
    }
    if (!ok) {  // podmanager.go:142-160: 1 try + 3 retries, 1 s apart
      const std::string path = "/api/v1/pods?fieldSelector=spec.nodeName%3D" + kube_->node_name + "%2Cstatus.phase%3DPending";
      for (int attempt = 0; attempt < 4 && !ok; attempt++) {
        ok = kube_->call("GET", path, "", "", &list, err);
        if (!ok && attempt < 3) std::this_thread::sleep_for(std::chrono::milliseconds(retry_sleep_ms_));
      }
      if (!ok) {
        *err = "failed to get Pods assigned to node " + kube_->node_name;
        return false;
      }
    }
    build_table(list, kube_->node_name, pending_only, &table_);
    reconcile_claims(list_started);
    table_.stamp = std::chrono::steady_clock::now();
    table_.valid = true;
    return true;
  }
  // A LIST is a snapshot that can pre-date a PATCH still in flight (the lock is not held across the PATCH), and a
  // watch event can be older than the table. So a pod handed out by this daemon is never a candidate again, in any
  // rebuilt or updated table, for as long as it is a pending pod of this node: the claim is dropped only when the
  // PATCH fails, when the pod is DELETED on the watch, or when a LIST issued AFTER the claim no longer contains it.
  // Caller holds amu_.
  void reconcile_claims(std::chrono::steady_clock::time_point list_started) {
    for (auto it = claimed_.begin(); it != claimed_.end();) {
      auto row = table_.by_uid.find(it->first);
      if (row == table_.by_uid.end()) {
        if (it->second < list_started) it = claimed_.erase(it);  // gone from the pending set for good
        else ++it;                                               // the snapshot may simply pre-date the pod
        continue;
      }
      table_.pods[row->second].assigned_is_false = 0;
      ++it;
    }
  }
  bool cache_fresh() const {
    if (synced_ && table_.valid && !resync_) return true;  // kept current by the watch stream
    return table_.valid && f_.pod_cache_ttl > 0 &&
           std::chrono::duration<double>(std::chrono::steady_clock::now() - table_.stamp).count() < f_.pod_cache_ttl;
  }
  int decide(const std::string &req, std::string *resp, int32_t *pod_index, uint32_t *pod_req) {
    resp->resize(1 << 16);
    size_t n = 0;
    actx_.pods_unique = table_.unique;  // a uid-keyed table: podmanager.go's dedupe would be a no-op
    const int kind = gsb_allocate(&actx_, table_.pods.data(), (uint32_t)table_.pods.size(), (const uint8_t *)req.data(),
                                  req.size(), (uint8_t *)&(*resp)[0], resp->size(), &n, pod_index, pod_req);
    resp->resize(kind > 0 ? n : 0);
    return kind;
  }
  std::string err_response(const std::string &req) {  // buildErrResponse (allocate.go:24-39)
    std::string out(1 << 16, '\0');
    size_t n = 0;
    if (gsb_allocate_err_response(&actx_, (const uint8_t *)req.data(), req.size(), (uint8_t *)&out[0], out.size(), &n) != GSB_OK)
      n = 0;
    out.resize(n);
    return out;
  }

  std::string allocate(const std::string &req) {  // allocate.go:42-198
    // --serialize-allocate: m.Lock(); defer m.Unlock() around the whole call, PATCH included (allocate.go:59-60)
    std::unique_lock<std::mutex> whole(ref_mu_, std::defer_lock);
    if (f_.serialize_allocate) whole.lock();
    VLOG(1, "----Allocating GPU for gpu mem is started----");
    std::string resp, name, ns, err, claimed_uid;
    int32_t pidx = -1;
    uint32_t pod_req = 0;
    int kind;
    {
      std::lock_guard<std::mutex> lk(amu_);  // held for list + decide + claim, not for the PATCH
      const bool was_cached = cache_fresh();
      if (!was_cached && !load_pods(&err)) {
        table_.valid = false;
        INFO("invalid allocation requst: Failed to find candidate pods due to %s", err.c_str());
        return err_response(req);
      }
      kind = decide(req, &resp, &pidx, &pod_req);
      // the cache may be older than the pod being started: anything but a match (the error response AND, on a
      // one-GPU node, the single-GPU shortcut of allocate.go:151-177, which would otherwise answer without ever
      // PATCHing the pod the reference would have found by LISTing) is re-decided on a fresh LIST
      if (kind != GSB_ALLOC_MATCHED && kind > 0 && was_cached) {
        if (!load_pods(&err)) {
          table_.valid = false;
          return err_response(req);
        }
        kind = decide(req, &resp, &pidx, &pod_req);
      }
      if (kind < 0) {
        WARN("Allocate: %s", last_error().c_str());
        return "";
      }
      VLOG(1, "RequestPodGPUs: %u", pod_req);
      if (kind == GSB_ALLOC_MATCHED) {
        name = table_.recs[pidx]->name;
        ns = table_.recs[pidx]->ns;
        table_.pods[pidx].assigned_is_false = 0;  // claimed: hidden from the next request
        claimed_uid = table_.recs[pidx]->uid;
        claimed_[claimed_uid] = std::chrono::steady_clock::now();
      }
    }
    if (kind == GSB_ALLOC_MATCHED) {
      VLOG(1, "Found Assumed GPU shared Pod %s in ns %s with GPU Memory %u", name.c_str(), ns.c_str(), pod_req);
      char body[256];
      timespec ts;
      clock_gettime(CLOCK_REALTIME, &ts);
      gsb_patch_assigned_body((uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec, body, sizeof body);
      const std::string path = "/api/v1/namespaces/" + ns + "/pods/" + name;
      const char *ct = "application/strategic-merge-patch+json";
      bool ok = kube_->call("PATCH", path, body, ct, nullptr, &err);
      if (!ok && err == kOptimisticLockErrorMsg) ok = kube_->call("PATCH", path, body, ct, nullptr, &err);  // one retry
      if (!ok) {
        WARN("Failed due to %s", err.c_str());
        std::lock_guard<std::mutex> lk(amu_);
        table_.valid = false;  // drop the cache: it no longer reflects the apiserver
        claimed_.erase(claimed_uid);  // this pod is a candidate again; other claims in flight stay
        resync_ = true;        // and make the informer start over from a fresh LIST
        {
          std::lock_guard<std::mutex> wl(wmu_);
          if (watch_conn_) watch_conn_->abort();
        }
        return err_response(req);
      }
      VLOG(1, "----Allocating GPU for gpu mem for %s is ended----", name.c_str());
    } else if (kind == GSB_ALLOC_ERR_RESPONSE) {
      WARN("invalid allocation requst: request GPU memory %u can't be satisfied.", pod_req);
    }
    return resp;
  }

 public:
  void configure_kubelet(std::string *err) {
    std::string token = f_.token;
    if (f_.client_cert.empty() && f_.client_key.empty() && token.empty())
      token = read_file("/var/run/secrets/kubernetes.io/serviceaccount/token");  // main.go:29-36
    http::Client::TlsExtra extra;  // main.go:40-46: TLSClientConfig{CertFile, KeyFile}; server verification off
    extra.cert_file = f_.client_cert;
    extra.key_file = f_.client_key;
    kubelet_.configure(f_.kubelet_scheme + "://" + f_.kubelet_address + ":" + std::to_string(f_.kubelet_port), token, "",
                       true, f_.timeout, err, &extra);
  }
  void set_retry_sleep_ms(int ms) { retry_sleep_ms_ = ms; }
  size_t n_gpus() const { return uuids_.size(); }
  // gsb_fault_report_text of GPU idx's FIRST / LAST report; empty when there is none (or no driver: --fake-inventory)
  std::string fault_report_line(uint32_t idx, uint32_t which) {
    gsb_fault_report r;
    if (idx >= uuids_.size() || gsb_fault_report_get(idx, which, &r) != GSB_OK || !r.valid) return "";
    return text_of([&](char *buf, size_t cap) { return gsb_fault_report_text(&r, uuids_[idx].c_str(), buf, cap); });
  }
  static const char *ecc_condition_name(uint64_t c) {
    switch (c) {
      case GSB_ECC_REMAP_PENDING: return "row remap pending (the GPU needs a reset)";
      case GSB_ECC_REMAP_FAILURE: return "row remap failure (no spare rows left)";
      case GSB_ECC_UNCORRECTED: return "uncorrected ECC error";
      default: return "ECC condition ?";
    }
  }
  // the GPU's place in uuids_; uuids_.size() when it has none
  uint32_t gpu_index(const std::string &uuid) const {
    uint32_t i = 0;
    while (i < uuids_.size() && uuids_[i] != uuid) i++;
    return i;
  }
  // gsb_ecc_status_text of GPU `uuid`'s live status; every field "unknown" when it cannot be read (--fake-inventory)
  std::string ecc_status_line(const std::string &uuid) {
    gsb_ecc_status st;
    memset(&st, 0, sizeof st);
    if (gsb_ecc_status_get(gpu_index(uuid), &st) != GSB_OK) memset(&st, 0, sizeof st);
    return text_of([&](char *buf, size_t cap) { return gsb_ecc_status_text(&st, uuid.c_str(), buf, cap); });
  }
  std::string dump() {
    std::lock_guard<std::mutex> lk(hmu_);
    std::ostringstream o;
    o << "gsbd state\nsocket " << socket_ << "\ngpus " << uuids_.size() << " slices " << slices_ << "\n";
    for (size_t g = 0; g < uuids_.size(); g++) {
      size_t bad = 0;
      for (uint32_t j = 0; j < slices_; j++) bad += (bits_[(g * slices_ + j) >> 3] >> ((g * slices_ + j) & 7)) & 1;
      o << uuids_[g] << " minor " << minors_[g] << " unhealthy_slices " << bad << "\n";
    }
    for (size_t g = 0; g < uuids_.size(); g++) {  // HBM fault reports: only GPUs that have one
      const std::string first = fault_report_line((uint32_t)g, GSB_FAULT_REPORT_FIRST);
      if (!first.empty()) o << "fault first " << first << "\n";
      const std::string last = fault_report_line((uint32_t)g, GSB_FAULT_REPORT_LAST);
      if (!last.empty()) o << "fault last " << last << "\n";
    }
    if (f_.health_ecc) {  // per GPU: what the prober attributed, then the live status
      for (size_t g = 0; g < uuids_.size(); g++) {
        o << "ecc " << uuids_[g];
        gsb_ecc_stats es;
        if (gsb_ecc_stats_get((uint32_t)g, &es) == GSB_OK)
          o << " walks " << es.cycles << " bytes_walked " << es.bytes_walked << " corrected_in_walks "
            << es.corrected_in_walks << " uncorrected_in_walks " << es.uncorrected_in_walks << " corrected_between_walks "
            << es.corrected_between_walks << " last_corrected " << es.last_corrected << " at 0x" << std::hex
            << es.last_window_offset << " +0x" << es.last_window_bytes << std::dec << ";";
        o << " " << ecc_status_line(uuids_[g]) << "\n";
      }
    }
    for (const Check &c : kChecks) {  // per GPU and check that is on: the probes so far, then the most recent one's line
      if (f_.*c.every <= 0) continue;
      for (size_t g = 0; g < uuids_.size(); g++) {
        const Probed p = c.probed((uint32_t)g, uuids_[g]);
        o << c.keyword << " " << uuids_[g] << p.counters << "; " << p.line << "\n";
      }
    }
    o << "health events queued " << pending_.size() << "\n";
    return o.str();
  }

 private:
  Flags f_;
  Kube *kube_;
  http::Client kubelet_;
  std::string socket_;
  std::vector<std::string> uuids_;
  std::vector<const char *> uuid_ptrs_;
  std::vector<uint32_t> minors_;
  uint32_t slices_ = 0;
  int disable_cgpu_ = 0;
  gsb_allocate_ctx actx_;
  std::unique_ptr<h2::Server> srv_;
  std::atomic<bool> stopping_{false};
  std::thread health_thread_;
  // health: bitset over fake devices + event log with per-stream cursors (never blocks without a stream)
  std::mutex hmu_;
  std::condition_variable hcv_;
  std::vector<uint8_t> bits_;
  std::vector<long long> pending_;  // i >= 0: device i Unhealthy; ~i: device i Healthy again (recovery flag)
  // Allocate
  std::mutex amu_;
  PodTable table_;
  std::thread informer_thread_;
  std::atomic<bool> synced_{false}, resync_{false};
  std::unordered_map<std::string, std::chrono::steady_clock::time_point> claimed_;  // uid -> when it was handed out
  std::mutex wmu_;
  http::Conn *watch_conn_ = nullptr;
  int retry_sleep_ms_ = 1000;
  std::mutex ref_mu_;  // --serialize-allocate only
};

}  // namespace

// ---------------------------------------------------------------- main + manager loop (gpumanager.go:33-111)
int main(int argc, char **argv) {
  Flags f;
  if (const int rc = parse_flags(argc, argv, &f)) return rc - 1;
  if (f.memory_unit != "GiB" && f.memory_unit != "MiB") {  // translatememoryUnits (main.go:67-78)
    WARN("Unsupported memory unit: %s, use memoryUnit Gi as default", f.memory_unit.c_str());
    f.memory_unit = "GiB";
  }
  if (f.fake_inventory > 0) {
    // test hook only: a synthetic node so the RPC surface can be exercised on a GPU-less builder. It never runs a
    // probe and never stands in for a GPU; refuse it unless the caller says so twice.
    const char *ok = getenv("GSBD_ALLOW_FAKE_INVENTORY");
    if (!ok || strcmp(ok, "1") != 0) {
      fprintf(stderr, "--fake-inventory is a test hook; set GSBD_ALLOW_FAKE_INVENTORY=1 to use it\n");
      return 2;
    }
    WARN("TEST MODE: advertising %d synthetic GPUs, no driver, no HBM probe", f.fake_inventory);
  }
  VLOG(1, "Start gpushare device plugin");
  const char *pd = getenv("GPUSHARE_PLUGIN_DIR");
  std::string plugin_dir = pd ? pd : kDevicePluginPath;
  if (plugin_dir.back() != '/') plugin_dir += '/';
  const char *dd = getenv("GPUSHARE_DUMP_DIR");
  const std::string dump_dir = dd ? dd : "/etc/kubernetes/";

  // signals are consumed through a signalfd by the manager loop (newOSWatcher, watchers.go:27-32)
  sigset_t mask;
  sigemptyset(&mask);
  sigaddset(&mask, SIGHUP);
  sigaddset(&mask, SIGINT);
  sigaddset(&mask, SIGTERM);
  sigaddset(&mask, SIGQUIT);
  pthread_sigmask(SIG_BLOCK, &mask, nullptr);
  {  // one fd per connection: lift the soft limit to the hard one (a container's default soft limit can be 1024)
    rlimit rl;
    if (getrlimit(RLIMIT_NOFILE, &rl) == 0 && rl.rlim_cur < rl.rlim_max) {
      rl.rlim_cur = rl.rlim_max;
      setrlimit(RLIMIT_NOFILE, &rl);
    }
  }
  signal(SIGPIPE, SIG_IGN);
  g_log.start();      // after the mask: every thread must inherit it, or a signal would land outside the signalfd
  atexit(log_flush);  // every _exit() below follows a WARN, which is written synchronously

  Kube kube;
  std::string err;
  if (!kube.init(f, &err)) {  // kubeInit: log.Fatalf
    logf('F', "Failed due to %s", err.c_str());
    return 255;
  }

  VLOG(1, "Loading NVML");
  if (f.fake_inventory == 0) {
    if (gsb_init() != GSB_OK) {  // gpumanager.go:36-40: park forever, no crash loop
      VLOG(1, "Failed to initialize NVML: %s.", last_error().c_str());
      VLOG(1, "If this is a GPU node, did you set the docker default runtime to `nvidia`?");
      for (;;) pause();
    }
    VLOG(1, "Fetching devices.");
    uint32_t n = 0;
    if (gsb_device_count(&n) != GSB_OK || n == 0) {
      VLOG(1, "No devices found. Waiting indefinitely.");
      for (;;) pause();
    }
  }

  VLOG(1, "Starting FS watcher.");
  const int ifd = inotify_init1(IN_NONBLOCK | IN_CLOEXEC);
  if (ifd < 0 || inotify_add_watch(ifd, plugin_dir.c_str(), IN_CREATE | IN_DELETE) < 0) {
    VLOG(1, "Failed to created FS watcher.");
    logf('F', "Failed due to inotify on %s: %s", plugin_dir.c_str(), strerror(errno));
    return 255;
  }
  VLOG(1, "Starting OS watcher.");
  const int sfd = signalfd(-1, &mask, SFD_NONBLOCK | SFD_CLOEXEC);

  const std::string kubelet_sock = plugin_dir + "kubelet.sock";
  const std::string socket = plugin_dir + kServerSockName;
  std::unique_ptr<Plugin> plugin;
  bool restart = true;
  int rc = 0;
  for (;;) {
    if (restart) {
      if (plugin) plugin->stop();
      plugin.reset(new Plugin(f, &kube, socket));
      if (!plugin->build(&err)) {
        WARN("Failed to get device plugin due to %s", err.c_str());
        _exit(1);  // gpumanager.go:73
      }
      plugin->configure_kubelet(&err);
      if (getenv("GPUSHARE_RETRY_SLEEP_MS")) plugin->set_retry_sleep_ms(atoi(getenv("GPUSHARE_RETRY_SLEEP_MS")));
      if (!plugin->start(&err)) {
        INFO("Could not start device plugin: %s", err.c_str());
        WARN("Failed to start device plugin due to %s", err.c_str());
        _exit(2);  // gpumanager.go:76
      }
      INFO("Starting to serve on %s", socket.c_str());
      if (!plugin->register_with(kubelet_sock, &err)) {
        INFO("Could not register device plugin: %s", err.c_str());
        plugin->stop();
        WARN("Failed to start device plugin due to %s", err.c_str());
        _exit(2);
      }
      INFO("Registered device plugin with Kubelet");
      restart = false;
    }
    pollfd fds[2] = {{ifd, POLLIN, 0}, {sfd, POLLIN, 0}};
    if (poll(fds, 2, -1) < 0) continue;
    if (fds[0].revents & POLLIN) {
      alignas(inotify_event) char buf[4096];
      ssize_t n;
      while ((n = read(ifd, buf, sizeof buf)) > 0) {
        for (char *p = buf; p < buf + n;) {
          inotify_event *ev = reinterpret_cast<inotify_event *>(p);
          if (ev->len && (ev->mask & IN_CREATE) && strcmp(ev->name, "kubelet.sock") == 0) {
            VLOG(1, "inotify: %s created, restarting.", kubelet_sock.c_str());  // gpumanager.go:83-87
            restart = true;
          }
          p += sizeof(inotify_event) + ev->len;
        }
      }
    }
    if (fds[1].revents & POLLIN) {
      signalfd_siginfo si;
      while (read(sfd, &si, sizeof si) == (ssize_t)sizeof si) {
        if (si.ssi_signo == SIGHUP) {
          VLOG(1, "Received SIGHUP, restarting.");
          restart = true;
        } else if (si.ssi_signo == SIGQUIT) {  // gpumanager.go:97-101: dump, keep running
          INFO("generate core dump");
          char ts[32];
          time_t now = time(nullptr);
          tm t;
          localtime_r(&now, &t);
          strftime(ts, sizeof ts, "%Y%m%d%H%M%S", &t);
          // composed before the file is created (the per-GPU health lines query NVML): a reader that finds the file
          // never finds it empty
          const std::string text = plugin->dump();
          std::ofstream(dump_dir + (dump_dir.back() == '/' ? "" : "/") + "go_" + ts + ".txt") << text;
        } else {
          VLOG(1, "Received signal \"%s\", shutting down.", strsignal((int)si.ssi_signo));
          plugin->stop();
          goto out;
        }
      }
    }
  }
out:
  if (f.fake_inventory == 0) {
    const int s = gsb_shutdown();
    VLOG(1, "Shutdown of NVML returned: %s", s == GSB_OK ? "<nil>" : gsb_strerror(s));
  }
  return rc;
}
