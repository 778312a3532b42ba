// gsbd: command line (cmd/nvidia/main.go:15-26 + glog's flags), Go flag-package behaviour
// Private to gsbd.cc (one translation unit): everything lives in an unnamed namespace.
#ifndef GSBD_FLAGS_HPP_
#define GSBD_FLAGS_HPP_
#include <stdio.h>
#include <stdlib.h>
#include <sys/stat.h>

#include <fstream>
#include <sstream>
#include <string>

#include "gsbd_log.hpp"

namespace {

struct Flags {
  bool mps = false, health_check = false, query_kubelet = false;
  std::string memory_unit = "GiB", kubelet_address = "0.0.0.0", client_cert, client_key, token;
  int kubelet_port = 10250, timeout = 10;
  // additions (active probe, test hooks); none changes the wire contract
  int probe_period_ms = 1000, probe_window_mib = 1024, probe_arena_mib = 0, probe_keep_free_mib = 1024, fake_inventory = 0;
  int probe_watchdog_ms = 2000, inventory_refresh_ms = 5000, probe_sweep_every = 0;
  int health_recovery_cycles = 0;  // 0 = the reference's sticky Unhealthy
  bool startup_full_walk = false, coalesce_health = true, pod_informer = true;
  bool startup_memtest = false;  // March C- of every GPU before serving (gsb_memtest)
  bool health_ecc = false;  // ECC and row-remapper health (GSB_OPT_ECC_HEALTH)
  int probe_link_every = 0;  // PCIe link probe every N prober cycles (GSB_OPT_LINK_PROBE_EVERY_CYCLES); 0 = off
  int probe_sm_every = 0;    // SM compute probe every N prober cycles (GSB_OPT_SM_PROBE_EVERY_CYCLES); 0 = off
  int probe_cluster_every = 0;  // SM-to-SM probe every N prober cycles (GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES); 0 = off
  int probe_atomic_every = 0;   // L2 atomic probe every N prober cycles (GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES); 0 = off
  int probe_tensor_every = 0;   // tensor-core format probe every N prober cycles (GSB_OPT_TENSOR_PROBE_EVERY_CYCLES); 0 = off
  int probe_sfu_every = 0;      // SM special-function probe every N prober cycles (GSB_OPT_SFU_PROBE_EVERY_CYCLES); 0 = off
  int probe_l1_every = 0;       // L1 and constant-cache probe every N prober cycles (GSB_OPT_L1_PROBE_EVERY_CYCLES); 0 = off
  int probe_order_every = 0;    // memory-ordering probe every N prober cycles (GSB_OPT_ORDER_PROBE_EVERY_CYCLES); 0 = off
  int probe_sparse_every = 0;   // sparse tensor-core probe every N prober cycles (GSB_OPT_SPARSE_PROBE_EVERY_CYCLES); 0 = off
  int probe_shared_atomic_every = 0;  // shared-memory atomic probe every N prober cycles (GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES); 0 = off
  int startup_stress_ms = 0; // SM stress of every GPU for N ms before serving (gsb_sm_stress); 0 = off
  int probe_copy_every = 0;  // copy-engine probe every N prober cycles (GSB_OPT_COPY_PROBE_EVERY_CYCLES); 0 = off
  bool serialize_allocate = false;  // the reference's plugin-wide lock across the whole Allocate, PATCH included
  double pod_cache_ttl = 1.0;
  std::string kube_api_url, kubelet_scheme = "https";
};

bool parse_bool(const std::string &v) { return v == "" || v == "1" || v == "t" || v == "T" || v == "true" || v == "TRUE" || v == "True"; }

// What Go's flag package prints for -h / an undefined flag (PrintDefaults: sorted by name, "  -name type" then a
// tab-indented description with the non-zero default). The first ten are cmd/nvidia/main.go:15-26 verbatim.
void usage(const char *prog) {
  fprintf(stderr, "Usage of %s:\n", prog);
  static const char *const lines[][2] = {
      {"-client-cert string", "Kubelet TLS client certificate"},
      {"-client-key string", "Kubelet TLS client key"},
      {"-coalesce-health", "Fold the health events already queued into one ListAndWatch resend; false = one resend per fake device, as the reference (default true)"},
      {"-health-check", "Enable or disable Health check"},
      {"-health-ecc", "Also watch the GPUs' ECC counters and row-remapper state: a pending row remap, a remap failure or a new uncorrected error marks the GPU unhealthy; corrected errors are counted, per probe walk and between walks"},
      {"-health-recovery-cycles int", "Consecutive clean probe cycles after which a probe-faulted GPU is Healthy again; 0 = sticky Unhealthy, as the reference"},
      {"-inventory-refresh-ms int", "Period of the off-path NVML re-query that guards the inventory snapshot while health runs; 0 = never (default 5000)"},
      {"-kube-api-url string", "Apiserver base URL instead of KUBECONFIG / in-cluster discovery"},
      {"-kubelet-address string", "Kubelet IP Address (default \"0.0.0.0\")"},
      {"-kubelet-port uint", "Kubelet listened Port (default 10250)"},
      {"-kubelet-scheme string", "http or https for the kubelet /pods/ client (default \"https\")"},
      {"-memory-unit string", "Set memoryUnit of the GPU Memroy, support 'GiB' and 'MiB' (default \"GiB\")"},
      {"-mps", "Enable or Disable MPS"},
      {"-pod-cache-ttl float", "Seconds a pending-pod LIST may be reused when the watch informer is off or down; 0 = LIST on every Allocate (default 1)"},
      {"-pod-informer", "Keep the pending-pod table current from a LIST + watch stream instead of LISTing inside Allocate (default true)"},
      {"-probe-arena-mib int", "Standing HBM probe arena per GPU in MiB, held by the plugin and not available to tenants; 0 = hold nothing, probe a transient window per cycle (default 0)"},
      {"-probe-keep-free-mib int", "Free HBM per GPU that no probe allocation (window, arena or start-up walk) ever takes (default 1024)"},
      {"-probe-period-ms int", "Period of the HBM health probe per GPU (default 1000)"},
      {"-probe-sweep-every int", "Every Nth probe cycle of a GPU without a standing arena walks ALL HBM that is allocatable at that moment (minus -probe-keep-free-mib) instead of one window, then gives it back; 0 = never (default 0)"},
      {"-probe-watchdog-ms int", "A probe launch still running after this long (+1 ms per 10 MB of window) marks the GPU unhealthy; 0 = wait for ever (default 2000)"},
      {"-probe-window-mib int", "HBM bytes verified and re-written per probe cycle (default 1024)"},
      {"-query-kubelet", "Query pending pods from kubelet instead of kube-apiserver"},
      {"-serialize-allocate", "Hold one lock across the whole Allocate, apiserver PATCH included, as the reference does; with -pod-informer=false -pod-cache-ttl 0 this is the reference's Allocate in compiled code"},
      {"-startup-full-walk", "Verify the whole arena once before serving"},
      {"-timeout int", "Kubelet client http timeout duration (default 10)"},
      {"-token string", "Kubelet client bearer token"},
      {"-v value", "log level for V logs (glog)"},
  };
  for (auto &l : lines) fprintf(stderr, "  %s\n    \t%s\n", l[0], l[1]);
}

// Go's flag syntax: -f, --f, -f=v, -f v (non-boolean). Returns 0 = go on, otherwise the process exit code + 1.
int parse_flags(int argc, char **argv, Flags *f) {
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i];
    if (a.size() < 2 || a[0] != '-') {
      fprintf(stderr, "unexpected argument %s\n", a.c_str());
      return 3;
    }
    a.erase(0, a[1] == '-' ? 2 : 1);
    std::string name = a, val;
    bool has_val = false;
    const size_t eq = a.find('=');
    if (eq != std::string::npos) {
      name = a.substr(0, eq);
      val = a.substr(eq + 1);
      has_val = true;
    }
    if (name == "h" || name == "help") {  // flag.ErrHelp: usage, exit status 0
      usage(argv[0]);
      return 1;
    }
    auto need = [&]() -> bool {
      if (has_val) return true;
      if (i + 1 >= argc) {
        fprintf(stderr, "flag needs an argument: -%s\n", name.c_str());
        usage(argv[0]);
        return false;
      }
      val = argv[++i];
      return true;
    };
    auto boolean = [&](bool *dst) { *dst = has_val ? parse_bool(val) : true; };
    if (name == "mps") boolean(&f->mps);
    else if (name == "health-check") boolean(&f->health_check);
    else if (name == "health-ecc") boolean(&f->health_ecc);
    else if (name == "query-kubelet") boolean(&f->query_kubelet);
    else if (name == "startup-full-walk") boolean(&f->startup_full_walk);
    // not listed by usage(): the -h listing is pinned by tests/test_ecc_health.py; DESIGN.md §11 documents the flag
    else if (name == "startup-memtest") boolean(&f->startup_memtest);
    else if (name == "probe-link-every") { if (!need()) return 3; f->probe_link_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-copy-every") { if (!need()) return 3; f->probe_copy_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-sm-every") { if (!need()) return 3; f->probe_sm_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-cluster-every") { if (!need()) return 3; f->probe_cluster_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-atomic-every") { if (!need()) return 3; f->probe_atomic_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-tensor-every") { if (!need()) return 3; f->probe_tensor_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-sfu-every") { if (!need()) return 3; f->probe_sfu_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-l1-every") { if (!need()) return 3; f->probe_l1_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-order-every") { if (!need()) return 3; f->probe_order_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-sparse-every") { if (!need()) return 3; f->probe_sparse_every = atoi(val.c_str()); }  // likewise
    else if (name == "probe-shared-atomic-every") { if (!need()) return 3; f->probe_shared_atomic_every = atoi(val.c_str()); }  // likewise
    else if (name == "startup-stress-ms") { if (!need()) return 3; f->startup_stress_ms = atoi(val.c_str()); }  // likewise
    else if (name == "coalesce-health") boolean(&f->coalesce_health);
    else if (name == "pod-informer") boolean(&f->pod_informer);
    else if (name == "serialize-allocate") boolean(&f->serialize_allocate);
    else if (name == "logtostderr" || name == "alsologtostderr") { bool ignored; boolean(&ignored); }
    else if (name == "memory-unit") { if (!need()) return 3; f->memory_unit = val; }
    else if (name == "kubelet-address") { if (!need()) return 3; f->kubelet_address = val; }
    else if (name == "kubelet-port") { if (!need()) return 3; f->kubelet_port = atoi(val.c_str()); }
    else if (name == "client-cert") { if (!need()) return 3; f->client_cert = val; }
    else if (name == "client-key") { if (!need()) return 3; f->client_key = val; }
    else if (name == "token") { if (!need()) return 3; f->token = val; }
    else if (name == "timeout") { if (!need()) return 3; f->timeout = atoi(val.c_str()); }
    else if (name == "v") { if (!need()) return 3; g_v = atoi(val.c_str()); }
    else if (name == "stderrthreshold" || name == "log_dir" || name == "vmodule" || name == "log_backtrace_at") { if (!need()) return 3; }
    else if (name == "probe-period-ms") { if (!need()) return 3; f->probe_period_ms = atoi(val.c_str()); }
    else if (name == "probe-window-mib") { if (!need()) return 3; f->probe_window_mib = atoi(val.c_str()); }
    else if (name == "probe-arena-mib") { if (!need()) return 3; f->probe_arena_mib = atoi(val.c_str()); }
    else if (name == "probe-keep-free-mib") { if (!need()) return 3; f->probe_keep_free_mib = atoi(val.c_str()); }
    else if (name == "probe-sweep-every") { if (!need()) return 3; f->probe_sweep_every = atoi(val.c_str()); }
    else if (name == "probe-watchdog-ms") { if (!need()) return 3; f->probe_watchdog_ms = atoi(val.c_str()); }
    else if (name == "inventory-refresh-ms") { if (!need()) return 3; f->inventory_refresh_ms = atoi(val.c_str()); }
    else if (name == "health-recovery-cycles") { if (!need()) return 3; f->health_recovery_cycles = atoi(val.c_str()); }
    else if (name == "pod-cache-ttl") { if (!need()) return 3; f->pod_cache_ttl = atof(val.c_str()); }
    else if (name == "kube-api-url") { if (!need()) return 3; f->kube_api_url = val; }
    else if (name == "kubelet-scheme") { if (!need()) return 3; f->kubelet_scheme = val; }
    else if (name == "fake-inventory") { if (!need()) return 3; f->fake_inventory = atoi(val.c_str()); }
    else {
      fprintf(stderr, "flag provided but not defined: -%s\n", name.c_str());
      usage(argv[0]);
      return 3;  // flag.ExitOnError: exit status 2
    }
  }
  return 0;
}

std::string read_file(const std::string &p) {
  std::ifstream f(p);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}
bool file_exists(const std::string &p) {
  struct stat st;
  return !p.empty() && stat(p.c_str(), &st) == 0;
}


}  // namespace

#endif  // GSBD_FLAGS_HPP_
