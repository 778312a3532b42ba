"""Process entry — mirror of cmd/nvidia/main.go: same flags, same defaults.

    python -m gpushare_device_plugin_b200.cmd.nvidia -logtostderr --v=5 --memory-unit=GiB

(the DaemonSet command line, device-plugin-ds.yaml:29-33, is accepted unchanged; glog's flags are
parsed and mapped onto `logging`)."""
from __future__ import annotations

import argparse
import logging
import sys

from ..kubelet.client import KubeletClientConfig, NewKubeletClient
from ..nvidia import const, podmanager
from ..nvidia.gpumanager import NewSharedGPUManager

log = logging.getLogger("gpushare")


def _bool(v):
    return str(v).lower() in ("1", "t", "true", "")


def parse(argv):
    p = argparse.ArgumentParser(prog="gpushare-device-plugin-v2", allow_abbrev=False)
    b = dict(nargs="?", const=True, type=_bool)  # Go flag: -x, -x=true, --x=false
    for dash in ("-", "--"):
        pass
    def add(name, **kw):
        p.add_argument("-" + name, "--" + name, dest=name.replace("-", "_"), **kw)
    add("mps", default=False, help="Enable or Disable MPS", **b)
    add("health-check", default=False, help="Enable or disable Health check", **b)
    add("memory-unit", default="GiB", help="Set memoryUnit of the GPU Memroy, support 'GiB' and 'MiB'")
    add("query-kubelet", default=False, help="Query pending pods from kubelet instead of kube-apiserver", **b)
    add("kubelet-address", default="0.0.0.0", help="Kubelet IP Address")
    add("kubelet-port", default=10250, type=int, help="Kubelet listened Port")
    add("client-cert", default="", help="Kubelet TLS client certificate")
    add("client-key", default="", help="Kubelet TLS client key")
    add("token", default="", help="Kubelet client bearer token")
    add("timeout", default=10, type=int, help="Kubelet client http timeout duration")
    # glog flags the DaemonSet passes
    add("logtostderr", default=True, **b)
    add("alsologtostderr", default=False, **b)
    add("v", default=0, type=int)
    add("stderrthreshold", default="ERROR")
    add("log_dir", default="")
    add("vmodule", default="")
    add("log_backtrace_at", default="")
    # additions (not in the reference): active HBM probe cadence of the health watch
    add("probe-period-ms", default=1000, type=int)
    add("probe-window-mib", default=1024, type=int)
    add("probe-arena-mib", default=0, type=int)  # 0 = transient window per cycle, nothing held
    add("probe-keep-free-mib", default=1024, type=int)
    add("probe-watchdog-ms", default=2000, type=int)
    add("inventory-refresh-ms", default=5000, type=int)
    add("probe-sweep-every", default=0, type=int)
    add("startup-full-walk", default=False, **b)
    add("startup-memtest", default=False, **b)  # March C- of every GPU before registering
    add("health-recovery-cycles", default=0, type=int)
    add("health-ecc", default=False, **b)  # ECC and row-remapper health (opt-in)
    add("probe-link-every", default=0, type=int)  # PCIe link probe every N prober cycles; 0 = off
    add("probe-copy-every", default=0, type=int)  # copy-engine probe every N prober cycles; 0 = off
    add("probe-sm-every", default=0, type=int)  # SM compute probe every N prober cycles; 0 = off
    add("startup-stress-ms", default=0, type=int)  # SM stress of every GPU for N ms before registering; 0 = off
    add("probe-cluster-every", default=0, type=int)  # SM-to-SM probe every N prober cycles; 0 = off
    add("probe-atomic-every", default=0, type=int)  # L2 atomic probe every N prober cycles; 0 = off
    add("probe-tensor-every", default=0, type=int)  # tensor-core format probe every N prober cycles; 0 = off
    add("probe-sfu-every", default=0, type=int)  # SM special-function probe every N prober cycles; 0 = off
    add("probe-l1-every", default=0, type=int)  # L1 and constant-cache probe every N prober cycles; 0 = off
    add("probe-order-every", default=0, type=int)  # memory-ordering probe every N prober cycles; 0 = off
    add("probe-sparse-every", default=0, type=int)  # sparse tensor-core probe every N prober cycles; 0 = off
    add("probe-shared-atomic-every", default=0, type=int)  # shared-memory atomic probe every N prober cycles; 0 = off
    return p.parse_args(argv)


def buildKubeletClient(a):  # main.go:28-53
    token = a.token
    if a.client_cert == "" and a.client_key == "" and token == "":
        try:
            with open("/var/run/secrets/kubernetes.io/serviceaccount/token") as f:
                token = f.read()
        except OSError as e:
            raise SystemExit(f"panic: in cluster mode, find token failed, error: {e}")
    return NewKubeletClient(KubeletClientConfig(Address=a.kubelet_address, Port=a.kubelet_port, BearerToken=token,
                                                CertFile=a.client_cert, KeyFile=a.client_key,
                                                HTTPTimeout=float(a.timeout)))


def translatememoryUnits(value: str) -> str:  # main.go:67-78
    if value in (const.MiBPrefix, const.GiBPrefix):
        return value
    log.warning("Unsupported memory unit: %s, use memoryUnit Gi as default", value)
    return const.GiBPrefix


def main(argv=None) -> None:  # main.go:55-65
    a = parse(sys.argv[1:] if argv is None else argv)
    logging.basicConfig(stream=sys.stderr, level=logging.DEBUG if a.v >= 4 else logging.INFO,
                        format="%(levelname).1s%(asctime)s %(name)s] %(message)s")
    log.info("Start gpushare device plugin")
    podmanager.kubeInit()  # the reference does this in package init() (allocate.go:20-22)
    kubeletClient = buildKubeletClient(a)
    import os
    ngm = NewSharedGPUManager(a.mps, a.health_check, a.query_kubelet, translatememoryUnits(a.memory_unit),
                              kubeletClient, pluginDir=os.environ.get("GPUSHARE_PLUGIN_DIR", const.DevicePluginPath),
                              dumpDir=os.environ.get("GPUSHARE_DUMP_DIR", "/etc/kubernetes/"),
                              probe_period_ms=a.probe_period_ms, window_bytes=a.probe_window_mib << 20,
                              probe_arena_bytes=a.probe_arena_mib << 20, startup_full_walk=a.startup_full_walk,
                              health_recovery_cycles=a.health_recovery_cycles,
                              probe_keep_free_bytes=a.probe_keep_free_mib << 20, probe_watchdog_ms=a.probe_watchdog_ms,
                              inventory_refresh_ms=a.inventory_refresh_ms, probe_sweep_every=a.probe_sweep_every,
                              health_ecc=a.health_ecc, startup_memtest=a.startup_memtest,
                              probe_link_every=a.probe_link_every, probe_copy_every=a.probe_copy_every,
                              probe_sm_every=a.probe_sm_every, startup_stress_ms=a.startup_stress_ms,
                              probe_cluster_every=a.probe_cluster_every, probe_atomic_every=a.probe_atomic_every,
                              probe_tensor_every=a.probe_tensor_every, probe_sfu_every=a.probe_sfu_every,
                              probe_l1_every=a.probe_l1_every, probe_order_every=a.probe_order_every,
                              probe_sparse_every=a.probe_sparse_every,
                              probe_shared_atomic_every=a.probe_shared_atomic_every)
    ngm.Run()


if __name__ == "__main__":
    main()
