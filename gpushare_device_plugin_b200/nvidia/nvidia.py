"""Inventory + health watch — mirror of pkg/gpu/nvidia/nvidia.go over the C ABI.

Same functions, same argument meaning, same results as the reference; every value comes from
libgpushare_b200.so (one NVML memory query + identity cross-check per GPU instead of go-nvml's
11-getter NewDevice, and an event queue fed by the XID thread and the HBM prober instead of a
per-fake-device NVML registration). Nothing here computes inventory in Python.
"""
from __future__ import annotations

import logging
import threading
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

from .. import device
from .._abi import (COPY_CONDITION_NAMES, ECC_CONDITION_NAMES, GSB_EVENT_COPY, GSB_EVENT_ECC, GSB_EVENT_INVENTORY,
                    GSB_EVENT_LINK, GSB_EVENT_PROBE, GSB_EVENT_XID, GSB_FAULT_REPORT_FIRST, GSB_OPT_COPY_PROBE_EVERY_CYCLES,
                    GSB_OPT_ECC_HEALTH, GSB_OPT_LINK_PROBE_EVERY_CYCLES, GSB_PROBE_FAULT_MISMATCH, GSB_PROBE_RECOVERED,
                    GSB_EVENT_SM, GSB_OPT_SM_PROBE_EVERY_CYCLES, LINK_CONDITION_NAMES, SM_CONDITION_NAMES, CopyResult,
                    EccStatus, GsbError, LinkResult, SmResult, lib, CLUSTER_CONDITION_NAMES, GSB_EVENT_CLUSTER,
                    GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, ClusterResult, ATOMIC_CONDITION_NAMES, GSB_EVENT_ATOMIC,
                    GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, AtomicResult, TENSOR_CONDITION_NAMES, GSB_EVENT_TENSOR,
                    GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, TensorResult, SFU_CONDITION_NAMES, GSB_EVENT_SFU,
                    GSB_OPT_SFU_PROBE_EVERY_CYCLES, SfuResult, L1_CONDITION_NAMES, GSB_EVENT_L1,
                    GSB_OPT_L1_PROBE_EVERY_CYCLES, L1Result, ORDER_CONDITION_NAMES, GSB_EVENT_ORDER,
                    GSB_OPT_ORDER_PROBE_EVERY_CYCLES, OrderResult, SPARSE_CONDITION_NAMES, GSB_EVENT_SPARSE,
                    GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, SparseResult, SHARED_ATOMIC_CONDITION_NAMES,
                    GSB_EVENT_SHARED_ATOMIC, GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, SharedAtomicResult)
from . import const

log = logging.getLogger("gpushare.nvidia")

# process globals, as in nvidia.go:15-18 (gpuMemory is set once, from the first GPU, and never reset)
gpuMemory: int = 0
metric: str = const.GiBPrefix


@dataclass
class Device:
    """pluginapi.Device (v1beta1/api.proto:82-90)."""
    ID: str
    Health: str = const.Healthy


def check(err: Exception) -> None:
    """nvidia.go:20-24: any inventory error is fatal (log.Fatalln -> exit status 1)."""
    if err is not None:
        log.critical("Fatal: %s", err)
        raise SystemExit(1)


def generateFakeDeviceID(realID: str, fakeCounter: int) -> str:  # nvidia.go:26-28
    return device.fake_device_id(realID, fakeCounter)


def extractRealDeviceID(fakeDeviceID: str) -> str:  # nvidia.go:30-32
    return device.real_device_id(fakeDeviceID)


def setGPUMemory(raw: int) -> None:  # nvidia.go:34-41
    global gpuMemory
    gpuMemory = device.slices(raw, metric == const.GiBPrefix)
    log.info("set gpu memory: %d", gpuMemory)


def getGPUMemory() -> int:  # nvidia.go:43-45
    return gpuMemory


def getDeviceCount() -> int:  # nvidia.go:47-51
    try:
        return device.device_count()
    except GsbError as e:
        check(e)


def getDevices() -> Tuple[List[Device], Dict[str, int]]:
    """nvidia.go:53-89: fake devices in (GPU index asc, slice asc) order + UUID -> /dev/nvidia minor."""
    try:
        n = device.device_count()
        devs: List[Device] = []
        realDevNames: Dict[str, int] = {}
        for i in range(n):
            d = device.device_info(i)
            log.info("Deivce %s's Path is /dev/nvidia%d", d.uuid, d.minor)
            realDevNames[d.uuid] = d.minor
            log.info("# device Memory: %d", d.total_mib)
            if getGPUMemory() == 0:
                setGPUMemory(d.total_mib)
            for j in range(getGPUMemory()):
                devs.append(Device(ID=device.fake_device_id(d.uuid, j)))
        return devs, realDevNames
    except GsbError as e:
        check(e)


def deviceExists(devs: List[Device], id_: str) -> bool:  # nvidia.go:91-98
    return any(d.ID == id_ for d in devs)


def faultReportLine(uuid: str) -> Optional[str]:
    """The log line of the FIRST HBM fault report of GPU `uuid` (gsb_fault_report_text), or None when there is none."""
    try:
        for i in range(device.device_count()):
            info, _ = device.inventory_snapshot(i)
            if info.uuid == uuid:
                r = device.fault_report(i, GSB_FAULT_REPORT_FIRST)
                return device.fault_report_text(r, uuid) if r.valid else None
    except GsbError:
        pass
    return None


def eccStatusLine(uuid: str) -> str:
    """gsb_ecc_status_text of GPU `uuid`'s live ECC status; every field "unknown" when it cannot be read."""
    st = EccStatus()
    try:
        for i in range(device.device_count()):
            info, _ = device.inventory_snapshot(i)
            if info.uuid == uuid:
                st = device.ecc_status(i)
    except GsbError:
        st = EccStatus()
    return device.ecc_status_text(st, uuid)


@dataclass(frozen=True, eq=False)
class Check:
    """One periodic health check of the library (none is in the reference): what turns it on, what it raises and how
    its most recent probe reads."""
    option: int                          # GSB_OPT_*_PROBE_EVERY_CYCLES
    event: int                           # GSB_EVENT_*
    stats: Callable[[int], object]       # device.*_stats
    text: Callable[[object, str], str]   # device.*_text
    empty: Callable[[], object]          # the result of a probe that has not run
    conditions: Dict[int, str]           # the name of each condition bit
    label: str                           # in the warning
    what: str                            # "<what> condition ?" stands for a condition without a name


# in the order the library runs them, which is the order watchXIDs takes their cadences and logs them in
CHECKS = (
    Check(GSB_OPT_LINK_PROBE_EVERY_CYCLES, GSB_EVENT_LINK, device.link_stats, device.link_text, LinkResult,
          LINK_CONDITION_NAMES, "PCIe link health", "link"),
    Check(GSB_OPT_COPY_PROBE_EVERY_CYCLES, GSB_EVENT_COPY, device.copy_stats, device.copy_text, CopyResult,
          COPY_CONDITION_NAMES, "copy-engine health", "copy"),
    Check(GSB_OPT_SM_PROBE_EVERY_CYCLES, GSB_EVENT_SM, device.sm_stats, device.sm_text, SmResult,
          SM_CONDITION_NAMES, "SM compute health", "SM"),
    Check(GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, GSB_EVENT_CLUSTER, device.cluster_stats, device.cluster_text,
          ClusterResult, CLUSTER_CONDITION_NAMES, "SM-to-SM health", "SM-to-SM"),
    Check(GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_ATOMIC, device.atomic_stats, device.atomic_text, AtomicResult,
          ATOMIC_CONDITION_NAMES, "L2 atomic health", "L2 atomic"),
    Check(GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, GSB_EVENT_TENSOR, device.tensor_stats, device.tensor_text, TensorResult,
          TENSOR_CONDITION_NAMES, "tensor-core format health", "tensor"),
    Check(GSB_OPT_SFU_PROBE_EVERY_CYCLES, GSB_EVENT_SFU, device.sfu_stats, device.sfu_text, SfuResult,
          SFU_CONDITION_NAMES, "SM special-function health", "SFU"),
    Check(GSB_OPT_L1_PROBE_EVERY_CYCLES, GSB_EVENT_L1, device.l1_stats, device.l1_text, L1Result,
          L1_CONDITION_NAMES, "L1 and constant-cache health", "L1"),
    Check(GSB_OPT_ORDER_PROBE_EVERY_CYCLES, GSB_EVENT_ORDER, device.order_stats, device.order_text, OrderResult,
          ORDER_CONDITION_NAMES, "memory-ordering health", "memory-ordering"),
    Check(GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, GSB_EVENT_SPARSE, device.sparse_stats, device.sparse_text, SparseResult,
          SPARSE_CONDITION_NAMES, "sparse tensor-core health", "sparse"),
    Check(GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, GSB_EVENT_SHARED_ATOMIC, device.shared_atomic_stats,
          device.shared_atomic_text, SharedAtomicResult, SHARED_ATOMIC_CONDITION_NAMES, "shared-memory atomic health",
          "shared-atomic"),
)


def checkLine(check: Check, uuid: str) -> str:
    """The text of GPU `uuid`'s most recent probe of `check`; that of a probe that has not run when there is none."""
    r = check.empty()
    try:
        for i in range(device.device_count()):
            info, _ = device.inventory_snapshot(i)
            if info.uuid == uuid:
                r = check.stats(i).last
    except GsbError:
        r = check.empty()
    return check.text(r, uuid)


def watchXIDs(stop: threading.Event, devs: List[Device], xids: Callable[[List[Device]], None],
              probe_period_ms: int = 0, window_bytes: int = device.GiB,
              recovered: Optional[Callable[[Device], None]] = None, recovery_cycles: int = 0,
              ecc: bool = False, link_every: int = 0, copy_every: int = 0, sm_every: int = 0,
              cluster_every: int = 0, atomic_every: int = 0, tensor_every: int = 0, sfu_every: int = 0,
              l1_every: int = 0, order_every: int = 0, sparse_every: int = 0, shared_atomic_every: int = 0) -> None:
    """nvidia.go:100-152 with the event source replaced: gsb_health_wait delivers both XID critical
    errors (same NVML event type, registered once per GPU) and verdicts of the active HBM probe.
    The loop shape, the 5 s wait, the XID 31/43/45 filter, "empty UUID = every device" and "every
    fake device of that UUID" are the reference's. `xids` receives every fake device one event hits in one call, in
    the reference's order, so that a stream never sees half of one GPU's flip. `ecc` (not in the reference) turns on
    the library's ECC and row-remapper health: its events mark the GPU unhealthy, with the status logged. `link_every`
    (not in the reference) > 0 runs a PCIe link probe every that many prober cycles; its events do the same, and so do
    those of the copy-engine probe `copy_every` (not in the reference) > 0 runs, of the SM compute probe `sm_every`
    (not in the reference) > 0 runs, of the SM-to-SM probe `cluster_every` (not in the reference) > 0 runs, of the
    L2 atomic probe `atomic_every` (not in the reference) > 0 runs, of the tensor-core format probe `tensor_every`
    (not in the reference) > 0 runs, of the SM special-function probe `sfu_every` (not in the reference) > 0 runs,
    of the L1 and constant-cache probe `l1_every` (not in the reference) > 0 runs, of the memory-ordering probe
    `order_every` (not in the reference) > 0 runs, of the sparse tensor-core probe `sparse_every` (not in the
    reference) > 0 runs and of the shared-memory atomic probe `shared_atomic_every` (not in the reference) > 0
    runs."""
    lib.gsb_health_set_recovery(recovery_cycles if recovered is not None else 0)
    device.set_option(GSB_OPT_ECC_HEALTH, 1 if ecc else 0)
    every = dict(zip(CHECKS, (link_every, copy_every, sm_every, cluster_every, atomic_every, tensor_every, sfu_every,
                              l1_every, order_every, sparse_every, shared_atomic_every)))
    for check, n in every.items():
        device.set_option(check.option, max(0, n))
    device.health_start(probe_period_ms, window_bytes)
    try:
        seen = {check: {} for check in CHECKS}
        while not stop.is_set():
            e = device.health_wait(5000)  # nvidia.go:126
            for check in CHECKS:  # each GPU's most recent probe of every check that is on, logged once
                if every[check] <= 0:
                    continue
                try:
                    for i in range(len({extractRealDeviceID(d.ID) for d in devs})):
                        st = check.stats(i)
                        if st.probes > seen[check].get(i, 0):
                            seen[check][i] = st.probes
                            log.info("%s", check.text(st.last, device.inventory_snapshot(i)[0].uuid))
                except GsbError:
                    pass
            if e is None:
                continue
            raised = next((c for c in CHECKS if e.etype == c.event and every[c] > 0), None)
            if e.etype == GSB_EVENT_ECC and ecc:  # not in the reference: what the GPU records about its HBM
                log.warning("ECC health of %s: %s: marking it unhealthy", e.uuid.decode(),
                            ECC_CONDITION_NAMES.get(e.edata, "ECC condition ?"))
                log.warning("%s", eccStatusLine(e.uuid.decode()))
            elif raised is not None:
                log.warning("%s of %s: %s: marking it unhealthy", raised.label, e.uuid.decode(),
                            raised.conditions.get(e.edata, raised.what + " condition ?"))
                log.warning("%s", checkLine(raised, e.uuid.decode()))
            elif e.etype == GSB_EVENT_INVENTORY:  # the low-rate NVML refresh disagrees with what is advertised
                log.warning("inventory of %s changed under the plugin (%d): marking it unhealthy", e.uuid.decode(), e.edata)
            elif e.etype not in (GSB_EVENT_XID, GSB_EVENT_PROBE):  # nvidia.go:127-129
                continue
            if e.etype == GSB_EVENT_XID and lib.gsb_xid_is_benign(e.edata):  # nvidia.go:134-136
                continue
            uuid = e.uuid.decode()
            if e.etype == GSB_EVENT_PROBE and e.edata == GSB_PROBE_RECOVERED:
                # not in the reference (server.go:180 FIXME): only when --health-recovery-cycles > 0
                if recovered is not None and recovery_cycles > 0:
                    for d in devs:
                        if extractRealDeviceID(d.ID) == uuid:
                            recovered(d)
                continue
            if e.etype == GSB_EVENT_PROBE and e.edata == GSB_PROBE_FAULT_MISMATCH:
                line = faultReportLine(uuid)  # not in the reference: where the probe's verdict came from
                if line is not None:
                    log.warning("%s", line)
            if len(uuid) == 0:  # nvidia.go:138-144: all devices are unhealthy
                xids(list(devs))
                continue
            xids([d for d in devs if extractRealDeviceID(d.ID) == uuid])  # nvidia.go:146-150
    finally:
        device.health_stop()
