"""Device-plugin gRPC server — mirror of pkg/gpu/nvidia/server.go.

Wire surface unchanged: service v1beta1.DevicePlugin (GetDevicePluginOptions, ListAndWatch, Allocate,
PreStartContainer) on a unix socket, and a v1beta1.Registration/Register call to the kubelet with
{version "v1beta1", endpoint "aliyungpushare.sock", resource_name "aliyun.com/gpu-mem"}
(server.go:150-169). All message bytes are produced/consumed by the C ABI (gsb_encode_*,
gsb_allocate); grpcio is the HTTP/2 transport only (identity (de)serialisers, generic handlers — the
image has no protoc and no Go toolchain, see DESIGN.md).
"""
from __future__ import annotations

import logging
import os
import threading
from concurrent import futures
from typing import Dict, List, Optional

import grpc

from .. import device
from . import allocate as _allocate
from . import const, nvidia, podmanager

log = logging.getLogger("gpushare.nvidia")

_SERVICE = "v1beta1.DevicePlugin"


class NvidiaDevicePlugin:
    """server.go:19-35. `coalesce_health=False` reproduces the reference's stream exactly (one full
    resend per fake-device health event, server.go:179-182); True (default) folds the events that
    are already queued into one resend — same final list, 1 frame instead of S per GPU."""

    def __init__(self, mps: bool, healthCheck: bool, queryKubelet: bool, client, socket: str = const.serverSock,
                 coalesce_health: bool = True, probe_period_ms: int = 1000, window_bytes: int = device.GiB,
                 max_workers: int = 16, pod_cache_ttl: float = 1.0, inventory=None,
                 probe_arena_bytes: int = 0, startup_full_walk: bool = False,
                 health_recovery_cycles: int = 0, probe_keep_free_bytes: int = device.GiB,
                 probe_watchdog_ms: int = 2000, inventory_refresh_ms: int = 5000, probe_sweep_every: int = 0,
                 health_ecc: bool = False, startup_memtest: bool = False, probe_link_every: int = 0,
                 probe_copy_every: int = 0, probe_sm_every: int = 0, startup_stress_ms: int = 0,
                 probe_cluster_every: int = 0, probe_atomic_every: int = 0, probe_tensor_every: int = 0,
                 probe_sfu_every: int = 0, probe_l1_every: int = 0, probe_order_every: int = 0,
                 probe_sparse_every: int = 0, probe_shared_atomic_every: int = 0):
        # `inventory` = (devs, devNameMap) injects a synthetic node (tests, Allocate benchmark)
        self.devs, self.devNameMap = inventory if inventory is not None else nvidia.getDevices()  # server.go:39
        devList = list(self.devNameMap)
        log.info("Device Map: %s", self.devNameMap)
        log.info("Device List: %s", devList)
        podmanager.patchGPUCount(len(devList))  # server.go:49-52
        self.disableCGPUIsolation = podmanager.disableCGPUIsolationOrNot()  # server.go:53-56
        self.realDevNames = devList
        self.devIndxMap: Dict[int, str] = {}
        self.socket = socket
        self.mps, self.healthCheck, self.queryKubelet, self.kubeletClient = mps, healthCheck, queryKubelet, client
        self.coalesce_health = coalesce_health
        self.probe_period_ms, self.window_bytes = probe_period_ms, window_bytes
        self.probe_arena_bytes, self.startup_full_walk = probe_arena_bytes, startup_full_walk
        self.health_recovery_cycles = health_recovery_cycles
        self.probe_keep_free_bytes, self.probe_watchdog_ms = probe_keep_free_bytes, probe_watchdog_ms
        self.inventory_refresh_ms, self.probe_sweep_every = inventory_refresh_ms, probe_sweep_every
        self.health_ecc = health_ecc
        self.startup_memtest = startup_memtest
        self.probe_link_every = probe_link_every
        self.probe_copy_every = probe_copy_every
        self.probe_sm_every = probe_sm_every
        self.probe_cluster_every = probe_cluster_every
        self.probe_atomic_every = probe_atomic_every
        self.probe_tensor_every = probe_tensor_every
        self.probe_sfu_every = probe_sfu_every
        self.probe_l1_every = probe_l1_every
        self.probe_order_every = probe_order_every
        self.probe_sparse_every = probe_sparse_every
        self.probe_shared_atomic_every = probe_shared_atomic_every
        self.startup_stress_ms = startup_stress_ms
        self.max_workers = max_workers
        self.stop = threading.Event()
        self.lock = threading.RLock()  # sync.RWMutex of server.go:34; Allocate takes it exclusively
        self.server: Optional[grpc.Server] = None
        # health state: bitset over self.devs + a version counter instead of the reference's unbuffered
        # channel, so a health event never blocks when no ListAndWatch stream is attached
        self._uuids = list(self.devNameMap)  # NVML order == insertion order of getDevices
        self._slices = nvidia.getGPUMemory()
        self._index = {d.ID: i for i, d in enumerate(self.devs)}
        self._bits = bytearray((len(self.devs) + 7) // 8)
        self._cv = threading.Condition()
        self._pending: List[int] = []
        self.allocate_ctx = _allocate.AllocateContext(self.devNameMap, self._slices,
                                                      nvidia.metric == const.GiBPrefix, self.disableCGPUIsolation)
        self.pod_cache = _allocate.PendingPodCache(pod_cache_ttl)
        self._health_thread: Optional[threading.Thread] = None

    # ---- helpers -------------------------------------------------------------------------
    def GetDeviceNameByIndex(self, index: int):  # server.go:72-83
        if len(self.devIndxMap) == 0:
            self.devIndxMap = {v: k for k, v in self.devNameMap.items()}
            log.info("Get devIndexMap: %s", self.devIndxMap)
        name = self.devIndxMap.get(index)
        return name, name is not None

    def _list_bytes(self, bits=None) -> bytes:
        bits = self._bits if bits is None else bits
        return device.encode_list_and_watch(self._uuids, self._slices, bytes(bits) if any(bits) else None)

    def _apply(self, bits: bytearray, e: int, record: bool) -> None:
        if e >= 0:  # d.Health = Unhealthy (server.go:181)
            bits[e >> 3] |= 1 << (e & 7)
            if record:
                self.devs[e].Health = const.Unhealthy
        else:       # optional recovery (not in the reference): ~e is the device index
            i = ~e
            bits[i >> 3] &= ~(1 << (i & 7)) & 0xFF
            if record:
                self.devs[i].Health = const.Healthy

    # ---- RPC handlers (raw bytes in/out) ---------------------------------------------------
    def GetDevicePluginOptions(self, request: bytes, context) -> bytes:  # server.go:85-87
        return b""

    def PreStartContainer(self, request: bytes, context) -> bytes:  # server.go:191-193
        return b""

    def ListAndWatch(self, request: bytes, context):  # server.go:172-185
        # The node's health state (self._bits, devs[i].Health) is written by the PRODUCER of an event (unhealthy /
        # recovered), never by a stream: an event raised while no stream is attached is in the first frame of the
        # next one (the reference's unbuffered channel blocks the producer until a stream takes the event). Each
        # stream replays the events it has not sent yet onto its own copy, so the reference-exact mode (one resend
        # per fake device, each frame the state after that event) does not depend on how far a stream lags.
        with self._cv:
            mine = bytearray(self._bits)
            first = self._list_bytes(mine)
            cursor = len(self._pending)
        yield first  # never yield while holding the condition's lock
        while True:
            with self._cv:
                while cursor >= len(self._pending) and not self.stop.is_set() and context.is_active():
                    self._cv.wait(0.25)
                if self.stop.is_set() or not context.is_active():
                    return
                frames = []
                for e in self._pending[cursor:]:
                    self._apply(mine, e, False)
                    if not self.coalesce_health:
                        frames.append(self._list_bytes(mine))
                cursor = len(self._pending)
                if self.coalesce_health:
                    frames = [self._list_bytes(mine)]
            for f in frames:
                yield f

    def Allocate(self, request: bytes, context) -> bytes:
        # grpc-go decodes the request before the handler runs: what gogo's Unmarshal refuses fails the call
        # with INTERNAL and never reaches allocate.go
        if not _allocate.decodable(self.allocate_ctx, request):
            context.abort(grpc.StatusCode.INTERNAL, "grpc: error unmarshalling request")
        return _allocate.allocate(self, request)

    # ---- health plumbing (server.go:187-189, 203-221) ----------------------------------------
    def unhealthy(self, devs: List[nvidia.Device]) -> None:
        """The fake devices one health event hits, queued under one lock: a coalescing stream sends them in one frame,
        the reference-exact stream still one frame per device."""
        with self._cv:
            for dev in devs:
                e = self._index[dev.ID]
                self._apply(self._bits, e, True)
                self._pending.append(e)
            self._cv.notify_all()

    def setup_probe_arenas(self, keep_free_bytes: int = device.GiB) -> None:
        """The memory the active probe walks. Default (probe_arena_bytes == 0): none is held — each probe cycle
        allocates its window, walks it and frees it (gsb_cycle's transient window), so the advertised slices are not
        oversold by the plugin itself. A standing arena (probe_arena_bytes > 0) widens coverage but keeps that HBM
        from tenants while ListAndWatch still advertises it; the warning says how much. Optionally one walk of
        everything allocatable at start-up. No probe allocation takes the last `keep_free_bytes`."""
        from .._abi import GSB_OP_VERIFY, GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, GsbError
        device.set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, keep_free_bytes)
        for i, uuid in enumerate(self._uuids):
            try:
                if self.startup_full_walk:
                    nbytes = device.arena_create(i, keep_free_bytes=keep_free_bytes)  # FILL of every mapped byte happens inside
                    r = device.probe(i, GSB_OP_VERIFY, flags=3)  # timed + generation table
                    log.info("start-up walk of %s: %d bytes actually allocatable, %d mismatching words, %.1f ms", uuid,
                             nbytes, r.mismatch_words, r.kernel_ns / 1e6)
                    if r.mismatch_words:
                        device.health_inject(uuid, 0x100, 1)
                    device.arena_destroy(i)
                if self.probe_arena_bytes > 0:
                    # the start-up memtest's standing arena, refilled, serves as it is (unless the full walk replaced it)
                    held = self.startup_memtest and not self.startup_full_walk and self._arena_bytes(i)
                    nbytes = held or device.arena_create(i, max_bytes=self.probe_arena_bytes,
                                                         keep_free_bytes=keep_free_bytes)
                    log.warning("standing probe arena on %s: %d bytes held by the plugin and NOT available to tenants "
                                "(%s still advertises %d slices)", uuid, nbytes, const.resourceName, self._slices)
                else:
                    log.info("probe of %s: transient %d MiB window per cycle, nothing held between cycles", uuid,
                             self.window_bytes >> 20)
            except GsbError as e:
                log.warning("no probe arena on %s: %s", uuid, e)

    @staticmethod
    def _arena_bytes(i: int) -> int:
        from .._abi import GsbError
        try:
            return device.arena_bytes(i)
        except GsbError:
            return 0

    def run_startup_memtest(self) -> None:
        """--startup-memtest (not in the reference): March C- of every GPU before the plugin serves or registers, so a
        GPU it faults is Unhealthy in the first ListAndWatch frame. With a standing arena it tests that arena and leaves
        it, refilled, to the prober; otherwise all allocatable HBM but the keep-free margin, given back."""
        from .._abi import (GSB_FAULT_REPORT_FIRST, GSB_OPT_ECC_HEALTH, GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, GsbError,
                            last_error)
        device.set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, self.probe_keep_free_bytes)
        device.set_option(GSB_OPT_ECC_HEALTH, 1 if self.health_ecc else 0)
        prober_keeps_arena = self.healthCheck and self.probe_period_ms > 0
        for i, uuid in enumerate(self._uuids):
            standing = False
            if self.probe_arena_bytes > 0:
                try:
                    device.arena_create(i, max_bytes=self.probe_arena_bytes, keep_free_bytes=self.probe_keep_free_bytes)
                    standing = True
                except GsbError as e:
                    log.warning("memtest of %s: no standing arena (%s): testing a transient window", uuid, e)
            r = device.memtest(i, raise_on_error=False)
            if standing and not prober_keeps_arena:
                device.arena_destroy(i)
            if r.n_elements == 0:  # nothing was tested (no memory to allocate, no usable device)
                log.warning("memtest of %s skipped: %s", uuid, last_error())
                continue
            line = device.memtest_text(r, uuid)
            if r.status == 0 and not any(r.elements[k].mismatch_words for k in range(r.n_elements)):
                log.info("%s", line)
                continue
            log.warning("%s: marking it unhealthy", line)
            first = device.fault_report(i, GSB_FAULT_REPORT_FIRST)
            if first.valid:
                log.warning("%s", device.fault_report_text(first, uuid))
            self.unhealthy([d for d in self.devs if d.ID.startswith(uuid + "-_-")])

    def run_startup_stress(self) -> None:
        """--startup-stress-ms N (not in the reference): N ms of full-rate, bit-checked tensor-core load on every SM of
        every GPU before the plugin serves or registers (after --startup-memtest), so a GPU that computes a wrong
        product under load is Unhealthy in the first ListAndWatch frame. The GPUs run at once, one thread each."""
        from .._abi import GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, last_error
        device.set_option(GSB_OPT_TRANSIENT_KEEP_FREE_BYTES, self.probe_keep_free_bytes)
        results: Dict[int, tuple] = {}

        def run(i: int) -> None:
            r = device.sm_stress(i, self.startup_stress_ms, raise_on_error=False)
            results[i] = (r, last_error())  # the library's error text is per thread
        threads = [threading.Thread(target=run, args=(i,)) for i in range(len(self._uuids))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for i, uuid in enumerate(self._uuids):
            r, err = results[i]
            if r.slices == 0:  # nothing ran (no memory to allocate, no usable device, a bad duration)
                log.warning("SM stress of %s skipped: %s", uuid, err)
                continue
            line = device.stress_text(r, uuid)
            if device.stress_conditions(r) == 0:
                log.info("%s", line)
                continue
            log.warning("%s: marking it unhealthy", line)
            self.unhealthy([d for d in self.devs if d.ID.startswith(uuid + "-_-")])

    def recovered(self, dev: nvidia.Device) -> None:
        with self._cv:
            e = ~self._index[dev.ID]
            self._apply(self._bits, e, True)
            self._pending.append(e)
            self._cv.notify_all()

    def healthcheck(self) -> None:
        if self.healthCheck:
            if self.probe_period_ms > 0:
                self.setup_probe_arenas(self.probe_keep_free_bytes)
            from .._abi import GSB_OPT_INVENTORY_REFRESH_MS, GSB_OPT_SWEEP_EVERY_CYCLES, GSB_OPT_WATCHDOG_MS
            device.set_option(GSB_OPT_SWEEP_EVERY_CYCLES, max(0, self.probe_sweep_every))
            device.set_option(GSB_OPT_WATCHDOG_MS, self.probe_watchdog_ms)
            device.set_option(GSB_OPT_INVENTORY_REFRESH_MS, self.inventory_refresh_ms)
            nvidia.watchXIDs(self.stop, self.devs, self.unhealthy, self.probe_period_ms, self.window_bytes,
                             self.recovered, self.health_recovery_cycles, self.health_ecc, self.probe_link_every,
                             self.probe_copy_every, self.probe_sm_every, self.probe_cluster_every,
                             self.probe_atomic_every, self.probe_tensor_every, self.probe_sfu_every,
                             self.probe_l1_every, self.probe_order_every, self.probe_sparse_every,
                             self.probe_shared_atomic_every)
        else:
            self.stop.wait()

    # ---- lifecycle ---------------------------------------------------------------------------
    def cleanup(self) -> None:  # server.go:195-201
        try:
            os.remove(self.socket)
        except FileNotFoundError:
            pass

    def Start(self) -> None:  # server.go:106-134
        self.cleanup()
        if self.startup_memtest:
            self.run_startup_memtest()
        if self.startup_stress_ms > 0:
            self.run_startup_stress()
        handlers = {
            "GetDevicePluginOptions": grpc.unary_unary_rpc_method_handler(self.GetDevicePluginOptions),
            "ListAndWatch": grpc.unary_stream_rpc_method_handler(self.ListAndWatch),
            "Allocate": grpc.unary_unary_rpc_method_handler(self.Allocate),
            "PreStartContainer": grpc.unary_unary_rpc_method_handler(self.PreStartContainer),
        }
        self.server = grpc.server(futures.ThreadPoolExecutor(max_workers=self.max_workers))
        self.server.add_generic_rpc_handlers((grpc.method_handlers_generic_handler(_SERVICE, handlers),))
        self.server.add_insecure_port("unix://" + self.socket)
        self.server.start()
        # wait for the server to come up with a blocking self-dial, 5 s (server.go:122-127)
        ch = grpc.insecure_channel("unix://" + self.socket)
        try:
            grpc.channel_ready_future(ch).result(timeout=5)
        finally:
            ch.close()
        self._health_thread = threading.Thread(target=self.healthcheck, name="healthcheck", daemon=True)
        self._health_thread.start()

    def Stop(self) -> None:  # server.go:137-147
        if self.server is None:
            return
        self.stop.set()
        if self.healthCheck:
            device.health_stop()  # wakes watchXIDs out of its 5 s wait (the reference's ctx cancel)
        with self._cv:
            self._cv.notify_all()
        self.server.stop(0)
        self.server = None
        # the health thread may be in the middle of a start-up walk: let it finish before anyone shuts the
        # device layer down or a new plugin starts its own health thread
        if self._health_thread is not None and self._health_thread is not threading.current_thread():
            self._health_thread.join(timeout=60)
        self.cleanup()

    def Register(self, kubeletEndpoint: str, resourceName: str) -> None:  # server.go:150-169
        ch = grpc.insecure_channel("unix://" + kubeletEndpoint)
        try:
            grpc.channel_ready_future(ch).result(timeout=5)
            req = device.encode_register_request(const.Version, os.path.basename(self.socket), resourceName)
            ch.unary_unary("/v1beta1.Registration/Register")(req, timeout=5)
        finally:
            ch.close()

    def Serve(self, kubeletSocket: str = const.KubeletSocket) -> None:  # server.go:224-241
        try:
            self.Start()
        except Exception as e:  # noqa: BLE001
            log.info("Could not start device plugin: %s", e)
            raise
        log.info("Starting to serve on %s", self.socket)
        try:
            self.Register(kubeletSocket, const.resourceName)
        except Exception as e:  # noqa: BLE001
            log.info("Could not register device plugin: %s", e)
            self.Stop()
            raise
        log.info("Registered device plugin with Kubelet")


def NewNvidiaDevicePlugin(mps: bool, healthCheck: bool, queryKubelet: bool, client, **kw) -> NvidiaDevicePlugin:
    return NvidiaDevicePlugin(mps, healthCheck, queryKubelet, client, **kw)
