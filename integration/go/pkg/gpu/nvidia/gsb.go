// +build linux

package nvidia

// Thin cgo shim over libgpushare_b200.so (include/gpushare_b200.h). NOT compiled in this repository:
// there is no Go toolchain in the build image. The same entry points are exercised by the ctypes
// binding and by the native daemon.

// #cgo CFLAGS: -I${SRCDIR}/../../../include
// #cgo LDFLAGS: -L${SRCDIR}/../../../lib -lgpushare_b200 -Wl,-rpath,$ORIGIN/../lib
// #include <stdlib.h>
// #include "gpushare_b200.h"
import "C"

import (
	"errors"
	"fmt"
	"unsafe"
)

func gsbErr(rc C.int) error {
	if rc >= 0 {
		return nil
	}
	var buf [512]C.char
	C.gsb_last_error(&buf[0], C.size_t(len(buf)))
	if rc == C.GSB_ERR_LIBRARY_NOT_FOUND {
		// same text nvml.Init() returns (vendor/.../nvml/bindings.go:63)
		return errors.New("could not load NVML library")
	}
	return fmt.Errorf("%s: %s", C.GoString(C.gsb_strerror(rc)), C.GoString(&buf[0]))
}

// gsbInit / gsbShutdown replace nvml.Init / nvml.Shutdown (gpumanager.go:36,41).
func gsbInit() error     { return gsbErr(C.gsb_init()) }
func gsbShutdown() error { return gsbErr(C.gsb_shutdown()) }

func gsbDeviceCount() (uint, error) {
	var n C.uint32_t
	err := gsbErr(C.gsb_device_count(&n))
	return uint(n), err
}

// gsbDevice carries the three fields of nvml.Device the plugin consumes (nvidia.go:64-71).
type gsbDevice struct {
	UUID   string
	Path   string // "/dev/nvidia<minor>"
	Memory uint64 // MiB == *nvml.Device.Memory
}

func gsbNewDevice(idx uint) (*gsbDevice, error) {
	var info C.gsb_device_info
	if err := gsbErr(C.gsb_device_info_get(C.uint32_t(idx), &info)); err != nil {
		return nil, err
	}
	return &gsbDevice{
		UUID:   C.GoString(&info.uuid[0]),
		Path:   fmt.Sprintf("/dev/nvidia%d", uint(info.minor)),
		Memory: uint64(info.total_mib),
	}, nil
}

// gsbRefreshInventory re-reads every GPU's identity + memory from NVML into the library's snapshot. gsbNewDevice does
// that per device already, so a plugin that builds its list through gsbNewDevice at every (re)start — as
// NewNvidiaDevicePlugin does (server.go:39) — needs it only to force a refresh outside a restart.
func gsbRefreshInventory() error { return gsbErr(C.gsb_inventory_refresh(C.GSB_ALL_DEVICES)) }

// Options (include/gpushare_b200.h, GSB_OPT_*): inventory policy of the cycle, completion-wait spin budget, probe
// watchdog, off-path NVML refresh period, HBM a transient probe window never takes.
func gsbSetOption(key uint32, value uint64) error {
	return gsbErr(C.gsb_set_option(C.uint32_t(key), C.uint64_t(value)))
}

// gsbSlices is setGPUMemory's arithmetic (nvidia.go:34-41).
func gsbSlices(totalMiB uint64, gib bool) uint {
	unit := C.int(0)
	if gib {
		unit = 1
	}
	return uint(C.gsb_slices(C.uint64_t(totalMiB), unit))
}

type gsbEvent struct {
	UUID  string
	Etype uint64
	Edata uint64
}

const (
	gsbEventXID       = uint64(C.GSB_EVENT_XID)       // == nvml.XidCriticalError
	gsbEventProbe     = uint64(C.GSB_EVENT_PROBE)     // verdict of the active HBM probe (mismatch, failed launch, wedged)
	gsbEventInventory = uint64(C.GSB_EVENT_INVENTORY) // the off-path NVML refresh disagrees with what is advertised
	gsbEventECC       = uint64(C.GSB_EVENT_ECC)       // opt-in ECC health: Edata = one of the gsbECC* conditions below
	gsbEventLink      = uint64(C.GSB_EVENT_LINK)      // opt-in PCIe link health: Edata = one of the gsbLink* conditions below
	gsbEventCopy      = uint64(C.GSB_EVENT_COPY)      // opt-in copy-engine health: Edata = one of the gsbCopy* conditions below
	gsbEventSM        = uint64(C.GSB_EVENT_SM)        // opt-in SM compute health: Edata = one of the gsbSM* conditions below
	gsbEventCluster   = uint64(C.GSB_EVENT_CLUSTER)   // opt-in SM-to-SM health: Edata = one of the gsbCluster* conditions below
	gsbEventAtomic    = uint64(C.GSB_EVENT_ATOMIC)    // opt-in L2 atomic health: Edata = one of the gsbAtomic* conditions below
	gsbEventTensor    = uint64(C.GSB_EVENT_TENSOR)    // opt-in tensor-core format health: Edata = one of the gsbTensor* conditions below
	gsbEventSFU       = uint64(C.GSB_EVENT_SFU)       // opt-in SM special-function health: Edata = one of the gsbSFU* conditions below
	gsbEventL1        = uint64(C.GSB_EVENT_L1)        // opt-in L1 and constant-cache health: Edata = one of the gsbL1* conditions below
	gsbEventOrder     = uint64(C.GSB_EVENT_ORDER)     // opt-in memory-ordering health: Edata = one of the gsbOrder* conditions below
	gsbEventSparse    = uint64(C.GSB_EVENT_SPARSE)    // opt-in sparse tensor-core health: Edata = one of the gsbSparse* conditions below
	gsbEventSharedAtomic = uint64(C.GSB_EVENT_SHARED_ATOMIC) // opt-in shared-memory atomic health: Edata = one of the gsbSharedAtomic* conditions below
)

const (
	gsbLinkCorrupt       = uint64(C.GSB_LINK_CORRUPT)        // a link phase read back a word the GPU did not write
	gsbLinkFailed        = uint64(C.GSB_LINK_FAILED)         // a link phase failed or outlived the watchdog
	gsbLinkWidthDegraded = uint64(C.GSB_LINK_WIDTH_DEGRADED) // the width under load is below the link's maximum
	gsbLinkSpeedDegraded = uint64(C.GSB_LINK_SPEED_DEGRADED) // the generation under load is below the link's maximum
)

const (
	gsbCopyCorrupt = uint64(C.GSB_COPY_CORRUPT) // a DMA copy left a destination byte other than it must, in range or in a guard
	gsbCopyFailed  = uint64(C.GSB_COPY_FAILED)  // a copy or its verify failed or outlived the watchdog
)

const (
	gsbSMCorrupt = uint64(C.GSB_SM_CORRUPT) // a result word differs from its exact answer on some SM
	gsbSMFailed  = uint64(C.GSB_SM_FAILED)  // an SM-check launch failed or outlived the watchdog
)

const (
	gsbClusterCorrupt = uint64(C.GSB_CLUSTER_CORRUPT) // a word that crossed the SM-to-SM network differs from its pattern
	gsbClusterFailed  = uint64(C.GSB_CLUSTER_FAILED)  // a launch failed or outlived the watchdog, or a transfer never completed
)

const (
	gsbAtomicCorrupt = uint64(C.GSB_ATOMIC_CORRUPT) // a final word, a ticket or a ticket slot of an L2 atomic is wrong
	gsbAtomicFailed  = uint64(C.GSB_ATOMIC_FAILED)  // a launch failed or outlived the watchdog, or a CAS loop ran out
)

const (
	gsbTensorCorrupt = uint64(C.GSB_TENSOR_CORRUPT) // a D word of a tensor-core form differs from its exact answer on some SM
	gsbTensorFailed  = uint64(C.GSB_TENSOR_FAILED)  // a tensor-check launch failed or outlived the watchdog
)

const (
	gsbSFUCorrupt = uint64(C.GSB_SFU_CORRUPT) // a conversion, divide, warp-collective or MUFU result is wrong on some SM
	gsbSFUBound   = uint64(C.GSB_SFU_BOUND)   // a MUFU result every SM agrees on lies outside its envelope
	gsbSFUFailed  = uint64(C.GSB_SFU_FAILED)  // an SFU-check launch failed or outlived the watchdog
)

const (
	gsbL1Corrupt = uint64(C.GSB_L1_CORRUPT) // a word read through L1, texture, constant bank or kernel parameters is wrong on some SM
	gsbL1Failed  = uint64(C.GSB_L1_FAILED)  // an L1-check launch failed or outlived the watchdog
)

const (
	gsbOrderCorrupt   = uint64(C.GSB_ORDER_CORRUPT)   // a word read back between SMs is not one any writer stored
	gsbOrderForbidden = uint64(C.GSB_ORDER_FORBIDDEN) // an outcome the PTX memory model forbids at .gpu scope
	gsbOrderLost      = uint64(C.GSB_ORDER_LOST)      // a store not visible after the grid barrier
	gsbOrderTimeout   = uint64(C.GSB_ORDER_TIMEOUT)   // a grid barrier ran out: an SM stalled or a store never became visible
	gsbOrderFailed    = uint64(C.GSB_ORDER_FAILED)    // a memory-ordering launch failed or outlived the watchdog
	gsbSparseCorrupt  = uint64(C.GSB_SPARSE_CORRUPT)  // a sparse tensor-core D word differs from its exact answer on some SM
	gsbSparseFailed   = uint64(C.GSB_SPARSE_FAILED)   // a sparse tensor-core launch failed or outlived the watchdog
	gsbSharedAtomicCorrupt = uint64(C.GSB_SHARED_ATOMIC_CORRUPT) // a shared-memory atomic left a wrong word, slot, ticket or pair on some SM
	gsbSharedAtomicFailed  = uint64(C.GSB_SHARED_ATOMIC_FAILED)  // a shared-memory atomic launch failed, or a CAS loop or red.async wait ran out
)

const (
	gsbECCRemapPending = uint64(C.GSB_ECC_REMAP_PENDING) // a row remap waits for a GPU reset
	gsbECCRemapFailure = uint64(C.GSB_ECC_REMAP_FAILURE) // a row remap failed: no spare rows left
	gsbECCUncorrected  = uint64(C.GSB_ECC_UNCORRECTED)   // the volatile uncorrected count rose since the start
)

// gsbEnableECCHealth turns on ECC and row-remapper health; call it before gsbHealthStart.
func gsbEnableECCHealth() error { return gsbErr(C.gsb_set_option(C.GSB_OPT_ECC_HEALTH, 1)) }

// gsbECCStatusLine is the one log line of GPU idx's live ECC status ("unknown" for every field that cannot be read):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_ECC event.
func gsbECCStatusLine(idx uint, uuid string) string {
	var st C.gsb_ecc_status
	if C.gsb_ecc_status_get(C.uint32_t(idx), &st) != C.GSB_OK {
		st = C.gsb_ecc_status{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_ecc_status_text(&st, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_ecc_status_text(&st, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbECCStats is what the prober attributed to device idx since gsbHealthStart: corrected errors during its walks and
// between them, and the window of the last walk that surfaced any.
func gsbECCStats(idx uint) (C.gsb_ecc_stats, error) {
	var st C.gsb_ecc_stats
	err := gsbErr(C.gsb_ecc_stats_get(C.uint32_t(idx), &st))
	return st, err
}

// gsbMemtest runs March C- on GPU idx before it is advertised: the whole standing arena if one exists, otherwise all
// allocatable HBM but the keep-free margin. bad is true when an element found mismatches or failed; line is the one
// log line for the result, and first the FIRST fault report's line when bad (else "").
func gsbMemtest(idx uint, uuid string) (bad bool, line, first string, err error) {
	var cfg C.gsb_memtest_cfg
	var r C.gsb_memtest_result
	rc := C.gsb_memtest(C.uint32_t(idx), &cfg, &r)
	if r.n_elements == 0 {
		return false, "", "", gsbErr(rc)
	}
	bad = rc != C.GSB_OK
	for k := 0; k < int(r.n_elements); k++ {
		bad = bad || r.elements[k].mismatch_words != 0
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	if need := C.gsb_memtest_text(&r, cu, nil, 0); need > 0 {
		buf := make([]byte, int(need))
		if n := C.gsb_memtest_text(&r, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf))); n >= 0 {
			line = string(buf[:int(n)])
		}
	}
	if bad {
		var rep C.gsb_fault_report
		if C.gsb_fault_report_get(C.uint32_t(idx), C.GSB_FAULT_REPORT_FIRST, &rep) == C.GSB_OK && rep.valid != 0 {
			if need := C.gsb_fault_report_text(&rep, cu, nil, 0); need > 0 {
				buf := make([]byte, int(need))
				if n := C.gsb_fault_report_text(&rep, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf))); n >= 0 {
					first = string(buf[:int(n)])
				}
			}
		}
	}
	return bad, line, first, nil
}

// gsbHealthStart replaces NewEventSet + the RegisterEventForDevice loop (nvidia.go:101-117).
func gsbHealthStart(probePeriodMs uint, windowBytes uint64) error {
	return gsbErr(C.gsb_health_start(C.uint32_t(probePeriodMs), C.uint64_t(windowBytes)))
}

func gsbHealthStop() { C.gsb_health_stop() }

// gsbWaitForEvent replaces nvml.WaitForEvent (nvidia.go:126). (nil, nil) == timeout.
// cgo releases the P while the call blocks: one OS thread, like the reference's.
func gsbWaitForEvent(timeoutMs uint) (*gsbEvent, error) {
	var ev C.gsb_event
	rc := C.gsb_health_wait(C.uint32_t(timeoutMs), &ev)
	if rc == C.GSB_ERR_TIMEOUT || rc == C.GSB_ERR_STOPPED {
		return nil, nil
	}
	if err := gsbErr(rc); err != nil {
		return nil, err
	}
	return &gsbEvent{C.GoString(&ev.uuid[0]), uint64(ev.etype), uint64(ev.edata)}, nil
}

func gsbXidIsBenign(xid uint64) bool { return C.gsb_xid_is_benign(C.uint64_t(xid)) != 0 }

const (
	gsbProbeFaultMismatch = uint64(C.GSB_PROBE_FAULT_MISMATCH)
	gsbFaultReportFirst   = uint32(C.GSB_FAULT_REPORT_FIRST) // first fault since start (or since RECOVERED)
	gsbFaultReportLast    = uint32(C.GSB_FAULT_REPORT_LAST)  // most recent faulted launch
)

// gsbFaultReportLine is the one log line of GPU idx's FIRST or LAST HBM fault report ("" when there is none): what a
// plugin logs before marking a GPU unhealthy on a PROBE / GSB_PROBE_FAULT_MISMATCH event.
func gsbFaultReportLine(idx uint, which uint32, uuid string) string {
	var r C.gsb_fault_report
	if C.gsb_fault_report_get(C.uint32_t(idx), C.uint32_t(which), &r) != C.GSB_OK || r.valid == 0 {
		return ""
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_fault_report_text(&r, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_fault_report_text(&r, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbArenaCreate maps the memory the probe walks; returns what was actually allocatable.
func gsbArenaCreate(idx uint, maxBytes, keepFreeBytes uint64) (uint64, error) {
	var got C.uint64_t
	err := gsbErr(C.gsb_arena_create(C.uint32_t(idx), C.uint64_t(maxBytes), C.uint64_t(keepFreeBytes), &got))
	return uint64(got), err
}

// gsbCycle runs one inventory + health-probe cycle of one device; lw receives the ListAndWatchResponse bytes. With no
// arena on the device and windowBytes > 0 the cycle probes a transient window (allocate -> fill -> verify -> free).
func gsbCycle(idx uint, cycle uint64, windowBytes uint64, lw []byte) (healthy bool, lwLen int, err error) {
	var res C.gsb_cycle_result
	rc := C.gsb_cycle(C.uint32_t(idx), C.uint64_t(cycle), C.uint64_t(windowBytes), 1, C.GSB_VARIANT_AUTO,
		(*C.uint8_t)(unsafe.Pointer(&lw[0])), C.size_t(len(lw)), &res)
	return res.healthy == 1, int(res.lw_len), gsbErr(rc)
}

// gsbPod is the handful of fields Allocate's pod selection reads (podutils.go:37-131, podmanager.go:187-201).
type gsbPod struct {
	Name, Namespace, UID string
	GPUMemLimit          uint64 // sum of spec.containers[].resources.limits["aliyun.com/gpu-mem"]
	AssumeTime           uint64 // ALIYUN_COM_GPU_MEM_ASSUME_TIME, 0 when absent or unparsable
	GPUIdx               int32  // ALIYUN_COM_GPU_MEM_IDX, -1 when absent or unparsable
	HasAssumeTime        bool
	HasAssigned          bool
	AssignedIsFalse      bool
	OnNode               bool
}

const (
	gsbAllocMatched     = int(C.GSB_ALLOC_MATCHED)      // PATCH pods[podIndex], then answer with resp
	gsbAllocSingleGPU   = int(C.GSB_ALLOC_SINGLE_GPU)   // allocate.go:151-177
	gsbAllocErrResponse = int(C.GSB_ALLOC_ERR_RESPONSE) // allocate.go:24-39
)

// gsbAllocate is the optional fast path for allocate.go:54-128: request bytes in (the gogo-marshalled
// AllocateRequest), response bytes out, and which pending pod to PATCH. The LIST before it and the PATCH after it
// stay in Go (podmanager.go:125-160, allocate.go:130-149). uuids/minors are devNameMap in NVML order.
func gsbAllocate(uuids []string, minors []uint32, slices uint, gib, disableCGPU bool, pods []gsbPod, req []byte) (kind int, resp []byte, podIndex int, err error) {
	cu := make([]*C.char, len(uuids))
	for i, u := range uuids {
		cu[i] = C.CString(u)
		defer C.free(unsafe.Pointer(cu[i]))
	}
	cm := make([]C.uint32_t, len(minors))
	for i, m := range minors {
		cm[i] = C.uint32_t(m)
	}
	b2i := func(b bool) C.int32_t {
		if b {
			return 1
		}
		return 0
	}
	// C memory for everything the C side keeps pointers to during the call (cgo forbids Go pointers to Go pointers)
	ctx := (*C.gsb_allocate_ctx)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_allocate_ctx{}))))
	defer C.free(unsafe.Pointer(ctx))
	cuArr := (**C.char)(C.calloc(C.size_t(len(cu)+1), C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(cuArr))
	cmArr := (*C.uint32_t)(C.calloc(C.size_t(len(cm)+1), 4))
	defer C.free(unsafe.Pointer(cmArr))
	copy(unsafe.Slice(cuArr, len(cu)), cu)
	copy(unsafe.Slice(cmArr, len(cm)), cm)
	ctx.uuids, ctx.minors, ctx.n_gpus = cuArr, cmArr, C.uint32_t(len(uuids))
	ctx.slices, ctx.unit_gib, ctx.disable_cgpu_isolation = C.uint32_t(slices), b2i(gib), b2i(disableCGPU)

	cp := (*C.gsb_pod)(C.calloc(C.size_t(len(pods)+1), C.size_t(unsafe.Sizeof(C.gsb_pod{}))))
	defer C.free(unsafe.Pointer(cp))
	cps := unsafe.Slice(cp, len(pods))
	b2u := func(b bool) C.uint8_t {
		if b {
			return 1
		}
		return 0
	}
	for i, p := range pods {
		name, ns, uid := C.CString(p.Name), C.CString(p.Namespace), C.CString(p.UID)
		defer C.free(unsafe.Pointer(name))
		defer C.free(unsafe.Pointer(ns))
		defer C.free(unsafe.Pointer(uid))
		cps[i].name, cps[i].ns, cps[i].uid = name, ns, uid
		cps[i].gpu_mem_limit, cps[i].assume_time, cps[i].gpu_idx = C.uint64_t(p.GPUMemLimit), C.uint64_t(p.AssumeTime), C.int32_t(p.GPUIdx)
		cps[i].has_assume_time, cps[i].has_assigned = b2u(p.HasAssumeTime), b2u(p.HasAssigned)
		cps[i].assigned_is_false, cps[i].on_node = b2u(p.AssignedIsFalse), b2u(p.OnNode)
	}
	out := make([]byte, 64<<10)
	var n C.size_t
	var idx C.int32_t
	var podReq C.uint32_t
	var reqPtr *C.uint8_t
	if len(req) > 0 {
		reqPtr = (*C.uint8_t)(unsafe.Pointer(&req[0]))
	}
	rc := C.gsb_allocate(ctx, cp, C.uint32_t(len(pods)), reqPtr, C.size_t(len(req)),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), C.size_t(len(out)), &n, &idx, &podReq)
	if rc < 0 {
		return 0, nil, -1, gsbErr(rc)
	}
	return int(rc), out[:int(n)], int(idx), nil
}

// gsbEncodeListAndWatch produces the bytes gogo's Marshal would for the list getDevices() builds (server.go:173,182);
// unhealthy is a bitmap over (gpu*slices + j). Use with a raw-bytes grpc codec, or keep gogo: the bytes are identical.
func gsbEncodeListAndWatch(uuids []string, slices uint, unhealthy []byte) ([]byte, error) {
	cu := (**C.char)(C.calloc(C.size_t(len(uuids)+1), C.size_t(unsafe.Sizeof(uintptr(0)))))
	defer C.free(unsafe.Pointer(cu))
	for i, u := range uuids {
		s := C.CString(u)
		defer C.free(unsafe.Pointer(s))
		unsafe.Slice(cu, len(uuids))[i] = s
	}
	var bits *C.uint8_t
	if len(unhealthy) > 0 {
		bits = (*C.uint8_t)(unsafe.Pointer(&unhealthy[0]))
	}
	need := C.gsb_encode_list_and_watch(cu, C.uint32_t(len(uuids)), C.uint32_t(slices), bits, nil, 0)
	if need < 0 && C.int(need) != C.GSB_ERR_BUFFER_TOO_SMALL {
		return nil, gsbErr(C.int(need))
	}
	buf := make([]byte, (len(uuids)*int(slices))*64+16)
	n := C.gsb_encode_list_and_watch(cu, C.uint32_t(len(uuids)), C.uint32_t(slices), bits, (*C.uint8_t)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return nil, gsbErr(C.int(n))
	}
	return buf[:int(n)], nil
}

// gsbEnableLinkHealth turns on PCIe link health: each prober runs gsb_link_probe after its first cycle of a session and
// after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableLinkHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_LINK_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbLinkLine is the one log line of GPU idx's most recent link probe ("unknown" for every reading there is none of):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_LINK event.
func gsbLinkLine(idx uint, uuid string) string {
	var st C.gsb_link_stats
	if C.gsb_link_stats_get(C.uint32_t(idx), &st) != C.GSB_OK {
		st = C.gsb_link_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_link_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_link_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableCopyHealth turns on copy-engine health: each prober runs gsb_copy_probe after its first cycle of a session
// and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableCopyHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_COPY_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbCopyLine is the one log line of GPU idx's most recent copy probe ("not run" when there is none): what a plugin
// logs before marking a GPU unhealthy on a GSB_EVENT_COPY event.
func gsbCopyLine(idx uint, uuid string) string {
	var st C.gsb_copy_stats
	if C.gsb_copy_stats_get(C.uint32_t(idx), &st) != C.GSB_OK {
		st = C.gsb_copy_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_copy_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_copy_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableSMHealth turns on SM compute health: each prober runs gsb_sm_probe after its first cycle of a session and
// after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableSMHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_SM_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbSMLine is the one log line of GPU idx's most recent SM probe ("not run" when there is none): what a plugin logs
// before marking a GPU unhealthy on a GSB_EVENT_SM event.
func gsbSMLine(idx uint, uuid string) string {
	var st C.gsb_sm_stats
	if C.gsb_sm_stats_get(C.uint32_t(idx), &st) != C.GSB_OK {
		st = C.gsb_sm_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_sm_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_sm_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableClusterHealth turns on SM-to-SM health: each prober runs gsb_cluster_probe after its first cycle of a
// session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableClusterHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_CLUSTER_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbClusterLine is the one log line of GPU idx's most recent SM-to-SM probe ("not run" when there is none): what a
// plugin logs before marking a GPU unhealthy on a GSB_EVENT_CLUSTER event.
func gsbClusterLine(idx uint, uuid string) string {
	st := (*C.gsb_cluster_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_cluster_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_cluster_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_cluster_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_cluster_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_cluster_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableAtomicHealth turns on L2 atomic health: each prober runs gsb_atomic_probe after its first cycle of a
// session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableAtomicHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_ATOMIC_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbAtomicLine is the one log line of GPU idx's most recent L2 atomic probe ("not run" when there is none): what a
// plugin logs before marking a GPU unhealthy on a GSB_EVENT_ATOMIC event.
func gsbAtomicLine(idx uint, uuid string) string {
	st := (*C.gsb_atomic_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_atomic_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_atomic_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_atomic_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_atomic_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_atomic_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableTensorHealth turns on tensor-core format health: each prober runs gsb_tensor_probe after its first cycle
// of a session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableTensorHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_TENSOR_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbTensorLine is the one log line of GPU idx's most recent tensor-core format probe ("not run" when there is none):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_TENSOR event.
func gsbTensorLine(idx uint, uuid string) string {
	st := (*C.gsb_tensor_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_tensor_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_tensor_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_tensor_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_tensor_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_tensor_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableSFUHealth turns on SM special-function health: each prober runs gsb_sfu_probe after its first cycle of a
// session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableSFUHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_SFU_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbSFULine is the one log line of GPU idx's most recent SM special-function probe ("not run" when there is none):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_SFU event.
func gsbSFULine(idx uint, uuid string) string {
	st := (*C.gsb_sfu_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_sfu_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_sfu_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_sfu_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_sfu_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_sfu_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableL1Health turns on L1 and constant-cache health: each prober runs gsb_l1_probe after its first cycle of a
// session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableL1Health(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_L1_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbL1Line is the one log line of GPU idx's most recent L1 and constant-cache probe ("not run" when there is none):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_L1 event.
func gsbL1Line(idx uint, uuid string) string {
	st := (*C.gsb_l1_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_l1_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_l1_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_l1_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_l1_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_l1_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableOrderHealth turns on memory-ordering health: each prober runs gsb_order_probe after its first cycle of a
// session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableOrderHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_ORDER_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbOrderLine is the one log line of GPU idx's most recent memory-ordering probe ("not run" when there is none):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_ORDER event.
func gsbOrderLine(idx uint, uuid string) string {
	st := (*C.gsb_order_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_order_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_order_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_order_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_order_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_order_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableSparseHealth turns on sparse tensor-core health: each prober runs gsb_sparse_probe after its first cycle
// of a session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableSparseHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_SPARSE_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbSparseLine is the one log line of GPU idx's most recent sparse tensor-core probe ("not run" when there is none):
// what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_SPARSE event.
func gsbSparseLine(idx uint, uuid string) string {
	st := (*C.gsb_sparse_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_sparse_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_sparse_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_sparse_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_sparse_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_sparse_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbEnableSharedAtomicHealth turns on shared-memory atomic health: each prober runs gsb_shared_atomic_probe after its
// first cycle of a session and after every `every`-th cycle. Call it before gsbHealthStart.
func gsbEnableSharedAtomicHealth(every uint64) error {
	return gsbErr(C.gsb_set_option(C.GSB_OPT_SHARED_ATOMIC_PROBE_EVERY_CYCLES, C.uint64_t(every)))
}

// gsbSharedAtomicLine is the one log line of GPU idx's most recent shared-memory atomic probe ("not run" when there is
// none): what a plugin logs before marking a GPU unhealthy on a GSB_EVENT_SHARED_ATOMIC event.
func gsbSharedAtomicLine(idx uint, uuid string) string {
	st := (*C.gsb_shared_atomic_stats)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gsb_shared_atomic_stats{}))))
	defer C.free(unsafe.Pointer(st))
	if C.gsb_shared_atomic_stats_get(C.uint32_t(idx), st) != C.GSB_OK {
		*st = C.gsb_shared_atomic_stats{}
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_shared_atomic_text(&st.last, cu, nil, 0)
	if need <= 0 {
		return ""
	}
	buf := make([]byte, int(need))
	n := C.gsb_shared_atomic_text(&st.last, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf)))
	if n < 0 {
		return ""
	}
	return string(buf[:int(n)])
}

// gsbStress runs the SM stress on GPU idx for durationMs (full-rate tensor-core GEMMs on every SM, every result bit
// checked), as --startup-stress-ms does before Register: line is the log line, bad is true when the run found a wrong
// word or a slice failed. Run one goroutine per GPU so start-up grows by durationMs, not by GPUs x durationMs.
func gsbStress(idx uint, uuid string, durationMs uint32) (line string, bad bool, err error) {
	cfg := C.gsb_stress_cfg{duration_ms: C.uint32_t(durationMs)}
	var r C.gsb_stress_result
	rc := C.gsb_sm_stress(C.uint32_t(idx), &cfg, &r)
	if r.slices == 0 {
		return "", false, gsbErr(rc)
	}
	cu := C.CString(uuid)
	defer C.free(unsafe.Pointer(cu))
	need := C.gsb_stress_text(&r, cu, nil, 0)
	if need > 0 {
		buf := make([]byte, int(need))
		if n := C.gsb_stress_text(&r, cu, (*C.char)(unsafe.Pointer(&buf[0])), C.size_t(len(buf))); n >= 0 {
			line = string(buf[:int(n)])
		}
	}
	return line, C.gsb_stress_conditions(&r) != 0, nil
}
