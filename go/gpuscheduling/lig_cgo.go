// Package gpuscheduling is the Go side of the drop-in: a handlers.Scheduler backed by the
// H100 endpoint picker (include/lig.h) through cgo.
//
// UNVERIFIED IN THIS REPOSITORY'S BUILD IMAGE: there is no Go toolchain in it, so this package
// has never been compiled or run here.  It is written against the reference's interfaces at
// commit 8e96339 (handlers.Scheduler pkg/ext-proc/handlers/server.go:37-39,
// scheduling.PodMetricsProvider pkg/ext-proc/scheduling/scheduler.go:108-110) and against
// include/lig.h.  The natively compiled and GPU-tested counterpart of exactly this logic is the
// C++ host runtime in llm_instance_gateway_b200/csrc/host/ (see INTEGRATION.md).
package gpuscheduling

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../llm_instance_gateway_b200 -llig -Wl,-rpath,${SRCDIR}/../../llm_instance_gateway_b200
#include <stdlib.h>
#include "lig.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// ligError turns a negative lig_* return code into a Go error carrying lig_last_error().
func ligError(op string, rc C.int) error {
	if rc == 0 {
		return nil
	}
	return fmt.Errorf("%s: lig error %d: %s", op, int(rc), C.GoString(C.lig_last_error()))
}

// ctx wraps one lig_ctx (one CUDA device).
type ctx struct {
	p *C.lig_ctx
}

func newCtx(device, maxPods, maxAdapters, maxBatch int) (*ctx, error) {
	var p *C.lig_ctx
	if err := ligError("lig_create", C.lig_create(&p, C.int(device), C.int(maxPods), C.int(maxAdapters), C.int(maxBatch))); err != nil {
		return nil, err
	}
	return &ctx{p: p}, nil
}

func (c *ctx) close() {
	if c.p != nil {
		C.lig_destroy(c.p)
		c.p = nil
	}
}

// pinned is a page-locked, device-mapped buffer owned by the C side (lig_host_alloc); Go sees it
// as a slice but never hands Go-allocated memory to C, which keeps the cgo pointer rules trivial.
type pinned struct {
	ptr   unsafe.Pointer
	bytes int
}

func allocPinned(bytes int) (*pinned, error) {
	p := C.lig_host_alloc(C.size_t(bytes))
	if p == nil {
		return nil, fmt.Errorf("lig_host_alloc(%d): %s", bytes, C.GoString(C.lig_last_error()))
	}
	return &pinned{ptr: p, bytes: bytes}, nil
}

func (b *pinned) free() {
	if b.ptr != nil {
		C.lig_host_free(b.ptr)
		b.ptr = nil
	}
}

func (b *pinned) reqs(n int) []C.lig_req   { return unsafe.Slice((*C.lig_req)(b.ptr), n) }
func (b *pinned) picks(n int) []C.lig_pick { return unsafe.Slice((*C.lig_pick)(b.ptr), n) }

func (c *ctx) setThresholds(kv float64, qCritical, qLoRA int64) error {
	t := C.lig_thresholds{kv_cache_threshold: C.double(kv), queue_threshold_critical: C.int64_t(qCritical), queueing_threshold_lora: C.int64_t(qLoRA)}
	return ligError("lig_set_thresholds", C.lig_set_thresholds(c.p, &t))
}

// setFilterTree hands a caller flow chart to lig_set_filter_tree.  The node table is a Go slice of
// C structs without Go pointers, which cgo may pass for the duration of the call.
func (c *ctx) setFilterTree(nodes []FilterNode) error {
	cn := make([]C.lig_filter_node, len(nodes))
	for i, n := range nodes {
		cn[i] = C.lig_filter_node{kind: C.int32_t(n.Kind), next_on_success: C.int32_t(n.NextOnSuccess),
			next_on_failure: C.int32_t(n.NextOnFailure), next_on_success_or_failure: C.int32_t(n.NextOnSuccessOrFailure),
			queue_threshold: C.int64_t(n.QueueThreshold), kv_threshold: C.double(n.KVThreshold)}
	}
	return ligError("lig_set_filter_tree", C.lig_set_filter_tree(c.p, &cn[0], C.int(len(cn))))
}

// uploadSnapshot copies the packed columns into C memory for the duration of the call only
// (the library stages them into its own pinned blob before returning).
func (c *ctx) uploadSnapshot(epoch uint64, s *packedSnapshot) error {
	var kv *C.double
	var q *C.int32_t
	var na, ma *C.uint16_t
	var bm *C.uint32_t
	if s.P > 0 {
		kv = (*C.double)(unsafe.Pointer(&s.kv[0]))
		q = (*C.int32_t)(unsafe.Pointer(&s.q[0]))
		na = (*C.uint16_t)(unsafe.Pointer(&s.nActive[0]))
		ma = (*C.uint16_t)(unsafe.Pointer(&s.maxActive[0]))
		if len(s.bitmap) > 0 {
			bm = (*C.uint32_t)(unsafe.Pointer(&s.bitmap[0]))
		}
	}
	return ligError("lig_upload_snapshot", C.lig_upload_snapshot(c.p, C.uint64_t(epoch), C.int(s.P), C.int(s.A), kv, q, na, ma, bm))
}

func (c *ctx) scheduleBatch(epoch, seed uint64, in, out *pinned, n int) C.int {
	return C.lig_schedule_batch(c.p, C.uint64_t(epoch), C.uint64_t(seed), (*C.lig_req)(in.ptr), C.int(n), (*C.lig_pick)(out.ptr))
}

// scheduleBatchFeedbackChain is scheduleBatch through the load-feedback chain: windows of `window`
// requests counted across calls against one epoch (include/lig.h).
func (c *ctx) scheduleBatchFeedbackChain(epoch, seed uint64, in, out *pinned, n, window int) C.int {
	return C.lig_schedule_batch_feedback_chain(c.p, C.uint64_t(epoch), C.uint64_t(seed), (*C.lig_req)(in.ptr), C.int(n),
		(*C.lig_pick)(out.ptr), C.int(window), nil)
}
