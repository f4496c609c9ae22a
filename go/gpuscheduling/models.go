package gpuscheduling

/*
#include "lig.h"
*/
import "C"

import (
	"unsafe"

	"inference.networking.x-k8s.io/llm-instance-gateway/api/v1alpha1"
)

// UNVERIFIED (no Go toolchain in the build image), like the rest of this package.
//
// The model-id call: the resolve step of HandleRequestBody (pkg/ext-proc/handlers/request.go:42-56
// — FetchModelData, RandomWeightedDraw, IsCritical; pkg/ext-proc/backend/datastore.go:70-105) runs
// on the device.  A pending request is ONE uint32 model id; the answer is a 4-byte lig_mpick:
// pod index, status and the index of the drawn Spec.TargetModels entry (for the body's "model"
// rewrite, request.go:60-69).  4 + 4 bytes per decision over PCIe instead of 16 + 8.

// packedModels is the datastore's InferenceModels interned against one snapshot.
type packedModels struct {
	ids        map[string]uint32 // Spec.ModelName -> model id
	offsets    []int32           // CSR into the two target arrays, len = nModels+1
	adapterIDs []int32           // Spec.TargetModels[k].Name interned against the snapshot
	weights    []int32           // Spec.TargetModels[k].Weight
	critical   []uint8           // backend.IsCritical(model)
	selfIDs    []int32           // the model's own name interned (TargetModels empty, request.go:47)
	present    []uint8           // 0: requests for it get LIG_NO_MODEL
	targets    [][]string        // per model: TargetModels names, to map target_idx back to a name
	names      []string          // per model: the object's Name ("error getting target model name", request.go:49)
}

func packModels(models []*v1alpha1.InferenceModel, s *packedSnapshot) *packedModels {
	n := len(models)
	p := &packedModels{ids: make(map[string]uint32, n), offsets: make([]int32, n+1), critical: make([]uint8, n),
		selfIDs: make([]int32, n), present: make([]uint8, n), targets: make([][]string, n), names: make([]string, n)}
	for m, im := range models {
		p.ids[im.Spec.ModelName] = uint32(m)
		p.names[m] = im.Name
		p.present[m] = 1
		if im.Spec.Criticality != nil && *im.Spec.Criticality == v1alpha1.Critical { // datastore.go:100-105
			p.critical[m] = 1
		}
		p.selfIDs[m] = s.adapterID(im.Spec.ModelName)
		var sum int64
		for _, tm := range im.Spec.TargetModels {
			sum += int64(tm.Weight)
		}
		if len(im.Spec.TargetModels) > 0 && sum <= 0 {
			// Go's Int31n would panic (datastore.go:90); the CRD promises "no valid target model"
			p.present[m] = 0
		} else {
			for _, tm := range im.Spec.TargetModels {
				p.adapterIDs = append(p.adapterIDs, s.adapterID(tm.Name))
				p.weights = append(p.weights, tm.Weight)
				p.targets[m] = append(p.targets[m], tm.Name)
			}
		}
		p.offsets[m+1] = int32(len(p.adapterIDs))
	}
	return p
}

func i32ptr(v []int32) *C.int32_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&v[0]))
}

func u8ptr(v []uint8) *C.uint8_t {
	if len(v) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&v[0]))
}

// uploadModels attaches the model table to a resident snapshot epoch (once per refresh tick, or
// when the datastore changes).
func (c *ctx) uploadModels(epoch uint64, p *packedModels) error {
	return ligError("lig_upload_models", C.lig_upload_models(c.p, C.uint64_t(epoch), C.int(len(p.critical)),
		i32ptr(p.offsets), i32ptr(p.adapterIDs), i32ptr(p.weights), u8ptr(p.critical), i32ptr(p.selfIDs), u8ptr(p.present)))
}

func (b *pinned) modelIDs(n int) []C.uint32_t  { return unsafe.Slice((*C.uint32_t)(b.ptr), n) }
func (b *pinned) mpicks(n int) []C.lig_mpick   { return unsafe.Slice((*C.lig_mpick)(b.ptr), n) }

// scheduleModels is one flushed batch through the model-id call.  firstIndex makes the
// per-request random streams unique across flushes (rand_key = firstIndex + i).
func (c *ctx) scheduleModels(epoch, seed, firstIndex uint64, in, out *pinned, n int) C.int {
	return C.lig_schedule_models_batch(c.p, C.uint64_t(epoch), C.uint64_t(seed), C.uint64_t(firstIndex),
		(*C.uint32_t)(in.ptr), C.int(n), (*C.lig_mpick)(out.ptr))
}

// scheduleModelsFeedbackChain is scheduleModels inside the load-feedback chain (Options.LoadFeedbackWindow):
// model-id and descriptor requests share its windows.
func (c *ctx) scheduleModelsFeedbackChain(epoch, seed, firstIndex uint64, in, out *pinned, n, window int) C.int {
	return C.lig_schedule_models_batch_feedback_chain(c.p, C.uint64_t(epoch), C.uint64_t(seed), C.uint64_t(firstIndex),
		(*C.uint32_t)(in.ptr), C.int(n), (*C.lig_mpick)(out.ptr), C.int(window), nil)
}

// group wraps lig_group: ONE scheduler per ext-proc process owning several GPUs (main.go:137); the
// snapshot broadcast (NCCL) and the request sharding happen inside the library.
type group struct {
	p *C.lig_group
}

func newGroup(devices []int, maxPods, maxAdapters, maxBatch int) (*group, error) {
	devs := make([]C.int, len(devices))
	for i, d := range devices {
		devs[i] = C.int(d)
	}
	var p *C.lig_group
	if err := ligError("lig_group_create", C.lig_group_create(&p, &devs[0], C.int(len(devs)), C.int(maxPods), C.int(maxAdapters), C.int(maxBatch))); err != nil {
		return nil, err
	}
	return &group{p: p}, nil
}

func (g *group) close() {
	if g.p != nil {
		C.lig_group_destroy(g.p)
		g.p = nil
	}
}

func (g *group) uploadSnapshot(epoch uint64, s *packedSnapshot) error {
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
	return ligError("lig_group_upload_snapshot", C.lig_group_upload_snapshot(g.p, C.uint64_t(epoch), C.int(s.P), C.int(s.A), kv, q, na, ma, bm))
}

func (g *group) scheduleBatch(epoch, seed uint64, in, out *pinned, n int) C.int {
	return C.lig_group_schedule_batch(g.p, C.uint64_t(epoch), C.uint64_t(seed), (*C.lig_req)(in.ptr), C.int(n), (*C.lig_pick)(out.ptr))
}
