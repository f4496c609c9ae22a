package gpuscheduling

import (
	"math"

	"inference.networking.x-k8s.io/llm-instance-gateway/pkg/ext-proc/backend"
)

// packedSnapshot is one refresh tick of PodMetricsProvider.AllPodMetrics() in the column layout
// include/lig.h describes.  The slice order of the provider IS the pod index: picks come back as
// indices into pods.
type packedSnapshot struct {
	epoch      uint64
	P, A       int
	kv         []float64
	q          []int32
	nActive    []uint16
	maxActive  []uint16
	bitmap     []uint32 // adapter-major, A x ceil(P/32)
	adapterIDs map[string]int32
	pods       []backend.Pod
	excluded   int // pods left out of this snapshot: a metric did not fit the device record
	models     *packedModels // Options.InferenceModels interned against this epoch; nil: none
}

// packSnapshot interns adapter names (order of first appearance) and narrows the Go-width
// metrics to the device record.  A pod whose WaitingQueueSize does not fit int32 or that lists
// more than 65534 active models cannot be represented: it is LEFT OUT of this snapshot and
// counted (never a silent wrap, and never a failed tick that would freeze the whole pool on a
// stale snapshot).  MaxActiveModels saturates to [0, 65535], which cannot change
// len(ActiveModels) < MaxActiveModels because len(ActiveModels) <= 65534.
func packSnapshot(in []*backend.PodMetrics) (*packedSnapshot, error) {
	all := make([]*backend.PodMetrics, 0, len(in))
	for _, pm := range in {
		if pm.WaitingQueueSize > math.MaxInt32 || pm.WaitingQueueSize < math.MinInt32 || len(pm.ActiveModels) > 65534 {
			continue
		}
		all = append(all, pm)
	}
	P := len(all)
	W := (P + 31) / 32
	s := &packedSnapshot{
		P: P, kv: make([]float64, P), q: make([]int32, P), nActive: make([]uint16, P),
		maxActive: make([]uint16, P), adapterIDs: map[string]int32{}, pods: make([]backend.Pod, P),
		excluded: len(in) - len(all),
	}
	for i, pm := range all {
		s.pods[i] = pm.Pod
		s.kv[i] = pm.KVCacheUsagePercent
		s.q[i] = int32(pm.WaitingQueueSize)
		s.nActive[i] = uint16(len(pm.ActiveModels))
		switch m := pm.MaxActiveModels; {
		case m < 0:
			s.maxActive[i] = 0
		case m > 65535:
			s.maxActive[i] = 65535
		default:
			s.maxActive[i] = uint16(m)
		}
		for name := range pm.ActiveModels {
			if _, ok := s.adapterIDs[name]; !ok {
				s.adapterIDs[name] = int32(len(s.adapterIDs))
			}
		}
	}
	s.A = len(s.adapterIDs)
	s.bitmap = make([]uint32, s.A*W)
	for i, pm := range all {
		for name := range pm.ActiveModels {
			s.bitmap[int(s.adapterIDs[name])*W+i>>5] |= 1 << (uint(i) & 31)
		}
	}
	return s, nil
}

// adapterID resolves ResolvedTargetModel; a model in no pod's ActiveModels gets id A, which
// matches no bitmap row — the same outcome as the Go map miss in loRAAffinityPredicate.
func (s *packedSnapshot) adapterID(model string) int32 {
	if id, ok := s.adapterIDs[model]; ok {
		return id
	}
	return int32(s.A)
}
