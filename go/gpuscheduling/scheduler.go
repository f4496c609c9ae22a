package gpuscheduling

/*
#include "lig.h"
*/
import "C"

import (
	"fmt"
	"math/rand"
	"sort"
	"sync"
	"time"

	"google.golang.org/grpc/codes"
	"google.golang.org/grpc/status"
	klog "k8s.io/klog/v2"

	"inference.networking.x-k8s.io/llm-instance-gateway/api/v1alpha1"
	"inference.networking.x-k8s.io/llm-instance-gateway/pkg/ext-proc/backend"
	"inference.networking.x-k8s.io/llm-instance-gateway/pkg/ext-proc/scheduling"
)

// Options of the GPU scheduler.  Thresholds default to the reference's constants
// (pkg/ext-proc/scheduling/scheduler.go:15-24).
type Options struct {
	Device          int
	MaxPods         int
	MaxAdapters     int
	MaxBatch        int
	FlushSize       int           // flush when this many requests are pending ...
	BatchWindow     time.Duration // ... or when the oldest pending request is this old
	RefreshInterval time.Duration // snapshot re-pack period; use main.go's refreshMetricsInterval
	KVCacheThreshold       float64
	QueueThresholdCritical int64
	QueueingThresholdLoRA  int64
	// FilterTree replaces defaultFilter (scheduler.go:26-91) by a caller flow chart of the
	// reference's filter nodes (filter.go:17-73); nil = defaultFilter.  Its nodes carry their own
	// thresholds, so the three above then do not apply.  See lig_set_filter_tree in include/lig.h.
	FilterTree []FilterNode
	// LoadFeedbackWindow > 0 carries load feedback across flushes (lig_schedule_batch_feedback_chain
	// in include/lig.h): every window of this many requests, counted across flushes, adds its picks
	// to the pods' WaitingQueueSize before the next request is scheduled, until the next Refresh
	// uploads a new epoch.  The reference never writes pod metrics while scheduling
	// (scheduler.go:113-122), so 0 (off) is the reference's behaviour.
	LoadFeedbackWindow int
	// InferenceModels is backend.K8sDatastore.InferenceModels (datastore.go:26-31: Spec.ModelName ->
	// *v1alpha1.InferenceModel).  When set, every Refresh packs it into the new epoch's model table
	// and ScheduleModel resolves requests on the device.  Deviation from the reference: a change of
	// an InferenceModel applies from the next refresh tick, not from the next request.
	InferenceModels *sync.Map
}

// FilterKind names the filter functions of filter.go / scheduler.go a FilterNode runs.
type FilterKind int32

const (
	FilterCriticalRequest  FilterKind = iota // criticalRequestPredicate             filter.go:179-181
	FilterLowQueueing                        // WaitingQueueSize < QueueThreshold     filter.go:124-126
	FilterLoRAAffinity                       // loRAAffinityPredicate                filter.go:169-172
	FilterCanAcceptNewLoRA                   // canAcceptNewLoraPredicate            filter.go:175-177
	FilterLowLoRACost                        // lowLoRACostPredicate                 filter.go:163-166
	FilterNoQueueAndLowKV                    // noQueueAndLessThanKVCacheThresholdPredicate  filter.go:183-187
	FilterLeastQueuing                       // leastQueuingFilterFunc               filter.go:102-122
	FilterLeastKVCache                       // leastKVCacheFilterFunc               filter.go:134-154
	FilterDrop                               // the "drop request" func              scheduler.go:83-89
)

// FilterNode is one node of a caller flow chart (include/lig.h lig_filter_node).  Node 0 is the
// root; successors are indices of later nodes, -1 = nil, and a node may have several parents.
type FilterNode struct {
	Kind                   FilterKind
	NextOnSuccess          int32
	NextOnFailure          int32
	NextOnSuccessOrFailure int32
	QueueThreshold         int64   // FilterLowQueueing, FilterNoQueueAndLowKV
	KVThreshold            float64 // FilterNoQueueAndLowKV
}

func DefaultOptions() Options {
	return Options{MaxPods: 4096, MaxAdapters: 1024, MaxBatch: 1 << 16, FlushSize: 4096,
		BatchWindow: 20 * time.Microsecond, RefreshInterval: 50 * time.Millisecond,
		KVCacheThreshold: 0.8, QueueThresholdCritical: 5, QueueingThresholdLoRA: 50}
}

// A waiter carries a descriptor request (req) or a model name (ScheduleModel).
type waiter struct {
	req     *scheduling.LLMRequest
	model   string
	modelID int64 // flush-time id in the captured epoch's table; -1: answered on the host
	done    chan result
}

type result struct {
	pod      backend.Pod
	resolved string
	err      error
}

// GPUScheduler implements handlers.Scheduler (pkg/ext-proc/handlers/server.go:37-39).  Swap it
// in at pkg/ext-proc/main.go:137:
//
//	sched, err := gpuscheduling.NewGPUScheduler(pp, gpuscheduling.DefaultOptions())
//	handlers.NewServer(pp, sched, *targetPodHeader, datastore)
type GPUScheduler struct {
	pmp  scheduling.PodMetricsProvider
	opt  Options
	c    *ctx
	in   *pinned
	out  *pinned
	seed uint64
	rng  *rand.Rand
	// the model-id lane: ids in, lig_mpicks out, and the first_index of the next device call
	inIDs      *pinned
	outM       *pinned
	firstIndex uint64

	snapMu sync.RWMutex
	snap   *packedSnapshot
	epoch  uint64

	queue     chan *waiter
	stop      chan struct{}
	wg        sync.WaitGroup
	closeOnce sync.Once
}

// NewGPUScheduler mirrors scheduling.NewScheduler(pmp) (scheduler.go:93-99).
func NewGPUScheduler(pmp scheduling.PodMetricsProvider, opt Options) (*GPUScheduler, error) {
	if opt.LoadFeedbackWindow < 0 {
		return nil, fmt.Errorf("gpu scheduler: LoadFeedbackWindow must be >= 0, got %d", opt.LoadFeedbackWindow)
	}
	c, err := newCtx(opt.Device, opt.MaxPods, opt.MaxAdapters, opt.MaxBatch)
	if err != nil {
		return nil, err // no CPU fallback: without the GPU the caller keeps the stock scheduler
	}
	if err := c.setThresholds(opt.KVCacheThreshold, opt.QueueThresholdCritical, opt.QueueingThresholdLoRA); err != nil {
		c.close()
		return nil, err
	}
	if len(opt.FilterTree) > 0 { // before the first snapshot upload: every table is built with it
		if err := c.setFilterTree(opt.FilterTree); err != nil {
			c.close()
			return nil, err
		}
	}
	in, err := allocPinned(opt.MaxBatch * 16)
	if err != nil {
		c.close()
		return nil, err
	}
	out, err := allocPinned(opt.MaxBatch * 8)
	if err != nil {
		in.free()
		c.close()
		return nil, err
	}
	inIDs, err := allocPinned(opt.MaxBatch * 4)
	if err != nil {
		in.free()
		out.free()
		c.close()
		return nil, err
	}
	outM, err := allocPinned(opt.MaxBatch * 4)
	if err != nil {
		inIDs.free()
		in.free()
		out.free()
		c.close()
		return nil, err
	}
	g := &GPUScheduler{pmp: pmp, opt: opt, c: c, in: in, out: out, inIDs: inIDs, outM: outM, seed: rand.Uint64(),
		rng: rand.New(rand.NewSource(time.Now().UnixNano())), queue: make(chan *waiter, opt.MaxBatch), stop: make(chan struct{})}
	if err := g.Refresh(); err != nil {
		g.Close()
		return nil, err
	}
	g.wg.Add(2)
	go g.batcher()
	go g.refresher()
	return g, nil
}

// Close stops the batcher and the refresher, answers every request that was still queued (or that
// races in while the scheduler shuts down) with codes.Unavailable, then frees the pinned buffers
// and the device context.  No Schedule call is left blocked.
func (g *GPUScheduler) Close() {
	g.closeOnce.Do(func() {
		close(g.stop)
		g.wg.Wait() // batcher and refresher are gone: nobody reads g.queue any more
		for {
			select {
			case w := <-g.queue:
				w.done <- result{err: status.Error(codes.Unavailable, "gpu scheduler is shut down")}
				continue
			default:
			}
			break
		}
		g.in.free()
		g.out.free()
		g.inIDs.free()
		g.outM.free()
		g.c.close()
	})
}

// Refresh re-packs the provider's current slice and uploads it as a new epoch.  One pack per
// refresh tick replaces the two AllPodMetrics() materialisations per request of
// scheduler.go:114-115.
func (g *GPUScheduler) Refresh() error {
	s, err := packSnapshot(g.pmp.AllPodMetrics())
	if err != nil {
		return err
	}
	g.snapMu.Lock()
	defer g.snapMu.Unlock()
	g.epoch++
	s.epoch = g.epoch
	if err := g.c.uploadSnapshot(s.epoch, s); err != nil {
		return err
	}
	// The model table goes into the new epoch before the epoch is published: a flush that captures
	// it maps names against the table the device reads.  Models the device would refuse are left out
	// (and logged) before packing, so one bad InferenceModel cannot fail every refresh tick.
	if g.opt.InferenceModels != nil {
		s.models = packModels(uploadableModels(inferenceModels(g.opt.InferenceModels)), s)
		if err := g.c.uploadModels(s.epoch, s.models); err != nil {
			return err
		}
	}
	g.snap = s
	return nil
}

// uploadableModels drops, with a log line, the models lig_upload_models refuses with LIG_ERR_RANGE:
// more than 255 targets, a negative weight, or weights summing above 2^31-1.  A model whose weights
// sum to <= 0 stays: it is packed as absent.  Requests for a dropped model get "error finding a
// model object"; valid CRDs (at most 10 targets, weights in [0, 1e6]) never hit this.
func uploadableModels(models []*v1alpha1.InferenceModel) []*v1alpha1.InferenceModel {
	out := models[:0:0]
	for _, im := range models {
		var sum int64
		negative := false
		for _, tm := range im.Spec.TargetModels {
			sum += int64(tm.Weight)
			negative = negative || tm.Weight < 0
		}
		if len(im.Spec.TargetModels) > 0 && sum > 0 && (len(im.Spec.TargetModels) > 255 || negative || sum > 1<<31-1) {
			klog.Errorf("gpu scheduler: InferenceModel %s cannot be uploaded (%d targets, weights summing to %d); "+
				"requests for it are rejected", im.Spec.ModelName, len(im.Spec.TargetModels), sum)
			continue
		}
		out = append(out, im)
	}
	return out
}

// inferenceModels lists the datastore's models in ModelName order (model ids stay stable while the
// set of names does).
func inferenceModels(m *sync.Map) []*v1alpha1.InferenceModel {
	var out []*v1alpha1.InferenceModel
	m.Range(func(_, v any) bool {
		if im, ok := v.(*v1alpha1.InferenceModel); ok && im != nil {
			out = append(out, im)
		}
		return true
	})
	sort.Slice(out, func(i, j int) bool { return out[i].Spec.ModelName < out[j].Spec.ModelName })
	return out
}

func (g *GPUScheduler) refresher() {
	defer g.wg.Done()
	t := time.NewTicker(g.opt.RefreshInterval)
	defer t.Stop()
	for {
		select {
		case <-g.stop:
			return
		case <-t.C:
			if err := g.Refresh(); err != nil {
				klog.Errorf("gpu scheduler: snapshot refresh failed, keeping the previous one: %v", err)
			}
		}
	}
}

// Schedule finds the target pod based on metrics and the requested lora adapter
// (scheduler.go:113-122).  Goroutine-safe and blocking, like the reference's.
func (g *GPUScheduler) Schedule(req *scheduling.LLMRequest) (backend.Pod, error) {
	r := g.submit(&waiter{req: req, done: make(chan result, 1)})
	return r.pod, r.err
}

// ScheduleModel is the resolve step of HandleRequestBody (request.go:42-56) and Schedule in one
// call, resolved on the device against the model table of Options.InferenceModels.  It returns the
// resolved target model (the body's "model" rewrite, request.go:60-69) and the pod.  An unknown
// model, or one whose weights sum to <= 0, gets the reference's error and never reaches the device;
// errors of the pick are wrapped as request.go:73-75 wraps them.  Without Options.InferenceModels
// every model is unknown, so a handler calls it only when ResolvesModels reports true (patch 0004).
// Unverified, like the rest of this package: it has never been compiled.
func (g *GPUScheduler) ScheduleModel(model string) (string, backend.Pod, error) {
	r := g.submit(&waiter{model: model, done: make(chan result, 1)})
	return r.resolved, r.pod, r.err
}

// ResolvesModels reports whether ScheduleModel has a model table to resolve against
// (Options.InferenceModels is set).  Without one, the handler keeps the reference's resolve step.
func (g *GPUScheduler) ResolvesModels() bool { return g.opt.InferenceModels != nil }

func (g *GPUScheduler) submit(w *waiter) result {
	select {
	case g.queue <- w:
	case <-g.stop:
		return result{err: status.Error(codes.Unavailable, "gpu scheduler is shut down")}
	}
	// A request that slipped into the queue while Close was draining it is answered by the
	// second arm: stop is closed for good, so no waiter can block forever.
	select {
	case r := <-w.done:
		return r
	case <-g.stop:
		select {
		case r := <-w.done:
			return r
		case <-time.After(g.opt.BatchWindow + 10*time.Millisecond):
			return result{err: status.Error(codes.Unavailable, "gpu scheduler is shut down")}
		}
	}
}

func (g *GPUScheduler) batcher() {
	defer g.wg.Done()
	batch := make([]*waiter, 0, g.opt.FlushSize)
	for {
		batch = batch[:0]
		select {
		case <-g.stop:
			return
		case w := <-g.queue:
			batch = append(batch, w)
		}
		deadline := time.NewTimer(g.opt.BatchWindow)
	fill:
		for len(batch) < g.opt.FlushSize && len(batch) < g.opt.MaxBatch {
			select {
			case w := <-g.queue:
				batch = append(batch, w)
			case <-deadline.C:
				break fill
			}
		}
		deadline.Stop()
		g.flush(batch)
	}
}

// flush makes the descriptor call first, then the model-id call.
func (g *GPUScheduler) flush(all []*waiter) {
	var batch, models []*waiter
	for _, w := range all {
		if w.req != nil {
			batch = append(batch, w)
		} else {
			models = append(models, w)
		}
	}
	if len(batch) > 0 {
		g.flushDescriptors(batch)
	}
	if len(models) > 0 {
		g.flushModels(models)
	}
}

func (g *GPUScheduler) flushDescriptors(batch []*waiter) {
	n := len(batch)
	var snap *packedSnapshot
	var rc C.int
	for attempt := 0; attempt < 4; attempt++ {
		g.snapMu.RLock()
		snap = g.snap
		g.snapMu.RUnlock()
		reqs := g.in.reqs(n)
		for i, w := range batch {
			reqs[i].adapter_id = C.int32_t(snap.adapterID(w.req.ResolvedTargetModel))
			reqs[i].flags = 0
			if w.req.Critical {
				reqs[i].flags = C.LIG_REQ_CRITICAL
			}
			reqs[i].rand_key = C.uint64_t(g.rng.Uint64())
		}
		if g.opt.LoadFeedbackWindow > 0 {
			rc = g.c.scheduleBatchFeedbackChain(snap.epoch, g.seed, g.in, g.out, n, g.opt.LoadFeedbackWindow)
		} else {
			rc = g.c.scheduleBatch(snap.epoch, g.seed, g.in, g.out, n)
		}
		if rc != C.LIG_ERR_STALE_EPOCH {
			break
		}
	}
	if rc != 0 {
		err := status.Errorf(codes.Internal, "gpu scheduler: %v", ligError("lig_schedule_batch", rc))
		for _, w := range batch {
			w.done <- result{err: err}
		}
		return
	}
	picks := g.out.picks(n)
	for i, w := range batch {
		switch picks[i].status {
		case C.LIG_OK:
			w.done <- result{pod: snap.pods[int(picks[i].pod_idx)]}
		case C.LIG_DROP:
			// identical to the reference: the ResourceExhausted status error of scheduler.go:87
			// wrapped with %w like scheduler.go:117, so status.Code(err) is still ResourceExhausted
			// after request.go:74 wraps it again and server.go:97-109 answers 429.
			inner := status.Errorf(codes.ResourceExhausted, "dropping request due to limited backend resources")
			w.done <- result{err: fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, inner)}
		case C.LIG_NO_PODS_LEFT:
			// a FilterTree ended on a predicate node that kept no pod: toFilterFunc's error
			// (filter.go:88-90) wrapped like scheduler.go:117; status.Code(err) is Unknown
			w.done <- result{err: fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, fmt.Errorf("no pods left"))}
		default:
			var nilErr error
			w.done <- result{err: fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, nilErr)}
		}
	}
}

// flushModels maps names to model ids against the captured epoch's table (again after a stale
// epoch, with the same first index) and sends the ids the host cannot answer to the device.
func (g *GPUScheduler) flushModels(batch []*waiter) {
	var snap *packedSnapshot
	var rc C.int
	k := 0
	for attempt := 0; attempt < 4; attempt++ {
		g.snapMu.RLock()
		snap = g.snap
		g.snapMu.RUnlock()
		ids := g.inIDs.modelIDs(len(batch))
		k = 0
		for _, w := range batch {
			w.modelID = -1
			if snap.models == nil {
				continue
			}
			if id, ok := snap.models.ids[w.model]; ok && snap.models.present[id] != 0 {
				w.modelID = int64(id)
				ids[k] = C.uint32_t(id)
				k++
			}
		}
		if k == 0 {
			break
		}
		if g.opt.LoadFeedbackWindow > 0 {
			rc = g.c.scheduleModelsFeedbackChain(snap.epoch, g.seed, g.firstIndex, g.inIDs, g.outM, k, g.opt.LoadFeedbackWindow)
		} else {
			rc = g.c.scheduleModels(snap.epoch, g.seed, g.firstIndex, g.inIDs, g.outM, k)
		}
		if rc != C.LIG_ERR_STALE_EPOCH {
			break
		}
	}
	g.firstIndex += uint64(k)
	picks := g.outM.mpicks(k)
	j := 0
	for _, w := range batch {
		if w.modelID < 0 {
			if snap.models != nil {
				if id, ok := snap.models.ids[w.model]; ok { // request.go:48-51
					w.done <- result{err: fmt.Errorf("error getting target model name for model %v", snap.models.names[id])}
					continue
				}
			}
			w.done <- result{err: fmt.Errorf("error finding a model object in InferenceModel for input %v", w.model)} // request.go:42-45
			continue
		}
		pk := picks[j]
		j++
		if rc != 0 {
			w.done <- result{err: fmt.Errorf("failed to find target pod: %w",
				status.Errorf(codes.Internal, "gpu scheduler: %v", ligError("lig_schedule_models_batch", rc)))}
			continue
		}
		resolved := w.model // 255: TargetModels is empty, the name passes through (request.go:47)
		if pk.target_idx != 255 {
			resolved = snap.models.targets[w.modelID][int(pk.target_idx)]
		}
		var err error
		switch pk.status {
		case C.LIG_OK:
			w.done <- result{pod: snap.pods[int(pk.pod_idx)], resolved: resolved}
			continue
		case C.LIG_DROP:
			inner := status.Errorf(codes.ResourceExhausted, "dropping request due to limited backend resources")
			err = fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, inner)
		case C.LIG_NO_PODS_LEFT:
			err = fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, fmt.Errorf("no pods left"))
		case C.LIG_EMPTY:
			var nilErr error
			err = fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", 0, nilErr)
		default: // LIG_NO_MODEL: absent models are answered on the host and never sent
			err = status.Errorf(codes.Internal, "model id %d (%s) has no model entry on the device", w.modelID, w.model)
		}
		w.done <- result{resolved: resolved, err: fmt.Errorf("failed to find target pod: %w", err)} // request.go:73-75
	}
}
