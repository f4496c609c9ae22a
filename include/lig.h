/*
 * lig.h — C ABI of the H100-native endpoint picker (drop-in for the ext-proc scheduler hot path).
 *
 * This is the boundary a cgo shim binds (see INTEGRATION.md).  Every entry point below replaces a
 * piece of the reference's Go scheduling package; the reference location is cited per symbol as
 * <file>:<line> relative to the reference repository root (kubernetes-sigs/llm-instance-gateway
 * @ 8e96339).  Plain pointers and sizes only: no C++ types, no torch types, no Go pointers kept
 * after a call returns.
 *
 * Conventions
 *   - every function returning int returns 0 on success or a negative LIG_ERR_* code; the
 *     human-readable reason is available (thread-local) from lig_last_error();
 *   - per-request outcomes are NOT errors: they are reported in lig_pick.status
 *     (LIG_OK / LIG_DROP / LIG_EMPTY), mirroring Schedule()'s (pod, err) return;
 *   - there is no CPU fallback anywhere behind this header: without a CUDA device lig_create
 *     fails with LIG_ERR_CUDA.
 */
#ifndef LIG_H_
#define LIG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LIG_ABI_VERSION 7

/* ---- per-request status (lig_pick.status) ------------------------------------------------------
 * LIG_OK    Schedule returned a pod, nil                      pkg/ext-proc/scheduling/scheduler.go:120-121
 * LIG_DROP  the "drop request" leaf fired: the Go side must return
 *           status.Errorf(codes.ResourceExhausted, "dropping request due to limited backend
 *           resources") wrapped like scheduler.go:117         scheduler.go:83-89  -> 429 at handlers/server.go:97-109
 * LIG_EMPTY the tree returned ([], nil): "failed to apply filter, resulted 0 pods, this should
 *           never happen"                                      scheduler.go:116-118
 * LIG_NO_PODS_LEFT  (caller filter trees only, see lig_set_filter_tree) the tree ended on a
 *           predicate node that kept no pod: toFilterFunc's fmt.Errorf("no pods left")
 *           (filter.go:88-90) wrapped by Schedule: "failed to apply filter, resulted 0 pods, this
 *           should never happen: no pods left" (scheduler.go:116-118).  The built-in tree never
 *           ends this way: every predicate node in it has a failure successor.
 */
enum { LIG_OK = 0, LIG_DROP = 1, LIG_EMPTY = 2,
       /* only from the model entry points (lig_schedule_models_*): FetchModelData returned nil,
        * "error finding a model object in InferenceModel for input ..."  handlers/request.go:42-45 */
       LIG_NO_MODEL = 3,
       LIG_NO_PODS_LEFT = 4 };

/* ---- batch-level error codes (negative return values) ---------------------------------------- */
enum {
  LIG_ERR_INVALID     = -1, /* bad argument (null pointer, P/A/R out of the ctx capacity, ...)    */
  LIG_ERR_CUDA        = -2, /* CUDA runtime/driver failure, or no device                          */
  LIG_ERR_STALE_EPOCH = -3, /* the epoch passed to schedule is not a resident snapshot            */
  LIG_ERR_NO_SNAPSHOT = -4, /* schedule called before any snapshot upload                         */
  LIG_ERR_RANGE       = -5, /* a host value does not fit the device record (see lig_pack_pods)    */
  LIG_ERR_BUSY        = -6, /* no free ticket for an asynchronous submit (wait for one first)     */
  LIG_ERR_NCCL        = -7  /* NCCL missing (dlopen libnccl.so.2 failed) or an NCCL call failed   */
};

/* ---- request descriptor: 16 bytes, one int4 load on the device --------------------------------
 * Replaces scheduling.LLMRequest (pkg/ext-proc/scheduling/types.go:4-11).  The filter tree reads
 * only ResolvedTargetModel and Critical (filter.go:163-181); Model and TargetModels are unused on
 * the path.  ResolvedTargetModel is interned by the host layer into adapter_id: the index of the
 * adapter's row in the snapshot bitmap, or any value outside [0, A) for a model that no pod
 * lists in ActiveModels (the base model, or a never-loaded adapter) — such a request matches no
 * pod in loRAAffinityPredicate, exactly like a Go map lookup miss (filter.go:170).
 * rand_key keys the request's private random stream used for the final pick (see below).
 */
typedef struct lig_req {
  int32_t  adapter_id;
  uint32_t flags;      /* bit 0 = Critical (types.go:10); other bits must be 0 */
  uint64_t rand_key;
} lig_req;
#define LIG_REQ_CRITICAL 1u

/* ---- result: 8 bytes ---------------------------------------------------------------------------
 * pod_idx      index into the snapshot's pod order (= order of the slice the injected
 *              PodMetricsProvider returned at pack time, scheduler.go:108-115), -1 unless LIG_OK;
 *              the host maps it back to backend.Pod{Name,Address} (backend/types.go:8-11).
 * n_survivors  len(pods) after the filter tree (the argument of rand.Intn, scheduler.go:120).
 */
typedef struct lig_pick {
  int32_t  pod_idx;
  uint16_t status;
  uint16_t n_survivors;
} lig_pick;

/* ---- thresholds: the compile-time constants of scheduler.go:15-24, made parameters so the
 * reference's own predicate test (filter_test.go:304-338 uses (0, 0.8)) can be run on the GPU. */
typedef struct lig_thresholds {
  double  kv_cache_threshold;         /* kvCacheThreshold        = 0.8 */
  int64_t queue_threshold_critical;   /* queueThresholdCritical  = 5   */
  int64_t queueing_threshold_lora;    /* queueingThresholdLoRA   = 50  */
} lig_thresholds;

typedef struct lig_ctx lig_ctx; /* opaque; one per (process, device) */

/* Hard limits of the device records. */
#define LIG_MAX_PODS     32768   /* list entries and n_survivors are uint16 */
#define LIG_MAX_ADAPTERS 65534

/* ---- lifetime -------------------------------------------------------------------------------- */
/* Replaces scheduling.NewScheduler (scheduler.go:93-99): binds the scheduler to one CUDA device
 * and reserves HBM + pinned staging for snapshots of up to max_pods x max_adapters and host
 * batches of up to max_batch requests (device-pointer batches are not limited by max_batch). */
int  lig_create(lig_ctx** out, int device, int max_pods, int max_adapters, int max_batch);
void lig_destroy(lig_ctx* ctx);

/* With a caller filter tree set (lig_set_filter_tree) the thresholds are still stored but do not
 * affect the class-table build: every node of a caller tree carries its own thresholds.
 * Every value of the three fields is legal (Go's thresholds are int and float64): queue thresholds
 * are compared as int64, the KV threshold as binary64 (a NaN threshold keeps no pod).
 * Resident epochs whose tables the built-in tree built are rebuilt with the new thresholds before
 * the call returns; epochs a caller tree built keep their tables.  A rebuild waits for the work
 * already enqueued against the epoch (on any stream), which sees the old tables, so the call can
 * block until that work is done; everything enqueued after the return sees the new ones.  A
 * feedback chain keeps the thresholds it started with (see below). */
int  lig_set_thresholds(lig_ctx* ctx, const lig_thresholds* t);   /* scheduler.go:15-24 */
int  lig_get_thresholds(const lig_ctx* ctx, lig_thresholds* t);

/* ---- caller-defined filter trees ----------------------------------------------------------------
 * The reference's scheduler is a flow chart of `filter` nodes linked by nextOnSuccess,
 * nextOnFailure and nextOnSuccessOrFailure (filter.go:17-73); Scheduler holds it as a Filter field
 * (scheduler.go:101-104) and defaultFilter (scheduler.go:26-91) is one such chart.  A caller tree
 * is any chart of the node kinds below, given as a table whose node 0 is the root.  Routing is
 * (*filter).Filter (filter.go:44-73): success = no error AND a non-empty result; on success the
 * node's result goes to next_on_success if set, else next_on_success_or_failure; on failure the
 * node's INPUT goes to next_on_failure if set, else next_on_success_or_failure; when the chosen
 * field is -1 (nil) the node's own (result, error) is the tree's result.  Every kind depends on the
 * request only through (Critical, ResolvedTargetModel), so any tree still yields one survivor set
 * per request class and runs on the class tables of every entry point above and below. */
enum {                                   /* filter.go / scheduler.go names                         */
  LIG_F_CRITICAL_REQUEST = 0,            /* criticalRequestPredicate             filter.go:179-181 */
  LIG_F_LOW_QUEUEING,                    /* WaitingQueueSize < queue_threshold   filter.go:124-126 */
  LIG_F_LORA_AFFINITY,                   /* loRAAffinityPredicate                filter.go:169-172 */
  LIG_F_CAN_ACCEPT_NEW_LORA,             /* canAcceptNewLoraPredicate            filter.go:175-177 */
  LIG_F_LOW_LORA_COST,                   /* lowLoRACostPredicate                 filter.go:163-166 */
  LIG_F_NO_QUEUE_AND_LOW_KV,             /* q <= queue_threshold && kv <= kv_threshold
                                            noQueueAndLessThanKVCacheThresholdPredicate filter.go:183-187 */
  LIG_F_LEAST_QUEUING,                   /* leastQueuingFilterFunc               filter.go:102-122 */
  LIG_F_LEAST_KV_CACHE,                  /* leastKVCacheFilterFunc               filter.go:134-154 */
  LIG_F_DROP                             /* the "drop request" func: ([], ResourceExhausted)
                                                                                 scheduler.go:83-89 */
};
/* Predicate kinds (the first six) fail with "no pods left" when they keep no pod (toFilterFunc,
 * filter.go:79-93); the two range kinds never err, they fail only on an empty result. */
typedef struct lig_filter_node {         /* 32 bytes */
  int32_t kind;                          /* LIG_F_* */
  int32_t next_on_success, next_on_failure, next_on_success_or_failure;  /* node index, -1 = nil */
  int64_t queue_threshold;               /* LOW_QUEUEING, NO_QUEUE_AND_LOW_KV; ignored otherwise   */
  double  kv_threshold;                  /* NO_QUEUE_AND_LOW_KV; ignored otherwise                 */
} lig_filter_node;
#define LIG_MAX_FILTER_NODES 32
/* Use `nodes` for every class-table build enqueued after the call returns: lig_upload_snapshot
 * and its _async / _device forms, lig_update_snapshot, the lig_comm_* uploads and the per-window
 * rebuilds of lig_schedule_batch_feedback_device.  Resident epochs keep the tables they were built
 * with.  nodes == NULL with n_nodes == 0 restores the built-in tree (defaultFilter with the
 * lig_set_thresholds values).  LIG_ERR_INVALID, and the previous tree stays in force, when n_nodes
 * is outside [1, LIG_MAX_FILTER_NODES], a kind is unknown, or a successor of node i is neither -1
 * nor in (i, n_nodes): edges only point forward, so every table is acyclic, and a node may have
 * several parents (defaultFilter shares queueAndKVCacheFilter).  The direct scan
 * (lig_schedule_scan[_device]) restates the built-in tree only: it returns LIG_ERR_INVALID for an
 * epoch whose tables a caller tree built; lig_filter_batch and lig_read_class return a caller tree's
 * survivor sets, and lig_schedule_batch_excluding walks the tree that built the epoch, per request. */
int  lig_set_filter_tree(lig_ctx* ctx, const lig_filter_node* nodes, int n_nodes);

/* ---- snapshot = the value of PodMetricsProvider.AllPodMetrics() (scheduler.go:108-115,
 * backend/provider.go:38-46) frozen at one refresh tick, in device layout -----------------------
 *
 * Packed blob, W = ceil(P/32), Ppad = 32*W, every section 16-byte aligned, in this order:
 *   double   kv[Ppad]          Metrics.KVCacheUsagePercent           backend/types.go:24
 *   int32_t  q[Ppad]           Metrics.WaitingQueueSize              backend/types.go:23
 *   uint16_t n_active[Ppad]    len(Metrics.ActiveModels)             backend/types.go:19
 *   uint16_t max_active[Ppad]  Metrics.MaxActiveModels (saturated)   backend/types.go:21
 *   uint32_t bitmap[A][W]      bit (a, p) = adapter a in pod p's ActiveModels (adapter-major)
 * Padding pods (index >= P), their bits in the last word of each bitmap row and the bytes after
 * the bitmap are ignored by every kernel, whatever they hold.
 */
size_t lig_snapshot_bytes(int P, int A);

/* Pure host helper (no GPU): narrow Go-width pod metrics to the device record.
 *   q          must fit int32, else LIG_ERR_RANGE (never silently wrapped);
 *   n_active   must be in [0, LIG_MAX_ADAPTERS], else LIG_ERR_RANGE;
 *   max_active is saturated to [0, 65535]: canAcceptNewLoraPredicate (filter.go:175-177) is
 *              `n_active < max_active` and n_active <= 65534, so saturation cannot change it. */
int lig_pack_pods(int P, const int64_t* waiting_queue_size, const int64_t* n_active_models,
                  const int64_t* max_active_models, int32_t* q_out, uint16_t* n_active_out,
                  uint16_t* max_active_out);

/* Pure host helper (no GPU): lay the five arrays out as the packed blob described above, with
 * padding pods and tail bits zeroed.  LIG_ERR_INVALID for a null blob, P or A < 0, a null pod
 * column when P > 0 or a null bitmap when P > 0 and A > 0; LIG_ERR_RANGE when a pod's n_active
 * exceeds LIG_MAX_ADAPTERS.  Nothing is written when the call is refused. */
int lig_pack_snapshot(void* blob, int P, int A, const double* kv, const int32_t* q,
                      const uint16_t* n_active, const uint16_t* max_active,
                      const uint32_t* bitmap_adapter_major /* A x ceil(P/32) */);

/* Upload a snapshot from host arrays and build the per-class survivor tables on the device.
 * After it returns, `epoch` is resident; the previous epoch stays resident too (two slots), so
 * in-flight batches against it still complete.  Replaces the per-request
 * AllPodMetrics() materialisation of scheduler.go:114-115 by one pack per refresh tick.
 * Refused, before any slot is touched (both resident epochs and their model tables stay as they
 * were, also when `epoch` is one of them), for the reasons of lig_pack_snapshot and with
 * LIG_ERR_INVALID for P > max_pods or A > max_adapters.  The _async form and
 * lig_group_upload_snapshot refuse the same arguments the same way. */
int lig_upload_snapshot(lig_ctx* ctx, uint64_t epoch, int P, int A, const double* kv,
                        const int32_t* q, const uint16_t* n_active, const uint16_t* max_active,
                        const uint32_t* bitmap_adapter_major);
/* The same without waiting for the device: the arrays are copied into the ctx's pinned staging
 * before the call returns (the caller may reuse them at once), the H2D copy and the table build
 * are only enqueued.  `epoch` is resident immediately; batches against it are ordered behind the
 * build on the device, so the refresher goroutine (backend/provider.go:81-88) never blocks on the
 * GPU and a refresh + the next batch cost one synchronisation, not three.  A device-side failure
 * of the build surfaces at the next call that synchronises. */
int lig_upload_snapshot_async(lig_ctx* ctx, uint64_t epoch, int P, int A, const double* kv,
                              const int32_t* q, const uint16_t* n_active, const uint16_t* max_active,
                              const uint32_t* bitmap_adapter_major);

/* Delta form of lig_upload_snapshot for the refresh tick (backend/provider.go:134-179 re-scrapes
 * every pod, but between two ticks most pods report the same metrics): `new_epoch` becomes
 * `base_epoch` (which must be resident and stays so, untouched) with n_dirty pods replaced.  P
 * and A are those of the base.  For dirty pod i: pod_idx[i], its four column values, and its
 * COMPLETE ActiveModels as adapter ids adapter_ids[adapter_offsets[i] .. adapter_offsets[i+1]).
 * Only the delta crosses PCIe; the base blob is copied device-to-device, the dirty rows and
 * bitmap bits are patched by a kernel, and the class tables are rebuilt.  LIG_ERR_INVALID when
 * the base epoch is the slot the new epoch would have to overwrite (it is the older of the two
 * resident epochs): fall back to lig_upload_snapshot.  LIG_ERR_INVALID too, before anything is
 * written (both resident epochs stay as they were), when the delta is malformed:
 *   - a pod index is outside [0, P) or appears more than once in pod_idx;
 *   - adapter_offsets[0] != 0, or adapter_offsets decreases anywhere;
 *   - an adapter id is outside [0, A) of the base.
 * LIG_ERR_RANGE, likewise before anything is written, when a dirty pod's n_active exceeds
 * LIG_MAX_ADAPTERS.  The same id twice within one pod's list is allowed (it sets the same bit). */
int lig_update_snapshot(lig_ctx* ctx, uint64_t new_epoch, uint64_t base_epoch, int n_dirty,
                        const int32_t* pod_idx, const double* kv, const int32_t* q,
                        const uint16_t* n_active, const uint16_t* max_active,
                        const int32_t* adapter_offsets, const int32_t* adapter_ids);

/* ---- outlier ejection: schedule as if some pods had left the provider ----------------------------
 * A proxy that finds a pod refusing connections can keep it out of every later pick until it lets it
 * back, without waiting for the pod to leave the provider (readiness probes take seconds, and a dead
 * pod's scrape fails, so the provider keeps its last, often attractive, metrics).
 *
 * `new_epoch` becomes `base_epoch`'s snapshot (which must be resident and stays so, untouched) with
 * pod_idx[0 .. n) left out of the pool.  It keeps base's metric columns, bitmap, P, A and pod order.
 * On it, every call returns byte for byte what it returns on an epoch uploaded from the literally
 * reduced snapshot (the kept pods' columns in order, the ejected pods' bitmap columns dropped, A
 * unchanged), built with the filter tree and thresholds in force at this call, with every pod index
 * of the results (pod_idx, survivor lists, fallback rows, loads) mapped back to base's order.  The
 * mapping keeps order, so picks, rankings and lists keep their definitions.  That covers the plain,
 * queue, persistent and model-id picks, the doorbell, lig_filter_*, lig_read_class, the fallback
 * calls, the in-batch feedback call and every chain call (the chain's private copy carries the
 * pool: an ejected pod gets no pick and a load of 0).  A retry's pool is the epoch's pool minus the
 * request's row; a row entry that names an ejected pod leaves out nothing more.  Ejecting every pod
 * is legal: every call then gets the tree's answer for an empty slice (under the built-in tree
 * LIG_DROP for every request, as for an empty retry pool).
 *
 * The set carried by an epoch: the listed set REPLACES base's (n = 0 derives an epoch with every pod
 * back); lig_update_snapshot from an ejected base keeps base's set; full uploads
 * (lig_upload_snapshot[_async|_device], lig_comm_*, lig_group_upload_snapshot) start with none;
 * lig_set_thresholds rebuilds keep it.  Like every snapshot writer, the new epoch has no model
 * table until lig_upload_models.  The direct scan (lig_schedule_scan[_device]) returns
 * LIG_ERR_INVALID for an epoch with ejected pods.  Ranks of a communicator eject the same pods each
 * on its own ctx.
 *
 * Only the pool mask crosses PCIe: the base blob is copied device-to-device and the class tables are
 * rebuilt from the pool.  Blocks like lig_update_snapshot, takes the upload lock and waits for the
 * readers of the slot it overwrites.  Refused with nothing written, both resident epochs as they
 * were: LIG_ERR_INVALID for new_epoch == base_epoch, n < 0, n > P, a null list with n > 0, an index
 * outside [0, P) or listed twice, and when base is the slot the new epoch would overwrite (the rule
 * of lig_update_snapshot); LIG_ERR_STALE_EPOCH / LIG_ERR_NO_SNAPSHOT when base is not resident. */
int lig_eject_pods(lig_ctx* ctx, uint64_t new_epoch, uint64_t base_epoch, const int32_t* pod_idx, int n);

/* Same, but the packed blob is already in HBM (e.g. the receive buffer of an NCCL broadcast of
 * the snapshot).  The blob is copied into the ctx on `stream` (a cudaStream_t, may be NULL =
 * legacy default stream); table build is enqueued on the same stream, nothing is synchronised.
 * The blob is taken as it is: padding pods may hold anything (they are ignored), and every real
 * pod's n_active <= LIG_MAX_ADAPTERS is the caller's contract (lig_pack_snapshot checks it on the
 * host; this form and lig_comm_upload_snapshot_device do not read the blob on the host). */
int lig_upload_snapshot_device(lig_ctx* ctx, uint64_t epoch, int P, int A, const void* d_blob,
                               void* stream);

/* ---- the hot path ------------------------------------------------------------------------------
 * Replaces R calls of Scheduler.Schedule (scheduler.go:113-122) == R walks of the defaultFilter
 * tree (scheduler.go:26-91, filter.go:44-187) followed by rand.Intn(len(pods)).
 *
 * The random pick.  The reference draws from Go's auto-seeded global source, so its pick is not
 * reproducible; this ABI defines it as what `rand.New(src).Intn(n)` returns (math/rand, Go 1.22:
 * Intn -> Int31n; Int31() = Int63()>>32) when src is a SplitMix64 source private to the request:
 *     state = seed ^ rand_key;
 *     next(): state += 0x9E3779B97F4A7C15; z = state;
 *             z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9; z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *             return z ^ (z >> 31);
 *     Int63() = next() >> 1            (so Int31() = next() >> 33)
 *     Int31n(n): if n is a power of two: Int31() & (n-1)
 *                else max = 2^31 - 1 - (2^31 % n); v = Int31(); while (v > max) v = Int31();
 *                     return v % n
 * and pod_idx is the k-th survivor in ascending pod index (= slice order, pods[i] scheduler.go:121).
 */

/* Page-locked, device-mapped host memory for request / pick buffers (what the Go shim exposes
 * to callers as unsafe.Slice, see INTEGRATION.md).  Buffers from here (or any cudaHostAlloc /
 * cudaHostRegister memory) are read and written by the kernel in place; ordinary pageable
 * memory also works but bounces through the ctx's own pinned buffers. */
void* lig_host_alloc(size_t bytes);
void  lig_host_free(void* p);

/* Host buffers in, host buffers out.  Nothing is staged through HBM: the pick kernel reads the
 * descriptors from, and writes the picks to, page-locked host memory over PCIe directly.  Blocks
 * until `out` is complete.  The kernels read a lig_req with one 16-byte load: a request array that
 * is not 16-byte aligned is staged like pageable memory. */
int lig_schedule_batch(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                       lig_pick* out);

/* Asynchronous submit for the one-goroutine-per-stream caller model (handlers/server.go:51, up to
 * 40 000 concurrent streams, pkg/manifests/ext_proc.yaml:102-105): many threads may have batches
 * in flight on one ctx at once.  `reqs` and `out` MUST be page-locked (lig_host_alloc /
 * cudaHostAlloc / cudaHostRegister) and stay untouched until the wait returns.  On success
 * *ticket identifies the in-flight batch; lig_schedule_wait blocks until its picks are complete and
 * releases the ticket.  The ctx lock is held only while the work is enqueued, never while waiting.
 * LIG_ERR_BUSY when all LIG_MAX_TICKETS tickets are in flight; LIG_ERR_INVALID when `reqs` is not
 * 16-byte aligned. */
#define LIG_MAX_TICKETS 256
int lig_schedule_batch_async(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                             lig_pick* out, int* ticket);
int lig_schedule_wait(lig_ctx* ctx, int ticket);

/* HBM-resident batch: d_reqs / d_out are device pointers (16-byte / 8-byte aligned); the work is
 * enqueued on `stream` and NOT synchronised.  This is the class-table fast path. */
int lig_schedule_batch_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                              int R, lig_pick* d_out, void* stream);

/* A queue of n_batches HBM-resident batches of R requests each against one epoch, enqueued
 * back to back on `stream` with one pass through the ABI (the micro-batcher's flush of several
 * pending batches).  Batch b uses seed `seed + b` (mod 2^64: a seed near 2^64 wraps to 0), reads
 * d_reqs[b] and writes d_out[b]; the two pointer arrays are host arrays of device pointers.
 * Equivalent to n_batches calls of lig_schedule_batch_device, however long the queue (the library
 * splits it into several launches where it must). */
int lig_schedule_batches_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                const lig_req* const* d_reqs, int R, lig_pick* const* d_out,
                                int n_batches, void* stream);

/* ---- streaming micro-batches without a kernel launch ---------------------------------------------
 * lig_stream_open parks one persistent CTA on the device that polls a mailbox in page-locked host
 * memory; lig_stream_submit writes up to lig_stream_capacity() descriptors + a doorbell ticket
 * into it and spins until the picks and the completion ticket are back: two PCIe crossings, no
 * launch, no stream synchronisation (Scheduler.Schedule under a sustained request stream,
 * handlers/request.go:72).  Same results as lig_schedule_batch for the same (epoch, seed, reqs).
 * While a stream is open nothing in the process may synchronise the whole device
 * (cudaDeviceSynchronize, cudaFree): the resident kernel never finishes until lig_stream_close.
 * A submit holds the ctx's upload lock for its whole round trip, and every snapshot and model
 * upload takes that lock: no table the resident kernel reads can be overwritten during a submit,
 * and submits of one ctx run one at a time. */
int lig_stream_capacity(void);
int lig_stream_open(lig_ctx* ctx);
int lig_stream_submit(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int n,
                      lig_pick* out);
/* (lig_stream_submit_models, the model-id form, is declared with the model entry points below.) */
int lig_stream_close(lig_ctx* ctx);

/* Direct scan: every request walks the whole tree over all P pods itself (one warp per request,
 * no class tables).  d_masks, when not NULL, receives the survivor set of every request as
 * R x ceil(P/32) words (bit p%32 of word p/32 = pod p survives) — the GPU analogue of
 * Filter.Filter's return value (filter.go:12-15, 44-73), used by the parity tests. */
int lig_schedule_scan_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                             int R, lig_pick* d_out, uint32_t* d_masks, void* stream);

/* Host-buffer wrapper of the direct scan (test hook; masks may be NULL). */
int lig_schedule_scan(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                      lig_pick* out, uint32_t* masks);

/* Read back one class table entry of a resident snapshot (test hook): the survivor list the
 * fast path uses for requests (critical, adapter_id).  `list` must hold P entries. */
int lig_read_class(lig_ctx* ctx, uint64_t epoch, int critical, int adapter_id, int* status,
                   int* n_survivors, uint16_t* list);

/* ---- the step before Schedule, on the device ------------------------------------------------------
 * Replaces, per request, the resolve step of HandleRequestBody (handlers/request.go:42-56):
 * datastore.FetchModelData(model) (backend/datastore.go:70-76), backend.RandomWeightedDraw over
 * Spec.TargetModels (datastore.go:78-98) and backend.IsCritical (datastore.go:100-105).  The host
 * interns the InferenceModel names to dense model ids once per datastore change and the request
 * shrinks to ONE 32-bit model id; the device looks the model up, draws the target model, derives
 * Critical and schedules — one pass over the batch, 4 bytes in and 4 bytes out per decision.
 *
 * The model table belongs to a resident snapshot epoch: target models are given as adapter ids
 * interned against that snapshot (an id outside [0, A) = a model no pod lists in ActiveModels).
 *   target_offsets[n_models + 1]   CSR offsets into the two target arrays (TargetModels order)
 *   target_adapter_ids / weights   Spec.TargetModels[k].Name (interned) / .Weight
 *   critical[n_models]             IsCritical(model)
 *   self_adapter_ids[n_models]     the model's own name interned: used when TargetModels is empty
 *                                  (request.go:47: modelName stays the requested model)
 *   present[n_models] (nullable)   0 = FetchModelData returns nil for this id -> LIG_NO_MODEL
 * Weights must be >= 0 and sum to [1, 2^31-1] for every model with targets (Go's Int31n panics on
 * a non-positive sum, a negative weight makes the reference's loop ill-defined), at most 255
 * targets per model: LIG_ERR_RANGE otherwise.
 *
 * The draw.  The reference draws from rand.NewSource(rand.Int63()) (request.go:48 passes seed 0):
 * unseeded, not reproducible.  As for the pick, this ABI defines it on a SplitMix64 source private
 * to the request: state = seed ^ rand_key ^ LIG_DRAW_DOMAIN, randomVal = Int31n(sum of weights)
 * (Go 1.22 algorithm, see below), target = first k with randomVal < Weight[k], else
 * randomVal -= Weight[k] (datastore.go:91-97).  A model with exactly one target skips the draw
 * (its result cannot depend on it).  The pick then uses state = seed ^ rand_key as always, so
 * lig_schedule_models_batch(ids) == lig_schedule_batch(descriptors resolved on the host).
 * rand_key of request i of a call is first_index + i, mod 2^64 (a counter-based key: shards of one
 * batch pass their offset and get the single-device result; a first_index near 2^64 wraps to 0
 * inside the batch). */
#define LIG_DRAW_DOMAIN 0xA0761D6478BD642Full
typedef struct lig_mpick {
  int16_t pod_idx;     /* as lig_pick.pod_idx (-1 unless LIG_OK)                                  */
  uint8_t status;      /* LIG_OK / LIG_DROP / LIG_EMPTY / LIG_NO_MODEL / LIG_NO_PODS_LEFT         */
  uint8_t target_idx;  /* index of the drawn Spec.TargetModels entry (the body's "model" rewrite,
                          request.go:61-69); 255 = TargetModels empty, the model name passes through */
} lig_mpick;
int lig_upload_models(lig_ctx* ctx, uint64_t epoch, int n_models, const int32_t* target_offsets,
                      const int32_t* target_adapter_ids, const int32_t* target_weights,
                      const uint8_t* critical, const int32_t* self_adapter_ids, const uint8_t* present);
/* Same, enqueued only (see lig_upload_snapshot_async). */
int lig_upload_models_async(lig_ctx* ctx, uint64_t epoch, int n_models, const int32_t* target_offsets,
                            const int32_t* target_adapter_ids, const int32_t* target_weights,
                            const uint8_t* critical, const int32_t* self_adapter_ids, const uint8_t* present);
/* Host buffers (page-locked ones are read / written over PCIe in place), blocking. */
int lig_schedule_models_batch(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                              const uint32_t* model_ids, int R, lig_mpick* out);
/* HBM-resident queue of n_batches batches of R model ids (4-byte aligned; 16-byte aligned buffers
 * take the TMA path), batch b with seed + b (mod 2^64) and the same first_index; enqueued on
 * `stream`, not synchronised. */
int lig_schedule_models_batches_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                       const uint32_t* const* d_model_ids, int R,
                                       lig_mpick* const* d_out, int n_batches, void* stream);
/* Test hook: only the resolve step, returning the 16-byte descriptor the device built for every
 * request (adapter_id, Critical, rand_key = first_index + i) and its status (LIG_OK / LIG_NO_MODEL)
 * and target index in `out`. */
int lig_resolve_models(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                       const uint32_t* model_ids, int R, lig_req* reqs_out, lig_mpick* out);
/* The doorbell round trip (lig_stream_open / lig_stream_submit) for model-id requests: up to
 * lig_stream_capacity() 4-byte ids in, as many 4-byte lig_mpicks out, byte for byte those of
 * lig_schedule_models_batch(ctx, epoch, seed, first_index, model_ids, n) (rand_key = first_index + i),
 * with the same contract as lig_stream_submit: it blocks, and one round trip of either kind runs
 * at a time.  Resolved against the model table of `epoch` as it stands at the call; it waits for
 * an enqueued upload of that table (lig_upload_models_async) as lig_stream_submit waits for the
 * class tables.  The submit holds the ctx's upload lock for its whole round trip and every model
 * upload takes that lock, so the table cannot be overwritten while the resident kernel reads it.
 * Model tables may be uploaded before or after lig_stream_open.  An upload that has to allocate
 * the slot's table (the first one for the slot, or one larger than the allocation, which is twice
 * the table that caused it) stops the resident kernel, reallocates and relaunches it: the stream
 * stays open, and no round trip is in flight meanwhile.
 * LIG_ERR_NO_SNAPSHOT when `epoch` has no model table, LIG_ERR_STALE_EPOCH when it is not
 * resident, LIG_ERR_INVALID before lig_stream_open, for n outside [0, capacity] or a null buffer.
 * Submits of both kinds may alternate on one open stream. */
int lig_stream_submit_models(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                             const uint32_t* model_ids, int n, lig_mpick* out);

/* ---- the survivor sets of a whole batch: Filter.Filter (filter.go:12-15) next to the pick --------
 * Each call makes the pick of the call it mirrors, byte for byte in `out`, and also returns every
 * request's survivor list (the slice the filter tree returned, filter.go:44-73) in CSR form:
 *   - request i's survivors are pods[offsets[i] .. offsets[i+1]): pod indices in ascending order,
 *     the order of Go's filtered slice.  offsets[0] = 0.  Offsets are int64: the sum can exceed 2^31.
 *   - LIG_DROP, LIG_EMPTY, LIG_NO_PODS_LEFT and LIG_NO_MODEL requests get an empty list.
 *   - pod entries at or beyond `capacity` are never written, but `out` and `offsets` are always
 *     complete, so a first call with capacity = 0 sizes the buffer (pods may then be NULL).  The
 *     host forms return LIG_ERR_INVALID, after filling `out` and `offsets`, when offsets[R] >
 *     capacity; the device forms leave that check to the caller.
 *   - the lists are read from the resident epoch's class tables, whichever build made them (the
 *     built-in tree, a caller filter tree, compact or strided tables), never from a feedback
 *     chain's private copy: the survivor sets of the scraped metrics.
 *   - refused like the call each form mirrors: stale epoch, null buffers, R > max_batch on the host
 *     forms; the model forms also with LIG_ERR_NO_SNAPSHOT when the epoch has no model table.
 * Host forms: page-locked buffers are read and written in place, pageable ones (and a request
 * array that is not 16-byte aligned) are staged; they block until everything is back.  Device forms: device pointers, enqueued on `stream` (a
 * cudaStream_t, NULL = legacy default stream), not synchronised. */
/* descriptors: out is byte for byte lig_schedule_batch(ctx, epoch, seed, reqs, R, out) */
int lig_filter_batch(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                     lig_pick* out, int64_t* offsets /* R + 1 */, uint16_t* pods, int64_t capacity);
int lig_filter_batch_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs, int R,
                            lig_pick* d_out, int64_t* d_offsets, uint16_t* d_pods, int64_t capacity,
                            void* stream);
/* model ids: out is byte for byte lig_schedule_models_batch(ctx, epoch, seed, first_index, ids, R,
 * out).  Resolved against the epoch's model table as lig_schedule_models_batch does: the call is
 * ordered behind the table's upload and registers as a reader of the slot, so a later model upload
 * waits on the device for it. */
int lig_filter_models_batch(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                            const uint32_t* model_ids, int R, lig_mpick* out, int64_t* offsets,
                            uint16_t* pods, int64_t capacity);
int lig_filter_models_batch_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                   const uint32_t* d_model_ids, int R, lig_mpick* d_out, int64_t* d_offsets,
                                   uint16_t* d_pods, int64_t capacity, void* stream);

/* ---- fallback endpoints: the pick and up to LIG_MAX_FALLBACKS more distinct survivors --------------
 * Schedule returns one pod (scheduler.go:113-122).  When that pod refuses the connection, was evicted
 * or is overloaded, a proxy can walk the request's fallback row instead of scheduling again: distinct
 * members of the same survivor set, in an order defined on the request's own random stream.
 *
 * The ranking.  Take a LIG_OK request with survivor list L of n pods (ascending pod order, the list
 * lig_read_class and lig_filter_batch return) and its pick stream state = seed ^ rand_key (rand_key =
 * first_index + i for model ids).  m = min(n, 1 + n_fallbacks).  perm starts as the identity on
 * [0, n).
 *   step 0: r_0 = Int31n(n), the pick's own draws and rejections; ranked entry 0 = L[r_0] = the pick.
 *   step j = 1 .. m-1: r_j = j + Int31n(n - j) on the stream continued after the last value the
 *           previous step drew (a power of two masks, otherwise v > 2^31-1-(2^31 % (n-j)) is
 *           rejected and v % (n-j) taken: Go 1.22, as for the pick).
 *   every step j swaps perm[j] and perm[r_j]; ranked entry j = L[perm[j]] (a partial Fisher-Yates
 *   shuffle: over keys every ordered choice of m distinct survivors is equally likely).
 * Request i's row is fallbacks[i * n_fallbacks .. (i + 1) * n_fallbacks): ranked entries 1 .. m-1 as
 * pod indices, then -1 to the end of the row.  Requests that are not LIG_OK (DROP, EMPTY,
 * NO_PODS_LEFT, NO_MODEL) get a row of -1.  The row for n_fallbacks = k is a prefix of the row for any
 * k' > k.  The lists of these four calls come from the resident epoch's class tables, whichever
 * build made them, never from a feedback chain's private copy; they neither end nor advance a
 * feedback chain.  Under a chain, lig_schedule_[models_]batch_feedback_chain_fallbacks below rank
 * the same way on the chain's own tables.
 *
 * `out` is byte for byte what the call each form mirrors returns.  LIG_ERR_INVALID for n_fallbacks
 * outside [1, LIG_MAX_FALLBACKS], null buffers, R > max_batch on the host forms, and device buffers
 * not aligned to their element (requests 16 bytes, picks 8 / 4, rows 2); a stale epoch and a missing
 * snapshot as the mirrored calls report them; the model forms also LIG_ERR_NO_SNAPSHOT when the
 * epoch has no model table.  Host forms: page-locked buffers are read and written in place,
 * pageable or misaligned ones are staged; they block until everything is back.  Device forms: device
 * pointers, enqueued on `stream` (NULL = legacy default stream), not synchronised.  The model forms
 * are ordered behind the table's upload and register as readers of the slot, as
 * lig_filter_models_batch does. */
#define LIG_MAX_FALLBACKS 8
/* descriptors: out is byte for byte lig_schedule_batch(ctx, epoch, seed, reqs, R, out) */
int lig_schedule_batch_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                 lig_pick* out, int n_fallbacks, int16_t* fallbacks);
int lig_schedule_batch_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                        int R, lig_pick* d_out, int n_fallbacks, int16_t* d_fallbacks,
                                        void* stream);
/* model ids: out is byte for byte lig_schedule_models_batch(ctx, epoch, seed, first_index, ids, R, out) */
int lig_schedule_models_batch_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                        const uint32_t* model_ids, int R, lig_mpick* out, int n_fallbacks,
                                        int16_t* fallbacks);
int lig_schedule_models_batch_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                               const uint32_t* d_model_ids, int R, lig_mpick* d_out,
                                               int n_fallbacks, int16_t* d_fallbacks, void* stream);

/* ---- session affinity: requests that share a key go to the same surviving pod -----------------------
 * Every other pick is a fresh draw, so two turns of one conversation rarely meet the pod that holds the
 * conversation's KV cache.  These calls replace the draw by rendezvous (highest random weight) hashing
 * on a caller key.  The reference picks with rand.Intn on an unseeded source (scheduler.go:120), so
 * any survivor is a legal outcome; an affinity pick is a member of exactly the survivor set the plain
 * call computes.
 *
 * Pod keys.  lig_upload_pod_keys gives epoch E a stable 64-bit identity per pod (pod_key[P], in E's
 * pod order; the schedulers use FNV-1a 64 over Name, a zero byte, then Address).  With mix the
 * SplitMix64 finalizer of the pick's stream, z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 * z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31), the device stores h_p = mix(pod_key[p]).
 * The table belongs to E like its model table: the upload is staged through the slot's pinned memory,
 * copied on the upload stream behind the slot's readers and recorded as an event every affinity call
 * on E is ordered behind.  lig_set_thresholds / lig_set_filter_tree rebuilds keep it; every writer that
 * makes a new epoch (full uploads, lig_update_snapshot, lig_eject_pods, lig_comm_*, the group upload)
 * leaves that epoch without keys.  LIG_ERR_INVALID when P differs from E's P or keys is null with
 * P > 0; a missing or stale epoch as every call reports it.  Refused uploads keep E's keys.
 *
 * The definition.  A request with affinity key k (lig_req.rand_key, or keys[i] for model ids) gives
 * survivor p the score s(k, p) = mix(k ^ h_p).  mix and ^k are bijections of 64-bit words, so distinct
 * pod keys give distinct scores, and the ranking is a strict order that does not depend on where a
 * pod sits in the snapshot.  Equal pod keys tie; ties break to the lower pod index, and the order
 * independence then holds only among distinct keys.
 *   - class, status and n_survivors are the plain call's (same class entry); for a LIG_OK request
 *     pod_idx is the member of its survivor list L with the highest score; otherwise -1.
 *   - the row, fallbacks[i * n_fallbacks .. (i + 1) * n_fallbacks): with m = min(n, 1 + n_fallbacks),
 *     entries 1 .. m-1 are the next members of L in descending score, then -1; a request that is not
 *     LIG_OK gets a row of -1.  The row for k fallbacks is a prefix of the row for any k' > k.
 *   - model ids resolve as in lig_schedule_models_batch, except that the target draw's state is
 *     k ^ LIG_DRAW_DOMAIN (no seed, no first_index), so a session keeps its target while the model's
 *     targets and weights stay the same.  target_idx is reported as there; a model that does not
 *     resolve gives {-1, LIG_NO_MODEL, 255} and a row of -1.
 *   - there is no seed and no counter: a request's output depends only on E's tables, its pod keys and
 *     the request, not on its place in the batch, how a batch is split or which ctx answers.  Two
 *     gateway replicas holding the same snapshot and keys agree.
 * Consistency: when L shrinks and still holds a key's pod, the key keeps it; when that pod leaves,
 * only its keys move.
 *
 * The calls read the resident epoch's tables, whichever build made them (built-in tree, caller tree,
 * an ejected epoch's pool, compact or strided lists), never a feedback chain's copy; they neither end
 * nor advance a chain.  Under a chain, lig_schedule_[models_]batch_feedback_chain_affinity below ranks
 * the chain's load-adjusted lists.  n_fallbacks = 0 means no row (fallbacks may then be NULL).  Refused, with
 * nothing written: LIG_ERR_INVALID for n_fallbacks outside [0, LIG_MAX_FALLBACKS], null buffers,
 * R > max_batch on the host forms and device buffers not aligned to their element (requests 16
 * bytes, picks 8 / 4, keys 8, rows 2); a stale epoch and a missing snapshot as lig_schedule_batch
 * reports them; LIG_ERR_NO_SNAPSHOT when E has no pod keys, and for the model forms when E has no
 * model table.  Host forms read and write page-locked buffers in place and stage pageable or
 * misaligned ones, as the fallback calls do, and block.  Device forms are enqueued on `stream` (NULL
 * = legacy default stream), not synchronised, and register as readers of the slot. */
int lig_upload_pod_keys(lig_ctx* ctx, uint64_t epoch, int P, const uint64_t* keys);
int lig_schedule_batch_affinity(lig_ctx* ctx, uint64_t epoch, const lig_req* reqs, int R, lig_pick* out,
                                int n_fallbacks, int16_t* fallbacks);
int lig_schedule_batch_affinity_device(lig_ctx* ctx, uint64_t epoch, const lig_req* d_reqs, int R, lig_pick* d_out,
                                       int n_fallbacks, int16_t* d_fallbacks, void* stream);
int lig_schedule_models_batch_affinity(lig_ctx* ctx, uint64_t epoch, const uint32_t* model_ids, const uint64_t* keys,
                                       int R, lig_mpick* out, int n_fallbacks, int16_t* fallbacks);
int lig_schedule_models_batch_affinity_device(lig_ctx* ctx, uint64_t epoch, const uint32_t* d_model_ids,
                                              const uint64_t* d_keys, int R, lig_mpick* d_out, int n_fallbacks,
                                              int16_t* d_fallbacks, void* stream);

/* ---- retry scheduling: schedule again without the pods a request already tried ------------------------
 * A fallback row runs out within a class's few survivors.  When every pod a proxy tried refused, the
 * reference's answer is Scheduler.Schedule over AllPodMetrics() without those pods (what it schedules
 * once they leave the provider): the range filters are recomputed over the remaining pods, so the
 * pick can be a pod outside the original survivor set.
 *
 * The definition.  Request i comes with row excluded[i * n_excluded .. (i + 1) * n_excluded) of int16
 * pod indices (the element type of a fallback row, so a proxy can pass back the pick and the row
 * entries it tried).  Its pool is the epoch's pods in their order minus the distinct entries of the
 * row that lie in [0, P); entries outside [0, P), -1 padding included, exclude nothing (as an
 * adapter_id outside [0, A) is a miss, not an error).  The result is Schedule (scheduler.go:113-122)
 * on that pool: the epoch's tree (the built-in tree with the ctx's thresholds, or the caller tree
 * that built the epoch, whatever lig_set_filter_tree has set since), n_survivors the size of the
 * reduced survivor set, the pick Int31n(n) on state seed ^ rand_key taking that survivor in pod
 * order, pod_idx an index into the epoch's full pod order.  Statuses are those of the schedule
 * calls; an empty pool runs as Go does with an empty slice (under the built-in tree: LIG_DROP for
 * critical and sheddable requests alike).  A row that excludes nothing gives lig_schedule_batch's
 * result byte for byte.  The calls read the resident epoch, never a feedback chain's copy; under a
 * chain, lig_schedule_batch_feedback_chain_excluding below walks the chain's copy.
 *
 * One warp per request walks the tree from its own pool (the direct scan's formulation).
 * LIG_ERR_INVALID, with nothing written, for n_excluded outside [1, LIG_MAX_EXCLUDED], null buffers
 * when R > 0, R > max_batch on the host form, and device buffers not aligned to their element
 * (requests 16 bytes, picks 8, rows 2); a stale epoch and a missing snapshot as lig_schedule_batch
 * reports them.  Host form: page-locked buffers are read and written in place, pageable or
 * misaligned ones (a request array at an odd 8 bytes included) are staged; it blocks until the picks
 * are back.  Device form: device pointers, enqueued on `stream` (NULL = legacy default stream), not
 * synchronised.  Both register as readers of the epoch's slot. */
#define LIG_MAX_EXCLUDED 32     /* one lane of the request's warp per entry */
int lig_schedule_batch_excluding(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                 const int16_t* excluded, int n_excluded, lig_pick* out);
int lig_schedule_batch_excluding_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                        int R, const int16_t* d_excluded, int n_excluded, lig_pick* d_out,
                                        void* stream);

/* ---- retry scheduling with fallback rows: the retry's pick and up to LIG_MAX_FALLBACKS more survivors ----
 * A retry returns one pod, so once a proxy has used up the first fallback row every further attempt
 * costs a whole retry call.  These calls return, with the retry's pick, a fallback row of the reduced
 * survivor set, so one round trip serves up to 1 + n_fallbacks attempts.
 *
 * The definition.  Request i, with its descriptor, its excluded row (format and rules of
 * lig_schedule_batch_excluding), seed and n_fallbacks = k:
 *   out[i] is what lig_schedule_batch_excluding returns for it, byte for byte: the same pool, the
 *   same tree (the epoch's built-in tree with the ctx's thresholds, or the caller tree that built
 *   the epoch), the same status and n_survivors.
 *   Its row, fallbacks[i * k .. (i + 1) * k), is the fallback ranking of the section above applied to
 *   L' = the reduced survivor set in ascending pod order (the set the retry's pick drew from), with
 *   n' = n_survivors: step 0 is the pick's own Int31n(n') draws on state seed ^ rand_key, rejections
 *   included; steps j = 1 .. m-1 (m = min(n', 1 + k)) draw j + Int31n(n' - j) on the continued
 *   stream, each swapping in a partial Fisher-Yates shuffle.  The row holds L'[perm[1]] ..
 *   L'[perm[m-1]] as pod indices in the epoch's pod order, then -1 up to k entries.  A request that is
 *   not LIG_OK gets a row of -1.
 * So no row entry is an excluded pod, entries are distinct, the row for k is a prefix of the row for
 * any k' > k, and a row that excludes nothing gives lig_schedule_batch_fallbacks's out and row byte
 * for byte (the reduced set is then the class's list).  The calls read the resident epoch only and
 * neither end nor advance a feedback chain.
 *
 * LIG_ERR_INVALID, with nothing written, for every reason either parent call refuses: n_excluded
 * outside [1, LIG_MAX_EXCLUDED], n_fallbacks outside [1, LIG_MAX_FALLBACKS], null buffers when R > 0,
 * R > max_batch on the host form, and device buffers not aligned to their element (requests 16
 * bytes, picks 8, both kinds of row 2); a stale epoch and a missing snapshot as lig_schedule_batch
 * reports them.  Host form: page-locked, aligned buffers are used in place, pageable or misaligned
 * ones (a request array at an odd 8 bytes included) are staged; it blocks until picks and rows are
 * back.  Device form: device pointers, enqueued on `stream` (NULL = legacy default stream), not
 * synchronised.  Both register as readers of the epoch's slot. */
int lig_schedule_batch_excluding_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                           const int16_t* excluded, int n_excluded, lig_pick* out,
                                           int n_fallbacks, int16_t* fallbacks);
int lig_schedule_batch_excluding_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                                  int R, const int16_t* d_excluded, int n_excluded, lig_pick* d_out,
                                                  int n_fallbacks, int16_t* d_fallbacks, void* stream);

/* ---- model-id retries: keep the drawn target, resolve on the device ------------------------------
 * A model-id request that needs a retry already went out rewritten to its drawn target, so a retry
 * must not draw again (a second draw could move it to another adapter and count it twice against
 * the traffic split).  These calls take the target index the first attempt returned
 * (lig_mpick.target_idx) and resolve it without a draw, so a caller of lig_schedule_models_batch
 * never interns adapter names or looks up criticality on the host to retry.
 *
 * The definition.  Request i is model_ids[i], targets[i] (a target_idx returned earlier), the
 * excluded row excluded[i * n_excluded ..) in the format and with the rules of
 * lig_schedule_batch_excluding, and rand_key = first_index + i (mod 2^64).  Fixed-target resolve
 * against E's model table as it stands at the call (no draw; LIG_DRAW_DOMAIN is not used): the
 * request is LIG_NO_MODEL when m >= n_models, present[m] == 0, the model has no TargetModels and
 * t != 255, or it has TargetModels and t >= their count.  Otherwise adapter_id = self_adapter_ids[m]
 * when t == 255, else target_adapter_ids[offset[m] + t], and Critical = critical[m].  out[i] is
 * lig_schedule_batch_excluding's pick for the descriptor {adapter_id, Critical, rand_key}, packed as
 * a lig_mpick {pod_idx, status, target_idx = t}; a LIG_NO_MODEL request gets {-1, LIG_NO_MODEL, 255}.
 * The pool, the tree, an ejected epoch's pool and the statuses are the descriptor retry's.  The
 * _fallbacks forms add lig_schedule_batch_excluding_fallbacks's row over the reduced survivor set;
 * a request that is not LIG_OK gets a row of -1.  The table re-interns target names at every
 * upload, so a target index stays valid across a refresh that gives adapters new ids.
 * So, with the target_idx values lig_schedule_models_batch[_fallbacks] returned for the same
 * (seed, first_index) and rows that exclude nothing, out and the rows are that call's byte for byte
 * (the pick stream seed ^ rand_key does not depend on the draw), and a model retry equals the
 * descriptor retry on host-built descriptors.
 *
 * Refused for every reason the descriptor counterpart is refused, with LIG_ERR_NO_SNAPSHOT when E
 * has no model table and LIG_ERR_INVALID for a null `targets` when R > 0; a bad id or target is
 * data (LIG_NO_MODEL), not a refusal.  Ordered behind the table's upload, both forms register as
 * readers of E's slot.  Host forms stage pageable or misaligned buffers; device forms refuse buffers
 * not aligned to their element (ids 4, picks 4, rows 2). */
int lig_schedule_models_batch_excluding(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                        const uint32_t* model_ids, const uint8_t* targets, int R,
                                        const int16_t* excluded, int n_excluded, lig_mpick* out);
int lig_schedule_models_batch_excluding_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                               const uint32_t* d_model_ids, const uint8_t* d_targets, int R,
                                               const int16_t* d_excluded, int n_excluded, lig_mpick* d_out,
                                               void* stream);
int lig_schedule_models_batch_excluding_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                                  const uint32_t* model_ids, const uint8_t* targets, int R,
                                                  const int16_t* excluded, int n_excluded, lig_mpick* out,
                                                  int n_fallbacks, int16_t* fallbacks);
int lig_schedule_models_batch_excluding_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                         uint64_t first_index, const uint32_t* d_model_ids,
                                                         const uint8_t* d_targets, int R, const int16_t* d_excluded,
                                                         int n_excluded, lig_mpick* d_out, int n_fallbacks,
                                                         int16_t* d_fallbacks, void* stream);

/* ---- in-batch load feedback (opt-in; the default path never mutates the snapshot) ----------------
 * The reference schedules every request against the scraped metrics as they are
 * (scheduler.go:113-122 never writes them), so all requests of one class that arrive inside a
 * 50 ms scrape window land on the same handful of survivors.  The simulator does account for
 * load per pick (simulations/llm_ig_simulation/src/loadbalancer.py:608-625: the chosen pod's
 * prefill queue grows immediately).  This entry point does the same at sub-batch granularity:
 * the batch is cut into windows of `sub_batch` requests; after every window the number of picks
 * each pod received — summed over all ranks with one ncclAllReduce(int32[P]) when the ctx has a
 * communicator (lig_comm_init_rank) — is added to that pod's WaitingQueueSize in a PRIVATE copy of
 * the snapshot, the class tables are rebuilt, and the next window is scheduled against them.
 *   n_windows <= 0: ceil(R / sub_batch) windows; ranks of one communicator must pass the same
 *   n_windows (trailing windows may be empty).  d_hist (nullable): int32[P], receives the total
 *   picks per pod of this call (all ranks).  Resident epochs are not modified.  Enqueued on
 *   `stream`, not synchronised.  Ends any feedback chain of the ctx (see below).  Defined
 *   sequentially in oracle/feedback.py. */
int lig_schedule_batch_feedback_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                       int R, lig_pick* d_out, int sub_batch, int n_windows,
                                       int32_t* d_hist, void* stream);

/* ---- load feedback across calls: the feedback chain (opt-in) ------------------------------------
 * A deployed scheduler sends a stream of small micro-batches, one per flush, against one scraped
 * epoch (refreshMetricsInterval = 50 ms, main.go:39); the herd of scheduler.go:113-122 forms
 * ACROSS those calls, where the in-batch call above cannot see it.  A chain carries the feedback
 * from call to call until the next metrics refresh replaces the epoch.
 *
 * A ctx holds at most one chain: a resident epoch E, a window size W >= 1, a private copy of E's
 * snapshot whose WaitingQueueSize column grows, and the requests counted so far.  Take the requests
 * of all chain calls against E, in call order, as one sequence and cut it into windows of W
 * requests; window boundaries ignore call boundaries.  Every request is scheduled against the
 * private copy's current tables with its own call's seed and its own rand_key, exactly as
 * lig_schedule_batch would on those tables.  When a window fills, its picks per pod are added to
 * WaitingQueueSize (saturating at INT32_MAX) and the tables are rebuilt before the next request;
 * DROP, EMPTY and NO_PODS_LEFT results count toward the window but add no pick.  So a chain of
 * calls with one seed gives the same picks as ONE lig_schedule_batch_feedback_device call over
 * their concatenation with sub_batch = W, however the requests are split into calls.
 *
 * A call starts a new chain (copies E afresh, zero loads) when its epoch differs from the chain's
 * or E was uploaded again since (the next scrape supersedes the estimate; lig_update_snapshot
 * makes a new epoch too), when its window differs, after lig_feedback_chain_reset, and after an
 * in-batch feedback call on the ctx (the two share one private copy).  The filter tree and the
 * thresholds in force when a chain starts rebuild all of its windows: a later lig_set_filter_tree
 * or lig_set_thresholds takes effect at the next chain start.  Resident epochs are never written.
 *
 * `window` is W; `loads` (nullable, int32[P]) receives the picks per pod since the chain began,
 * closed windows plus the open one; R = 0 with `loads` reads them without scheduling.  A call that
 * returns LIG_ERR_* for a bad argument (window < 1, R < 0, a null buffer, R > max_batch on the host
 * form), a stale epoch (E must be resident at every call), a ctx with a communicator, or a doorbell
 * stream open before the first feedback call allocated the private copy, leaves the chain exactly
 * as it was; after LIG_ERR_CUDA the next call starts a new chain.  Calls are serialised on the
 * chain; the order in which they take its lock is the sequence, so a reproducible sequence needs
 * one calling thread.  Calls may alternate between the two forms and between streams: each is
 * ordered behind the previous one on the device.  A ctx with a communicator (lig_comm_init_rank)
 * returns LIG_ERR_INVALID: per-rank micro-batch streams share no window boundaries.  Defined
 * sequentially in the tests' chain oracle (tests/feedback_chain_ref.py). */
/* host buffers (page-locked ones are used in place, pageable ones bounce like lig_schedule_batch);
 * blocks until `out` and `loads` are complete */
int lig_schedule_batch_feedback_chain(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                                      int R, lig_pick* out, int window, int32_t* loads);
/* device pointers, enqueued on `stream`, not synchronised */
int lig_schedule_batch_feedback_chain_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                             int R, lig_pick* d_out, int window, int32_t* d_loads, void* stream);
/* The same chain for model-id requests (see lig_schedule_models_batch).  A model-id call is one more
 * chain call: its R requests join the same sequence and the same windows as descriptor calls, and
 * the two kinds of call may alternate without restarting the chain; the restart rules above are
 * unchanged.  Request i of the call has rand_key = first_index + i; it is resolved against E's
 * model table as that table stands at the call, then picked on the chain's current private tables
 * with the call's seed.  So while no window has closed the picks equal lig_schedule_models_batch
 * byte for byte.  The model table is read from E's resident slot, never copied into the chain: a
 * lig_upload_models[_async] for E does not restart the chain (loads belong to pods, not to
 * models) and the next chain call resolves against the new table.  A call is ordered on the device
 * behind the table's upload, and a later model upload waits on the device for the calls that read
 * the table before it overwrites it, whatever their stream.  LIG_NO_MODEL, LIG_DROP, LIG_EMPTY and
 * LIG_NO_PODS_LEFT count toward the window and add no pick.  A call is refused, leaving the chain
 * exactly as it was, for the reasons above and with LIG_ERR_NO_SNAPSHOT when E has no model table. */
/* host buffers (page-locked ones used in place, pageable ones bounce); blocks */
int lig_schedule_models_batch_feedback_chain(lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                             const uint32_t* model_ids, int R, lig_mpick* out,
                                             int window, int32_t* loads);
/* device pointers, enqueued on `stream`, not synchronised */
int lig_schedule_models_batch_feedback_chain_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                    uint64_t first_index, const uint32_t* d_model_ids, int R,
                                                    lig_mpick* d_out, int window, int32_t* d_loads, void* stream);
/* Fallback rows under the chain.  A chain fallback call is a chain call of its kind in every
 * respect, plus a row per request:
 *   1. Picks and loads do not change: the R requests join the chain's sequence and windows exactly
 *      as a plain chain call's would, each is picked on the private copy's current tables with the
 *      call's seed and its rand_key, and only the pick is counted (row entries add no load: a
 *      fallback pod is loaded only if the proxy retries, and the chain's estimate must not depend on
 *      n_fallbacks).  So `out` and `loads` are byte for byte the plain chain call's on the same
 *      sequence, and calls with and without rows, of either kind, may alternate in one chain.
 *   2. Request i's row is the ranking of the fallback calls above, applied to the survivor list of
 *      its class in the chain's private tables at its position in the sequence: the list its pick
 *      drew from.  So entry 0 is the pick, the entries are distinct members of the load-adjusted
 *      survivor set, and the row for k is a prefix of the row for k' > k.  A row depends only on
 *      (seed, rand_key, the tables at its position): split invariance carries over, and while no
 *      window of the chain has closed `out` and the rows equal lig_schedule_[models_]batch_fallbacks
 *      on E byte for byte.
 *   3. Refused, with nothing written and the chain exactly as it was, for every reason the chain
 *      call is refused, and for n_fallbacks outside [1, LIG_MAX_FALLBACKS] or a null row buffer when
 *      R > 0; the device forms also for a row buffer that is not 2-byte aligned.
 * Host forms: page-locked, aligned rows are written in place; pageable or misaligned ones are staged
 * in a pinned area of max_batch * LIG_MAX_FALLBACKS int16 that the ctx allocates at first use. */
int lig_schedule_batch_feedback_chain_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                                                int R, lig_pick* out, int n_fallbacks, int16_t* fallbacks,
                                                int window, int32_t* loads);
int lig_schedule_batch_feedback_chain_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                       const lig_req* d_reqs, int R, lig_pick* d_out,
                                                       int n_fallbacks, int16_t* d_fallbacks, int window,
                                                       int32_t* d_loads, void* stream);
int lig_schedule_models_batch_feedback_chain_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                       uint64_t first_index, const uint32_t* model_ids, int R,
                                                       lig_mpick* out, int n_fallbacks, int16_t* fallbacks,
                                                       int window, int32_t* loads);
int lig_schedule_models_batch_feedback_chain_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                              uint64_t first_index, const uint32_t* d_model_ids,
                                                              int R, lig_mpick* d_out, int n_fallbacks,
                                                              int16_t* d_fallbacks, int window, int32_t* d_loads,
                                                              void* stream);
/* Session affinity under the chain.  Affinity alone sends every turn of a hot session, and every
 * key whose top pod is the same pod, to that pod for a whole scrape window.  Under the chain, the
 * pod's counts grow, the least-queuing filters drop it from the load-adjusted survivor set, and by
 * the consistency property of the ranking only the keys whose top was that pod move, each to its
 * next-ranked pod; the next scrape starts a new chain and they come back (bounded-load consistent
 * hashing).  A chain affinity call is a chain call in every respect except the choice among
 * survivors:
 *   1. Sequence and windows: the R requests join the ctx's one chain sequence and its windows
 *      exactly as a plain chain call's would; descriptor and model-id calls, with or without rows,
 *      of every chain kind (plain, fallback, retry, affinity), may alternate in one chain, and the
 *      restart rules are unchanged.
 *   2. The pick: request j takes the class entry of its class in the chain's private tables at its
 *      position in the sequence (the table a plain chain request at that position reads); status and
 *      n_survivors come from that entry.  For a LIG_OK request, pod_idx is the member of that list
 *      with the highest mix(k ^ h_p), ties to the lower pod index: the ranking of
 *      lig_schedule_batch_affinity applied to the load-adjusted list.  k is rand_key for descriptors
 *      and keys[i] for model ids; h_p are E's pod keys, read from E's resident slot.
 *   3. Counting: only the pick adds one to its pod in the open window; row entries add none.  DROP,
 *      EMPTY, NO_PODS_LEFT and NO_MODEL count toward the window and add no pick.
 *   4. Rows: n_fallbacks in [0, LIG_MAX_FALLBACKS], 0 = no row (fallbacks may then be NULL).  Entries
 *      1 .. m-1 (m = min(n, 1 + n_fallbacks)) are the next members of the same load-adjusted list in
 *      descending score, then -1; a request that is not LIG_OK gets a row of -1.  The row for k is a
 *      prefix of the row for any k' > k.
 *   5. Model ids resolve as in lig_schedule_models_batch_affinity (draw state k ^ LIG_DRAW_DOMAIN, no
 *      seed, no first_index) against E's model table as it stands at the call.  Neither a model
 *      upload nor a pod-key upload for E restarts the chain (loads belong to pods, and the keys to
 *      the same pods); a later upload of either waits on the device for the chain calls that read the
 *      old table.
 * So while no window of the chain has closed, `out` and the rows are lig_schedule_[models_]batch_affinity's
 * on E byte for byte; how requests are split into calls changes neither `out`, the rows nor `loads`;
 * and, like the resident affinity calls, the calls take no seed.  Refused, with nothing written and
 * the chain exactly as it was (not started, not restarted), for every reason a chain call is refused,
 * n_fallbacks outside [0, LIG_MAX_FALLBACKS], null buffers when R > 0, device buffers not aligned to
 * their element (requests 16 bytes, picks 8 / 4, keys 8, rows 2), and LIG_ERR_NO_SNAPSHOT when E has
 * no pod keys (and, for the model forms, no model table).  Host forms: page-locked, aligned buffers
 * are used in place; pageable or misaligned requests and picks bounce as for the plain chain call,
 * rows are staged as for the chain fallback calls, keys in stream-ordered device memory; they block.
 * Device forms: device pointers, enqueued on `stream`, not synchronised. */
int lig_schedule_batch_feedback_chain_affinity(lig_ctx* ctx, uint64_t epoch, const lig_req* reqs, int R,
                                               lig_pick* out, int n_fallbacks, int16_t* fallbacks, int window,
                                               int32_t* loads);
int lig_schedule_batch_feedback_chain_affinity_device(lig_ctx* ctx, uint64_t epoch, const lig_req* d_reqs, int R,
                                                      lig_pick* d_out, int n_fallbacks, int16_t* d_fallbacks,
                                                      int window, int32_t* d_loads, void* stream);
int lig_schedule_models_batch_feedback_chain_affinity(lig_ctx* ctx, uint64_t epoch, const uint32_t* model_ids,
                                                      const uint64_t* keys, int R, lig_mpick* out, int n_fallbacks,
                                                      int16_t* fallbacks, int window, int32_t* loads);
int lig_schedule_models_batch_feedback_chain_affinity_device(lig_ctx* ctx, uint64_t epoch,
                                                             const uint32_t* d_model_ids, const uint64_t* d_keys,
                                                             int R, lig_mpick* d_out, int n_fallbacks,
                                                             int16_t* d_fallbacks, int window, int32_t* d_loads,
                                                             void* stream);
/* Retries under the chain.  A chain retry call is a descriptor chain call in every respect, plus a
 * row of excluded pods per request in the format of lig_schedule_batch_excluding (int16, n_excluded
 * in [1, LIG_MAX_EXCLUDED], entries outside [0, P), -1 included, exclude nothing):
 *   1. Sequence and windows: the R requests join the chain's sequence and windows exactly as a plain
 *      chain call's would; window boundaries ignore call boundaries, retry calls may alternate with
 *      plain, model-id and fallback chain calls, and the restart rules are unchanged.
 *   2. Request i gets what lig_schedule_batch_excluding would return for it on the chain's private
 *      copy at its position in the sequence, with the call's seed and its rand_key, except that the
 *      pool is the chain's (its WaitingQueueSize has grown by every window closed so far) and the
 *      tree is the one the chain's windows are rebuilt with (the caller tree and thresholds in force
 *      when the chain started, not the epoch's own tree and not the ctx's current thresholds).
 *      pod_idx is in E's pod order; empty pools and statuses are the resident retry's.
 *   3. Only a LIG_OK pick adds one to its pod in the open window; DROP, EMPTY and NO_PODS_LEFT count
 *      toward the window's length.  `loads` as for the other chain calls.
 *   So rows that exclude nothing give the plain chain call's `out` and `loads` byte for byte; while
 *   no window has closed, and the chain's tree and thresholds are those E was built with, `out` is
 *   lig_schedule_batch_excluding's on E byte for byte; and results do not depend on how the requests
 *   are split into calls.  A retry segment reads no class table, so it never rebuilds the tables of
 *   a closed window: the next table-reading segment does, once.
 *   4. Refused, with nothing written and the chain exactly as it was, for every reason a chain call
 *      is refused and every reason lig_schedule_batch_excluding is refused (n_excluded, null buffers
 *      when R > 0, R > max_batch on the host form, device buffers not aligned to their element).
 * Host form: page-locked, aligned buffers are used in place; pageable or misaligned requests and
 * picks bounce as for the plain chain call, and such rows are staged in stream-ordered device memory;
 * it blocks.  Device form: device pointers, enqueued on `stream`, not synchronised. */
int lig_schedule_batch_feedback_chain_excluding(lig_ctx* ctx, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                                                int R, const int16_t* excluded, int n_excluded, lig_pick* out,
                                                int window, int32_t* loads);
int lig_schedule_batch_feedback_chain_excluding_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                       const lig_req* d_reqs, int R, const int16_t* d_excluded,
                                                       int n_excluded, lig_pick* d_out, int window,
                                                       int32_t* d_loads, void* stream);
/* Retries with fallback rows under the chain.  A chain retry call with rows is
 * lig_schedule_batch_feedback_chain_excluding in every respect, plus a fallback row per request, as
 * lig_schedule_batch_feedback_chain_fallbacks adds rows to the plain chain call:
 *   1. Sequence, windows, picks and loads do not change: request i's `out` is what
 *      lig_schedule_batch_feedback_chain_excluding returns for it at the same position, byte for byte
 *      (the chain's private copy, the tree and thresholds the chain started with, the call's seed and
 *      its rand_key).  Only a LIG_OK pick adds load; row entries add none, so `loads` does not depend
 *      on n_fallbacks.  Calls with and without rows, of every kind (plain, model-id, fallback,
 *      retry), may alternate in one chain, and the restart rules are unchanged.
 *   2. Request i's row is the ranking of lig_schedule_batch_excluding_fallbacks applied to the
 *      chain's pool instead of the epoch's: L' = the reduced survivor set of that walk in ascending
 *      pod order, n' = n_survivors; step 0 is the pick's own Int31n(n') draws on seed ^ rand_key,
 *      steps j = 1 .. m-1 draw j + Int31n(n' - j) on the continued stream; entries are pod indices in
 *      E's pod order, padded with -1 up to k; a request that is not LIG_OK gets a row of -1.
 *   So no row entry is an excluded pod, the entries are distinct, the row for k is a prefix of the
 *   row for k' > k, and results do not depend on how the requests are split into calls.  Rows that
 *   exclude nothing give lig_schedule_batch_feedback_chain_fallbacks's `out`, rows and `loads` byte
 *   for byte; while no window has closed, and the chain's tree and thresholds are those E was built
 *   with, `out` and the rows are lig_schedule_batch_excluding_fallbacks's on E byte for byte.  Like a
 *   chain retry segment, a segment of this call reads no class table.
 *   3. Refused, with nothing written and the chain exactly as it was, for every reason the chain
 *      retry call is refused and every reason the chain fallback calls are refused (n_fallbacks
 *      outside [1, LIG_MAX_FALLBACKS], a null row buffer when R > 0, a device row buffer that is not
 *      2-byte aligned).
 * Host form: excluded rows are staged as for the chain retry call, fallback rows as for the chain
 * fallback calls; it blocks.  Device form: device pointers, enqueued on `stream`, not synchronised. */
int lig_schedule_batch_feedback_chain_excluding_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                          const lig_req* reqs, int R, const int16_t* excluded,
                                                          int n_excluded, lig_pick* out, int n_fallbacks,
                                                          int16_t* fallbacks, int window, int32_t* loads);
int lig_schedule_batch_feedback_chain_excluding_fallbacks_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                                 const lig_req* d_reqs, int R,
                                                                 const int16_t* d_excluded, int n_excluded,
                                                                 lig_pick* d_out, int n_fallbacks,
                                                                 int16_t* d_fallbacks, int window,
                                                                 int32_t* d_loads, void* stream);
/* Model-id retries under the chain: the model-id retries above (fixed-target resolve, then the
 * descriptor's retry) as chain calls in every respect.  The requests join the chain's sequence and
 * windows, and calls of every kind (descriptor and model, plain, fallback and retry) may alternate.
 * The walk uses the chain's private copy and the tree and thresholds the chain started with.  Only a
 * LIG_OK pick adds load; LIG_NO_MODEL, DROP, EMPTY and NO_PODS_LEFT count toward the window's length
 * and add none, and row entries add none.  The model table is read from E's resident slot, as
 * lig_schedule_models_batch_feedback_chain reads it.  So with the target_idx values the plain model
 * chain call returned at the same positions and rows that exclude nothing, picks, rows and loads are
 * that call's byte for byte.  Refused, leaving the chain exactly as it was, for every reason the
 * descriptor chain retry calls are refused, with LIG_ERR_NO_SNAPSHOT when E has no model table, and
 * with LIG_ERR_INVALID for a null `targets` when R > 0.  Host forms stage pageable targets in
 * stream-ordered device memory, as they stage excluded rows. */
int lig_schedule_models_batch_feedback_chain_excluding(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                       uint64_t first_index, const uint32_t* model_ids,
                                                       const uint8_t* targets, int R, const int16_t* excluded,
                                                       int n_excluded, lig_mpick* out, int window, int32_t* loads);
int lig_schedule_models_batch_feedback_chain_excluding_device(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                              uint64_t first_index, const uint32_t* d_model_ids,
                                                              const uint8_t* d_targets, int R,
                                                              const int16_t* d_excluded, int n_excluded,
                                                              lig_mpick* d_out, int window, int32_t* d_loads,
                                                              void* stream);
int lig_schedule_models_batch_feedback_chain_excluding_fallbacks(lig_ctx* ctx, uint64_t epoch, uint64_t seed,
                                                                 uint64_t first_index, const uint32_t* model_ids,
                                                                 const uint8_t* targets, int R,
                                                                 const int16_t* excluded, int n_excluded,
                                                                 lig_mpick* out, int n_fallbacks, int16_t* fallbacks,
                                                                 int window, int32_t* loads);
int lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device(
    lig_ctx* ctx, uint64_t epoch, uint64_t seed, uint64_t first_index, const uint32_t* d_model_ids,
    const uint8_t* d_targets, int R, const int16_t* d_excluded, int n_excluded, lig_mpick* d_out, int n_fallbacks,
    int16_t* d_fallbacks, int window, int32_t* d_loads, void* stream);
/* The next chain call starts a new chain. */
int lig_feedback_chain_reset(lig_ctx* ctx);

/* ---- several GPUs, one process (the reference runs ONE scheduler per process, main.go:137) ------
 * A lig_group owns one lig_ctx per listed CUDA device and an NCCL communicator over them
 * (ncclCommInitAll).  The request batch shards BY REQUEST (decisions are independent given a
 * frozen snapshot: Schedule never mutates pod metrics, scheduler.go:113-122); the snapshot is
 * replicated with one ncclBroadcast per refresh tick, received directly into every member's
 * resident snapshot slot and consumed in place by the class-table build.  Picks need no
 * collective: device g owns the contiguous shard [R*g/G, R*(g+1)/G) of the result. */
typedef struct lig_group lig_group;
int  lig_group_create(lig_group** out, const int* devices, int n_devices, int max_pods,
                      int max_adapters, int max_batch);
void lig_group_destroy(lig_group* g);
int  lig_group_size(const lig_group* g);
lig_ctx* lig_group_ctx(lig_group* g, int member);   /* member ctx, e.g. for the device-pointer API */
int  lig_group_set_thresholds(lig_group* g, const lig_thresholds* t);
/* lig_set_filter_tree on every member (validated once: an invalid table changes no member). */
int  lig_group_set_filter_tree(lig_group* g, const lig_filter_node* nodes, int n_nodes);
/* lig_upload_snapshot for the whole group: one pack, one H2D to member 0, one ncclBroadcast over
 * NVLink, one class-table build per member.  Resident on every member when it returns. */
int  lig_group_upload_snapshot(lig_group* g, uint64_t epoch, int P, int A, const double* kv,
                               const int32_t* q, const uint16_t* n_active,
                               const uint16_t* max_active, const uint32_t* bitmap_adapter_major);
/* lig_schedule_batch over the group: contiguous request shards, results in request order.  The
 * pick of a request depends on (seed, rand_key) only, so the result equals the single-device
 * result bit for bit.  Page-locked buffers must be portable (lig_host_alloc is). */
int  lig_group_schedule_batch(lig_group* g, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                              int R, lig_pick* out);

/* ---- several GPUs, one process per GPU (torchrun-style launch) ----------------------------------
 * Rank 0 calls lig_comm_unique_id and ships the LIG_COMM_ID_BYTES to the other ranks by any means
 * (a file, an env var, the launcher's store); every rank then calls lig_comm_init_rank on its own
 * ctx.  lig_comm_upload_snapshot_device replicates the root's packed blob (device memory on the
 * root; ignored elsewhere) into every rank's snapshot slot with one ncclBroadcast enqueued on
 * `stream`, followed by the class-table build on the same stream; nothing is synchronised.
 * lig_comm_upload_snapshot is the blocking host-array form (arrays read on the root only). */
#define LIG_COMM_ID_BYTES 128
int lig_comm_unique_id(void* id /* LIG_COMM_ID_BYTES */);
int lig_comm_init_rank(lig_ctx* ctx, int n_ranks, int rank, const void* id);
int lig_comm_upload_snapshot_device(lig_ctx* ctx, uint64_t epoch, int P, int A, const void* d_blob,
                                    int root, void* stream);
int lig_comm_upload_snapshot(lig_ctx* ctx, uint64_t epoch, int P, int A, const double* kv,
                             const int32_t* q, const uint16_t* n_active, const uint16_t* max_active,
                             const uint32_t* bitmap_adapter_major, int root);
/* In-place sum of an int32 vector over the ranks (ncclAllReduce on `stream`): the per-pod pick
 * histogram of the load-feedback mode. */
int lig_comm_allreduce_i32(lig_ctx* ctx, int32_t* d_values, int n, void* stream);

/* ---- introspection ------------------------------------------------------------------------- */
const char* lig_last_error(void);            /* thread-local, never NULL */
const char* lig_version(void);
int         lig_abi_version(void);
int         lig_device_count(void);          /* 0 when no CUDA device / driver */
uint64_t    lig_kernel_launches(const lig_ctx* ctx);  /* kernels this ctx launched so far */
int         lig_sm_count(const lig_ctx* ctx);
/* The pick kernel a device-resident queue launches against `epoch` right now: its name, resident
 * grid and block size (bench.py checks its committed ncu capture against this), and the size of
 * the compact tables (0 = not available / strided tables in use). */
int         lig_pick_kernel_info(lig_ctx* ctx, uint64_t epoch, char* name, int name_len, int* grid,
                                 int* threads, int* table_bytes, int* tables_in_smem);
/* The pick kernel of this ctx's most recent pick launch and its template arguments: what the
 * LIG_* knobs, the buffers' alignment and the table sizes selected for it (0 where a field does
 * not apply).  Recorded at the launch; kernel is LIG_KERNEL_NONE before the first one. */
#define LIG_KERNEL_NONE         0
#define LIG_KERNEL_PERSISTENT   1   /* lig_pick_persistent_kernel<groups, stages, bulk_store, tables_in_smem> */
#define LIG_KERNEL_LOOP         2   /* lig_pick_loop_kernel<tables_in_smem> */
#define LIG_KERNEL_PLAIN        3   /* lig_pick_stream_kernel<per_thread> */
#define LIG_KERNEL_QUEUE        4   /* lig_pick_queue_kernel<per_thread>: the merged queue */
#define LIG_KERNEL_MODELS       5   /* lig_pick_models_kernel<groups, stages, tables_in_smem> */
#define LIG_KERNEL_MODELS_PLAIN 6   /* lig_pick_models_stream_kernel */
typedef struct lig_launch_info {
  int32_t kernel, groups, stages, bulk_store, tables_in_smem, per_thread;
} lig_launch_info;
int         lig_last_pick_launch(lig_ctx* ctx, lig_launch_info* info);

#ifdef __cplusplus
}
#endif
#endif /* LIG_H_ */
