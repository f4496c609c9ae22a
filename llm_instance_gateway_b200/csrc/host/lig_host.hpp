// lig_host.hpp — native host side above the C ABI (include/lig.h): the C++ counterpart of the Go
// adapter a maintainer adds to the reference (INTEGRATION.md).  It mirrors the reference's
// scheduling-package interface for the hot path — same names, argument meaning, error behaviour:
//
//   backend::Pod / Metrics / PodMetrics     pkg/ext-proc/backend/types.go:8-31
//   scheduling::LLMRequest                   pkg/ext-proc/scheduling/types.go:4-11
//   scheduling::PodMetricsProvider           pkg/ext-proc/scheduling/scheduler.go:108-110
//   scheduling::NewScheduler / Scheduler     pkg/ext-proc/scheduling/scheduler.go:93-122
//
// Scheduler::Schedule is goroutine-style safe: many threads call it concurrently and block for
// their pick (one caller per Envoy stream, pkg/ext-proc/handlers/request.go:72); a batcher thread
// folds the concurrent calls into one lig_schedule_batch call per flush.  The snapshot is
// re-packed once per refresh tick (refreshMetricsInterval, pkg/ext-proc/main.go:39) instead of
// once per request.  No CPU scheduling path exists here: without liblig.so + a CUDA device,
// NewScheduler fails.
//
// Model requests.  ScheduleModel(datastore, ...) resolves a request on the caller's thread
// (FetchModelData, RandomWeightedDraw, IsCritical) and sends the resolved descriptor through
// Schedule.  ScheduleModel(model, ...) sends only the model name: SetInferenceModels gives the
// scheduler the datastore's InferenceModels, every snapshot epoch carries them as a device model
// table (lig_upload_models, target names interned against that epoch's adapter ids), and the
// batcher maps names to model ids at flush time and lets the device resolve, draw and pick in one
// call (lig_schedule_models_batch, lig_stream_submit_models with use_doorbell, or
// lig_schedule_models_batch_feedback_chain with load_feedback_window).  Pods, adapter ids and the
// model table always change together, in one published epoch.
#pragma once

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../../include/lig.h"

struct lig_ctx;
struct lig_group;
struct lig_req;
struct lig_pick;

namespace lig {

namespace backend {

struct Pod {                         // backend/types.go:8-11
  std::string Name;
  std::string Address;
  std::string String() const { return Name + ":" + Address; }   // types.go:13-15
};

struct Metrics {                     // backend/types.go:17-26
  std::map<std::string, int> ActiveModels;
  int64_t MaxActiveModels = 0;
  int64_t RunningQueueSize = 0;
  int64_t WaitingQueueSize = 0;
  double KVCacheUsagePercent = 0.0;
  int64_t KvCacheMaxTokenCapacity = 0;
};

struct PodMetrics {                  // backend/types.go:28-31
  Pod pod;
  Metrics metrics;
};

// api/v1alpha1/inferencemodel_types.go: the fields the request path reads
struct TargetModel {
  std::string Name;
  int32_t Weight = 0;
};
struct InferenceModel {
  std::string ModelName;             // Spec.ModelName: the key requests carry in "model"
  bool Critical = false;             // Spec.Criticality != nil && *Spec.Criticality == Critical
  std::vector<TargetModel> TargetModels;
};

class ModelDataStore {               // handlers/server.go:47-49
 public:
  virtual ~ModelDataStore() = default;
  virtual std::shared_ptr<const InferenceModel> FetchModelData(const std::string& modelName) = 0;
};

// A rand.Source over SplitMix64: the injected source include/lig.h defines the draw and the pick on.
struct SplitMixSource {
  uint64_t state;
  uint64_t Uint64();
  int32_t Int31() { return (int32_t)(Uint64() >> 33); }          // Int63() >> 32
  int32_t Int31n(int32_t n);                                      // math/rand (Go 1.22)
};

// RandomWeightedDraw(model, seed)                                 backend/datastore.go:78-98
// Returns "" like the reference when no target is hit; weights summing to <= 0 (where Go's
// Int31n panics) also return "".
std::string RandomWeightedDraw(const InferenceModel& model, SplitMixSource source);

}  // namespace backend

namespace scheduling {

struct LLMRequest {                  // scheduling/types.go:4-11
  std::string Model;
  std::map<std::string, int> TargetModels;
  std::string ResolvedTargetModel;
  bool Critical = false;
};

// google.golang.org/grpc/codes values the path can produce.
enum Code : int { OK = 0, Unknown = 2, InvalidArgument = 3, ResourceExhausted = 8, Internal = 13 };

struct Status {                      // a Go `error` carrying a gRPC status code
  int code = OK;
  std::string message;
  bool ok() const { return code == OK; }
};

class PodMetricsProvider {           // scheduling/scheduler.go:108-110
 public:
  virtual ~PodMetricsProvider() = default;
  virtual std::vector<std::shared_ptr<const backend::PodMetrics>> AllPodMetrics() = 0;
};

struct Options {
  int device = 0;
  // More than one entry: ONE scheduler owns all listed GPUs (lig_group_*): the snapshot is
  // replicated by an in-library ncclBroadcast per refresh, every flushed batch is sharded by request.
  std::vector<int> devices;
  int max_pods = 4096;
  int max_adapters = 1024;
  int max_batch = 1 << 16;
  // A batch is flushed when it has flush_size requests or its oldest request is batch_window old.
  int flush_size = 4096;
  std::chrono::microseconds batch_window{50};
  uint64_t seed = 0;                 // 0 = seed from std::random_device (Go's auto-seeded source)
  // >0: a refresher thread re-packs the provider's snapshot at this period.
  std::chrono::milliseconds refresh_interval{0};
  // Latency knobs: the batcher thread polls its queue instead of sleeping on a condition
  // variable, and callers spin this long on their result before blocking in the kernel.
  // Flush micro-batches through the persistent doorbell kernel (lig_stream_submit) instead of a
  // kernel launch per flush.  Nothing else in the process may then synchronise the whole device.
  bool use_doorbell = false;
  bool busy_poll = false;
  std::chrono::microseconds caller_spin{0};
  double kv_cache_threshold = 0.8;   // scheduler.go:15-24
  int64_t queue_threshold_critical = 5;
  int64_t queueing_threshold_lora = 50;
  // A caller flow chart of the reference's filter nodes (lig_set_filter_tree, node 0 = root)
  // instead of defaultFilter; empty = the built-in tree.  Its nodes carry their own thresholds.
  std::vector<lig_filter_node> filter;
  // >0: in-batch load feedback carried across flushes (lig_schedule_batch_feedback_chain): every
  // window of this many requests adds its picks to the pods' WaitingQueueSize before the next
  // request is scheduled, until the next refresh replaces the snapshot (each refresh restarts the
  // chain on the new epoch).  0 = off, the reference's behaviour.  Single device, no doorbell.
  int load_feedback_window = 0;
  // With load_feedback_window > 0: let ScheduleWithFallbacks and ScheduleModelWithFallbacks run as
  // feedback-chain calls (lig_schedule_[models_]batch_feedback_chain_fallbacks), whose rows rank the
  // survivors in the chain's load-adjusted tables, the set the pick itself drew from.  Picks and
  // feedback windows are the same with or without it.  Off by default only because those calls have
  // always been refused under feedback with InvalidArgument and that refusal is relied upon; without
  // it they still are.  No effect without load_feedback_window.  Together with feedback_retries it
  // also lets ScheduleRetryWithFallbacks run under the chain (see there).
  bool feedback_fallbacks = false;
  // With load_feedback_window > 0: let ScheduleRetry run as feedback-chain calls
  // (lig_schedule_batch_feedback_chain_excluding): a retry is scheduled on the chain's load-adjusted
  // copy without the pods it tried, and its pick counts toward the chain's windows like any other.
  // Off by default because ScheduleRetry has always been refused under feedback with InvalidArgument;
  // without it, it still is.  No effect without load_feedback_window.  Together with
  // feedback_fallbacks it also lets ScheduleRetryWithFallbacks run under the chain (see there).
  bool feedback_retries = false;
  // Upload the pods' keys (PodKey) with every epoch the scheduler publishes (full, delta and ejected),
  // so that ScheduleAffinity and its relatives can place requests by a caller key
  // (lig_schedule_[models_]batch_affinity).  Off: those calls are refused and nothing else changes.
  bool affinity = false;
  // With affinity and load_feedback_window > 0: let the affinity calls run as feedback-chain calls
  // (lig_schedule_[models_]batch_feedback_chain_affinity): a request takes the top-scoring pod of the
  // chain's load-adjusted survivors, and its pick counts toward the chain's windows like any other, so
  // a hot key moves off a pod the chain has loaded out of the survivor set until the next refresh.  Off
  // by default because those calls have always been refused under feedback with InvalidArgument;
  // without it they still are.  No effect without load_feedback_window.
  bool feedback_affinity = false;
};

// A pod's affinity identity: FNV-1a 64 over Name, a zero byte, then Address (the provider's own
// identity of a pod, so a pod keeps its key whatever order the provider lists it in).
uint64_t PodKey(const backend::Pod& pod);

struct Stats {
  uint64_t scheduled = 0;      // Schedule calls completed
  uint64_t batches = 0;        // lig_schedule_batch calls issued
  uint64_t max_batch = 0;      // largest batch flushed
  uint64_t refreshes = 0;      // snapshots uploaded
  uint64_t stale_retries = 0;  // batches and Filter calls re-resolved after LIG_ERR_STALE_EPOCH
  uint64_t delta_refreshes = 0;    // refreshes that went through lig_update_snapshot (dirty pods only)
  uint64_t last_dirty_pods = 0;    // pods whose metrics changed at the last refresh
  uint64_t failed_refreshes = 0;   // Refresh() calls that kept the previous snapshot (see last_refresh_error)
  uint64_t excluded_pods = 0;      // pods left out of the last snapshot: a metric did not fit the device record
  uint64_t feedback_windows = 0;   // load-feedback windows closed (Options::load_feedback_window)
  uint64_t feedback_restarts = 0;  // feedback chains restarted on a new epoch after the first one
  uint64_t model_scheduled = 0;    // ScheduleModel(model, ...) calls completed (host-answered ones included)
  uint64_t model_batches = 0;      // device calls issued for model-id requests
  uint64_t fallback_scheduled = 0; // ScheduleWithFallbacks and ScheduleModelWithFallbacks calls completed
  uint64_t retry_scheduled = 0;    // ScheduleRetry, ScheduleModelRetry and their WithFallbacks calls completed
  uint64_t ejected_pods = 0;       // pods of the current snapshot left out of the pool (EjectPods)
  uint64_t eject_publishes = 0;    // epochs derived with lig_eject_pods and published
  uint64_t affinity_scheduled = 0; // ScheduleAffinity, ScheduleModelAffinity and their WithFallbacks calls completed
  double last_pack_us = 0;     // last Refresh: provider slice -> columns + bitmap (host)
  double last_upload_us = 0;   // last Refresh: lig_upload_snapshot (H2D + class tables)
  double max_device_call_us = 0;   // slowest single lig_schedule_batch call (launch + kernel + synchronise)
  double max_flush_us = 0;         // slowest Flush: resolve + device call + waking the callers
  uint64_t slowest_call_batch = 0; // which batch (0-based count of device calls) that slowest call was
  double slowest_call_cpu_us = 0;  // CPU time the batcher thread burnt inside that call: ~ its wall time when it
                                   // was spinning on a busy device, far less when the thread itself was descheduled
};

class Scheduler {
 public:
  ~Scheduler();
  Scheduler(const Scheduler&) = delete;
  Scheduler& operator=(const Scheduler&) = delete;

  // Schedule finds the target pod based on metrics and the requested lora adapter.
  // Returns OK and fills *targetPod, or: ResourceExhausted "dropping request due to limited
  // backend resources" wrapped exactly like scheduler.go:117 (-> HTTP 429 at
  // handlers/server.go:97-109); Unknown for the "resulted 0 pods" case; Internal for a
  // batch-level (CUDA) failure.                                       scheduler.go:113-122
  Status Schedule(const LLMRequest& req, backend::Pod* targetPod);

  // Schedule plus up to n fallback endpoints (1 <= n <= LIG_MAX_FALLBACKS): fills *pods with the pick
  // (pods[0], the pod Schedule would have returned for the same rand_key) and then up to n more
  // distinct survivors in the order a proxy should retry them (include/lig.h, fallback endpoints).
  // Goes through the micro-batcher and takes the next rand_key like Schedule; errors are Schedule's.
  // A flush in which any caller asked for fallbacks makes its device call with
  // lig_schedule_batch_fallbacks (the largest n asked in that flush); plain Schedule callers in it get
  // the same picks.  With load_feedback_window > 0 and Options::feedback_fallbacks, that call is
  // lig_schedule_batch_feedback_chain_fallbacks in place of the chain call: same picks and windows,
  // rows from the chain's tables.  InvalidArgument for n outside [1, LIG_MAX_FALLBACKS], with
  // load_feedback_window > 0 and no feedback_fallbacks (the picks come from the feedback chain's
  // copy), and with several devices.
  Status ScheduleWithFallbacks(const LLMRequest& req, int n, std::vector<backend::Pod>* pods);

  // Schedule again without the pods already tried: Schedule over the current epoch's pods minus
  // `tried` (lig_schedule_batch_excluding), what Schedule returns once those pods have left the
  // provider.  Tried pods are matched by value (Name and Address) against the snapshot current at
  // flush time, so a retry after a refresh still excludes the right pods; pods no longer in it are
  // ignored.  Goes through the micro-batcher and takes the next rand_key from the same sequence as
  // Schedule, in flush order; a flush's retries make one device call after its plain descriptor
  // requests, never through the doorbell.  Errors are Schedule's.  InvalidArgument with more than
  // LIG_MAX_EXCLUDED (32) tried pods, with load_feedback_window > 0 unless Options::feedback_retries
  // (then the flush's retries make one lig_schedule_batch_feedback_chain_excluding call instead, and a
  // waiter refused on the host is left out of it, so it loads no pod) and with several devices.  A handler that used
  // ScheduleModel retries with ScheduleModelRetry.
  Status ScheduleRetry(const LLMRequest& req, const std::vector<backend::Pod>& tried, backend::Pod* targetPod);

  // ScheduleRetry plus up to n fallback endpoints (1 <= n <= LIG_MAX_FALLBACKS): fills *pods with the
  // retry's pick (pods[0], the pod ScheduleRetry would have returned for the same rand_key and tried
  // pods) and then up to n more distinct survivors of the same reduced pool, none of them tried, in the
  // order a proxy should try them (lig_schedule_batch_excluding_fallbacks), so one call serves several
  // attempts.  Goes through the retry lane like ScheduleRetry: a flush whose retry lane holds any such
  // caller makes one lig_schedule_batch_excluding_fallbacks call at the largest n asked in it, and plain
  // ScheduleRetry callers in it get the same picks.  Never through the doorbell; counted in
  // Stats::retry_scheduled.  Errors are Schedule's.  With load_feedback_window > 0 and both
  // Options::feedback_retries and Options::feedback_fallbacks, that call is
  // lig_schedule_batch_feedback_chain_excluding_fallbacks in place of the chain retry call: same picks
  // and windows (rows add no load), rows from the reduced pool of the chain's load-adjusted copy, and a
  // waiter refused on the host is left out of it.  InvalidArgument for n outside [1, LIG_MAX_FALLBACKS],
  // more than LIG_MAX_EXCLUDED tried pods, load_feedback_window > 0 without both of those options, and
  // several devices.
  Status ScheduleRetryWithFallbacks(const LLMRequest& req, const std::vector<backend::Pod>& tried, int n,
                                    std::vector<backend::Pod>* pods);

  // The reference's Filter interface (filter.go:12-15) run on the current epoch: fills *pods with
  // the survivors of req's walk of the filter tree (the built-in one or Options::filter), in slice
  // order.  One blocking lig_filter_batch call on the caller's thread, outside the micro-batcher; no
  // rand_key is taken.  Errors are the tree's own: ResourceExhausted "dropping request due to
  // limited backend resources" for the drop leaf, Unknown "no pods left" when a caller tree ends on a
  // predicate that kept no pod, Internal for a device failure; an empty result is OK with no pods.
  // A scheduler over several devices refuses it with InvalidArgument.
  Status Filter(const LLMRequest& req, std::vector<backend::Pod>* pods);

  // The resolve step of HandleRequestBody (handlers/request.go:42-56) followed by Schedule:
  // FetchModelData, RandomWeightedDraw when TargetModels is non-empty, IsCritical.  Fills
  // *resolvedTargetModel (the body's "model" is rewritten with it, request.go:60-69).  Errors as the
  // reference: Unknown "error finding a model object in InferenceModel for input <model>" /
  // "error getting target model name for model <name>".
  Status ScheduleModel(backend::ModelDataStore& datastore, const std::string& model, std::string* resolvedTargetModel,
                       backend::Pod* targetPod);

  // The same step resolved on the device, against the list last given to SetInferenceModels (none
  // given: every model is unknown, like an empty datastore).  The batcher maps the name to the
  // captured epoch's model id at flush time; the device draws the target and picks the pod.
  // Unknown models and models whose weights sum to <= 0 are answered on the host with the errors
  // above and take no rand_key and no place in a feedback window.  Other errors are those of
  // Schedule, prefixed "failed to find target pod: " (request.go:73-75).  Request k that reaches
  // the device (counted from 0 per scheduler) has rand_key = k: the draw and the pick are those of
  // lig_schedule_models_batch with first_index = k.  Neither rand_key sequence of the two calls
  // above is touched.
  Status ScheduleModel(const std::string& model, std::string* resolvedTargetModel, backend::Pod* targetPod);

  // ScheduleModel(model, ...) plus up to n fallback endpoints: *pods gets the pick (the pod
  // ScheduleModel would have returned for the same rand_key) and then up to n more distinct survivors
  // in retry order.  Host-answered errors, *resolvedTargetModel and the rand_key sequence are
  // ScheduleModel's.  A model-id flush with any such caller makes its device call with
  // lig_schedule_models_batch_fallbacks at the largest n asked among the requests it sends (under
  // load_feedback_window with Options::feedback_fallbacks, the chain-fallback model call) and skips
  // the doorbell.  Refused like ScheduleWithFallbacks.
  Status ScheduleModelWithFallbacks(const std::string& model, int n, std::string* resolvedTargetModel,
                                    std::vector<backend::Pod>* pods);

  // The retry of a ScheduleModel(model, ...) request without the pods it tried, keeping the target it
  // drew: resolvedTargetModel is the name ScheduleModel returned, so the retry does not draw again (the
  // body went out rewritten to it).  At flush time, against the captured epoch's list, the batcher maps
  // model to its id and resolvedTargetModel to the first TargetModels entry of that name, or, for a
  // model without TargetModels, to its own name; the device resolves that target and schedules as
  // ScheduleRetry does (lig_schedule_models_batch_excluding).  Tried pods are matched by value as in
  // ScheduleRetry.  Answered on the host, with no rand_key and no place in a feedback window: an
  // unknown model or one whose weights sum to <= 0 with ScheduleModel's Unknown errors, a name that is
  // not a target of the model in the current list and tried pods matching more than LIG_MAX_EXCLUDED
  // pods of the snapshot with InvalidArgument.  Requests that reach the device take their rand_keys
  // from ScheduleModel's sequence, after the flush's ScheduleModel requests.  Other errors are
  // ScheduleModel's.  Never through the doorbell; counted in Stats::retry_scheduled, its device calls
  // in Stats::model_batches.  InvalidArgument for more than LIG_MAX_EXCLUDED tried pods, with
  // load_feedback_window > 0 unless Options::feedback_retries (then the call is
  // lig_schedule_models_batch_feedback_chain_excluding), and with several devices.
  Status ScheduleModelRetry(const std::string& model, const std::string& resolvedTargetModel,
                            const std::vector<backend::Pod>& tried, backend::Pod* targetPod);

  // ScheduleModelRetry plus up to n fallback endpoints (1 <= n <= LIG_MAX_FALLBACKS), as
  // ScheduleRetryWithFallbacks adds them to ScheduleRetry: a flush whose model-retry lane holds any such
  // caller makes one lig_schedule_models_batch[_feedback_chain]_excluding_fallbacks call at the largest
  // n asked.  Under load_feedback_window it needs both Options::feedback_retries and
  // Options::feedback_fallbacks; refused otherwise like ScheduleModelRetry.
  Status ScheduleModelRetryWithFallbacks(const std::string& model, const std::string& resolvedTargetModel,
                                         const std::vector<backend::Pod>& tried, int n,
                                         std::vector<backend::Pod>* pods);

  // Replace the InferenceModels that ScheduleModel(model, ...) resolves against; of two models
  // with one ModelName the later wins (the reference's datastore is a map).  Publishes a new epoch
  // through Refresh, so the list applies from that epoch on, and like every new epoch it restarts
  // the load-feedback chain.  A list the device cannot take (a model with more than 255 targets, a
  // negative weight, weights summing above 2^31-1) or a failed refresh leaves the previous list and
  // snapshot in force; the error names the model.  Single device only (InvalidArgument otherwise).
  Status SetInferenceModels(std::vector<std::shared_ptr<const backend::InferenceModel>> models);

  // Re-read the provider and upload a new snapshot epoch (call on every metrics refresh).  With a
  // model list set, the list is re-interned against the new epoch and uploaded into it before the
  // epoch is published: a target model that no pod listed matches once a pod loads it.
  // A refresh uploads only the dirty pods (lig_update_snapshot) when the previous epoch is its base.
  // A refresh that fails (a refused upload, more than max_pods pods, a refused model table) keeps the
  // previous epoch for scheduling but not as a delta base: the per-pod memo has already moved to the
  // refused tick, so the next refresh uploads in full.
  Status Refresh();

  // Outlier ejection: schedule as if `pods` had left the provider, until a later call lets them back.
  // `pods` is the complete ejected set (an empty list lets every pod back), matched by value (Name +
  // Address) against the snapshot; pods it does not hold are ignored.  Before it returns, a derived
  // epoch (lig_eject_pods, with the model table when a list is set) is published, so every Schedule*
  // call that starts after the return avoids the ejected pods.  Every later refresh keeps them out: a
  // delta tick inherits the set, and after a full upload (or when the pods' positions moved) one more
  // epoch is derived and published.  Single device only (InvalidArgument otherwise).
  Status EjectPods(const std::vector<backend::Pod>& pods);

  // Session affinity: Schedule with the random pick replaced by rendezvous hashing on `key`
  // (lig_schedule_batch_affinity): of req's survivors, the pod with the highest score
  // mix(key ^ mix(PodKey(pod))).  A key keeps its pod while that pod survives, and the answer does not
  // depend on the provider's pod order, on flushes or on the seed.  Goes through the micro-batcher in a
  // lane of its own and takes no rand_key; never through the doorbell; counted in
  // Stats::affinity_scheduled.  Errors are Schedule's.  InvalidArgument without Options::affinity, with
  // load_feedback_window > 0 unless Options::feedback_affinity is set (affinity picks would bypass the
  // chain's per-pod counts; with it they are chain calls, counted in the feedback_* stats) and with
  // several devices.
  Status ScheduleAffinity(const LLMRequest& req, uint64_t key, backend::Pod* targetPod);
  // ScheduleAffinity plus up to n (1..LIG_MAX_FALLBACKS) more survivors in descending score: the
  // session's retry order.  A flush asks the lane's largest n; rows are prefixes of longer rows.
  Status ScheduleAffinityWithFallbacks(const LLMRequest& req, uint64_t key, int n, std::vector<backend::Pod>* pods);
  // ScheduleModel(model, ...) placed by `key` (lig_schedule_models_batch_affinity): the target is drawn on
  // key ^ LIG_DRAW_DOMAIN, so a session keeps its target while the model's targets and weights stay.
  // Host-answered errors as ScheduleModel; takes no rand_key; refused like ScheduleAffinity.
  Status ScheduleModelAffinity(const std::string& model, uint64_t key, std::string* resolvedTargetModel,
                               backend::Pod* targetPod);
  Status ScheduleModelAffinityWithFallbacks(const std::string& model, uint64_t key, int n,
                                            std::string* resolvedTargetModel, std::vector<backend::Pod>* pods);
 private:
  struct ModelList;
  Status RefreshImpl(const std::shared_ptr<const ModelList>& models);
  Status RecordRefresh(Status st);
 public:

  Stats stats() const;
  std::string last_refresh_error() const;

 private:
  friend Status NewScheduler(std::shared_ptr<PodMetricsProvider>, const Options&,
                             std::unique_ptr<Scheduler>*);
  Scheduler() = default;

  using InternTable = std::unordered_map<std::string, int>;
  struct Snapshot {
    uint64_t epoch = 0;
    int A = 0;
    std::shared_ptr<const InternTable> adapter_ids;   // shared between snapshots until a name is added
    std::vector<backend::Pod> pods;
    std::shared_ptr<const ModelList> models;          // the list this epoch's model table was packed from
    std::vector<int32_t> ejected;                     // pods left out of this epoch's pool (ascending)
  };
  // The list SetInferenceModels accepted: dense model id -> InferenceModel, and the name map.
  struct ModelList {
    std::vector<std::shared_ptr<const backend::InferenceModel>> models;
    std::unordered_map<std::string, uint32_t> ids;    // Spec.ModelName -> model id
    std::vector<uint8_t> present;                     // 0: weights sum to <= 0, no target can be drawn
  };
  // EjectPods' set as indices into `pods` (ascending); caller holds refresh_mu_
  std::vector<int32_t> EjectedIndices(const std::vector<backend::Pod>& pods) const;
  // pack (when the list or the adapter ids changed) and upload the model table into snap.epoch
  Status UploadModelTable(const Snapshot& snap, const std::shared_ptr<const ModelList>& models);
  // lig_upload_pod_keys for snap.epoch (Options::affinity only)
  Status UploadPodKeys(const Snapshot& snap);
  // The last model table packed for lig_upload_models, reused while neither the list nor the
  // adapter-id table changed (guarded by refresh_mu_).
  struct PackedModelTable {
    std::shared_ptr<const ModelList> list;
    std::shared_ptr<const InternTable> adapter_ids;
    std::vector<int32_t> target_offsets, target_adapter_ids, target_weights, self_adapter_ids;
    std::vector<uint8_t> critical;
  };
  // Packer state kept between refreshes (guarded by refresh_mu_): adapter ids are stable while
  // the table fits max_adapters, and a pod whose ActiveModels keys did not change since the last
  // tick reuses its encoded ids (sequential string compares instead of hash lookups).
  struct PodMemo {
    std::vector<std::string> names;
    std::vector<int> ids;
  };
  // last uploaded columns, to find the dirty pods of a tick (delta upload)
  std::vector<double> prev_kv_;
  std::vector<int32_t> prev_q_;
  std::vector<uint16_t> prev_na_, prev_ma_;
  int prev_A_ = -1;
  uint64_t prev_epoch_ = 0;
  std::vector<int32_t> prev_ejected_;         // the pods prev_epoch_ left out: a delta from it inherits them
  std::vector<backend::Pod> ejected_;         // EjectPods' set (guarded by refresh_mu_)
  std::atomic<uint64_t> model_draws_{0};
  std::shared_ptr<InternTable> intern_;
  std::vector<PodMemo> memo_;
  std::shared_ptr<const ModelList> models_;   // SetInferenceModels' list (guarded by refresh_mu_); null: none set
  PackedModelTable packed_models_;
  // Lives on the caller's stack.  `done` goes 0 -> 1 (result published, the caller may read it)
  // -> 2 (the notifier will not touch the Waiter again, the caller may return and destroy it).
  // Carries a descriptor request (req) or a model name (model).
  struct Waiter {
    const LLMRequest* req = nullptr;
    const std::string* model = nullptr;
    int fallbacks = 0;           // *WithFallbacks: the n asked for (0: Schedule / ScheduleModel)
    std::vector<backend::Pod>* pods = nullptr;   // *WithFallbacks: receives the pick and its row
    const std::vector<backend::Pod>* tried = nullptr;   // ScheduleRetry: the pods to leave out
    const std::string* target = nullptr;   // ScheduleModelRetry: the resolved target model to keep
    bool affinity = false;       // Schedule[Model]Affinity*: placed by `key`, no rand_key
    uint64_t key = 0;
    int64_t model_id = -1;       // flush-time id in the captured epoch's table; -1: answered on the host
    std::string resolved;        // model requests: the resolved target model
    Status status;
    backend::Pod pod;
    std::atomic<uint32_t> done{0};
  };

  void BatcherLoop();
  void RefresherLoop();
  void Submit(Waiter& w);
  struct CallTime {
    double us = 0, cpu_us = 0;   // wall time of a device call, and the batcher thread's CPU time inside it
  };
  void Flush(std::vector<Waiter*>& batch);
  // one lane of a flush; `timing` (may be null) keeps its slowest device call
  void FlushLane(std::vector<Waiter*>& lane, CallTime* timing);
  int LaneCall(uint64_t epoch, bool models, bool retry, bool affinity, int k, int nf, int width, const char** call);
  Status MapModel(const Snapshot& snap, Waiter* w, int* target);
  // The tried pods of batch[0 .. n) as indices into snap.pods, matched by value; *width is the widest
  // row of at most LIG_MAX_EXCLUDED entries (at least 1)
  static void TriedRows(const Snapshot& snap, Waiter* const* batch, int n, std::vector<std::vector<int16_t>>* rows,
                        int* width);
  void CountFeedback(uint64_t epoch, int n);
  bool AwaitPublication(int rc, uint64_t writes_seen, int attempt);
  void FinishWrite();
  Status CheckRequest(const char* fn, const Waiter& w) const;

  std::shared_ptr<PodMetricsProvider> pmp_;
  Options opt_;
  lig_ctx* ctx_ = nullptr;
  lig_group* group_ = nullptr;     // set instead of ctx_ when Options::devices lists several GPUs
  lig_req* h_reqs_ = nullptr;      // pinned, device-mapped (lig_host_alloc)
  lig_pick* h_picks_ = nullptr;
  int16_t* h_fallbacks_ = nullptr;    // pinned, max_batch x LIG_MAX_FALLBACKS rows
  uint32_t* h_model_ids_ = nullptr;   // pinned, max_batch entries each: the model-id lane
  lig_mpick* h_mpicks_ = nullptr;
  uint64_t model_index_ = 0;          // first_index of the next model-id device call
  // a flush split by kind: descriptors, retries, model ids, model-id retries, affinity descriptors,
  // affinity model ids (batcher thread only)
  std::vector<Waiter*> lanes_[6];
  uint64_t* h_keys_ = nullptr;        // pinned, max_batch affinity keys of the model-id affinity lane (first use)
  std::vector<uint8_t> model_targets_;   // the model-retry lane's target indices (batcher thread only)
  int16_t* h_excluded_ = nullptr;     // pinned, max_batch x LIG_MAX_EXCLUDED rows (first retry flush)
  uint64_t seed_ = 0;
  uint64_t rng_state_ = 0;
  // the feedback chain as the batcher thread sees it (the library's window count is deterministic)
  uint64_t fb_epoch_ = 0;
  int fb_filled_ = 0;

  mutable std::mutex snap_mu_;
  std::shared_ptr<const Snapshot> snap_;
  // Refresh, SetInferenceModels and EjectPods calls finished, published or not (guarded by snap_mu_);
  // a call refused with a stale epoch waits on writes_cv_ for the next one (AwaitPublication)
  uint64_t writes_done_ = 0;
  std::condition_variable writes_cv_;
  uint64_t next_epoch_ = 1;
  std::mutex refresh_mu_;

  std::mutex mu_;
  std::condition_variable cv_;
  std::vector<Waiter*> pending_;
  std::atomic<int> pending_count_{0};
  std::chrono::steady_clock::time_point oldest_;
  bool stop_ = false;
  std::atomic<bool> stop_flag_{false};
  std::thread batcher_, refresher_;

  mutable std::mutex stats_mu_;
  Stats stats_;
  std::string last_refresh_error_;
};

// NewScheduler                                                        scheduler.go:93-99
Status NewScheduler(std::shared_ptr<PodMetricsProvider> pmp, const Options& opt,
                    std::unique_ptr<Scheduler>* out);

}  // namespace scheduling
}  // namespace lig
