// lig_host.cpp — see lig_host.hpp.  Talks to the device only through the C ABI of include/lig.h.
#include "lig_host.hpp"

#include <time.h>
#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>
#include <random>
#include <unordered_set>

#include "../../../include/lig.h"

namespace lig {
namespace scheduling {

namespace {

Status Errorf(int code, const std::string& msg) { return Status{code, msg}; }

Status LigFailure(const char* what) {
  return Errorf(Internal, std::string(what) + ": " + lig_last_error());
}

// status.Errorf(codes.ResourceExhausted, ...) printed through %w            scheduler.go:87,117
const char kDropInner[] =
    "rpc error: code = ResourceExhausted desc = dropping request due to limited backend resources";

// Schedule's error for a pick that is not LIG_OK                            scheduler.go:117
Status PickError(uint16_t status) {
  if (status == LIG_DROP)
    return Errorf(ResourceExhausted, std::string("failed to apply filter, resulted 0 pods, this should never "
                                                 "happen: ") + kDropInner);
  if (status == LIG_NO_PODS_LEFT)   // a caller tree's predicate leaf kept no pod     filter.go:88-90
    return Errorf(Unknown, "failed to apply filter, resulted 0 pods, this should never happen: no pods left");
  return Errorf(Unknown, "failed to apply filter, resulted 0 pods, this should never happen: %!w(<nil>)");
}

// A model request's error for a device pick that is not LIG_OK: Schedule's, prefixed as
// request.go:73-75 wraps it.
constexpr const char* kModelPrefix = "failed to find target pod: ";
Status ModelPickError(uint16_t status, int64_t model_id, const std::string& model) {
  if (status == LIG_NO_MODEL)   // absent models and targets are answered on the host and never sent
    return Errorf(Internal, std::string(kModelPrefix) + "rpc error: code = Internal desc = model id " +
                                std::to_string(model_id) + " (" + model + ") has no model entry on the device");
  Status st = PickError(status);
  st.message = kModelPrefix + st.message;
  return st;
}

inline uint64_t splitmix_next(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// A stale epoch is re-resolved and tried again up to this many attempts in all (AwaitPublication).
constexpr int kStaleAttempts = 4;

double ThreadCpuUs() {
  timespec ts;
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &ts);
  return (double)ts.tv_sec * 1e6 + (double)ts.tv_nsec * 1e-3;
}

template <class F>
struct OnExit {
  F f;
  ~OnExit() { f(); }
};

}  // namespace

Status NewScheduler(std::shared_ptr<PodMetricsProvider> pmp, const Options& opt,
                    std::unique_ptr<Scheduler>* out) {
  if (!pmp || !out) return Errorf(Internal, "NewScheduler: nil provider");
  std::unique_ptr<Scheduler> s(new Scheduler());
  s->pmp_ = std::move(pmp);
  s->opt_ = opt;
  lig_thresholds t{opt.kv_cache_threshold, opt.queue_threshold_critical, opt.queueing_threshold_lora};
  if (opt.load_feedback_window < 0) return Errorf(Internal, "NewScheduler: load_feedback_window must be >= 0");
  if (opt.load_feedback_window > 0 && opt.devices.size() > 1)
    return Errorf(Internal, "NewScheduler: load_feedback_window needs a single device (the feedback chain has no "
                            "cross-device windows)");
  if (opt.load_feedback_window > 0 && opt.use_doorbell)
    return Errorf(Internal, "NewScheduler: load_feedback_window cannot be combined with use_doorbell (the doorbell "
                            "kernel schedules against the resident epoch only)");
  if (opt.devices.size() > 1) {
    if (opt.use_doorbell) return Errorf(Internal, "the doorbell stream is a single-device mode");
    if (lig_group_create(&s->group_, opt.devices.data(), (int)opt.devices.size(), opt.max_pods, opt.max_adapters,
                         opt.max_batch) != 0)
      return LigFailure("lig_group_create");
    if (lig_group_set_thresholds(s->group_, &t) != 0) return LigFailure("lig_group_set_thresholds");
    if (!opt.filter.empty() && lig_group_set_filter_tree(s->group_, opt.filter.data(), (int)opt.filter.size()) != 0)
      return LigFailure("lig_group_set_filter_tree");
  } else {
    const int dev = opt.devices.size() == 1 ? opt.devices[0] : opt.device;
    if (lig_create(&s->ctx_, dev, opt.max_pods, opt.max_adapters, opt.max_batch) != 0)
      return LigFailure("lig_create");
    if (lig_set_thresholds(s->ctx_, &t) != 0) return LigFailure("lig_set_thresholds");
    if (!opt.filter.empty() && lig_set_filter_tree(s->ctx_, opt.filter.data(), (int)opt.filter.size()) != 0)
      return LigFailure("lig_set_filter_tree");
  }
  s->h_reqs_ = static_cast<lig_req*>(lig_host_alloc((size_t)opt.max_batch * sizeof(lig_req)));
  s->h_picks_ = static_cast<lig_pick*>(lig_host_alloc((size_t)opt.max_batch * sizeof(lig_pick)));
  s->h_fallbacks_ = static_cast<int16_t*>(lig_host_alloc((size_t)opt.max_batch * LIG_MAX_FALLBACKS * sizeof(int16_t)));
  s->h_model_ids_ = static_cast<uint32_t*>(lig_host_alloc((size_t)opt.max_batch * sizeof(uint32_t)));
  s->h_mpicks_ = static_cast<lig_mpick*>(lig_host_alloc((size_t)opt.max_batch * sizeof(lig_mpick)));
  if (!s->h_reqs_ || !s->h_picks_ || !s->h_fallbacks_ || !s->h_model_ids_ || !s->h_mpicks_)
    return LigFailure("lig_host_alloc");
  uint64_t seed = opt.seed;
  if (seed == 0) {
    std::random_device rd;
    seed = ((uint64_t)rd() << 32) ^ rd();
  }
  s->seed_ = seed;
  s->rng_state_ = seed ^ 0xD1B54A32D192ED03ull;
  Status st = s->Refresh();
  if (!st.ok()) return st;
  if (opt.use_doorbell && lig_stream_open(s->ctx_) != 0) return LigFailure("lig_stream_open");
  s->batcher_ = std::thread(&Scheduler::BatcherLoop, s.get());
  if (opt.refresh_interval.count() > 0) s->refresher_ = std::thread(&Scheduler::RefresherLoop, s.get());
  *out = std::move(s);
  return Status{};
}

Scheduler::~Scheduler() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    stop_ = true;
    stop_flag_.store(true);
  }
  cv_.notify_all();
  if (batcher_.joinable()) batcher_.join();
  if (refresher_.joinable()) refresher_.join();
  if (ctx_ && opt_.use_doorbell) lig_stream_close(ctx_);
  if (h_reqs_) lig_host_free(h_reqs_);
  if (h_picks_) lig_host_free(h_picks_);
  if (h_fallbacks_) lig_host_free(h_fallbacks_);
  if (h_excluded_) lig_host_free(h_excluded_);
  if (h_keys_) lig_host_free(h_keys_);
  if (h_model_ids_) lig_host_free(h_model_ids_);
  if (h_mpicks_) lig_host_free(h_mpicks_);
  if (ctx_) lig_destroy(ctx_);
  if (group_) lig_group_destroy(group_);
}

// One pack per refresh tick replaces the per-request AllPodMetrics() of scheduler.go:114-115.
// A failed refresh keeps the previous snapshot — like a failed scrape keeps stale metrics
// (backend/provider.go:151-156) — but never silently: it is counted and its reason kept.
// Its end is counted (FinishWrite): calls refused with a stale epoch meanwhile wait for it.
Status Scheduler::Refresh() {
  std::lock_guard<std::mutex> rk(refresh_mu_);
  const OnExit finish{[this] { FinishWrite(); }};
  return RecordRefresh(RefreshImpl(models_));
}

Status Scheduler::RecordRefresh(Status st) {
  if (!st.ok()) {
    std::lock_guard<std::mutex> sk(stats_mu_);
    stats_.failed_refreshes++;
    last_refresh_error_ = st.message;
    fprintf(stderr, "lig: snapshot refresh failed, keeping the previous one: %s\n", st.message.c_str());
  }
  return st;
}

std::string Scheduler::last_refresh_error() const {
  std::lock_guard<std::mutex> sk(stats_mu_);
  return last_refresh_error_;
}

// Called with refresh_mu_ held.  `models` (null: no list set) is packed against the new epoch.
Status Scheduler::RefreshImpl(const std::shared_ptr<const ModelList>& models) {
  const auto t_begin = std::chrono::steady_clock::now();
  auto pods = pmp_->AllPodMetrics();
  // A pod whose metrics do not fit the device record (WaitingQueueSize outside int32,
  // len(ActiveModels) above the record's limit) is left out of this snapshot and counted; one bad
  // scrape must not freeze the whole pool on a stale snapshot.
  uint64_t excluded = 0;
  {
    size_t keep = 0;
    for (size_t i = 0; i < pods.size(); ++i) {
      const auto& m = pods[i]->metrics;
      const bool fits = m.WaitingQueueSize >= INT32_MIN && m.WaitingQueueSize <= INT32_MAX &&
                        m.ActiveModels.size() <= (size_t)LIG_MAX_ADAPTERS;
      if (fits) pods[keep++] = pods[i];
      else ++excluded;
    }
    pods.resize(keep);
  }
  const int P = (int)pods.size();
  const int W = (P + 31) / 32;
  auto snap = std::make_shared<Snapshot>();
  snap->pods.reserve(P);
  std::vector<double> kv(P);
  std::vector<int64_t> q(P), na(P), ma(P);
  if (!intern_) intern_ = std::make_shared<InternTable>();
  // From here on the memo (and the intern table) describe this tick.  A return before the epoch is
  // published leaves the device on an older epoch the memo no longer matches, so that epoch must not
  // be a delta base: a pod whose names changed would look clean and keep its old bitmap row.
  struct DeltaBaseReset {
    uint64_t* base;
    ~DeltaBaseReset() { if (base) *base = 0; }   // the next refresh uploads in full
  } reset_base{&prev_epoch_};
  bool table_changed = false;
  std::vector<char> memo_dirty;
  for (int attempt = 0; attempt < 2; ++attempt) {
    memo_.resize((size_t)P);
    memo_dirty.assign((size_t)P, 0);
    snap->pods.clear();
    for (int p = 0; p < P; ++p) {
      const backend::PodMetrics& pm = *pods[p];
      snap->pods.push_back(pm.pod);
      kv[p] = pm.metrics.KVCacheUsagePercent;
      q[p] = pm.metrics.WaitingQueueSize;
      na[p] = (int64_t)pm.metrics.ActiveModels.size();
      ma[p] = pm.metrics.MaxActiveModels;
      PodMemo& m = memo_[(size_t)p];
      bool same = m.names.size() == pm.metrics.ActiveModels.size();
      if (same) {
        size_t k = 0;
        for (const auto& kvp : pm.metrics.ActiveModels)     // std::map: ordered keys
          if (m.names[k++] != kvp.first) { same = false; break; }
      }
      if (same) continue;
      memo_dirty[(size_t)p] = 1;
      m.names.clear();
      m.ids.clear();
      for (const auto& kvp : pm.metrics.ActiveModels) {
        auto it = intern_->find(kvp.first);
        if (it == intern_->end()) {
          if (!table_changed) {                              // copy on write: older snapshots keep theirs
            intern_ = std::make_shared<InternTable>(*intern_);
            table_changed = true;
          }
          it = intern_->emplace(kvp.first, (int)intern_->size()).first;
        }
        m.names.push_back(kvp.first);
        m.ids.push_back(it->second);
      }
    }
    if ((int)intern_->size() <= opt_.max_adapters || attempt == 1) break;
    // the grow-only table outgrew the device capacity (adapters churned): re-intern from scratch
    intern_ = std::make_shared<InternTable>();
    table_changed = true;
    memo_.clear();
  }
  const int A = (int)intern_->size();
  snap->A = A;
  snap->adapter_ids = intern_;
  std::vector<uint32_t> bitmap((size_t)A * W, 0u);
  for (int p = 0; p < P; ++p)
    for (int id : memo_[(size_t)p].ids) bitmap[(size_t)id * W + (p >> 5)] |= 1u << (p & 31);
  std::vector<int32_t> q32(P);
  std::vector<uint16_t> na16(P), ma16(P);
  if (lig_pack_pods(P, q.data(), na.data(), ma.data(), q32.data(), na16.data(), ma16.data()) != 0)
    return LigFailure("lig_pack_pods");
  snap->epoch = next_epoch_++;
  const auto t_packed = std::chrono::steady_clock::now();
  // Which pods changed since the last uploaded tick?  With the adapter table and the pool size
  // unchanged and few dirty pods, only the delta crosses PCIe (lig_update_snapshot); the base is
  // the previous epoch, still resident in the other slot.
  std::vector<int32_t> dirty;
  const bool comparable = !group_ && prev_epoch_ != 0 && !table_changed && prev_A_ == A && (int)prev_q_.size() == P;
  if (comparable) {
    for (int p = 0; p < P; ++p)
      if (memo_dirty[(size_t)p] || prev_q_[(size_t)p] != q32[(size_t)p] || prev_na_[(size_t)p] != na16[(size_t)p] ||
          prev_ma_[(size_t)p] != ma16[(size_t)p] || memcmp(&prev_kv_[(size_t)p], &kv[(size_t)p], sizeof(double)) != 0)
        dirty.push_back(p);
  }
  bool used_delta = false;
  if (comparable && (int)dirty.size() * 4 <= P) {
    std::vector<double> dkv(dirty.size());
    std::vector<int32_t> dq(dirty.size()), doff(dirty.size() + 1, 0), dids;
    std::vector<uint16_t> dna(dirty.size()), dma(dirty.size());
    for (size_t i = 0; i < dirty.size(); ++i) {
      const size_t p = (size_t)dirty[i];
      dkv[i] = kv[p]; dq[i] = q32[p]; dna[i] = na16[p]; dma[i] = ma16[p];
      dids.insert(dids.end(), memo_[p].ids.begin(), memo_[p].ids.end());
      doff[i + 1] = (int32_t)dids.size();
    }
    const int rc = lig_update_snapshot(ctx_, snap->epoch, prev_epoch_, (int)dirty.size(), dirty.data(), dkv.data(),
                                       dq.data(), dna.data(), dma.data(), doff.data(), dids.data());
    if (rc == 0) used_delta = true;
    else if (rc != LIG_ERR_INVALID && rc != LIG_ERR_STALE_EPOCH) return LigFailure("lig_update_snapshot");
  }
  if (!used_delta) {
    const int rc = group_ ? lig_group_upload_snapshot(group_, snap->epoch, P, A, kv.data(), q32.data(), na16.data(),
                                                      ma16.data(), bitmap.data())
                          : lig_upload_snapshot(ctx_, snap->epoch, P, A, kv.data(), q32.data(), na16.data(),
                                                ma16.data(), bitmap.data());
    if (rc != 0) return LigFailure(group_ ? "lig_group_upload_snapshot" : "lig_upload_snapshot");
  }
  // The ejected set: a delta epoch inherits its base's; when that is not the set EjectPods asks for on
  // this tick's pods (a full upload has none, or the pods moved), one more epoch is derived from it.
  // That derive evicts the published epoch until snap_ moves on; calls refused meanwhile wait for the
  // end of this write (AwaitPublication) before they re-resolve.
  snap->ejected = used_delta ? prev_ejected_ : std::vector<int32_t>{};
  bool derived = false;
  {
    std::vector<int32_t> want = EjectedIndices(snap->pods);
    if (want != snap->ejected) {
      const uint64_t e = next_epoch_++;
      if (lig_eject_pods(ctx_, e, snap->epoch, want.data(), (int)want.size()) != 0) return LigFailure("lig_eject_pods");
      snap->epoch = e;
      snap->ejected = std::move(want);
      derived = true;
    }
  }
  // So do the pod keys (a delta or derived epoch starts without them) and the model table: a flush
  // that captures the epoch always finds the keys and the table its requests were mapped against.
  if (opt_.affinity && !group_)
    if (Status st = UploadPodKeys(*snap); !st.ok()) return st;
  if (models)
    if (Status st = UploadModelTable(*snap, models); !st.ok()) return st;
  snap->models = models;
  prev_kv_ = kv;
  prev_q_ = q32;
  prev_na_ = na16;
  prev_ma_ = ma16;
  prev_A_ = A;
  reset_base.base = nullptr;
  prev_epoch_ = snap->epoch;
  prev_ejected_ = snap->ejected;
  const uint64_t n_ejected = snap->ejected.size();
  {
    std::lock_guard<std::mutex> lk(snap_mu_);
    snap_ = std::move(snap);
  }
  const auto t_done = std::chrono::steady_clock::now();
  std::lock_guard<std::mutex> sk(stats_mu_);
  stats_.refreshes++;
  stats_.delta_refreshes += used_delta ? 1 : 0;
  stats_.last_dirty_pods = comparable ? dirty.size() : (uint64_t)P;
  stats_.excluded_pods = excluded;
  stats_.ejected_pods = n_ejected;
  stats_.eject_publishes += derived ? 1 : 0;
  stats_.last_pack_us = std::chrono::duration<double, std::micro>(t_packed - t_begin).count();
  stats_.last_upload_us = std::chrono::duration<double, std::micro>(t_done - t_packed).count();
  return Status{};
}

Status Scheduler::UploadModelTable(const Snapshot& snap, const std::shared_ptr<const ModelList>& models) {
  const int A = snap.A;
  PackedModelTable& t = packed_models_;
  if (t.list != models || t.adapter_ids != snap.adapter_ids) {
    const size_t n = models->models.size();
    t.target_offsets.assign(n + 1, 0);
    t.target_adapter_ids.clear();
    t.target_weights.clear();
    t.self_adapter_ids.resize(n);
    t.critical.resize(n);
    // a name no pod lists, or one interned after this epoch's table (>= A), is id A: no pod matches
    auto intern = [&](const std::string& name) {
      auto it = snap.adapter_ids->find(name);
      return (it == snap.adapter_ids->end() || it->second >= A) ? A : it->second;
    };
    for (size_t m = 0; m < n; ++m) {
      const backend::InferenceModel& im = *models->models[m];
      t.critical[m] = im.Critical ? 1 : 0;
      t.self_adapter_ids[m] = intern(im.ModelName);
      if (models->present[m])
        for (const backend::TargetModel& tm : im.TargetModels) {
          t.target_adapter_ids.push_back(intern(tm.Name));
          t.target_weights.push_back(tm.Weight);
        }
      t.target_offsets[m + 1] = (int32_t)t.target_adapter_ids.size();
    }
    t.list = models;
    t.adapter_ids = snap.adapter_ids;
  }
  if (lig_upload_models(ctx_, snap.epoch, (int)models->models.size(), t.target_offsets.data(),
                        t.target_adapter_ids.data(), t.target_weights.data(), t.critical.data(),
                        t.self_adapter_ids.data(), models->present.data()) != 0)
    return LigFailure("lig_upload_models");
  return Status{};
}

uint64_t PodKey(const backend::Pod& pod) {
  uint64_t h = 0xCBF29CE484222325ull;
  auto feed = [&h](const std::string& s) {
    for (unsigned char c : s) h = (h ^ c) * 0x100000001B3ull;
  };
  feed(pod.Name);
  h = (h ^ 0u) * 0x100000001B3ull;
  feed(pod.Address);
  return h;
}

Status Scheduler::UploadPodKeys(const Snapshot& snap) {
  std::vector<uint64_t> keys(snap.pods.size());
  for (size_t p = 0; p < keys.size(); ++p) keys[p] = PodKey(snap.pods[p]);
  if (lig_upload_pod_keys(ctx_, snap.epoch, (int)keys.size(), keys.data()) != 0) return LigFailure("lig_upload_pod_keys");
  return Status{};
}

std::vector<int32_t> Scheduler::EjectedIndices(const std::vector<backend::Pod>& pods) const {
  std::vector<int32_t> idx;
  if (ejected_.empty()) return idx;
  std::unordered_set<std::string> gone;                 // Name + '\0' + Address, as the retry lane matches
  for (const backend::Pod& p : ejected_) gone.insert(p.Name + '\0' + p.Address);
  for (size_t p = 0; p < pods.size(); ++p)
    if (gone.count(pods[p].Name + '\0' + pods[p].Address)) idx.push_back((int32_t)p);
  return idx;
}

Status Scheduler::EjectPods(const std::vector<backend::Pod>& pods) {
  if (group_)
    return Errorf(InvalidArgument, "EjectPods: a scheduler over several devices has no ejection call (lig_group)");
  std::lock_guard<std::mutex> rk(refresh_mu_);
  const OnExit finish{[this] { FinishWrite(); }};
  ejected_ = pods;
  std::shared_ptr<const Snapshot> cur;
  {
    std::lock_guard<std::mutex> lk(snap_mu_);
    cur = snap_;
  }
  if (!cur) return Status{};                            // the first refresh applies the set
  std::vector<int32_t> want = EjectedIndices(cur->pods);
  if (want != cur->ejected) {
    // derived from the published epoch, the newest resident one: the slot it overwrites is the other
    auto snap = std::make_shared<Snapshot>(*cur);
    snap->epoch = next_epoch_++;
    if (lig_eject_pods(ctx_, snap->epoch, cur->epoch, want.data(), (int)want.size()) != 0)
      return LigFailure("lig_eject_pods");
    if (opt_.affinity)
      if (Status st = UploadPodKeys(*snap); !st.ok()) return st;
    if (snap->models)
      if (Status st = UploadModelTable(*snap, snap->models); !st.ok()) return st;
    snap->ejected = std::move(want);
    if (prev_epoch_ == cur->epoch) {                    // same columns: the next delta starts from it
      prev_epoch_ = snap->epoch;
      prev_ejected_ = snap->ejected;
    }
    const uint64_t n = snap->ejected.size();
    {
      std::lock_guard<std::mutex> lk(snap_mu_);
      snap_ = std::move(snap);
    }
    std::lock_guard<std::mutex> sk(stats_mu_);
    stats_.ejected_pods = n;
    stats_.eject_publishes++;
  }
  return Status{};
}

Status Scheduler::SetInferenceModels(std::vector<std::shared_ptr<const backend::InferenceModel>> models) {
  if (group_)
    return Errorf(InvalidArgument, "SetInferenceModels: model requests need a single device (lig_group has no "
                                   "model-table calls)");
  auto list = std::make_shared<ModelList>();
  for (auto& m : models) {
    if (!m) return Errorf(InvalidArgument, "SetInferenceModels: nil InferenceModel");
    auto ins = list->ids.emplace(m->ModelName, (uint32_t)list->models.size());
    if (ins.second) list->models.push_back(std::move(m));
    else list->models[ins.first->second] = std::move(m);          // the later one wins
  }
  list->present.assign(list->models.size(), 1);
  for (size_t i = 0; i < list->models.size(); ++i) {
    const backend::InferenceModel& im = *list->models[i];
    int64_t total = 0;
    bool negative = false;
    for (const backend::TargetModel& tm : im.TargetModels) {
      total += tm.Weight;
      negative |= tm.Weight < 0;
    }
    if (im.TargetModels.empty()) continue;
    // no target can be drawn (Go's Int31n panics on 0): "error getting target model name"
    if (total <= 0) {
      list->present[i] = 0;
      continue;
    }
    // what lig_upload_models refuses with LIG_ERR_RANGE
    if (im.TargetModels.size() > 255)
      return Errorf(InvalidArgument, "SetInferenceModels: model " + im.ModelName + " has " +
                                         std::to_string(im.TargetModels.size()) + " target models (at most 255)");
    if (negative) return Errorf(InvalidArgument, "SetInferenceModels: model " + im.ModelName + " has a negative weight");
    if (total > INT32_MAX)
      return Errorf(InvalidArgument, "SetInferenceModels: the weights of model " + im.ModelName + " sum to " +
                                         std::to_string(total) + " (at most 2^31-1)");
  }
  std::shared_ptr<const ModelList> next = std::move(list);
  std::lock_guard<std::mutex> rk(refresh_mu_);
  const OnExit finish{[this] { FinishWrite(); }};
  Status st = RecordRefresh(RefreshImpl(next));
  if (st.ok()) models_ = std::move(next);
  return st;
}

void Scheduler::RefresherLoop() {
  std::unique_lock<std::mutex> lk(mu_);
  while (!stop_) {
    cv_.wait_for(lk, opt_.refresh_interval, [&] { return stop_; });
    if (stop_) break;
    lk.unlock();
    Refresh();   // failures are counted and logged there
    lk.lock();
  }
}

Status Scheduler::Schedule(const LLMRequest& req, backend::Pod* targetPod) {
  Waiter w;
  w.req = &req;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

// The refusals of the Schedule* calls that ask for more than Schedule: fallback rows (w.pods), a retry
// (w.tried) or both, checked in this order before the waiter is queued.
Status Scheduler::CheckRequest(const char* fn, const Waiter& w) const {
  const bool rows = w.pods != nullptr, retry = w.tried != nullptr;
  if (rows && (w.fallbacks < 1 || w.fallbacks > LIG_MAX_FALLBACKS))
    return Errorf(InvalidArgument, std::string(fn) + ": n=" + std::to_string(w.fallbacks) + " outside [1, " +
                                       std::to_string(LIG_MAX_FALLBACKS) + "]");
  if (w.affinity) {
    if (!opt_.affinity)
      return Errorf(InvalidArgument, std::string(fn) + ": the scheduler was built without Options::affinity (it "
                                                       "uploads the pods' keys)");
    if (opt_.load_feedback_window > 0 && !opt_.feedback_affinity)
      return Errorf(InvalidArgument, std::string(fn) + ": not defined under load_feedback_window (affinity picks "
                                                       "would bypass the feedback chain's per-pod counts)");
    if (group_)
      return Errorf(InvalidArgument, std::string(fn) + ": a scheduler over several devices has no affinity call");
    return Status{};
  }
  if (retry && w.tried->size() > (size_t)LIG_MAX_EXCLUDED)
    return Errorf(InvalidArgument, std::string(fn) + ": " + std::to_string(w.tried->size()) + " tried pods (at most " +
                                       std::to_string(LIG_MAX_EXCLUDED) + ")");
  if (opt_.load_feedback_window > 0 && ((retry && !opt_.feedback_retries) || (rows && !opt_.feedback_fallbacks))) {
    const char* needs = retry && rows ? "feedback_retries and feedback_fallbacks"
                        : retry       ? "feedback_retries"
                                      : "feedback_fallbacks";
    const char* these = retry && rows ? "these" : retry ? "a retry" : "the fallbacks";
    return Errorf(InvalidArgument, std::string(fn) + ": not defined under load_feedback_window without " + needs +
                                       " (the picks come from the feedback chain's copy of the snapshot, " + these +
                                       " would not)");
  }
  if (group_)
    return Errorf(InvalidArgument, std::string(fn) + ": a scheduler over several devices has no " +
                                       (retry ? "retry" : "fallback") + " call");
  return Status{};
}

Status Scheduler::ScheduleWithFallbacks(const LLMRequest& req, int n, std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.req = &req;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  return w.status;
}

Status Scheduler::ScheduleRetry(const LLMRequest& req, const std::vector<backend::Pod>& tried,
                                backend::Pod* targetPod) {
  Waiter w;
  w.req = &req;
  w.tried = &tried;
  if (Status st = CheckRequest("ScheduleRetry", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

Status Scheduler::ScheduleRetryWithFallbacks(const LLMRequest& req, const std::vector<backend::Pod>& tried, int n,
                                             std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.req = &req;
  w.tried = &tried;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleRetryWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  return w.status;
}

Status Scheduler::ScheduleModel(const std::string& model, std::string* resolvedTargetModel, backend::Pod* targetPod) {
  Waiter w;
  w.model = &model;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  if (resolvedTargetModel) *resolvedTargetModel = std::move(w.resolved);
  return w.status;
}

Status Scheduler::ScheduleModelWithFallbacks(const std::string& model, int n, std::string* resolvedTargetModel,
                                             std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.model = &model;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleModelWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  if (resolvedTargetModel) *resolvedTargetModel = std::move(w.resolved);
  return w.status;
}

Status Scheduler::ScheduleModelRetry(const std::string& model, const std::string& resolvedTargetModel,
                                     const std::vector<backend::Pod>& tried, backend::Pod* targetPod) {
  Waiter w;
  w.model = &model;
  w.target = &resolvedTargetModel;
  w.tried = &tried;
  if (Status st = CheckRequest("ScheduleModelRetry", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

Status Scheduler::ScheduleModelRetryWithFallbacks(const std::string& model, const std::string& resolvedTargetModel,
                                                  const std::vector<backend::Pod>& tried, int n,
                                                  std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.model = &model;
  w.target = &resolvedTargetModel;
  w.tried = &tried;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleModelRetryWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  return w.status;
}

Status Scheduler::ScheduleAffinity(const LLMRequest& req, uint64_t key, backend::Pod* targetPod) {
  Waiter w;
  w.req = &req;
  w.affinity = true;
  w.key = key;
  if (Status st = CheckRequest("ScheduleAffinity", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

Status Scheduler::ScheduleAffinityWithFallbacks(const LLMRequest& req, uint64_t key, int n,
                                                std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.req = &req;
  w.affinity = true;
  w.key = key;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleAffinityWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  return w.status;
}

Status Scheduler::ScheduleModelAffinity(const std::string& model, uint64_t key, std::string* resolvedTargetModel,
                                        backend::Pod* targetPod) {
  Waiter w;
  w.model = &model;
  w.affinity = true;
  w.key = key;
  if (Status st = CheckRequest("ScheduleModelAffinity", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  if (resolvedTargetModel) *resolvedTargetModel = std::move(w.resolved);
  return w.status;
}

Status Scheduler::ScheduleModelAffinityWithFallbacks(const std::string& model, uint64_t key, int n,
                                                     std::string* resolvedTargetModel,
                                                     std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.model = &model;
  w.affinity = true;
  w.key = key;
  w.fallbacks = n;
  w.pods = &ranked;
  if (Status st = CheckRequest("ScheduleModelAffinityWithFallbacks", w); !st.ok()) return st;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  if (resolvedTargetModel) *resolvedTargetModel = std::move(w.resolved);
  return w.status;
}

Status Scheduler::Filter(const LLMRequest& req, std::vector<backend::Pod>* pods) {
  if (group_)
    return Errorf(InvalidArgument, "Filter: a scheduler over several devices has no survivor-list call");
  if (pods) pods->clear();
  lig_req r{};
  lig_pick pick{};
  int64_t offsets[2] = {0, 0};
  std::vector<uint16_t> list;
  std::shared_ptr<const Snapshot> snap;
  int rc = 0;
  uint64_t writes_seen = 0;
  for (int attempt = 0; attempt < kStaleAttempts; ++attempt) {
    {
      std::lock_guard<std::mutex> lk(snap_mu_);
      snap = snap_;
        writes_seen = writes_done_;
    }
    if (!snap) return Errorf(Internal, "Filter: no snapshot uploaded yet");
    auto it = snap->adapter_ids->find(req.ResolvedTargetModel);   // interned as in Flush
    r.adapter_id = (it == snap->adapter_ids->end() || it->second >= snap->A) ? snap->A : it->second;
    r.flags = req.Critical ? LIG_REQ_CRITICAL : 0u;
    list.resize(std::max<size_t>(snap->pods.size(), 1));   // a survivor list never exceeds P
    rc = lig_filter_batch(ctx_, snap->epoch, seed_, &r, 1, &pick, offsets, list.data(), (int64_t)list.size());
    if (!AwaitPublication(rc, writes_seen, attempt)) break;
  }
  if (rc != 0) return LigFailure("lig_filter_batch");
  if (pick.status == LIG_DROP)                                               // scheduler.go:83-89
    return Errorf(ResourceExhausted, "dropping request due to limited backend resources");
  if (pick.status == LIG_NO_PODS_LEFT)                                       // filter.go:88-90
    return Errorf(Unknown, "no pods left");
  if (pods)
    for (int64_t k = offsets[0]; k < offsets[1]; ++k) pods->push_back(snap->pods[list[(size_t)k]]);
  return Status{};
}

// Whether a call refused with `rc` is tried again.  LIG_ERR_STALE_EPOCH means its epoch was evicted
// after it was captured, by a write that may still be in progress: a refresh that derives an ejected
// set evicts the published epoch before the derived one is published.  Every eviction happens inside
// Refresh, SetInferenceModels or EjectPods, and each of them counts writes_done_ when it ends, so the
// call waits until writes_done_ moves past the count it captured with its epoch: for the write in
// flight only, not for a later one still scraping the provider (a provider that calls back into the
// scheduler cannot deadlock here).  The last attempt does not wait.  The wait is bounded so that a
// refusal no write of this scheduler caused cannot hold a flush for good.
bool Scheduler::AwaitPublication(int rc, uint64_t writes_seen, int attempt) {
  if (rc != LIG_ERR_STALE_EPOCH) return false;
  {
    std::lock_guard<std::mutex> sk(stats_mu_);
    stats_.stale_retries++;
  }
  if (attempt + 1 >= kStaleAttempts) return false;
  std::unique_lock<std::mutex> lk(snap_mu_);
  writes_cv_.wait_for(lk, std::chrono::seconds(1), [&] { return writes_done_ != writes_seen; });
  return true;
}

void Scheduler::FinishWrite() {
  {
    std::lock_guard<std::mutex> lk(snap_mu_);
    writes_done_++;
  }
  writes_cv_.notify_all();
}

// Queue the waiter for the batcher and block until its result is published.
void Scheduler::Submit(Waiter& w) {
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (stop_) {
      w.status = Errorf(Internal, "scheduler is shut down");
      return;
    }
    if (pending_.empty()) oldest_ = std::chrono::steady_clock::now();
    pending_.push_back(&w);
    pending_count_.store((int)pending_.size(), std::memory_order_release);
  }
  if (!opt_.busy_poll) cv_.notify_all();
  if (opt_.caller_spin.count() > 0) {
    const auto until = std::chrono::steady_clock::now() + opt_.caller_spin;
    while (w.done.load(std::memory_order_acquire) == 0 && std::chrono::steady_clock::now() < until) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
  }
  w.done.wait(0, std::memory_order_acquire);
  // the notifier may still be inside notify_one() on this stack object: leave only once it says
  // it is finished (done == 2); a handful of spins at most
  while (w.done.load(std::memory_order_acquire) != 2) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
}

void Scheduler::BatcherLoop() {
  std::vector<Waiter*> batch;
  std::unique_lock<std::mutex> lk(mu_);
  for (;;) {
    if (opt_.busy_poll) {
      lk.unlock();
      while (pending_count_.load(std::memory_order_acquire) == 0) {
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
        if (stop_flag_.load(std::memory_order_relaxed)) break;
      }
      lk.lock();
      if (pending_.empty()) {
        if (stop_) break;
        continue;
      }
      const auto deadline = oldest_ + opt_.batch_window;
      while ((int)pending_.size() < opt_.flush_size && std::chrono::steady_clock::now() < deadline && !stop_) {
        lk.unlock();
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
        lk.lock();
      }
    } else {
      cv_.wait(lk, [&] { return stop_ || !pending_.empty(); });
      if (pending_.empty() && stop_) break;
      const auto deadline = oldest_ + opt_.batch_window;
      cv_.wait_until(lk, deadline, [&] { return stop_ || (int)pending_.size() >= opt_.flush_size; });
    }
    batch.clear();
    batch.swap(pending_);
    pending_count_.store(0, std::memory_order_release);
    lk.unlock();
    Flush(batch);
    lk.lock();
  }
}

void Scheduler::CountFeedback(uint64_t epoch, int n) {
  // the chain restarts on every new epoch: "until the next metrics refresh" (Refresh never reuses an
  // epoch number)
  const int W = opt_.load_feedback_window;
  std::lock_guard<std::mutex> sk(stats_mu_);
  if (epoch != fb_epoch_) {
    if (fb_epoch_ != 0) stats_.feedback_restarts++;
    fb_epoch_ = epoch;
    fb_filled_ = 0;
  }
  stats_.feedback_windows += (uint64_t)((fb_filled_ + (int64_t)n) / W);
  fb_filled_ = (int)((fb_filled_ + (int64_t)n) % W);
}

// A flush makes its calls lane by lane: descriptors, retries, model ids, model-id retries, affinity
// descriptors, affinity model ids.  Under load_feedback_window this is the order of the flush's
// requests in the feedback chain.
void Scheduler::Flush(std::vector<Waiter*>& all) {
  for (std::vector<Waiter*>& lane : lanes_) lane.clear();
  for (Waiter* w : all)
    lanes_[w->affinity ? (w->model ? 5 : 4) : (w->model ? 2 : 0) + (w->tried ? 1 : 0)].push_back(w);
  const auto flush_t0 = std::chrono::steady_clock::now();
  CallTime slowest;   // the descriptor lane's slowest device call
  for (int l = 0; l < 6; ++l) FlushLane(lanes_[l], l == 0 ? &slowest : nullptr);
  const double flush_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - flush_t0).count();
  std::lock_guard<std::mutex> sk(stats_mu_);
  if (slowest.us > stats_.max_device_call_us) {
    stats_.max_device_call_us = slowest.us;
    stats_.slowest_call_cpu_us = slowest.cpu_us;
    stats_.slowest_call_batch = stats_.batches ? stats_.batches - 1 : 0;
  }
  stats_.max_flush_us = std::max(stats_.max_flush_us, flush_us);
}

void Scheduler::TriedRows(const Snapshot& snap, Waiter* const* batch, int n, std::vector<std::vector<int16_t>>* rows,
                          int* width) {
  std::unordered_map<std::string, std::vector<int16_t>> where;   // Name + '\0' + Address -> pod indices
  for (size_t p = 0; p < snap.pods.size(); ++p) where[snap.pods[p].Name + '\0' + snap.pods[p].Address].push_back((int16_t)p);
  rows->assign((size_t)n, {});
  *width = 1;
  for (int i = 0; i < n; ++i) {
    std::vector<int16_t>& row = (*rows)[(size_t)i];
    for (const backend::Pod& t : *batch[i]->tried) {
      auto it = where.find(t.Name + '\0' + t.Address);
      if (it != where.end()) row.insert(row.end(), it->second.begin(), it->second.end());
    }
    // only pods listed more than once in the slice get past 32: that caller is refused
    if ((int)row.size() <= LIG_MAX_EXCLUDED) *width = std::max(*width, (int)row.size());
  }
}

// A model waiter's id in the captured epoch's list and, for a retry, the index of its resolved target
// among the model's TargetModels (the first of that name; 255 for a model without TargetModels whose
// own name it is).  A waiter the list alone answers gets the error it is answered with.
Status Scheduler::MapModel(const Snapshot& snap, Waiter* w, int* target) {
  w->model_id = -1;
  const ModelList* list = snap.models.get();
  auto it = list ? list->ids.find(*w->model) : decltype(list->ids)::const_iterator{};
  if (!list || it == list->ids.end())                                                   // request.go:42-45
    return Errorf(Unknown, "error finding a model object in InferenceModel for input " + *w->model);
  const backend::InferenceModel& im = *list->models[it->second];
  if (!list->present[it->second])                                                       // request.go:48-51
    return Errorf(Unknown, "error getting target model name for model " + im.ModelName);
  if (w->target) {
    *target = -1;
    if (im.TargetModels.empty()) {
      if (*w->target == *w->model) *target = 255;                                       // request.go:47
    } else {
      for (size_t j = 0; j < im.TargetModels.size() && *target < 0; ++j)
        if (im.TargetModels[j].Name == *w->target) *target = (int)j;
    }
    if (*target < 0)
      return Errorf(InvalidArgument, "ScheduleModelRetry: " + *w->target + " is not a target model of " + *w->model);
  }
  w->model_id = it->second;
  return Status{};
}

// The library call for k mapped requests of one lane.  *call receives the name LigFailure reports: the
// entry point's own, except that the group and the doorbell report as lig_schedule_batch.
#define LIG_LANE_CALL(fn, ...) (*call = #fn, fn(__VA_ARGS__))
int Scheduler::LaneCall(uint64_t epoch, bool models, bool retry, bool affinity, int k, int nf, int width,
                        const char** call) {
  const int W = opt_.load_feedback_window;
  const uint64_t first = model_index_;
  const uint8_t* targets = model_targets_.data();
  if (affinity && models && W > 0)
    return LIG_LANE_CALL(lig_schedule_models_batch_feedback_chain_affinity, ctx_, epoch, h_model_ids_, h_keys_, k,
                         h_mpicks_, nf, h_fallbacks_, W, nullptr);
  if (affinity && models)
    return LIG_LANE_CALL(lig_schedule_models_batch_affinity, ctx_, epoch, h_model_ids_, h_keys_, k, h_mpicks_, nf,
                         h_fallbacks_);
  if (affinity && W > 0)
    return LIG_LANE_CALL(lig_schedule_batch_feedback_chain_affinity, ctx_, epoch, h_reqs_, k, h_picks_, nf,
                         h_fallbacks_, W, nullptr);
  if (affinity)
    return LIG_LANE_CALL(lig_schedule_batch_affinity, ctx_, epoch, h_reqs_, k, h_picks_, nf, h_fallbacks_);
  if (models && retry) {
    if (nf > 0 && W > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_feedback_chain_excluding_fallbacks, ctx_, epoch, seed_, first,
                           h_model_ids_, targets, k, h_excluded_, width, h_mpicks_, nf, h_fallbacks_, W, nullptr);
    if (nf > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_excluding_fallbacks, ctx_, epoch, seed_, first, h_model_ids_,
                           targets, k, h_excluded_, width, h_mpicks_, nf, h_fallbacks_);
    if (W > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_feedback_chain_excluding, ctx_, epoch, seed_, first, h_model_ids_,
                           targets, k, h_excluded_, width, h_mpicks_, W, nullptr);
    return LIG_LANE_CALL(lig_schedule_models_batch_excluding, ctx_, epoch, seed_, first, h_model_ids_, targets, k,
                         h_excluded_, width, h_mpicks_);
  }
  if (models) {
    if (nf > 0 && W > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_feedback_chain_fallbacks, ctx_, epoch, seed_, first, h_model_ids_,
                           k, h_mpicks_, nf, h_fallbacks_, W, nullptr);
    if (nf > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_fallbacks, ctx_, epoch, seed_, first, h_model_ids_, k, h_mpicks_,
                           nf, h_fallbacks_);
    if (W > 0)
      return LIG_LANE_CALL(lig_schedule_models_batch_feedback_chain, ctx_, epoch, seed_, first, h_model_ids_, k,
                           h_mpicks_, W, nullptr);
    if (opt_.use_doorbell && k <= lig_stream_capacity())
      return LIG_LANE_CALL(lig_stream_submit_models, ctx_, epoch, seed_, first, h_model_ids_, k, h_mpicks_);
    return LIG_LANE_CALL(lig_schedule_models_batch, ctx_, epoch, seed_, first, h_model_ids_, k, h_mpicks_);
  }
  if (retry) {
    if (nf > 0 && W > 0)
      return LIG_LANE_CALL(lig_schedule_batch_feedback_chain_excluding_fallbacks, ctx_, epoch, seed_, h_reqs_, k,
                           h_excluded_, width, h_picks_, nf, h_fallbacks_, W, nullptr);
    if (nf > 0)
      return LIG_LANE_CALL(lig_schedule_batch_excluding_fallbacks, ctx_, epoch, seed_, h_reqs_, k, h_excluded_, width,
                           h_picks_, nf, h_fallbacks_);
    if (W > 0)
      return LIG_LANE_CALL(lig_schedule_batch_feedback_chain_excluding, ctx_, epoch, seed_, h_reqs_, k, h_excluded_,
                           width, h_picks_, W, nullptr);
    return LIG_LANE_CALL(lig_schedule_batch_excluding, ctx_, epoch, seed_, h_reqs_, k, h_excluded_, width, h_picks_);
  }
  if (nf > 0 && W > 0)
    return LIG_LANE_CALL(lig_schedule_batch_feedback_chain_fallbacks, ctx_, epoch, seed_, h_reqs_, k, h_picks_, nf,
                         h_fallbacks_, W, nullptr);
  if (nf > 0)
    return LIG_LANE_CALL(lig_schedule_batch_fallbacks, ctx_, epoch, seed_, h_reqs_, k, h_picks_, nf, h_fallbacks_);
  *call = "lig_schedule_batch";
  if (group_) return lig_group_schedule_batch(group_, epoch, seed_, h_reqs_, k, h_picks_);
  if (W > 0)
    return LIG_LANE_CALL(lig_schedule_batch_feedback_chain, ctx_, epoch, seed_, h_reqs_, k, h_picks_, W, nullptr);
  if (opt_.use_doorbell && k <= lig_stream_capacity()) return lig_stream_submit(ctx_, epoch, seed_, h_reqs_, k, h_picks_);
  return lig_schedule_batch(ctx_, epoch, seed_, h_reqs_, k, h_picks_);
}
#undef LIG_LANE_CALL

// One lane of a flush: its waiters are all of one kind, a descriptor (req) or a model name (model),
// a first attempt or a retry (tried).  Each chunk of at most max_batch waiters captures the epoch, maps
// every waiter to a device request or to the answer the host gives it, makes one library call
// (LaneCall) for the mapped requests, maps again on a stale epoch (AwaitPublication), then answers,
// counts and wakes its waiters.  A retry's tried pods become a row of their indices, -1 padded to the
// widest row of the call; one that matches more than LIG_MAX_EXCLUDED pods is answered on the host.
// Fallback rows are asked at the largest n of the lane's waiters (rows are prefixes of longer rows, the
// picks are the plain call's).  rand_keys: each descriptor waiter, sent or not, takes the next splitmix
// key on every attempt; the k model requests sent have rand_key = model_index_ + k on every attempt,
// and model_index_ moves past them once per chunk.  Host-answered model waiters take no key.  An
// affinity lane takes no rand_key either: each request carries its waiter's key.
void Scheduler::FlushLane(std::vector<Waiter*>& lane, CallTime* timing) {
  if (lane.empty()) return;
  const bool models = lane[0]->model != nullptr, retry = lane[0]->tried != nullptr, affinity = lane[0]->affinity;
  const int W = opt_.load_feedback_window;
  Status failure;   // a retry or affinity lane's failure also answers its later chunks, which make no call
  if (retry && !h_excluded_) {
    h_excluded_ = static_cast<int16_t*>(lig_host_alloc((size_t)opt_.max_batch * LIG_MAX_EXCLUDED * sizeof(int16_t)));
    if (!h_excluded_) failure = LigFailure("lig_host_alloc");
  }
  if (affinity && models && !h_keys_) {
    h_keys_ = static_cast<uint64_t*>(lig_host_alloc((size_t)opt_.max_batch * sizeof(uint64_t)));
    if (!h_keys_) failure = LigFailure("lig_host_alloc");
  }
  if (models && retry) model_targets_.resize((size_t)opt_.max_batch);
  std::vector<std::vector<int16_t>> rows;
  std::vector<int> slot;   // waiter i's request in the call, -1 when answered on the host
  for (size_t done = 0; done < lane.size();) {
    Waiter* const* batch = lane.data() + done;
    const int n = (int)std::min(lane.size() - done, (size_t)opt_.max_batch);
    if (!retry && !affinity) failure = Status{};
    std::shared_ptr<const Snapshot> snap;
    int rc = 0, k = 0, nf = 0, width = 1;
    const char* call = "";
    uint64_t writes_seen = 0;
    slot.assign((size_t)n, -1);
    for (int attempt = 0; failure.ok() && attempt < kStaleAttempts; ++attempt) {
      {
        std::lock_guard<std::mutex> lk(snap_mu_);
        snap = snap_;
        writes_seen = writes_done_;
      }
      if (retry) TriedRows(*snap, batch, n, &rows, &width);
      k = 0;
      nf = 0;
      for (int i = 0; i < n; ++i) {
        Waiter* w = batch[i];
        uint64_t key = 0;
        int target = 0;
        if (w->model) {
          w->status = MapModel(*snap, w, &target);
        } else {
          key = affinity ? w->key : splitmix_next(rng_state_);
          nf = std::max(nf, w->fallbacks);   // every descriptor waiter's n counts, sent or not
          w->status = Status{};
        }
        if (w->status.ok() && retry && rows[(size_t)i].size() > (size_t)LIG_MAX_EXCLUDED)
          w->status = Errorf(InvalidArgument, std::string(models ? "ScheduleModelRetry" : "ScheduleRetry") +
                                                  ": the tried pods match more than " +
                                                  std::to_string(LIG_MAX_EXCLUDED) + " pods of the snapshot");
        slot[(size_t)i] = w->status.ok() ? k : -1;
        if (!w->status.ok()) continue;
        if (w->model) {
          h_model_ids_[k] = (uint32_t)w->model_id;
          if (retry) model_targets_[(size_t)k] = (uint8_t)target;
          if (affinity) h_keys_[k] = w->key;
          nf = std::max(nf, w->fallbacks);   // model rows only for the requests the device sees
        } else {
          auto it = snap->adapter_ids->find(w->req->ResolvedTargetModel);
          // a model in no pod's ActiveModels: id A matches no pod, like a Go map miss (filter.go:170).
          // An id interned after this snapshot was packed (>= A) is equally "in no pod" for it.
          h_reqs_[k].adapter_id = (it == snap->adapter_ids->end() || it->second >= snap->A) ? snap->A : it->second;
          h_reqs_[k].flags = w->req->Critical ? LIG_REQ_CRITICAL : 0u;
          h_reqs_[k].rand_key = key;
        }
        if (retry) {
          const std::vector<int16_t>& ex = rows[(size_t)i];
          int16_t* row = h_excluded_ + (size_t)k * (size_t)width;
          for (int j = 0; j < width; ++j) row[j] = j < (int)ex.size() ? ex[(size_t)j] : (int16_t)-1;
        }
        ++k;
      }
      const auto call_t0 = std::chrono::steady_clock::now();
      const double cpu_t0 = timing ? ThreadCpuUs() : 0;
      rc = k > 0 ? LaneCall(snap->epoch, models, retry, affinity, k, nf, width, &call) : 0;
      // a descriptor retry chunk refused on the host as a whole still moves the chain to its epoch
      if (rc == 0 && W > 0 && (k > 0 || !models)) CountFeedback(snap->epoch, k);
      if (timing) {
        const double us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - call_t0).count();
        if (us > timing->us) *timing = CallTime{us, ThreadCpuUs() - cpu_t0};
      }
      if (!AwaitPublication(rc, writes_seen, attempt)) break;
    }
    if (models && !affinity) model_index_ += (uint64_t)k;
    if (failure.ok() && rc != 0) failure = LigFailure(call);
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[i];
      const int s = slot[(size_t)i];
      if (!failure.ok()) {
        if (w->model && !w->status.ok()) continue;   // a model answered on the host keeps that answer
        w->status = failure;
        if (w->model && s >= 0) w->status.message = kModelPrefix + w->status.message;
        continue;
      }
      if (s < 0) continue;
      const uint16_t status = models ? h_mpicks_[s].status : h_picks_[s].status;
      if (models && !retry) {
        const lig_mpick& pk = h_mpicks_[s];   // 255: TargetModels is empty and the name passes through (request.go:47)
        w->resolved = pk.target_idx == 255 ? *w->model
                                           : snap->models->models[(size_t)w->model_id]->TargetModels[pk.target_idx].Name;
      }
      if (status != LIG_OK) {
        w->status = models ? ModelPickError(status, w->model_id, *w->model) : PickError(status);
        continue;
      }
      w->pod = snap->pods[(size_t)(models ? h_mpicks_[s].pod_idx : h_picks_[s].pod_idx)];   // scheduler.go:121
      if (w->fallbacks > 0) {
        w->pods->push_back(w->pod);
        const int16_t* row = h_fallbacks_ + (size_t)s * (size_t)nf;
        for (int j = 0; j < w->fallbacks && row[j] >= 0; ++j) w->pods->push_back(snap->pods[(size_t)row[j]]);
      }
    }
    {
      std::lock_guard<std::mutex> sk(stats_mu_);
      if (affinity) {
        stats_.affinity_scheduled += (uint64_t)n;
      } else if (!models) {
        stats_.scheduled += (uint64_t)n;
        stats_.batches++;
        stats_.max_batch = std::max<uint64_t>(stats_.max_batch, (uint64_t)n);
      }
      if (retry) stats_.retry_scheduled += (uint64_t)n;
      if (models && !retry && !affinity) stats_.model_scheduled += (uint64_t)n;
      if (!retry && !affinity)
        for (int i = 0; i < n; ++i) stats_.fallback_scheduled += batch[i]->fallbacks > 0 ? 1 : 0;
      if (models && !affinity) stats_.model_batches += k > 0 ? 1 : 0;
    }
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[i];
      w->done.store(1, std::memory_order_release);
      w->done.notify_one();
      w->done.store(2, std::memory_order_release);   // last access: the caller may now destroy *w
    }
    done += (size_t)n;
  }
}

Status Scheduler::ScheduleModel(backend::ModelDataStore& datastore, const std::string& model,
                                std::string* resolvedTargetModel, backend::Pod* targetPod) {
  auto modelObj = datastore.FetchModelData(model);                              // request.go:42-45
  if (!modelObj) return Errorf(Unknown, "error finding a model object in InferenceModel for input " + model);
  std::string modelName = model;
  if (!modelObj->TargetModels.empty()) {                                        // request.go:46-51
    const uint64_t key = model_draws_.fetch_add(1, std::memory_order_relaxed) + 1;
    modelName = backend::RandomWeightedDraw(*modelObj, backend::SplitMixSource{seed_ ^ key ^ LIG_DRAW_DOMAIN});
    if (modelName.empty()) return Errorf(Unknown, "error getting target model name for model " + modelObj->ModelName);
  }
  LLMRequest req;                                                               // request.go:52-56
  req.Model = model;
  req.ResolvedTargetModel = modelName;
  req.Critical = modelObj->Critical;
  Status st = Schedule(req, targetPod);
  if (!st.ok()) st.message = "failed to find target pod: " + st.message;        // request.go:73-75 (%w keeps the code)
  if (resolvedTargetModel) *resolvedTargetModel = modelName;
  return st;
}

Stats Scheduler::stats() const {
  std::lock_guard<std::mutex> sk(stats_mu_);
  return stats_;
}

}  // namespace scheduling

namespace backend {

uint64_t SplitMixSource::Uint64() {
  uint64_t z = (state += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

int32_t SplitMixSource::Int31n(int32_t n) {            // math/rand (Go 1.22) Rand.Int31n; n > 0
  if ((n & (n - 1)) == 0) return Int31() & (n - 1);
  const int32_t mx = (int32_t)((1u << 31) - 1 - (uint32_t)((1ull << 31) % (uint64_t)n));
  int32_t v = Int31();
  while (v > mx) v = Int31();
  return v % n;
}

std::string RandomWeightedDraw(const InferenceModel& model, SplitMixSource source) {   // datastore.go:78-98
  int32_t weights = 0;
  for (const TargetModel& tm : model.TargetModels) weights = (int32_t)((uint32_t)weights + (uint32_t)tm.Weight);
  if (weights <= 0) return "";                          // Go's Int31n panics here
  int32_t randomVal = source.Int31n(weights);
  for (const TargetModel& tm : model.TargetModels) {
    if (randomVal < tm.Weight) return tm.Name;
    randomVal -= tm.Weight;
  }
  return "";
}

}  // namespace backend
}  // namespace lig
