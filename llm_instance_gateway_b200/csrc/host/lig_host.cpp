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

inline uint64_t splitmix_next(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// A stale epoch is re-resolved and tried again up to this many attempts in all (AwaitPublication).
constexpr int kStaleAttempts = 4;

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
  // The model table goes into the published epoch before it is published, so a flush that captures
  // the epoch always finds the table its names were mapped against.
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

Status Scheduler::CheckFallbacks(const char* fn, int n) const {
  if (n < 1 || n > LIG_MAX_FALLBACKS)
    return Errorf(InvalidArgument, std::string(fn) + ": n=" + std::to_string(n) + " outside [1, " +
                                       std::to_string(LIG_MAX_FALLBACKS) + "]");
  if (opt_.load_feedback_window > 0 && !opt_.feedback_fallbacks)
    return Errorf(InvalidArgument, std::string(fn) + ": not defined under load_feedback_window (the picks come "
                                   "from the feedback chain's copy of the snapshot, the fallbacks would not)");
  if (group_)
    return Errorf(InvalidArgument, std::string(fn) + ": a scheduler over several devices has no fallback call");
  return Status{};
}

Status Scheduler::ScheduleWithFallbacks(const LLMRequest& req, int n, std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  if (Status st = CheckFallbacks("ScheduleWithFallbacks", n); !st.ok()) return st;
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.req = &req;
  w.fallbacks = n;
  w.pods = &ranked;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  return w.status;
}

Status Scheduler::ScheduleRetry(const LLMRequest& req, const std::vector<backend::Pod>& tried,
                                backend::Pod* targetPod) {
  if (tried.size() > (size_t)LIG_MAX_EXCLUDED)
    return Errorf(InvalidArgument, "ScheduleRetry: " + std::to_string(tried.size()) + " tried pods (at most " +
                                       std::to_string(LIG_MAX_EXCLUDED) + ")");
  if (opt_.load_feedback_window > 0 && !opt_.feedback_retries)
    return Errorf(InvalidArgument, "ScheduleRetry: not defined under load_feedback_window (the picks come from the "
                                   "feedback chain's copy of the snapshot, a retry would not)");
  if (group_)
    return Errorf(InvalidArgument, "ScheduleRetry: a scheduler over several devices has no retry call");
  Waiter w;
  w.req = &req;
  w.tried = &tried;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

Status Scheduler::ScheduleRetryWithFallbacks(const LLMRequest& req, const std::vector<backend::Pod>& tried, int n,
                                             std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  if (n < 1 || n > LIG_MAX_FALLBACKS)
    return Errorf(InvalidArgument, "ScheduleRetryWithFallbacks: n=" + std::to_string(n) + " outside [1, " +
                                       std::to_string(LIG_MAX_FALLBACKS) + "]");
  if (tried.size() > (size_t)LIG_MAX_EXCLUDED)
    return Errorf(InvalidArgument, "ScheduleRetryWithFallbacks: " + std::to_string(tried.size()) +
                                       " tried pods (at most " + std::to_string(LIG_MAX_EXCLUDED) + ")");
  if (opt_.load_feedback_window > 0 && !(opt_.feedback_retries && opt_.feedback_fallbacks))
    return Errorf(InvalidArgument, "ScheduleRetryWithFallbacks: not defined under load_feedback_window without "
                                   "feedback_retries and feedback_fallbacks (the picks come from the feedback "
                                   "chain's copy of the snapshot, these would not)");
  if (group_)
    return Errorf(InvalidArgument, "ScheduleRetryWithFallbacks: a scheduler over several devices has no retry call");
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.req = &req;
  w.tried = &tried;
  w.fallbacks = n;
  w.pods = &ranked;
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
  if (Status st = CheckFallbacks("ScheduleModelWithFallbacks", n); !st.ok()) return st;
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.model = &model;
  w.fallbacks = n;
  w.pods = &ranked;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
  if (resolvedTargetModel) *resolvedTargetModel = std::move(w.resolved);
  return w.status;
}

Status Scheduler::ScheduleModelRetry(const std::string& model, const std::string& resolvedTargetModel,
                                     const std::vector<backend::Pod>& tried, backend::Pod* targetPod) {
  if (tried.size() > (size_t)LIG_MAX_EXCLUDED)
    return Errorf(InvalidArgument, "ScheduleModelRetry: " + std::to_string(tried.size()) + " tried pods (at most " +
                                       std::to_string(LIG_MAX_EXCLUDED) + ")");
  if (opt_.load_feedback_window > 0 && !opt_.feedback_retries)
    return Errorf(InvalidArgument, "ScheduleModelRetry: not defined under load_feedback_window without "
                                   "feedback_retries (the picks come from the feedback chain's copy of the "
                                   "snapshot, a retry would not)");
  if (group_)
    return Errorf(InvalidArgument, "ScheduleModelRetry: a scheduler over several devices has no retry call");
  Waiter w;
  w.model = &model;
  w.target = &resolvedTargetModel;
  w.tried = &tried;
  Submit(w);
  if (w.status.ok() && targetPod) *targetPod = std::move(w.pod);
  return w.status;
}

Status Scheduler::ScheduleModelRetryWithFallbacks(const std::string& model, const std::string& resolvedTargetModel,
                                                  const std::vector<backend::Pod>& tried, int n,
                                                  std::vector<backend::Pod>* pods) {
  if (pods) pods->clear();
  if (n < 1 || n > LIG_MAX_FALLBACKS)
    return Errorf(InvalidArgument, "ScheduleModelRetryWithFallbacks: n=" + std::to_string(n) + " outside [1, " +
                                       std::to_string(LIG_MAX_FALLBACKS) + "]");
  if (tried.size() > (size_t)LIG_MAX_EXCLUDED)
    return Errorf(InvalidArgument, "ScheduleModelRetryWithFallbacks: " + std::to_string(tried.size()) +
                                       " tried pods (at most " + std::to_string(LIG_MAX_EXCLUDED) + ")");
  if (opt_.load_feedback_window > 0 && !(opt_.feedback_retries && opt_.feedback_fallbacks))
    return Errorf(InvalidArgument, "ScheduleModelRetryWithFallbacks: not defined under load_feedback_window without "
                                   "feedback_retries and feedback_fallbacks (the picks come from the feedback "
                                   "chain's copy of the snapshot, these would not)");
  if (group_)
    return Errorf(InvalidArgument,
                  "ScheduleModelRetryWithFallbacks: a scheduler over several devices has no retry call");
  std::vector<backend::Pod> ranked;
  Waiter w;
  w.model = &model;
  w.target = &resolvedTargetModel;
  w.tried = &tried;
  w.fallbacks = n;
  w.pods = &ranked;
  Submit(w);
  if (w.status.ok() && pods) *pods = std::move(ranked);
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

// A flush that holds both kinds makes the descriptor calls first, then the model-id calls.
void Scheduler::Flush(std::vector<Waiter*>& all) {
  desc_lane_.clear();
  model_lane_.clear();
  retry_lane_.clear();
  model_retry_lane_.clear();
  for (Waiter* w : all)
    (w->model ? (w->tried ? model_retry_lane_ : model_lane_) : w->tried ? retry_lane_ : desc_lane_).push_back(w);
  std::vector<Waiter*>& batch = desc_lane_;
  size_t done = 0;
  const auto flush_t0 = std::chrono::steady_clock::now();
  double device_us = 0, device_cpu_us = 0;
  auto thread_cpu_us = [] {
    timespec ts;
    clock_gettime(CLOCK_THREAD_CPUTIME_ID, &ts);
    return (double)ts.tv_sec * 1e6 + (double)ts.tv_nsec * 1e-3;
  };
  while (done < batch.size()) {
    const int n = (int)std::min(batch.size() - done, (size_t)opt_.max_batch);
    // any ScheduleWithFallbacks caller in this call: one lig_schedule_batch_fallbacks call with the
    // largest n asked (rows are prefixes of longer rows, picks are lig_schedule_batch's)
    int nf = 0;
    for (int i = 0; i < n; ++i) nf = std::max(nf, batch[done + i]->fallbacks);
    std::shared_ptr<const Snapshot> snap;
    Status failure;
    int rc = 0;
    uint64_t writes_seen = 0;
  for (int attempt = 0; attempt < kStaleAttempts; ++attempt) {
      {
        std::lock_guard<std::mutex> lk(snap_mu_);
        snap = snap_;
        writes_seen = writes_done_;
      }
      for (int i = 0; i < n; ++i) {
        const LLMRequest& r = *batch[done + i]->req;
        auto it = snap->adapter_ids->find(r.ResolvedTargetModel);
        // a model in no pod's ActiveModels: id A matches no pod, like a Go map miss (filter.go:170).
        // An id interned after this snapshot was packed (>= A) is equally "in no pod" for it.
        h_reqs_[i].adapter_id = (it == snap->adapter_ids->end() || it->second >= snap->A) ? snap->A : it->second;
        h_reqs_[i].flags = r.Critical ? LIG_REQ_CRITICAL : 0u;
        h_reqs_[i].rand_key = splitmix_next(rng_state_);
      }
      const auto call_t0 = std::chrono::steady_clock::now();
      const double cpu_t0 = thread_cpu_us();
      const int W = opt_.load_feedback_window;
      rc = nf > 0 && W > 0
               ? lig_schedule_batch_feedback_chain_fallbacks(ctx_, snap->epoch, seed_, h_reqs_, n, h_picks_, nf,
                                                             h_fallbacks_, W, nullptr)
           : nf > 0 ? lig_schedule_batch_fallbacks(ctx_, snap->epoch, seed_, h_reqs_, n, h_picks_, nf, h_fallbacks_)
           : group_ ? lig_group_schedule_batch(group_, snap->epoch, seed_, h_reqs_, n, h_picks_)
           : W > 0 ? lig_schedule_batch_feedback_chain(ctx_, snap->epoch, seed_, h_reqs_, n, h_picks_, W, nullptr)
           : (opt_.use_doorbell && n <= lig_stream_capacity())
               ? lig_stream_submit(ctx_, snap->epoch, seed_, h_reqs_, n, h_picks_)
               : lig_schedule_batch(ctx_, snap->epoch, seed_, h_reqs_, n, h_picks_);
      if (rc == 0 && W > 0) CountFeedback(snap->epoch, n);
      const double call_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - call_t0).count();
      if (call_us > device_us) {
        device_us = call_us;
        device_cpu_us = thread_cpu_us() - cpu_t0;
      }
      if (!AwaitPublication(rc, writes_seen, attempt)) break;
    }
    if (rc != 0)
      failure = LigFailure(nf > 0 && opt_.load_feedback_window > 0 ? "lig_schedule_batch_feedback_chain_fallbacks"
                           : nf > 0                         ? "lig_schedule_batch_fallbacks"
                           : opt_.load_feedback_window > 0 ? "lig_schedule_batch_feedback_chain" : "lig_schedule_batch");
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      if (rc != 0) {
        w->status = failure;
      } else if (h_picks_[i].status == LIG_OK) {
        w->pod = snap->pods[(size_t)h_picks_[i].pod_idx];          // pods[i].Pod  scheduler.go:121
        if (w->fallbacks > 0) {
          w->pods->push_back(w->pod);
          const int16_t* row = h_fallbacks_ + (size_t)i * (size_t)nf;
          for (int j = 0; j < w->fallbacks && row[j] >= 0; ++j) w->pods->push_back(snap->pods[(size_t)row[j]]);
        }
      } else {
        w->status = PickError(h_picks_[i].status);
      }
    }
    {
      std::lock_guard<std::mutex> sk(stats_mu_);
      stats_.scheduled += (uint64_t)n;
      for (int i = 0; i < n; ++i) stats_.fallback_scheduled += batch[done + i]->fallbacks > 0 ? 1 : 0;
      stats_.batches++;
      stats_.max_batch = std::max<uint64_t>(stats_.max_batch, (uint64_t)n);
    }
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      w->done.store(1, std::memory_order_release);
      w->done.notify_one();
      w->done.store(2, std::memory_order_release);   // last access: the caller may now destroy *w
    }
    done += (size_t)n;
  }
  FlushRetries(retry_lane_);
  FlushModels(model_lane_);
  FlushModelRetries(model_retry_lane_);
  const double flush_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - flush_t0).count();
  std::lock_guard<std::mutex> sk(stats_mu_);
  if (device_us > stats_.max_device_call_us) {
    stats_.max_device_call_us = device_us;
    stats_.slowest_call_cpu_us = device_cpu_us;
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

// The retry lane: one lig_schedule_batch_excluding call per max_batch waiters (under
// load_feedback_window, lig_schedule_batch_feedback_chain_excluding; with a ScheduleRetryWithFallbacks
// caller among them, lig_schedule_batch_[feedback_chain_]excluding_fallbacks at the largest n asked,
// whose picks, and under the chain whose windows, are the same).  Each waiter's tried pods are
// matched by value against the captured snapshot; its row holds their indices, -1 padded to the
// widest row of the call.  Every waiter takes a rand_key; under the chain a waiter refused on the
// host is left out of the call, since its pick would load a pod and shift every later window.
void Scheduler::FlushRetries(std::vector<Waiter*>& batch) {
  if (batch.empty()) return;
  Status failure;
  if (!h_excluded_) {
    h_excluded_ = static_cast<int16_t*>(lig_host_alloc((size_t)opt_.max_batch * LIG_MAX_EXCLUDED * sizeof(int16_t)));
    if (!h_excluded_) failure = LigFailure("lig_host_alloc");
  }
  std::vector<std::vector<int16_t>> rows;
  std::vector<int> slot;   // waiter i's request in the call, -1 when left out
  const int W = opt_.load_feedback_window;
  size_t done = 0;
  while (done < batch.size()) {
    const int n = (int)std::min(batch.size() - done, (size_t)opt_.max_batch);
    int nf = 0;   // ScheduleRetryWithFallbacks callers: the largest n asked
    for (int i = 0; i < n; ++i) nf = std::max(nf, batch[done + i]->fallbacks);
    std::shared_ptr<const Snapshot> snap;
    int rc = 0, width = 1, k = 0;
    uint64_t writes_seen = 0;
    for (int attempt = 0; failure.ok() && attempt < kStaleAttempts; ++attempt) {
      {
        std::lock_guard<std::mutex> lk(snap_mu_);
        snap = snap_;
        writes_seen = writes_done_;
      }
      TriedRows(*snap, batch.data() + done, n, &rows, &width);
      slot.assign((size_t)n, -1);
      k = 0;
      for (int i = 0; i < n; ++i) {
        const LLMRequest& r = *batch[done + i]->req;
        const uint64_t key = splitmix_next(rng_state_);
        const std::vector<int16_t>& ex = rows[(size_t)i];
        if (W > 0 && ex.size() > (size_t)LIG_MAX_EXCLUDED) continue;
        slot[(size_t)i] = k;
        auto it = snap->adapter_ids->find(r.ResolvedTargetModel);   // interned as in Flush
        h_reqs_[k].adapter_id = (it == snap->adapter_ids->end() || it->second >= snap->A) ? snap->A : it->second;
        h_reqs_[k].flags = r.Critical ? LIG_REQ_CRITICAL : 0u;
        h_reqs_[k].rand_key = key;
        int16_t* row = h_excluded_ + (size_t)k * (size_t)width;
        const int m = (int)ex.size() <= width ? (int)ex.size() : 0;
        for (int j = 0; j < width; ++j) row[j] = j < m ? ex[(size_t)j] : (int16_t)-1;
        ++k;
      }
      if (W > 0) {
        rc = k == 0   ? 0
             : nf > 0 ? lig_schedule_batch_feedback_chain_excluding_fallbacks(ctx_, snap->epoch, seed_, h_reqs_, k,
                                                                              h_excluded_, width, h_picks_, nf,
                                                                              h_fallbacks_, W, nullptr)
                      : lig_schedule_batch_feedback_chain_excluding(ctx_, snap->epoch, seed_, h_reqs_, k, h_excluded_,
                                                                    width, h_picks_, W, nullptr);
        if (rc == 0) CountFeedback(snap->epoch, k);
      } else if (nf > 0) {
        rc = lig_schedule_batch_excluding_fallbacks(ctx_, snap->epoch, seed_, h_reqs_, n, h_excluded_, width, h_picks_,
                                                    nf, h_fallbacks_);
      } else {
        rc = lig_schedule_batch_excluding(ctx_, snap->epoch, seed_, h_reqs_, n, h_excluded_, width, h_picks_);
      }
      if (!AwaitPublication(rc, writes_seen, attempt)) break;
    }
    if (failure.ok() && rc != 0)
      failure = LigFailure(W > 0 && nf > 0 ? "lig_schedule_batch_feedback_chain_excluding_fallbacks"
                           : W > 0         ? "lig_schedule_batch_feedback_chain_excluding"
                           : nf > 0        ? "lig_schedule_batch_excluding_fallbacks"
                                           : "lig_schedule_batch_excluding");
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      const lig_pick* pk = failure.ok() && slot[(size_t)i] >= 0 ? &h_picks_[slot[(size_t)i]] : nullptr;
      if (!failure.ok()) w->status = failure;
      else if (rows[(size_t)i].size() > (size_t)LIG_MAX_EXCLUDED)
        w->status = Errorf(InvalidArgument, "ScheduleRetry: the tried pods match more than " +
                                                std::to_string(LIG_MAX_EXCLUDED) + " pods of the snapshot");
      else if (pk->status == LIG_OK) {
        w->pod = snap->pods[(size_t)pk->pod_idx];
        if (w->fallbacks > 0) {
          w->pods->push_back(w->pod);
          const int16_t* row = h_fallbacks_ + (size_t)slot[(size_t)i] * (size_t)nf;
          for (int j = 0; j < w->fallbacks && row[j] >= 0; ++j) w->pods->push_back(snap->pods[(size_t)row[j]]);
        }
      } else {
        w->status = PickError(pk->status);
      }
    }
    {
      std::lock_guard<std::mutex> sk(stats_mu_);
      stats_.scheduled += (uint64_t)n;
      stats_.retry_scheduled += (uint64_t)n;
      stats_.batches++;
      stats_.max_batch = std::max<uint64_t>(stats_.max_batch, (uint64_t)n);
    }
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      w->done.store(1, std::memory_order_release);
      w->done.notify_one();
      w->done.store(2, std::memory_order_release);   // last access: the caller may now destroy *w
    }
    done += (size_t)n;
  }
}

// A model request's result from its device pick (and row), with ScheduleModel's errors.
static constexpr const char* kModelPrefix = "failed to find target pod: ";            // request.go:73-75

template <class Snap, class W>
static void ModelPickResult(const Snap& snap, const backend::InferenceModel& im, const lig_mpick& pk, const int16_t* row,
                            W* w) {
  const std::string prefix = kModelPrefix;
  if (pk.status == LIG_OK) {
    w->pod = snap.pods[(size_t)pk.pod_idx];
    if (w->fallbacks > 0) {
      w->pods->push_back(w->pod);
      for (int f = 0; f < w->fallbacks && row[f] >= 0; ++f) w->pods->push_back(snap.pods[(size_t)row[f]]);
    }
  } else if (pk.status == LIG_DROP) {
    w->status = Errorf(ResourceExhausted, prefix + "failed to apply filter, resulted 0 pods, this should never "
                                                   "happen: " + kDropInner);
  } else if (pk.status == LIG_NO_PODS_LEFT) {
    w->status = Errorf(Unknown, prefix + "failed to apply filter, resulted 0 pods, this should never happen: "
                                         "no pods left");
  } else if (pk.status == LIG_EMPTY) {
    w->status = Errorf(Unknown, prefix + "failed to apply filter, resulted 0 pods, this should never happen: "
                                         "%!w(<nil>)");
  } else {   // LIG_NO_MODEL: absent models and targets are answered on the host and never sent
    w->status = Errorf(Internal, prefix + "rpc error: code = Internal desc = model id " +
                                     std::to_string(w->model_id) + " (" + im.ModelName +
                                     ") has no model entry on the device");
  }
}

// The model-id lane: names are mapped to ids against the captured epoch's list; names the host can
// answer from that list alone never reach the device.  Request k that reaches the device has
// rand_key = model_index_ + k; a stale-epoch retry maps again and reuses the same first_index.
void Scheduler::FlushModels(std::vector<Waiter*>& batch) {
  size_t done = 0;
  while (done < batch.size()) {
    const int n = (int)std::min(batch.size() - done, (size_t)opt_.max_batch);
    std::shared_ptr<const Snapshot> snap;
    int rc = 0, k = 0, nf = 0;
    const char* call = "lig_schedule_models_batch";
    uint64_t writes_seen = 0;
  for (int attempt = 0; attempt < kStaleAttempts; ++attempt) {
      {
        std::lock_guard<std::mutex> lk(snap_mu_);
        snap = snap_;
        writes_seen = writes_done_;
      }
      const ModelList* list = snap->models.get();
      k = 0;
      nf = 0;
      for (int i = 0; i < n; ++i) {
        Waiter* w = batch[done + i];
        auto it = list ? list->ids.find(*w->model) : decltype(list->ids)::const_iterator{};
        if (!list || it == list->ids.end()) {                                       // request.go:42-45
          w->model_id = -1;
          w->status = Errorf(Unknown, "error finding a model object in InferenceModel for input " + *w->model);
        } else if (!list->present[it->second]) {                                     // request.go:48-51
          w->model_id = -1;
          w->status = Errorf(Unknown, "error getting target model name for model " +
                                          list->models[it->second]->ModelName);
        } else {
          w->model_id = it->second;
          w->status = Status{};   // a retry may map a name the previous epoch answered on the host
          h_model_ids_[k++] = it->second;
          nf = std::max(nf, w->fallbacks);   // rows only for the requests the device sees
        }
      }
      if (k == 0) break;
      const int W = opt_.load_feedback_window;
      // any ScheduleModelWithFallbacks caller among them: one fallback call at the largest n asked
      // (rows are prefixes of longer rows, picks are the plain call's); never the doorbell
      if (nf > 0 && W > 0) {
        call = "lig_schedule_models_batch_feedback_chain_fallbacks";
        rc = lig_schedule_models_batch_feedback_chain_fallbacks(ctx_, snap->epoch, seed_, model_index_, h_model_ids_,
                                                                k, h_mpicks_, nf, h_fallbacks_, W, nullptr);
      } else if (nf > 0) {
        call = "lig_schedule_models_batch_fallbacks";
        rc = lig_schedule_models_batch_fallbacks(ctx_, snap->epoch, seed_, model_index_, h_model_ids_, k, h_mpicks_,
                                                 nf, h_fallbacks_);
      } else if (W > 0) {
        call = "lig_schedule_models_batch_feedback_chain";
        rc = lig_schedule_models_batch_feedback_chain(ctx_, snap->epoch, seed_, model_index_, h_model_ids_, k,
                                                      h_mpicks_, W, nullptr);
      } else if (opt_.use_doorbell && k <= lig_stream_capacity()) {
        call = "lig_stream_submit_models";
        rc = lig_stream_submit_models(ctx_, snap->epoch, seed_, model_index_, h_model_ids_, k, h_mpicks_);
      } else {
        rc = lig_schedule_models_batch(ctx_, snap->epoch, seed_, model_index_, h_model_ids_, k, h_mpicks_);
      }
      if (rc == 0 && W > 0) CountFeedback(snap->epoch, k);
      if (!AwaitPublication(rc, writes_seen, attempt)) break;
    }
    if (k > 0) model_index_ += (uint64_t)k;
    const Status failure = rc != 0 ? LigFailure(call) : Status{};
    const std::string prefix = kModelPrefix;
    for (int i = 0, j = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      if (w->model_id < 0) continue;
      const int16_t* row = h_fallbacks_ + (size_t)j * (size_t)nf;
      const lig_mpick& pk = h_mpicks_[j++];
      if (rc != 0) {
        w->status = failure;
        w->status.message = prefix + w->status.message;
        continue;
      }
      const backend::InferenceModel& im = *snap->models->models[(size_t)w->model_id];
      // 255: TargetModels is empty and the requested name passes through (request.go:47)
      w->resolved = pk.target_idx == 255 ? *w->model : im.TargetModels[pk.target_idx].Name;
      ModelPickResult(*snap, im, pk, row, w);
    }
    {
      std::lock_guard<std::mutex> sk(stats_mu_);
      stats_.model_scheduled += (uint64_t)n;
      for (int i = 0; i < n; ++i) stats_.fallback_scheduled += batch[done + i]->fallbacks > 0 ? 1 : 0;
      stats_.model_batches += k > 0 ? 1 : 0;
    }
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      w->done.store(1, std::memory_order_release);
      w->done.notify_one();
      w->done.store(2, std::memory_order_release);   // last access: the caller may now destroy *w
    }
    done += (size_t)n;
  }
}

// The model-retry lane: per max_batch waiters, names are mapped against the captured epoch's list (the
// model to its id, the resolved target to its index, 255 for a model without TargetModels), tried pods
// to their indices; waiters the host can answer never reach the device and take no rand_key.  Request k
// that reaches the device has rand_key = model_index_ + k.  One lig_schedule_models_batch_excluding call
// (with fallback rows at the largest n asked when any caller wants them; under load_feedback_window the
// chain forms); a stale-epoch retry maps again and reuses the same first_index.
void Scheduler::FlushModelRetries(std::vector<Waiter*>& batch) {
  if (batch.empty()) return;
  Status failure;
  if (!h_excluded_) {
    h_excluded_ = static_cast<int16_t*>(lig_host_alloc((size_t)opt_.max_batch * LIG_MAX_EXCLUDED * sizeof(int16_t)));
    if (!h_excluded_) failure = LigFailure("lig_host_alloc");
  }
  model_targets_.resize((size_t)opt_.max_batch);
  std::vector<std::vector<int16_t>> rows;
  const int W = opt_.load_feedback_window;
  size_t done = 0;
  while (done < batch.size()) {
    const int n = (int)std::min(batch.size() - done, (size_t)opt_.max_batch);
    std::shared_ptr<const Snapshot> snap;
    int rc = 0, k = 0, nf = 0, width = 1;
    bool mapped = false;   // the waiters were mapped against a snapshot (host answers are in place)
    const char* call = "lig_schedule_models_batch_excluding";
    uint64_t writes_seen = 0;
    for (int attempt = 0; failure.ok() && attempt < kStaleAttempts; ++attempt) {
      {
        std::lock_guard<std::mutex> lk(snap_mu_);
        snap = snap_;
        writes_seen = writes_done_;
      }
      const ModelList* list = snap->models.get();
      TriedRows(*snap, batch.data() + done, n, &rows, &width);
      mapped = true;
      k = 0;
      nf = 0;
      for (int i = 0; i < n; ++i) {
        Waiter* w = batch[done + i];
        w->model_id = -1;
        auto it = list ? list->ids.find(*w->model) : decltype(list->ids)::const_iterator{};
        if (!list || it == list->ids.end()) {                                       // request.go:42-45
          w->status = Errorf(Unknown, "error finding a model object in InferenceModel for input " + *w->model);
          continue;
        }
        if (!list->present[it->second]) {                                           // request.go:48-51
          w->status = Errorf(Unknown, "error getting target model name for model " +
                                          list->models[it->second]->ModelName);
          continue;
        }
        const backend::InferenceModel& im = *list->models[it->second];
        int t = -1;
        if (im.TargetModels.empty()) {
          if (*w->target == *w->model) t = 255;                                      // request.go:47
        } else {
          for (size_t j = 0; j < im.TargetModels.size() && t < 0; ++j)
            if (im.TargetModels[j].Name == *w->target) t = (int)j;
        }
        if (t < 0) {
          w->status = Errorf(InvalidArgument, "ScheduleModelRetry: " + *w->target + " is not a target model of " +
                                                  *w->model);
          continue;
        }
        const std::vector<int16_t>& ex = rows[(size_t)i];
        if (ex.size() > (size_t)LIG_MAX_EXCLUDED) {
          w->status = Errorf(InvalidArgument, "ScheduleModelRetry: the tried pods match more than " +
                                                  std::to_string(LIG_MAX_EXCLUDED) + " pods of the snapshot");
          continue;
        }
        w->model_id = it->second;
        w->status = Status{};   // a retry may map a name the previous epoch answered on the host
        w->resolved = *w->target;
        h_model_ids_[k] = it->second;
        model_targets_[(size_t)k] = (uint8_t)t;
        int16_t* row = h_excluded_ + (size_t)k * (size_t)width;
        for (int j = 0; j < width; ++j) row[j] = j < (int)ex.size() ? ex[(size_t)j] : (int16_t)-1;
        nf = std::max(nf, w->fallbacks);   // rows only for the requests the device sees
        ++k;
      }
      if (k == 0) break;
      if (nf > 0 && W > 0) {
        call = "lig_schedule_models_batch_feedback_chain_excluding_fallbacks";
        rc = lig_schedule_models_batch_feedback_chain_excluding_fallbacks(
            ctx_, snap->epoch, seed_, model_index_, h_model_ids_, model_targets_.data(), k, h_excluded_, width,
            h_mpicks_, nf, h_fallbacks_, W, nullptr);
      } else if (nf > 0) {
        call = "lig_schedule_models_batch_excluding_fallbacks";
        rc = lig_schedule_models_batch_excluding_fallbacks(ctx_, snap->epoch, seed_, model_index_, h_model_ids_,
                                                           model_targets_.data(), k, h_excluded_, width, h_mpicks_, nf,
                                                           h_fallbacks_);
      } else if (W > 0) {
        call = "lig_schedule_models_batch_feedback_chain_excluding";
        rc = lig_schedule_models_batch_feedback_chain_excluding(ctx_, snap->epoch, seed_, model_index_, h_model_ids_,
                                                                model_targets_.data(), k, h_excluded_, width,
                                                                h_mpicks_, W, nullptr);
      } else {
        rc = lig_schedule_models_batch_excluding(ctx_, snap->epoch, seed_, model_index_, h_model_ids_,
                                                 model_targets_.data(), k, h_excluded_, width, h_mpicks_);
      }
      if (rc == 0 && W > 0) CountFeedback(snap->epoch, k);
      if (!AwaitPublication(rc, writes_seen, attempt)) break;
    }
    if (k > 0) model_index_ += (uint64_t)k;
    if (failure.ok() && rc != 0) failure = LigFailure(call);
    for (int i = 0, j = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
      if (mapped && w->model_id < 0) continue;
      if (!failure.ok()) {
        w->status = failure;
        if (w->model_id >= 0) w->status.message = kModelPrefix + w->status.message;
        continue;
      }
      const int16_t* row = h_fallbacks_ + (size_t)j * (size_t)nf;
      const lig_mpick& pk = h_mpicks_[j++];
      ModelPickResult(*snap, *snap->models->models[(size_t)w->model_id], pk, row, w);
    }
    {
      std::lock_guard<std::mutex> sk(stats_mu_);
      stats_.retry_scheduled += (uint64_t)n;
      stats_.model_batches += k > 0 ? 1 : 0;
    }
    for (int i = 0; i < n; ++i) {
      Waiter* w = batch[done + i];
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
