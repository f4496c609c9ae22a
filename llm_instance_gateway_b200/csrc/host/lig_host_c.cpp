// lig_host_c.cpp — C entry points over lig_host.hpp (tests + streaming benchmark driver).
#include "lig_host_c.h"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <thread>

#include "lig_host.hpp"

using namespace lig;
using lig::scheduling::Scheduler;

struct ligh_provider : public scheduling::PodMetricsProvider {
  std::mutex mu;
  std::vector<std::shared_ptr<const backend::PodMetrics>> pods;
  std::vector<std::shared_ptr<const backend::PodMetrics>> AllPodMetrics() override {
    std::lock_guard<std::mutex> lk(mu);
    return pods;   // a fresh slice of pointers, like provider.go:38-46
  }
};

struct ligh_scheduler {
  std::shared_ptr<ligh_provider> provider;
  std::unique_ptr<Scheduler> sched;
  // the list last accepted by ligh_scheduler_set_models, to report which target a call resolved to
  std::map<std::string, std::shared_ptr<const backend::InferenceModel>> models_by_name;
};

struct ligh_datastore : public backend::ModelDataStore {     // backend/fake.go: FakeDataStore
  std::mutex mu;
  std::map<std::string, std::shared_ptr<const backend::InferenceModel>> res;
  std::shared_ptr<const backend::InferenceModel> FetchModelData(const std::string& name) override {
    std::lock_guard<std::mutex> lk(mu);
    auto it = res.find(name);
    return it == res.end() ? nullptr : it->second;
  }
};

namespace {
void put(char* dst, int cap, const std::string& s) {
  if (!dst || cap <= 0) return;
  snprintf(dst, (size_t)cap, "%s", s.c_str());
}
}  // namespace

extern "C" {

ligh_provider* ligh_provider_new(void) { return new ligh_provider(); }

static std::shared_ptr<ligh_provider> share(ligh_provider* raw) {
  // shared_from_this-free: build an aliasing non-owning shared_ptr; lifetime is managed by the
  // caller (ligh_provider_free must come after every scheduler using it is freed).
  return std::shared_ptr<ligh_provider>(std::shared_ptr<ligh_provider>(), raw);
}

void ligh_provider_free(ligh_provider* p) { delete p; }

int ligh_provider_set_pods(ligh_provider* p, int n, const char* const* names, const char* const* addrs,
                           const int64_t* q, const double* kv, const int64_t* max_active,
                           const char* const* active_flat, const int* off) {
  if (!p || n < 0) return -1;
  std::vector<std::shared_ptr<const backend::PodMetrics>> v;
  v.reserve((size_t)n);
  for (int i = 0; i < n; ++i) {
    auto pm = std::make_shared<backend::PodMetrics>();
    pm->pod.Name = names ? names[i] : "";
    pm->pod.Address = addrs ? addrs[i] : "";
    pm->metrics.WaitingQueueSize = q[i];
    pm->metrics.KVCacheUsagePercent = kv[i];
    pm->metrics.MaxActiveModels = max_active[i];
    for (int k = off[i]; k < off[i + 1]; ++k) pm->metrics.ActiveModels[active_flat[k]] = 1;
    v.push_back(std::move(pm));
  }
  std::lock_guard<std::mutex> lk(p->mu);
  p->pods.swap(v);
  return 0;
}

ligh_scheduler* ligh_scheduler_new2(ligh_provider* p, int device, int max_pods, int max_adapters,
                                    int max_batch, int flush_size, int window_us, int refresh_ms,
                                    uint64_t seed, int busy_poll, int caller_spin_us,
                                    int use_doorbell, char* err, int err_cap) {
  scheduling::Options o;
  o.device = device;
  o.max_pods = max_pods;
  o.max_adapters = max_adapters;
  o.max_batch = max_batch;
  o.flush_size = flush_size;
  o.batch_window = std::chrono::microseconds(window_us);
  o.refresh_interval = std::chrono::milliseconds(refresh_ms);
  o.seed = seed;
  o.busy_poll = busy_poll != 0;
  o.caller_spin = std::chrono::microseconds(caller_spin_us);
  o.use_doorbell = use_doorbell != 0;
  auto* s = new ligh_scheduler();
  s->provider = share(p);
  scheduling::Status st = scheduling::NewScheduler(s->provider, o, &s->sched);
  if (!st.ok()) {
    put(err, err_cap, st.message);
    delete s;
    return nullptr;
  }
  return s;
}

ligh_scheduler* ligh_scheduler_new_devices(ligh_provider* p, const int* devices, int n_devices, int max_pods,
                                           int max_adapters, int max_batch, int flush_size, int window_us,
                                           int refresh_ms, uint64_t seed, char* err, int err_cap) {
  scheduling::Options o;
  o.devices.assign(devices, devices + n_devices);
  o.max_pods = max_pods;
  o.max_adapters = max_adapters;
  o.max_batch = max_batch;
  o.flush_size = flush_size;
  o.batch_window = std::chrono::microseconds(window_us);
  o.refresh_interval = std::chrono::milliseconds(refresh_ms);
  o.seed = seed;
  auto* s = new ligh_scheduler();
  s->provider = share(p);
  scheduling::Status st = scheduling::NewScheduler(s->provider, o, &s->sched);
  if (!st.ok()) {
    put(err, err_cap, st.message);
    delete s;
    return nullptr;
  }
  return s;
}

ligh_datastore* ligh_datastore_new(void) { return new ligh_datastore(); }
void ligh_datastore_free(ligh_datastore* d) { delete d; }

int ligh_datastore_set_model(ligh_datastore* d, const char* model_name, int critical, int n_targets,
                             const char* const* target_names, const int32_t* weights) {
  if (!d || !model_name || n_targets < 0) return -1;
  auto m = std::make_shared<backend::InferenceModel>();
  m->ModelName = model_name;
  m->Critical = critical != 0;
  for (int k = 0; k < n_targets; ++k) m->TargetModels.push_back(backend::TargetModel{target_names[k], weights[k]});
  std::lock_guard<std::mutex> lk(d->mu);
  d->res[model_name] = std::move(m);
  return 0;
}

int ligh_schedule_model(ligh_scheduler* s, ligh_datastore* d, const char* model, char* resolved, int resolved_cap,
                        char* name, int name_cap, char* addr, int addr_cap, char* err, int err_cap) {
  backend::Pod pod;
  std::string target;
  scheduling::Status st = s->sched->ScheduleModel(*d, model ? model : "", &target, &pod);
  put(resolved, resolved_cap, target);
  if (st.ok()) {
    put(name, name_cap, pod.Name);
    put(addr, addr_cap, pod.Address);
  } else {
    put(err, err_cap, st.message);
  }
  return st.code;
}

int ligh_scheduler_set_models(ligh_scheduler* s, ligh_datastore* d, char* err, int err_cap) {
  std::vector<std::shared_ptr<const backend::InferenceModel>> models;
  {
    std::lock_guard<std::mutex> lk(d->mu);
    for (const auto& kv : d->res) models.push_back(kv.second);
  }
  std::map<std::string, std::shared_ptr<const backend::InferenceModel>> by_name;
  for (const auto& m : models) by_name[m->ModelName] = m;
  scheduling::Status st = s->sched->SetInferenceModels(std::move(models));
  if (st.ok()) s->models_by_name.swap(by_name);
  else put(err, err_cap, st.message);
  return st.code;
}

int ligh_schedule_model_device(ligh_scheduler* s, const char* model, char* resolved, int resolved_cap, char* name,
                               int name_cap, char* addr, int addr_cap, char* err, int err_cap) {
  backend::Pod pod;
  std::string target;
  scheduling::Status st = s->sched->ScheduleModel(std::string(model ? model : ""), &target, &pod);
  put(resolved, resolved_cap, target);
  if (st.ok()) {
    put(name, name_cap, pod.Name);
    put(addr, addr_cap, pod.Address);
  } else {
    put(err, err_cap, st.message);
  }
  return st.code;
}

int ligh_schedule_model_with_fallbacks(ligh_scheduler* s, const char* model, int n, char* resolved, int resolved_cap,
                                       char* names, int names_cap, int* n_pods, char* err, int err_cap) {
  std::string target;
  std::vector<backend::Pod> pods;
  scheduling::Status st = s->sched->ScheduleModelWithFallbacks(std::string(model ? model : ""), n, &target, &pods);
  put(resolved, resolved_cap, target);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

void ligh_model_stats(ligh_scheduler* s, uint64_t out[2]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.model_scheduled;
  out[1] = st.model_batches;
}

ligh_scheduler* ligh_scheduler_new(ligh_provider* p, int device, int max_pods, int max_adapters,
                                   int max_batch, int flush_size, int window_us, int refresh_ms,
                                   uint64_t seed, char* err, int err_cap) {
  return ligh_scheduler_new2(p, device, max_pods, max_adapters, max_batch, flush_size, window_us,
                             refresh_ms, seed, 0, 0, 0, err, err_cap);
}

ligh_scheduler* ligh_scheduler_new_tree(ligh_provider* p, int device, const int* devices, int n_devices,
                                        int max_pods, int max_adapters, int max_batch, int flush_size,
                                        int window_us, int refresh_ms, uint64_t seed, int busy_poll,
                                        int caller_spin_us, int use_doorbell, const lig_filter_node* nodes,
                                        int n_nodes, char* err, int err_cap) {
  return ligh_scheduler_new_feedback(p, device, devices, n_devices, max_pods, max_adapters, max_batch, flush_size,
                                     window_us, refresh_ms, seed, busy_poll, caller_spin_us, use_doorbell, nodes,
                                     n_nodes, 0, 0, 0, err, err_cap);
}

ligh_scheduler* ligh_scheduler_new_feedback(ligh_provider* p, int device, const int* devices, int n_devices,
                                            int max_pods, int max_adapters, int max_batch, int flush_size,
                                            int window_us, int refresh_ms, uint64_t seed, int busy_poll,
                                            int caller_spin_us, int use_doorbell, const lig_filter_node* nodes,
                                            int n_nodes, int load_feedback_window, int feedback_fallbacks,
                                            int feedback_retries, char* err, int err_cap) {
  return ligh_scheduler_new_affinity(p, device, devices, n_devices, max_pods, max_adapters, max_batch, flush_size,
                                     window_us, refresh_ms, seed, busy_poll, caller_spin_us, use_doorbell, nodes,
                                     n_nodes, load_feedback_window, feedback_fallbacks, feedback_retries, 0, err,
                                     err_cap);
}

ligh_scheduler* ligh_scheduler_new_affinity(ligh_provider* p, int device, const int* devices, int n_devices,
                                            int max_pods, int max_adapters, int max_batch, int flush_size,
                                            int window_us, int refresh_ms, uint64_t seed, int busy_poll,
                                            int caller_spin_us, int use_doorbell, const lig_filter_node* nodes,
                                            int n_nodes, int load_feedback_window, int feedback_fallbacks,
                                            int feedback_retries, int affinity, char* err, int err_cap) {
  return ligh_scheduler_new_feedback_affinity(p, device, devices, n_devices, max_pods, max_adapters, max_batch,
                                              flush_size, window_us, refresh_ms, seed, busy_poll, caller_spin_us,
                                              use_doorbell, nodes, n_nodes, load_feedback_window, feedback_fallbacks,
                                              feedback_retries, affinity, 0, err, err_cap);
}

ligh_scheduler* ligh_scheduler_new_feedback_affinity(ligh_provider* p, int device, const int* devices,
                                                     int n_devices, int max_pods, int max_adapters, int max_batch,
                                                     int flush_size, int window_us, int refresh_ms, uint64_t seed,
                                                     int busy_poll, int caller_spin_us, int use_doorbell,
                                                     const lig_filter_node* nodes, int n_nodes,
                                                     int load_feedback_window, int feedback_fallbacks,
                                                     int feedback_retries, int affinity, int feedback_affinity,
                                                     char* err, int err_cap) {
  scheduling::Options o;
  o.affinity = affinity != 0;
  o.feedback_affinity = feedback_affinity != 0;
  o.load_feedback_window = load_feedback_window;
  o.feedback_fallbacks = feedback_fallbacks != 0;
  o.feedback_retries = feedback_retries != 0;
  o.device = device;
  if (devices && n_devices > 1) o.devices.assign(devices, devices + n_devices);
  o.busy_poll = busy_poll != 0;
  o.caller_spin = std::chrono::microseconds(caller_spin_us);
  o.use_doorbell = use_doorbell != 0;
  o.max_pods = max_pods;
  o.max_adapters = max_adapters;
  o.max_batch = max_batch;
  o.flush_size = flush_size;
  o.batch_window = std::chrono::microseconds(window_us);
  o.refresh_interval = std::chrono::milliseconds(refresh_ms);
  o.seed = seed;
  if (nodes && n_nodes > 0) o.filter.assign(nodes, nodes + n_nodes);
  auto* s = new ligh_scheduler();
  s->provider = share(p);
  scheduling::Status st = scheduling::NewScheduler(s->provider, o, &s->sched);
  if (!st.ok()) {
    put(err, err_cap, st.message);
    delete s;
    return nullptr;
  }
  return s;
}

void ligh_scheduler_free(ligh_scheduler* s) { delete s; }

int ligh_schedule(ligh_scheduler* s, const char* model, const char* resolved, int critical,
                  char* name, int name_cap, char* addr, int addr_cap, char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.Model = model ? model : "";
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  backend::Pod pod;
  scheduling::Status st = s->sched->Schedule(req, &pod);
  if (st.ok()) {
    put(name, name_cap, pod.Name);
    put(addr, addr_cap, pod.Address);
  } else {
    put(err, err_cap, st.message);
  }
  return st.code;
}

int ligh_schedule_with_fallbacks(ligh_scheduler* s, const char* resolved, int critical, int n, char* names,
                                 int names_cap, int* n_pods, char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  std::vector<backend::Pod> pods;
  scheduling::Status st = s->sched->ScheduleWithFallbacks(req, n, &pods);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

uint64_t ligh_fallback_scheduled(ligh_scheduler* s) { return s->sched->stats().fallback_scheduled; }

int ligh_schedule_retry(ligh_scheduler* s, const char* resolved, int critical, const char* const* tried_names,
                        const char* const* tried_addrs, int n_tried, char* name, int name_cap, char* addr, int addr_cap,
                        char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  std::vector<backend::Pod> tried;
  for (int i = 0; i < n_tried; ++i)
    tried.push_back(backend::Pod{tried_names[i] ? tried_names[i] : "", tried_addrs[i] ? tried_addrs[i] : ""});
  backend::Pod pod;
  scheduling::Status st = s->sched->ScheduleRetry(req, tried, &pod);
  if (st.ok()) {
    put(name, name_cap, pod.Name);
    put(addr, addr_cap, pod.Address);
  } else {
    put(err, err_cap, st.message);
  }
  return st.code;
}

int ligh_schedule_retry_with_fallbacks(ligh_scheduler* s, const char* resolved, int critical,
                                       const char* const* tried_names, const char* const* tried_addrs, int n_tried,
                                       int n, char* names, int names_cap, int* n_pods, char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  std::vector<backend::Pod> tried;
  for (int i = 0; i < n_tried; ++i)
    tried.push_back(backend::Pod{tried_names[i] ? tried_names[i] : "", tried_addrs[i] ? tried_addrs[i] : ""});
  std::vector<backend::Pod> pods;
  scheduling::Status st = s->sched->ScheduleRetryWithFallbacks(req, tried, n, &pods);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

uint64_t ligh_retry_scheduled(ligh_scheduler* s) { return s->sched->stats().retry_scheduled; }

int ligh_schedule_affinity(ligh_scheduler* s, const char* resolved, int critical, uint64_t key, int n, char* names,
                           int names_cap, int* n_pods, char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  std::vector<backend::Pod> pods(1);
  scheduling::Status st = n == 0 ? s->sched->ScheduleAffinity(req, key, &pods[0])
                                 : s->sched->ScheduleAffinityWithFallbacks(req, key, n, &pods);
  if (!st.ok()) pods.clear();
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

int ligh_schedule_model_affinity(ligh_scheduler* s, const char* model, uint64_t key, int n, char* resolved,
                                 int resolved_cap, char* names, int names_cap, int* n_pods, char* err, int err_cap) {
  std::string target;
  std::vector<backend::Pod> pods(1);
  const std::string m(model ? model : "");
  scheduling::Status st = n == 0 ? s->sched->ScheduleModelAffinity(m, key, &target, &pods[0])
                                 : s->sched->ScheduleModelAffinityWithFallbacks(m, key, n, &target, &pods);
  if (!st.ok()) pods.clear();
  put(resolved, resolved_cap, target);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

uint64_t ligh_affinity_scheduled(ligh_scheduler* s) { return s->sched->stats().affinity_scheduled; }

uint64_t ligh_pod_key(const char* name, const char* address) {
  return scheduling::PodKey(backend::Pod{name ? name : "", address ? address : ""});
}

int ligh_schedule_model_retry(ligh_scheduler* s, const char* model, const char* resolved,
                              const char* const* tried_names, const char* const* tried_addrs, int n_tried, char* name,
                              int name_cap, char* addr, int addr_cap, char* err, int err_cap) {
  std::vector<backend::Pod> tried;
  for (int i = 0; i < n_tried; ++i)
    tried.push_back(backend::Pod{tried_names[i] ? tried_names[i] : "", tried_addrs[i] ? tried_addrs[i] : ""});
  backend::Pod pod;
  scheduling::Status st =
      s->sched->ScheduleModelRetry(std::string(model ? model : ""), std::string(resolved ? resolved : ""), tried, &pod);
  if (st.ok()) {
    put(name, name_cap, pod.Name);
    put(addr, addr_cap, pod.Address);
  } else {
    put(err, err_cap, st.message);
  }
  return st.code;
}

int ligh_schedule_model_retry_with_fallbacks(ligh_scheduler* s, const char* model, const char* resolved,
                                             const char* const* tried_names, const char* const* tried_addrs,
                                             int n_tried, int n, char* names, int names_cap, int* n_pods, char* err,
                                             int err_cap) {
  std::vector<backend::Pod> tried;
  for (int i = 0; i < n_tried; ++i)
    tried.push_back(backend::Pod{tried_names[i] ? tried_names[i] : "", tried_addrs[i] ? tried_addrs[i] : ""});
  std::vector<backend::Pod> pods;
  scheduling::Status st = s->sched->ScheduleModelRetryWithFallbacks(
      std::string(model ? model : ""), std::string(resolved ? resolved : ""), tried, n, &pods);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

int ligh_eject_pods(ligh_scheduler* s, const char* const* names, const char* const* addrs, int n, char* err,
                    int err_cap) {
  std::vector<backend::Pod> pods;
  for (int i = 0; i < n; ++i) pods.push_back(backend::Pod{names[i] ? names[i] : "", addrs[i] ? addrs[i] : ""});
  scheduling::Status st = s->sched->EjectPods(pods);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

void ligh_eject_stats(ligh_scheduler* s, uint64_t out[2]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.ejected_pods;
  out[1] = st.eject_publishes;
}

int ligh_filter(ligh_scheduler* s, const char* resolved, int critical, char* names, int names_cap, int* n_pods,
                char* err, int err_cap) {
  scheduling::LLMRequest req;
  req.ResolvedTargetModel = resolved ? resolved : "";
  req.Critical = critical != 0;
  std::vector<backend::Pod> pods;
  scheduling::Status st = s->sched->Filter(req, &pods);
  std::string joined;
  for (size_t i = 0; i < pods.size(); ++i) joined += (i ? "\n" : "") + pods[i].Name;
  if (n_pods) *n_pods = (int)pods.size();
  put(names, names_cap, joined);
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

int ligh_refresh(ligh_scheduler* s, char* err, int err_cap) {
  scheduling::Status st = s->sched->Refresh();
  if (!st.ok()) put(err, err_cap, st.message);
  return st.code;
}

void ligh_stats(ligh_scheduler* s, uint64_t out[9]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.scheduled; out[1] = st.batches; out[2] = st.max_batch; out[3] = st.refreshes;
  out[4] = st.stale_retries; out[5] = st.failed_refreshes; out[6] = st.excluded_pods;
  out[7] = st.delta_refreshes; out[8] = st.last_dirty_pods;
}

void ligh_feedback_stats(ligh_scheduler* s, uint64_t out[2]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.feedback_windows;
  out[1] = st.feedback_restarts;
}

void ligh_refresh_timing(ligh_scheduler* s, double out[2]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.last_pack_us;
  out[1] = st.last_upload_us;
}

void ligh_flush_timing(ligh_scheduler* s, double out[4]) {
  scheduling::Stats st = s->sched->stats();
  out[0] = st.max_device_call_us;
  out[1] = st.max_flush_us;
  out[2] = (double)st.slowest_call_batch;
  out[3] = st.slowest_call_cpu_us;
}

int ligh_schedule_concurrent(ligh_scheduler* s, int n_threads, int per_thread,
                             const char* const* models, const int* critical, int n_models,
                             int* out_codes, int* out_pod) {
  if (!s || n_threads < 1 || per_thread < 0 || n_models < 1) return -1;
  auto pods = s->provider->AllPodMetrics();
  std::unordered_map<std::string, int> index;
  for (size_t i = 0; i < pods.size(); ++i) index[pods[i]->pod.Name + "\n" + pods[i]->pod.Address] = (int)i;
  std::vector<std::thread> th;
  for (int t = 0; t < n_threads; ++t) {
    th.emplace_back([&, t] {
      for (int k = 0; k < per_thread; ++k) {
        const int i = t * per_thread + k;
        const int m = i % n_models;
        scheduling::LLMRequest req;
        req.Model = req.ResolvedTargetModel = models[m];
        req.Critical = critical[m] != 0;
        backend::Pod pod;
        scheduling::Status st = s->sched->Schedule(req, &pod);
        out_codes[i] = st.code;
        if (st.ok()) {
          auto it = index.find(pod.Name + "\n" + pod.Address);
          out_pod[i] = it == index.end() ? -1 : it->second;
        } else {
          out_pod[i] = -1;
        }
      }
    });
  }
  for (auto& x : th) x.join();
  return 0;
}

int ligh_schedule_models_concurrent(ligh_scheduler* s, ligh_datastore* d, int n_threads, int per_thread,
                                    const char* const* models, int n_models, int* out_codes, int* out_pod,
                                    int* out_target) {
  if (!s || n_threads < 1 || per_thread < 0 || n_models < 1) return -1;
  auto pods = s->provider->AllPodMetrics();
  std::unordered_map<std::string, int> index;
  for (size_t i = 0; i < pods.size(); ++i) index[pods[i]->pod.Name + "\n" + pods[i]->pod.Address] = (int)i;
  std::vector<std::thread> th;
  for (int t = 0; t < n_threads; ++t) {
    th.emplace_back([&, t] {
      for (int k = 0; k < per_thread; ++k) {
        const int i = t * per_thread + k;
        const std::string model = models[i % n_models];
        std::string resolved;
        backend::Pod pod;
        scheduling::Status st = d ? s->sched->ScheduleModel(*d, model, &resolved, &pod)
                                  : s->sched->ScheduleModel(model, &resolved, &pod);
        out_codes[i] = st.code;
        out_pod[i] = -1;
        if (st.ok()) {
          auto it = index.find(pod.Name + "\n" + pod.Address);
          if (it != index.end()) out_pod[i] = it->second;
        }
        // which target the draw chose: its index in the model's TargetModels, 255 = passed through, -1 = none
        out_target[i] = -1;
        auto m = d ? d->FetchModelData(model) : nullptr;
        if (!d) {
          auto it = s->models_by_name.find(model);
          if (it != s->models_by_name.end()) m = it->second;
        }
        if (!resolved.empty() && m) {
          const auto& tms = m->TargetModels;
          for (size_t j = 0; j < tms.size(); ++j)
            if (tms[j].Name == resolved) { out_target[i] = (int)j; break; }
          if (out_target[i] < 0 && resolved == model) out_target[i] = 255;
        }
      }
    });
  }
  for (auto& x : th) x.join();
  return 0;
}

int ligh_stream_bench(ligh_scheduler* s, double rate, double seconds, int n_threads,
                      const char* const* models, const int* critical, int n_models, uint64_t seed,
                      float* lat_us, float* svc_us, int cap, int* n_done, int* n_errors) {
  if (!s || rate <= 0 || seconds <= 0 || n_threads < 1 || n_models < 1) return -1;
  using clock = std::chrono::steady_clock;
  std::atomic<int> slot{0}, errors{0};
  const auto t0 = clock::now() + std::chrono::milliseconds(5);
  std::vector<std::thread> th;
  for (int t = 0; t < n_threads; ++t) {
    th.emplace_back([&, t] {
      uint64_t st = seed ^ (0x9E3779B97F4A7C15ull * (uint64_t)(t + 1));
      auto next_u = [&st]() {   // xorshift64* -> (0,1]
        st ^= st >> 12; st ^= st << 25; st ^= st >> 27;
        return ((st * 2685821657736338717ull) >> 11) * (1.0 / 9007199254740992.0) + 1e-18;
      };
      const double thread_rate = rate / n_threads;
      double at = 0.0;   // seconds since t0 of this thread's next arrival
      uint64_t k = 0;
      for (;;) {
        at += -std::log(next_u()) / thread_rate;   // exponential inter-arrival
        if (at >= seconds) break;
        const auto arrival = t0 + std::chrono::nanoseconds((int64_t)(at * 1e9));
        // sleep most of the way, spin the last stretch for microsecond precision
        auto now = clock::now();
        if (arrival - now > std::chrono::microseconds(200))
          std::this_thread::sleep_for(arrival - now - std::chrono::microseconds(100));
        while (clock::now() < arrival) {}
        const int m = (int)((k++ * (uint64_t)n_threads + (uint64_t)t) % (uint64_t)n_models);
        scheduling::LLMRequest req;
        req.Model = req.ResolvedTargetModel = models[m];
        req.Critical = critical[m] != 0;
        backend::Pod pod;
        const auto called = clock::now();     // >= arrival: the generator itself may run late
        scheduling::Status stt = s->sched->Schedule(req, &pod);
        const auto done = clock::now();
        if (!stt.ok() && stt.code != scheduling::ResourceExhausted) errors++;
        const int i = slot.fetch_add(1);
        if (i < cap) {
          // from the SCHEDULED arrival (no coordinated omission: a late generator counts against us)
          lat_us[i] = (float)(std::chrono::duration<double, std::micro>(done - arrival).count());
          // from the moment Schedule was actually called (the scheduler's own share)
          if (svc_us) svc_us[i] = (float)(std::chrono::duration<double, std::micro>(done - called).count());
        }
      }
    });
  }
  for (auto& x : th) x.join();
  *n_done = std::min(slot.load(), cap);
  *n_errors = errors.load();
  return 0;
}

}  // extern "C"
