/* lig_host_c.h — C entry points over the C++ host runtime (lig_host.hpp), for ctypes-driven tests
 * and the streaming benchmark.  Not part of the drop-in boundary (that is include/lig.h). */
#ifndef LIG_HOST_C_H_
#define LIG_HOST_C_H_
#include <stdint.h>

#include "../../../include/lig.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct ligh_provider ligh_provider;   /* a mutable fake PodMetricsProvider (backend/fake.go:10-21 analogue) */
typedef struct ligh_scheduler ligh_scheduler;

ligh_provider* ligh_provider_new(void);
void ligh_provider_free(ligh_provider*);
/* Replace the provider's slice.  active_flat holds all pods' ActiveModels keys back to back;
 * pod i owns active_flat[active_offsets[i] .. active_offsets[i+1]). */
int ligh_provider_set_pods(ligh_provider*, int n, const char* const* names, const char* const* addrs,
                           const int64_t* waiting_queue_size, const double* kv_cache_usage_percent,
                           const int64_t* max_active_models, const char* const* active_flat,
                           const int* active_offsets);

ligh_scheduler* ligh_scheduler_new(ligh_provider*, int device, int max_pods, int max_adapters,
                                   int max_batch, int flush_size, int batch_window_us,
                                   int refresh_interval_ms, uint64_t seed, char* err, int err_cap);
/* Same, plus the latency knobs: busy_poll (batcher polls instead of sleeping), caller_spin_us,
 * use_doorbell (flush through the persistent doorbell kernel instead of a launch per flush). */
ligh_scheduler* ligh_scheduler_new2(ligh_provider*, int device, int max_pods, int max_adapters,
                                    int max_batch, int flush_size, int batch_window_us,
                                    int refresh_interval_ms, uint64_t seed, int busy_poll,
                                    int caller_spin_us, int use_doorbell, char* err, int err_cap);
/* ligh_scheduler_new2 / _new_devices with a caller filter tree (Options::filter; see
 * lig_set_filter_tree): n_devices > 1 lists the GPUs of one scheduler (then `device` is ignored). */
ligh_scheduler* ligh_scheduler_new_tree(ligh_provider*, int device, const int* devices, int n_devices,
                                        int max_pods, int max_adapters, int max_batch, int flush_size,
                                        int batch_window_us, int refresh_interval_ms, uint64_t seed,
                                        int busy_poll, int caller_spin_us, int use_doorbell,
                                        const lig_filter_node* nodes, int n_nodes, char* err, int err_cap);
/* ligh_scheduler_new_tree plus Options::load_feedback_window (0 = off; > 0 flushes through
 * lig_schedule_batch_feedback_chain; refused with several devices or use_doorbell) and
 * Options::feedback_fallbacks (nonzero: the *WithFallbacks calls run under the chain) and
 * Options::feedback_retries (nonzero: ScheduleRetry runs under the chain; with both nonzero,
 * ScheduleRetryWithFallbacks does too). */
ligh_scheduler* ligh_scheduler_new_feedback(ligh_provider*, int device, const int* devices, int n_devices,
                                            int max_pods, int max_adapters, int max_batch, int flush_size,
                                            int batch_window_us, int refresh_interval_ms, uint64_t seed,
                                            int busy_poll, int caller_spin_us, int use_doorbell,
                                            const lig_filter_node* nodes, int n_nodes, int load_feedback_window,
                                            int feedback_fallbacks, int feedback_retries, char* err, int err_cap);
/* ligh_scheduler_new_feedback plus Options::affinity (nonzero: every published epoch carries the pods'
 * keys, and ligh_schedule_affinity / ligh_schedule_model_affinity are served). */
ligh_scheduler* ligh_scheduler_new_affinity(ligh_provider*, int device, const int* devices, int n_devices,
                                            int max_pods, int max_adapters, int max_batch, int flush_size,
                                            int batch_window_us, int refresh_interval_ms, uint64_t seed,
                                            int busy_poll, int caller_spin_us, int use_doorbell,
                                            const lig_filter_node* nodes, int n_nodes, int load_feedback_window,
                                            int feedback_fallbacks, int feedback_retries, int affinity, char* err,
                                            int err_cap);
/* ligh_scheduler_new_affinity plus Options::feedback_affinity (nonzero, with affinity and
 * load_feedback_window: ligh_schedule_affinity / ligh_schedule_model_affinity run under the chain). */
ligh_scheduler* ligh_scheduler_new_feedback_affinity(ligh_provider*, int device, const int* devices, int n_devices,
                                                     int max_pods, int max_adapters, int max_batch, int flush_size,
                                                     int batch_window_us, int refresh_interval_ms, uint64_t seed,
                                                     int busy_poll, int caller_spin_us, int use_doorbell,
                                                     const lig_filter_node* nodes, int n_nodes,
                                                     int load_feedback_window, int feedback_fallbacks,
                                                     int feedback_retries, int affinity, int feedback_affinity,
                                                     char* err, int err_cap);
void ligh_scheduler_free(ligh_scheduler*);
/* Scheduler.Schedule: returns the gRPC code (0 OK, 8 ResourceExhausted, 2 Unknown, 13 Internal). */
int ligh_schedule(ligh_scheduler*, const char* model, const char* resolved_target_model, int critical,
                  char* name, int name_cap, char* addr, int addr_cap, char* err, int err_cap);
/* Scheduler::Filter: returns the gRPC code; names receives the survivors' pod names joined by '\n'
 * (slice order) and *n_pods their count. */
int ligh_filter(ligh_scheduler*, const char* resolved_target_model, int critical, char* names, int names_cap,
                int* n_pods, char* err, int err_cap);
/* Scheduler::ScheduleWithFallbacks: returns the gRPC code; names receives the pick and then up to n
 * fallback pods' names joined by '\n' (retry order) and *n_pods their count. */
int ligh_schedule_with_fallbacks(ligh_scheduler*, const char* resolved_target_model, int critical, int n,
                                 char* names, int names_cap, int* n_pods, char* err, int err_cap);
uint64_t ligh_fallback_scheduled(ligh_scheduler*);   /* Stats::fallback_scheduled */
/* Scheduler::ScheduleRetry: returns the gRPC code; the tried pods are given by value as n_tried
 * (name, address) pairs. */
int ligh_schedule_retry(ligh_scheduler*, const char* resolved_target_model, int critical, const char* const* tried_names,
                        const char* const* tried_addrs, int n_tried, char* name, int name_cap, char* addr, int addr_cap,
                        char* err, int err_cap);
/* Scheduler::ScheduleRetryWithFallbacks: returns the gRPC code; the tried pods as ligh_schedule_retry's;
 * names receives the retry's pick and then up to n fallback pods' names joined by '\n' (retry order)
 * and *n_pods their count. */
int ligh_schedule_retry_with_fallbacks(ligh_scheduler*, const char* resolved_target_model, int critical,
                                       const char* const* tried_names, const char* const* tried_addrs, int n_tried,
                                       int n, char* names, int names_cap, int* n_pods, char* err, int err_cap);
uint64_t ligh_retry_scheduled(ligh_scheduler*);      /* Stats::retry_scheduled */
/* Scheduler::ScheduleAffinity (n = 0) or ScheduleAffinityWithFallbacks (n fallbacks): returns the gRPC
 * code; names receives the pick and then the row's pods' names joined by '\n' and *n_pods their count. */
int ligh_schedule_affinity(ligh_scheduler*, const char* resolved_target_model, int critical, uint64_t key, int n,
                           char* names, int names_cap, int* n_pods, char* err, int err_cap);
/* Scheduler::ScheduleModelAffinity[WithFallbacks], as ligh_schedule_affinity; resolved receives the
 * resolved target model. */
int ligh_schedule_model_affinity(ligh_scheduler*, const char* model, uint64_t key, int n, char* resolved,
                                 int resolved_cap, char* names, int names_cap, int* n_pods, char* err, int err_cap);
uint64_t ligh_affinity_scheduled(ligh_scheduler*);   /* Stats::affinity_scheduled */
uint64_t ligh_pod_key(const char* name, const char* address);   /* scheduling::PodKey */
/* Scheduler::ScheduleModelRetry: returns the gRPC code; resolved_target_model is the name the model call
 * returned; the tried pods as ligh_schedule_retry's. */
int ligh_schedule_model_retry(ligh_scheduler*, const char* model, const char* resolved_target_model,
                              const char* const* tried_names, const char* const* tried_addrs, int n_tried, char* name,
                              int name_cap, char* addr, int addr_cap, char* err, int err_cap);
/* Scheduler::ScheduleModelRetryWithFallbacks: as ligh_schedule_retry_with_fallbacks, for a model request. */
int ligh_schedule_model_retry_with_fallbacks(ligh_scheduler*, const char* model, const char* resolved_target_model,
                                             const char* const* tried_names, const char* const* tried_addrs,
                                             int n_tried, int n, char* names, int names_cap, int* n_pods, char* err,
                                             int err_cap);
/* Scheduler::EjectPods: the complete ejected set as n (name, address) pairs (n = 0 lets every pod back);
 * returns the gRPC code, err receives the refusal. */
int ligh_eject_pods(ligh_scheduler*, const char* const* names, const char* const* addrs, int n, char* err,
                    int err_cap);
void ligh_eject_stats(ligh_scheduler*, uint64_t out[2]);  /* Stats::ejected_pods, Stats::eject_publishes */
int ligh_refresh(ligh_scheduler*, char* err, int err_cap);
/* several GPUs behind one scheduler (lig_group_*) */
ligh_scheduler* ligh_scheduler_new_devices(ligh_provider*, const int* devices, int n_devices, int max_pods,
                                           int max_adapters, int max_batch, int flush_size, int window_us,
                                           int refresh_ms, uint64_t seed, char* err, int err_cap);
/* a fake ModelDataStore (backend/fake.go) and the resolve + Schedule call of HandleRequestBody */
typedef struct ligh_datastore ligh_datastore;
ligh_datastore* ligh_datastore_new(void);
void ligh_datastore_free(ligh_datastore*);
int ligh_datastore_set_model(ligh_datastore*, const char* model_name, int critical, int n_targets,
                             const char* const* target_names, const int32_t* weights);
int ligh_schedule_model(ligh_scheduler*, ligh_datastore*, const char* model, char* resolved, int resolved_cap,
                        char* name, int name_cap, char* addr, int addr_cap, char* err, int err_cap);
/* Scheduler::SetInferenceModels with the datastore's current contents (the list is copied: later
 * ligh_datastore_set_model calls do not reach the scheduler until the next ligh_scheduler_set_models).
 * Returns the gRPC code; err receives the refusal. */
int ligh_scheduler_set_models(ligh_scheduler*, ligh_datastore*, char* err, int err_cap);
/* Scheduler::ScheduleModel(model, ...): resolved on the device against that list. */
int ligh_schedule_model_device(ligh_scheduler*, const char* model, char* resolved, int resolved_cap,
                               char* name, int name_cap, char* addr, int addr_cap, char* err, int err_cap);
/* Scheduler::ScheduleModelWithFallbacks: returns the gRPC code; resolved receives the resolved target
 * model, names the pick and then up to n fallback pods' names joined by '\n' and *n_pods their count. */
int ligh_schedule_model_with_fallbacks(ligh_scheduler*, const char* model, int n, char* resolved, int resolved_cap,
                                       char* names, int names_cap, int* n_pods, char* err, int err_cap);
void ligh_model_stats(ligh_scheduler*, uint64_t out[2]); /* model_scheduled, model_batches */
void ligh_stats(ligh_scheduler*, uint64_t out[9]); /* scheduled, batches, max_batch, refreshes, stale_retries */
void ligh_feedback_stats(ligh_scheduler*, uint64_t out[2]); /* feedback_windows, feedback_restarts */
void ligh_refresh_timing(ligh_scheduler*, double out[2]); /* last Refresh: host pack us, lig_upload_snapshot us */
void ligh_flush_timing(ligh_scheduler*, double out[4]);   /* slowest device call us, slowest Flush us, index of that call, thread CPU us inside it */

/* n_threads caller threads each issue `per_thread` blocking Schedule calls (model i of the
 * request table, round-robin); out_codes/out_pod (n_threads*per_thread) receive the code and the
 * index of the returned pod in the provider's slice (-1 on error). */
int ligh_schedule_concurrent(ligh_scheduler*, int n_threads, int per_thread,
                             const char* const* resolved_models, const int* critical, int n_models,
                             int* out_codes, int* out_pod);

/* The same for model requests: caller i sends models[i % n_models] through ligh_schedule_model_device
 * (datastore null) or ligh_schedule_model with the datastore.  out_target receives the index of the
 * resolved name in that model's TargetModels (255: the name passed through, -1: no resolved name). */
int ligh_schedule_models_concurrent(ligh_scheduler*, ligh_datastore* datastore, int n_threads, int per_thread,
                                    const char* const* models, int n_models, int* out_codes, int* out_pod,
                                    int* out_target);

/* Streaming load (BASELINE.json configs[4]): Poisson arrivals at `rate` req/s for `seconds`,
 * spread over n_threads caller threads; latency = completion - scheduled arrival.  Fills
 * lat_us[0..*n_done) (capacity cap).  Returns 0. */
int ligh_stream_bench(ligh_scheduler*, double rate, double seconds, int n_threads,
                      const char* const* resolved_models, const int* critical, int n_models,
                      uint64_t seed, float* lat_us, float* svc_us, int cap, int* n_done, int* n_errors);

#ifdef __cplusplus
}
#endif
#endif
