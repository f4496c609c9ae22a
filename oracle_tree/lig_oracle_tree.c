/*
 * lig_oracle_tree.c — caller filter trees for the CPU oracle.  TEST INFRASTRUCTURE ONLY (the
 * rules of oracle/lig_oracle.h apply: the product library never loads it).
 *
 * The oracle's port of the reference (oracle/lig_oracle.c) is compiled into this library as it
 * is: the node type with its three successor fields, (*filter).Filter (filter.go:44-73), every
 * node function (filter.go:79-187, scheduler.go:83-89) and the pick.  This file only adds what a
 * caller tree needs on top of it:
 *   - a table of nodes (the same 32-byte record as include/lig.h's lig_filter_node, restated so
 *     the oracle keeps no dependency on the product tree) turned into linked `filter` structs;
 *   - lowQueueingPodPredicate with a per-node threshold, the way the port's
 *     noQueueAndLessThanKVCacheThresholdPredicate closes over its thresholds;
 *   - Filter and Schedule entry points whose root is the caller's tree (NULL = defaultFilter).
 */
#include "../oracle/lig_oracle.c"

typedef struct {                     /* include/lig.h lig_filter_node, 32 bytes */
  int32_t kind;                      /* 0 critical, 1 low queueing, 2 LoRA affinity, 3 can accept LoRA,
                                        4 low LoRA cost, 5 no queue + low KV, 6 least queuing,
                                        7 least KV cache, 8 drop */
  int32_t next_on_success, next_on_failure, next_on_success_or_failure;   /* -1 = nil */
  int64_t queue_threshold;
  double kv_threshold;
} lig_oracle_filter_node;

#define LIGO_MAX_FILTER_NODES 32

/* filter.go:124-126 as a closure over the node's threshold */
static int lowQueueingNodePredicate(const filter* s, const LLMRequest* r, const PodMetrics* pod) {
  (void)r;
  int64_t qt = s->use_closure_thresholds ? s->queueThreshold : queueingThresholdLoRA;
  return pod->m.WaitingQueueSize < qt;
}

static filter tree_nodes[LIGO_MAX_FILTER_NODES];
static const filter* tree_root = &defaultFilter;

/* Use the table (node 0 = root) for every later lig_oracle_tree_* call; NULL = defaultFilter.
 * Returns -1, leaving the previous tree, for a table lig_set_filter_tree would refuse. */
int lig_oracle_set_filter_tree(const lig_oracle_filter_node* nodes, int n) {
  static const char* names[9] = {"critical request", "low queueing", "affinity LoRA",
                                 "can accept LoRA Adapter", "low cost LoRA",
                                 "no queue and low KV cache", "least queuing",
                                 "least KV cache percent", "drop request"};
  if (!nodes) {
    tree_root = &defaultFilter;
    return 0;
  }
  if (n < 1 || n > LIGO_MAX_FILTER_NODES) return -1;
  for (int i = 0; i < n; ++i) {
    const int32_t next[3] = {nodes[i].next_on_success, nodes[i].next_on_failure,
                             nodes[i].next_on_success_or_failure};
    if (nodes[i].kind < 0 || nodes[i].kind > 8) return -1;
    for (int k = 0; k < 3; ++k)
      if (next[k] != -1 && (next[k] <= i || next[k] >= n)) return -1;
  }
  for (int i = 0; i < n; ++i) {
    const lig_oracle_filter_node* nd = &nodes[i];
    filter* f = &tree_nodes[i];
    memset(f, 0, sizeof(*f));
    f->name = names[nd->kind];
    f->filter = predicate_filter;                                   /* toFilterFunc(pp) */
    switch (nd->kind) {
      case 0: f->pp = criticalRequestPredicate; break;
      case 1:
        f->pp = lowQueueingNodePredicate;
        f->use_closure_thresholds = 1;
        f->queueThreshold = nd->queue_threshold;
        break;
      case 2: f->pp = loRAAffinityPredicate; break;
      case 3: f->pp = canAcceptNewLoraPredicate; break;
      case 4: f->pp = lowLoRACostPredicate; break;
      case 5:
        f->pp = noQueueAndLessThanKVCacheThresholdPredicate;
        f->use_closure_thresholds = 1;
        f->queueThreshold = nd->queue_threshold;
        f->kvThreshold = nd->kv_threshold;
        break;
      case 6: f->filter = leastQueuingFilterFunc; break;
      case 7: f->filter = leastKVCacheFilterFunc; break;
      default: f->filter = dropRequestFilterFunc; break;
    }
    f->nextOnSuccess = nd->next_on_success >= 0 ? &tree_nodes[nd->next_on_success] : NULL;
    f->nextOnFailure = nd->next_on_failure >= 0 ? &tree_nodes[nd->next_on_failure] : NULL;
    f->nextOnSuccessOrFailure =
        nd->next_on_success_or_failure >= 0 ? &tree_nodes[nd->next_on_success_or_failure] : NULL;
  }
  tree_root = &tree_nodes[0];
  return 0;
}

/* Schedule's outcome as include/lig.h numbers it: 0 OK, 1 DROP (ResourceExhausted),
 * 2 EMPTY ([] with a nil error), 4 NO_PODS_LEFT (toFilterFunc's "no pods left"). */
static int tree_status(podslice s, const lig_err* e) {
  if (e == &ERR_RESOURCE_EXHAUSTED) return 1;
  if (e == &ERR_NO_PODS_LEFT) return 4;
  if (e) return -1;
  return s.len == 0 ? 2 : 0;
}

/* tree.Filter(req, AllPodMetrics()): survivors in slice order, the status as above. */
int lig_oracle_tree_filter(const lig_oracle_pool* pool, const char* model, int critical,
                           int32_t* out_idx, int* n_out) {
  garbage g = {{0}, 0};
  LLMRequest req = {model, model, critical};
  const lig_err* e = NULL;
  podslice s = filter_Filter(tree_root, &req, AllPodMetrics(pool, &g), &e, &g);
  emit_indices(pool, s, out_idx, n_out);
  int rc = tree_status(s, e);
  gc_release(&g);
  return rc;
}

/* Scheduler.Schedule (scheduler.go:113-122) with the caller's tree, over interned requests as in
 * lig_oracle_schedule_batch (ids outside [0, n_adapters) schedule `unknown`). */
int lig_oracle_tree_schedule_batch(const lig_oracle_pool* pool, const char* const* names, int n_adapters,
                                   const char* unknown, const lig_oracle_req* reqs, int R, uint64_t seed,
                                   lig_oracle_pick* out) {
  if (!pool || R < 0 || (R > 0 && (!reqs || !out))) return -1;
  for (int i = 0; i < R; ++i) {
    const lig_oracle_req* r = &reqs[i];
    const char* model = (r->adapter_id >= 0 && r->adapter_id < n_adapters) ? names[r->adapter_id]
                                                                          : (unknown ? unknown : "");
    LLMRequest req = {model, model, (int)(r->flags & 1u)};
    garbage g = {{0}, 0};
    const lig_err* e = NULL;
    podslice pods = filter_Filter(tree_root, &req, AllPodMetrics(pool, &g), &e, &g);
    int rc = tree_status(pods, e);
    out[i].status = (uint16_t)rc;
    out[i].pod_idx = -1;
    out[i].n_survivors = (uint16_t)(e ? 0 : pods.len);
    if (rc == 0) {
      uint64_t st = seed ^ r->rand_key;
      int32_t k = lig_oracle_int31n(&st, (int32_t)pods.len);       /* scheduler.go:120 */
      out[i].pod_idx = (int32_t)(pods.v[k] - pool->pods);           /* scheduler.go:121 */
    }
    gc_release(&g);
  }
  return 0;
}
