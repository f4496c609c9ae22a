// lig.cu — the C ABI of include/lig.h over the sm_90a kernels of lig_device.cuh.
//
// Host-side responsibilities only: context and HBM/pinned allocation, snapshot slots (two resident
// epochs), stream/event ordering, the host-buffer path, error reporting.  There is deliberately no
// CPU implementation of the scheduling path in this library: if CUDA is missing every entry point
// fails with LIG_ERR_CUDA.
#include <cuda_runtime.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <atomic>
#include <cctype>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

#include "lig_device.cuh"
#include "lig_internal.hpp"

using namespace lig;

namespace {
thread_local char g_err[512] = "";
}

namespace ligi {
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace ligi
using ligi::fail;

namespace {

#define CUDA_TRY(expr)                                                                      \
  do {                                                                                      \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      return fail(LIG_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),    \
                  __FILE__, __LINE__);                                                      \
  } while (0)

inline int words_for(int P) { return (P + 31) / 32; }

// Run STMT with the compile-time constant kPpt bound to the run-time requests-per-thread knob.
#define LIG_DISPATCH_PPT(ppt, STMT)                           \
  switch (ppt) {                                              \
    case 1:  { constexpr int kPpt = 1;  STMT; } break;        \
    case 2:  { constexpr int kPpt = 2;  STMT; } break;        \
    case 8:  { constexpr int kPpt = 8;  STMT; } break;        \
    case 16: { constexpr int kPpt = 16; STMT; } break;        \
    default: { constexpr int kPpt = 4;  STMT; } break;        \
  }

struct Layout {  // offsets into the packed blob
  size_t kv, q, na, ma, bitmap, total;
};

Layout layout_for(int P, int A) {
  const size_t Ppad = (size_t)words_for(P) * 32;
  Layout l;
  l.kv = 0;
  l.q = l.kv + Ppad * sizeof(double);
  l.na = l.q + Ppad * sizeof(int32_t);
  l.ma = l.na + Ppad * sizeof(uint16_t);
  l.bitmap = l.ma + Ppad * sizeof(uint16_t);
  l.total = l.bitmap + (size_t)A * words_for(P) * sizeof(uint32_t);
  l.total = (l.total + 15) & ~(size_t)15;
  if (l.total == 0) l.total = 16;
  return l;
}

struct Slot {
  bool valid = false;
  uint64_t epoch = 0;
  int P = 0, A = 0, W = 0;
  unsigned char* d_blob = nullptr;
  ClassEntry* d_cls = nullptr;
  uint16_t* d_lists = nullptr;
  unsigned char* d_ctab = nullptr;  // compact tables (CompactHeader blob): entries + packed lists
  uint32_t* d_counters = nullptr;   // pool cursor + finished-CTA counter of the build kernel
  uint32_t ctab_pool_capacity = 0;  // list entries the compact pool can hold
  CompactHeader* h_hdr = nullptr;   // pinned, device-mapped copy of the blob's header, valid once `ready` completed
  CompactHeader* d_hdr_alias = nullptr;   // its device-visible address
  unsigned char* h_blob = nullptr;  // pinned staging for host uploads
  // model table of this epoch (lig_upload_models), grown on demand
  unsigned char* d_mtab = nullptr;
  unsigned char* h_mtab = nullptr;  // pinned staging
  size_t mtab_capacity = 0;
  uint32_t mtab_bytes = 0, n_models = 0;
  bool models_valid = false;
  cudaEvent_t models_ready = nullptr;
  // pod keys of this epoch (lig_upload_pod_keys): h[p] = mix(pod_key[p]), max_pods entries
  uint64_t* d_podkeys = nullptr;
  uint64_t* h_podkeys = nullptr;    // pinned staging
  bool keys_valid = false;
  cudaEvent_t keys_ready = nullptr;
  cudaEvent_t ready = nullptr;      // class tables built
  // Batches that read this slot, possibly on different caller streams: a ring of events, one per
  // schedule call.  A writer (re-upload, threshold rebuild) waits on every event of the ring; when
  // the ring wraps, the new reader's stream first waits on the event it is about to re-record, so
  // the re-recorded event still covers the reader it replaces (transitively).
  static constexpr int kReaders = 8;
  cudaEvent_t readers[kReaders] = {};
  int next_reader = 0;
  uint64_t stamp = 0;               // upload order, to pick the slot to overwrite
  bool caller_tree = false;         // tables built with a caller filter tree (thresholds do not apply)
  FilterTree tree{};                // that tree (caller_tree only): the retry walk runs the epoch's own tree
  // lig_eject_pods: the epoch's pool, W words (bit p = pod p is in it), read only when n_ejected > 0.
  // Every class-table build and retry walk of the slot starts from it instead of every pod.
  uint32_t* d_pool = nullptr;
  int n_ejected = 0;
};

constexpr int kLanes = 8;   // streams of the host-buffer path; also the queue streams

}  // namespace

struct lig_ctx {
  int device = 0;
  int max_pods = 0, max_adapters = 0, max_batch = 0;
  int sm_count = 0;
  size_t smem_optin = 0;
  lig_thresholds thr{0.8, 5, 50};
  // caller filter tree (lig_set_filter_tree), guarded by upload_mu like every snapshot writer
  FilterTree tree{};
  bool has_tree = false;
  // mu guards the slot metadata, the reader rings, lanes/tickets and the item ring.  It is held
  // only while work is ENQUEUED, never across a host-device synchronisation.  upload_mu serialises
  // snapshot writers (uploads, threshold rebuilds) and is taken BEFORE mu.  bounce_mu serialises
  // pageable callers of the host-buffer path (they share the pinned bounce buffers).
  std::mutex mu;
  std::mutex upload_mu;
  std::mutex bounce_mu;
  std::atomic<uint64_t> launches{0};
  lig_launch_info last_pick{};               // lig_last_pick_launch (under mu)
  void* comm = nullptr;                      // ncclComm_t, owned by lig_multi.cpp

  // ---- snapshot deltas (lig_update_snapshot): pinned + device staging of one delta ----
  unsigned char* h_delta = nullptr;
  unsigned char* d_delta = nullptr;
  size_t delta_capacity = 0;

  // ---- load feedback (lig_schedule_batch_feedback_device): a private, mutable snapshot copy ----
  std::mutex fb_mu;
  Slot fb_scratch;                            // allocated at first use
  int32_t* d_fb_hist = nullptr;               // picks per pod of the current window
  int32_t* d_fb_total = nullptr;              // picks per pod of the chain's closed windows
  int32_t* h_fb_loads = nullptr;              // pinned, mapped: the chain's loads for pageable callers
  int16_t* h_fb_rows = nullptr;               // pinned, mapped: chain fallback rows for pageable callers
                                              // (max_batch x LIG_MAX_FALLBACKS, first use, bounce_mu)
  cudaStream_t s_fb = nullptr;                // host-buffer chain calls
  cudaEvent_t fb_free = nullptr;              // the previous feedback call has finished with the scratch
  // The feedback chain (lig_schedule_batch_feedback_chain) the scratch holds between calls; all
  // of it guarded by fb_mu.  chain_live is false before the first chain call, after
  // lig_feedback_chain_reset, an in-batch feedback call or a failed chain call.
  bool chain_live = false;
  uint64_t chain_epoch = 0, chain_stamp = 0;  // the epoch copied, and its upload (Slot::stamp)
  int chain_window = 0;
  int chain_filled = 0;                       // requests in the open window
  bool chain_stale = true;                    // a window closed since the scratch's tables were built
  bool chain_has_tree = false;                // the filter tree and thresholds of the chain's start
  FilterTree chain_tree{};
  Thr chain_thr{};

  // ---- snapshots: two resident epochs ----
  Slot slot[2];
  uint64_t stamp = 0;
  cudaStream_t s_up = nullptr;               // snapshot uploads + table builds

  // ---- host-buffer batches ----
  cudaStream_t s_lane[kLanes] = {};          // also the queue streams of the per-batch mode
  int next_lane = 0;
  cudaEvent_t ticket_ev[LIG_MAX_TICKETS] = {};
  std::vector<int> free_tickets;
  lig_req* d_reqs = nullptr;                 // device staging (scan test hook)
  lig_pick* d_out = nullptr;
  uint32_t* d_masks = nullptr;               // scan test hook staging (lazily sized)
  size_t d_masks_bytes = 0;
  lig_req* h_reqs = nullptr;                 // pinned, device-mapped bounce buffers for pageable callers
  lig_pick* h_out = nullptr;

  // ---- batch queues (lig_schedule_batches_device) ----
  cudaEvent_t fork = nullptr;
  cudaEvent_t join[kLanes] = {};
  // queues longer than kMaxInlineItems carry their item table through a small pinned ring
  static constexpr int kItemSlots = 4;
  static constexpr int kMaxItems = 65535;
  QueueItem* d_items[kItemSlots] = {};
  QueueItem* h_items[kItemSlots] = {};
  cudaEvent_t items_free[kItemSlots] = {};
  int item_slot = 0;
  // tile-claim counters of the persistent kernels (TileClaim): launches on different streams may
  // run at once, so each takes the next counter of a ring; claim_free[i] is recorded after the
  // kernel that last used counter i, and claim_base[i] is that counter's value once it has finished
  static constexpr int kClaimSlots = 16;
  uint32_t* d_claims = nullptr;
  uint32_t claim_base[kClaimSlots] = {};
  cudaEvent_t claim_free[kClaimSlots] = {};
  int claim_slot = 0;

  // ---- streaming doorbell (lig_stream_open): a persistent kernel polling a host mailbox ----
  Mailbox* mailbox = nullptr;       // pinned, device-mapped
  Mailbox* d_mailbox = nullptr;     // its device alias
  cudaStream_t s_doorbell = nullptr;
  uint32_t next_ticket = 1;
  bool stream_open = false;

  // ---- tuning knobs, read from the environment at lig_create (DESIGN.md section 3) ----
  // LIG_PICK_KERNEL = tma (default: persistent CTAs fed by a TMA bulk-copy ring) | loop (persistent
  // CTAs, LDG with register prefetch) | merged (round 1: one short-lived CTA per 1024 requests)
  int pick_kernel = 0;              // 0 tma, 1 loop, 2 merged
  int tma_groups = 2;               // LIG_TMA_GROUPS = 1|2|3 consumer groups of 8 warps per CTA
  int tma_stages = 2;               // LIG_TMA_STAGES = 2|3|4|6 ring stages of 16 KB per CTA (a multiple of the groups)
  bool tma_bulk_store = false;      // LIG_TMA_BULK_STORE=1: picks leave through TMA bulk stores
  bool fast_build = true;           // LIG_FAST_BUILD=0: always the general class-build kernel
  bool tab_smem = true;             // LIG_TAB_SMEM=0: never pull the compact tables into shared memory
  int models_groups = 2;            // LIG_MODELS_GROUPS = 1|2, LIG_MODELS_STAGES = 2|4|8 (4 KB stages)
  int models_stages = 4;
  int models_grid[2] = {0, 0};      // resident CTAs of the model-request kernel: [tables in smem?]
  int persist_ctas_req = 0;         // LIG_PERSIST_CTAS: resident CTAs per SM (0 = as many as fit)
  int persist_grid[2][2] = {};      // resident CTAs of the tma variant: [bulk stores?][tables in smem?]
  int loop_grid[2] = {0, 0};        // resident CTAs of the loop kernel: [tables in smem?]
  bool host_tma = false;            // LIG_HOST_TMA=1: host-buffer batches through the TMA kernel too
  int pick_per_thread = 4;          // LIG_PICK_PER_THREAD = 1|2|4 (plain) | 8|16 (software-pipelined)
  int queue_streams = 4;            // LIG_QUEUE_STREAMS   = 1..8 streams of the per-batch mode
  // LIG_MERGE_MAX (only with LIG_PICK_KERNEL=merged): largest R whose queues run as ONE merged launch
  // (blockIdx.y = batch); above it, one kernel per batch forked over the queue streams.
  int merge_max_requests = 0x7fffffff;
};

namespace {

SnapView view_of(const Slot& s) {
  const Layout l = layout_for(s.P, s.A);
  SnapView v;
  v.kv = reinterpret_cast<const double*>(s.d_blob + l.kv);
  v.q = reinterpret_cast<const int*>(s.d_blob + l.q);
  v.n_active = reinterpret_cast<const uint16_t*>(s.d_blob + l.na);
  v.max_active = reinterpret_cast<const uint16_t*>(s.d_blob + l.ma);
  v.bitmap = reinterpret_cast<const uint32_t*>(s.d_blob + l.bitmap);
  v.P = s.P;
  v.A = s.A;
  v.W = s.W;
  return v;
}

Thr thr_of(const lig_ctx* c) {
  return Thr{c->thr.kv_cache_threshold, (long long)c->thr.queue_threshold_critical,
             (long long)c->thr.queueing_threshold_lora};
}

Slot* find_slot(lig_ctx* c, uint64_t epoch) {
  for (auto& s : c->slot)
    if (s.valid && s.epoch == epoch) return &s;
  return nullptr;
}

int resolve_slot(lig_ctx* c, uint64_t epoch, Slot** out) {
  if (!c->slot[0].valid && !c->slot[1].valid)
    return fail(LIG_ERR_NO_SNAPSHOT, "no snapshot uploaded yet");
  Slot* s = find_slot(c, epoch);
  if (!s)
    return fail(LIG_ERR_STALE_EPOCH, "epoch %llu is not resident (resident: %llu%s, %llu%s)",
                (unsigned long long)epoch, (unsigned long long)c->slot[0].epoch,
                c->slot[0].valid ? "" : " [empty]", (unsigned long long)c->slot[1].epoch,
                c->slot[1].valid ? "" : " [empty]");
  *out = s;
  return 0;
}

// A batch on `st` reads slot s: record it in the slot's reader ring (see Slot::readers).
int note_reader(Slot& s, cudaStream_t st) {
  cudaEvent_t ev = s.readers[s.next_reader];
  s.next_reader = (s.next_reader + 1) % Slot::kReaders;
  CUDA_TRY(cudaStreamWaitEvent(st, ev, 0));   // no-op unless the ring wrapped onto a live reader
  CUDA_TRY(cudaEventRecord(ev, st));
  return 0;
}

// The direct scan restates the built-in tree over every pod only: it refuses an epoch whose class
// tables a caller filter tree built (lig_read_class reads those survivor sets) or that has ejected pods.
int check_scannable(const Slot& s, uint64_t epoch) {
  if (s.caller_tree)
    return fail(LIG_ERR_INVALID, "direct scan: epoch %llu was built with a caller filter tree; the scan "
                                 "walks the built-in tree only", (unsigned long long)epoch);
  if (s.n_ejected > 0)
    return fail(LIG_ERR_INVALID, "direct scan: epoch %llu has ejected pods; the scan walks every pod",
                (unsigned long long)epoch);
  return 0;
}

// `writer` must not touch slot s before every recorded reader has finished.
int wait_readers(Slot& s, cudaStream_t writer) {
  for (cudaEvent_t ev : s.readers) CUDA_TRY(cudaStreamWaitEvent(writer, ev, 0));
  return 0;
}

// Does the tree-walking kernel stage the pod columns in shared memory for this W?
bool staged_fits(const lig_ctx* c, int W) {
  return scratch_bytes(W) + staged_bytes(W) <= c->smem_optin;
}

// Enqueue the class-table build for slot s on `stream`: the caller's filter tree when `tree` is not
// null, else the built-in tree with the thresholds *thr (null: the ctx's current ones).
int launch_class_build(lig_ctx* c, Slot& s, cudaStream_t stream, const FilterTree* tree,
                       const Thr* thr = nullptr) {
  const SnapView v = view_of(s);
  const Thr th = thr ? *thr : thr_of(c);
  const int n_classes = 2 * (s.A + 1);
  const int W = s.W > 0 ? s.W : 1;
  // an epoch with ejected pods builds from its pool (the pool forms of the three builds)
  const bool pooled = s.n_ejected > 0;
  const int n_pool = s.P - s.n_ejected;
  s.caller_tree = tree != nullptr;
  if (tree) {
    s.tree = *tree;
    // one warp per class; the pod columns go to shared memory when they fit (P up to ~12 K pods)
    const bool staged = s.P > 0 && tree_fixed_bytes(W) + staged_bytes(W) <= c->smem_optin;
    const size_t smem = tree_fixed_bytes(W) + (staged ? staged_bytes(W) : 0);
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
        &per_sm, pooled ? (staged ? lig_class_build_tree_kernel<true, true> : lig_class_build_tree_kernel<false, true>)
                        : (staged ? lig_class_build_tree_kernel<true> : lig_class_build_tree_kernel<false>),
        kCtaThreads, smem));
    int grid = (n_classes + kWarpsPerCta - 1) / kWarpsPerCta;
    if (grid > c->sm_count * (per_sm > 0 ? per_sm : 1)) grid = c->sm_count * (per_sm > 0 ? per_sm : 1);
    const CompactOut co{s.d_ctab, s.d_counters, s.ctab_pool_capacity, s.d_hdr_alias, nullptr};
    const int stride = s.P > 0 ? s.P : 1;
    if (pooled && staged)
      lig_class_build_tree_kernel<true, true><<<grid, kCtaThreads, smem, stream>>>(v, *tree, s.d_cls, s.d_lists, stride, co,
                                                                                  s.d_pool, n_pool);
    else if (pooled)
      lig_class_build_tree_kernel<false, true><<<grid, kCtaThreads, smem, stream>>>(v, *tree, s.d_cls, s.d_lists, stride, co,
                                                                                   s.d_pool, n_pool);
    else if (staged)
      lig_class_build_tree_kernel<true><<<grid, kCtaThreads, smem, stream>>>(v, *tree, s.d_cls, s.d_lists, stride, co);
    else
      lig_class_build_tree_kernel<false><<<grid, kCtaThreads, smem, stream>>>(v, *tree, s.d_cls, s.d_lists, stride, co);
    CUDA_TRY(cudaGetLastError());
    c->launches++;
    return 0;
  }
  const bool staged = s.P > 0 && build_fixed_bytes(W) + staged_bytes(W) <= c->smem_optin;
  const size_t smem = build_fixed_bytes(W) + (staged ? staged_bytes(W) : 0);
  // every CTA repeats the shared stages, so no more CTAs than needed to give each warp a couple
  // of classes, and never more than one per SM
  int grid = (n_classes + 2 * kBuildWarps - 1) / (2 * kBuildWarps);
  if (grid > c->sm_count) grid = c->sm_count;
  if (grid < 1) grid = 1;
  const int stride = s.P > 0 ? s.P : 1;
  // the pool cursor / finished-CTA counters are zero at allocation and reset by the sealing CTA
  static unsigned long long* dbg = nullptr;   // LIG_BUILD_DEBUG=1: phase stamps of the fast build
  static bool dbg_on = getenv("LIG_BUILD_DEBUG") != nullptr;
  if (dbg_on && !dbg) {
    cudaHostAlloc(reinterpret_cast<void**>(&dbg), 16 * sizeof(unsigned long long), cudaHostAllocMapped);
    memset(dbg, 0, 16 * sizeof(unsigned long long));
  }
  if (dbg_on && dbg[7]) {
    fprintf(stderr, "lig build stamps (cycles): stage %llu | own pods %llu | counts %llu | crit stages %llu | masks+shed %llu | classes %llu | seal %llu | total %llu\n",
            dbg[1] - dbg[0], dbg[2] - dbg[1], dbg[3] - dbg[2], dbg[4] - dbg[3], dbg[5] - dbg[4], dbg[6] - dbg[5], dbg[7] - dbg[6], dbg[7] - dbg[0]);
    dbg[7] = 0;
  }
  const CompactOut co{s.d_ctab, s.d_counters, s.ctab_pool_capacity, s.d_hdr_alias, dbg};
  // an empty pool takes the general build's early path (every class LIG_DROP)
  const bool fast = c->fast_build && s.P > 0 && W <= kFastMaxWords &&
                    fast_fixed_bytes(W) + staged_bytes(W) <= c->smem_optin && (!pooled || n_pool > 0);
  if (fast) {
    // pools of up to 4096 pods: register-resident shared stages, one class per warp up to
    // 8 * SMs adapters, several per warp (round-robin) beyond
    int fgrid = (n_classes + kBuildWarps - 1) / kBuildWarps;
    if (fgrid > c->sm_count) fgrid = c->sm_count;
    if (pooled)
      lig_class_build_fast_kernel<true><<<fgrid, kBuildThreads, fast_fixed_bytes(W) + staged_bytes(W), stream>>>(
          v, th, s.d_cls, s.d_lists, stride, co, s.d_pool, n_pool);
    else
      lig_class_build_fast_kernel<<<fgrid, kBuildThreads, fast_fixed_bytes(W) + staged_bytes(W), stream>>>(
          v, th, s.d_cls, s.d_lists, stride, co);
  } else if (pooled && staged) {
    lig_class_build_kernel<true, true><<<grid, kBuildThreads, smem, stream>>>(v, th, s.d_cls, s.d_lists, stride, co,
                                                                             s.d_pool, n_pool);
  } else if (pooled) {
    lig_class_build_kernel<false, true><<<grid, kBuildThreads, smem, stream>>>(v, th, s.d_cls, s.d_lists, stride, co,
                                                                              s.d_pool, n_pool);
  } else if (staged) {
    lig_class_build_kernel<true><<<grid, kBuildThreads, smem, stream>>>(v, th, s.d_cls, s.d_lists, stride, co);
  } else {
    lig_class_build_kernel<false><<<grid, kBuildThreads, smem, stream>>>(v, th, s.d_cls, s.d_lists, stride, co);
  }
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  // the sealing CTA also writes the compact blob's header to s.h_hdr (mapped host memory): the
  // host reads it once `ready` has completed to decide whether the tables go to shared memory
  return 0;
}

// One kernel, one batch, one CTA per 1024 requests (plain LDG/STG): the host-buffer path (the
// pointers may be page-locked host memory read and written over PCIe in place) and the per-batch
// queue mode.
int launch_pick(lig_ctx* c, const Slot& s, uint64_t seed, const lig_req* d_reqs, int R,
                lig_pick* d_out, cudaStream_t stream) {
  if (R == 0) return 0;
  const int4* in = reinterpret_cast<const int4*>(d_reqs);
  int2* out = reinterpret_cast<int2*>(d_out);
  const uint4* cls = reinterpret_cast<const uint4*>(s.d_cls);
  const int per_cta = kPickThreads * c->pick_per_thread;
  const int grid = (R + per_cta - 1) / per_cta;
  LIG_DISPATCH_PPT(c->pick_per_thread,
                   (lig_pick_stream_kernel<kPpt><<<grid, kPickThreads, 0, stream>>>(in, out, R, cls, s.d_lists, s.A, seed)));
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  c->last_pick = lig_launch_info{LIG_KERNEL_PLAIN, 0, 0, 0, 0, c->pick_per_thread};
  return 0;
}

struct PersistVariant {
  const void* fn = nullptr;
  int threads = 0;
  size_t smem = 0;
};

template <int kGroups, int kStages, bool kBulk, bool kTab>
PersistVariant make_variant() {
  PersistVariant v;
  v.fn = reinterpret_cast<const void*>(&lig_pick_persistent_kernel<kGroups, kStages, kBulk, kTab>);
  v.threads = persist_threads(kGroups);
  v.smem = persist_smem_bytes(kGroups, kStages, kBulk, kTab);
  return v;
}

template <int kGroups, bool kBulk, bool kTab>
PersistVariant variant_for_stages(int stages) {
  switch (stages) {
    case 2: return make_variant<kGroups, 2, kBulk, kTab>();
    case 3: return make_variant<kGroups, 3, kBulk, kTab>();
    case 6: return make_variant<kGroups, 6, kBulk, kTab>();
    default: return make_variant<kGroups, 4, kBulk, kTab>();
  }
}

template <bool kTab>
PersistVariant variant_for_groups(int groups, int stages, bool bulk) {
  switch (groups * 2 + (bulk ? 1 : 0)) {
    case 1 * 2 + 0: return variant_for_stages<1, false, kTab>(stages);
    case 1 * 2 + 1: return variant_for_stages<1, true, kTab>(stages);
    case 3 * 2 + 0: return variant_for_stages<3, false, kTab>(stages);
    case 3 * 2 + 1: return variant_for_stages<3, true, kTab>(stages);
    case 2 * 2 + 1: return variant_for_stages<2, true, kTab>(stages);
    default:        return variant_for_stages<2, false, kTab>(stages);
  }
}

PersistVariant persist_variant(int groups, int stages, bool bulk, bool tab) {
  return tab ? variant_for_groups<true>(groups, stages, bulk) : variant_for_groups<false>(groups, stages, bulk);
}

PersistVariant loop_variant(bool tab) {
  PersistVariant v;
  v.fn = tab ? reinterpret_cast<const void*>(&lig_pick_loop_kernel<true>)
             : reinterpret_cast<const void*>(&lig_pick_loop_kernel<false>);
  v.threads = kLoopThreads;
  v.smem = tab ? (size_t)kTabBudget + 16 : 0;
  return v;
}

// May the class tables (and, with_models, the model table behind them) go to shared memory?
bool tables_fit_smem(const lig_ctx* c, const Slot& s, bool with_models) {
  if (!c->tab_smem) return false;
  const bool done = cudaEventQuery(s.ready) == cudaSuccess;
  cudaGetLastError();   // cudaErrorNotReady is not an error
  if (!done || s.h_hdr->bytes == 0 || s.h_hdr->n_classes != 2u * (uint32_t)(s.A + 1)) return false;
  const size_t need = (size_t)s.h_hdr->bytes + (with_models ? (size_t)s.mtab_bytes : 0);
  return need <= kTabBudget;
}

// Launch persistent kernel v (its last argument, *tc, is filled in here) with the next tile-claim
// counter of the ring.  On the device the launch first waits for the counter's previous kernel,
// whose claims the counter's base already counts.  Caller holds c->mu.
int launch_claimed(lig_ctx* c, const PersistVariant& v, int grid, int total_tiles, void** args, TileClaim* tc,
                   cudaStream_t st) {
  const int k = c->claim_slot;
  c->claim_slot = (k + 1) % lig_ctx::kClaimSlots;
  CUDA_TRY(cudaStreamWaitEvent(st, c->claim_free[k], 0));   // no-op unless the ring wrapped onto a live launch
  *tc = TileClaim{c->d_claims + k, c->claim_base[k]};
  CUDA_TRY(cudaLaunchKernel(v.fn, dim3((unsigned)grid), dim3((unsigned)v.threads), args, v.smem, st));
  c->claim_base[k] += (uint32_t)total_tiles + (uint32_t)grid;   // every CTA's producer fails one claim
  CUDA_TRY(cudaEventRecord(c->claim_free[k], st));
  return 0;
}

// The persistent TMA-pipelined pick over a queue of n batches of R requests (one launch per
// <= 2^30 tiles).  Caller holds c->mu.
int launch_persistent(lig_ctx* c, const Slot& s, uint64_t seed, const lig_req* const* reqs, int R,
                      lig_pick* const* outs, int n_batches, cudaStream_t st) {
  if (R == 0 || n_batches == 0) return 0;
  const uint4* cls = reinterpret_cast<const uint4*>(s.d_cls);
  const int tile = c->pick_kernel == 1 ? kLoopTile : kTile;
  const int tpb = (R + tile - 1) / tile;
  // the compact tables go to shared memory when their header is back (the build has completed)
  // and they fit the budget; otherwise the strided tables are read through L1 (same results)
  const bool tab = tables_fit_smem(c, s, false);
  int per_launch = (1 << 30) / tpb;
  if (per_launch > lig_ctx::kMaxItems) per_launch = lig_ctx::kMaxItems;
  if (per_launch < 1) per_launch = 1;
  for (int lo = 0; lo < n_batches; lo += per_launch) {
    const int n = (n_batches - lo) < per_launch ? (n_batches - lo) : per_launch;
    QueueParams qp;
    qp.n_batches = n;
    qp.R = R;
    qp.tiles_per_batch = tpb;
    qp.total_tiles = n * tpb;
    qp.dev_items = nullptr;
    bool aligned = true;   // TMA bulk stores need 16-byte aligned pick buffers (the ABI asks for 8)
    for (int b = 0; b < n; ++b)
      if (reinterpret_cast<uintptr_t>(outs[lo + b]) & 15u) aligned = false;
    int slot = -1;
    if (n <= kMaxInlineItems) {
      for (int b = 0; b < n; ++b)
        qp.items[b] = QueueItem{reinterpret_cast<const int4*>(reqs[lo + b]),
                                reinterpret_cast<int2*>(outs[lo + b]), seed + (uint64_t)(lo + b)};
    } else {
      slot = c->item_slot;
      c->item_slot = (slot + 1) % lig_ctx::kItemSlots;
      CUDA_TRY(cudaEventSynchronize(c->items_free[slot]));   // the kernel of 4 long queues ago is done
      for (int b = 0; b < n; ++b)
        c->h_items[slot][b] = QueueItem{reinterpret_cast<const int4*>(reqs[lo + b]),
                                        reinterpret_cast<int2*>(outs[lo + b]), seed + (uint64_t)(lo + b)};
      CUDA_TRY(cudaMemcpyAsync(c->d_items[slot], c->h_items[slot], sizeof(QueueItem) * (size_t)n,
                               cudaMemcpyHostToDevice, st));
      qp.dev_items = c->d_items[slot];
    }
    const uint16_t* lists = s.d_lists;
    int A = s.A;
    const unsigned char* ctab = s.d_ctab;
    uint32_t ctab_bytes = tab ? s.h_hdr->bytes : 0u;
    TileClaim tc{};
    void* args[7] = {&qp, &cls, &lists, &A, &ctab, &ctab_bytes, &tc};
    if (c->pick_kernel == 1) {
      const PersistVariant v = loop_variant(tab);
      const int cap = c->loop_grid[tab ? 1 : 0];
      const int grid = qp.total_tiles < cap ? qp.total_tiles : cap;
      CUDA_TRY(cudaLaunchKernel(v.fn, dim3((unsigned)grid), dim3((unsigned)v.threads), args, v.smem, st));
      c->last_pick = lig_launch_info{LIG_KERNEL_LOOP, 0, 0, 0, tab ? 1 : 0, 0};
    } else {
      const bool bulk = c->tma_bulk_store && aligned;
      const PersistVariant v = persist_variant(c->tma_groups, c->tma_stages, bulk, tab);
      const int cap = c->persist_grid[bulk ? 1 : 0][tab ? 1 : 0];
      const int grid = qp.total_tiles < cap ? qp.total_tiles : cap;
      if (int rc = launch_claimed(c, v, grid, qp.total_tiles, args, &tc, st)) return rc;
      c->last_pick = lig_launch_info{LIG_KERNEL_PERSISTENT, c->tma_groups, c->tma_stages, bulk ? 1 : 0, tab ? 1 : 0, 0};
    }
    c->launches++;
    if (slot >= 0) CUDA_TRY(cudaEventRecord(c->items_free[slot], st));   // after the kernel that reads the table
  }
  return 0;
}

template <int kGroups, bool kTab>
PersistVariant mvariant_for_stages(int stages) {
  PersistVariant v;
  v.threads = persist_threads(kGroups);
  switch (stages) {
    case 2: v.fn = reinterpret_cast<const void*>(&lig_pick_models_kernel<kGroups, 2, kTab>); v.smem = mpersist_smem_bytes(2, kTab); break;
    case 8: v.fn = reinterpret_cast<const void*>(&lig_pick_models_kernel<kGroups, 8, kTab>); v.smem = mpersist_smem_bytes(8, kTab); break;
    default: v.fn = reinterpret_cast<const void*>(&lig_pick_models_kernel<kGroups, 4, kTab>); v.smem = mpersist_smem_bytes(4, kTab); break;
  }
  return v;
}

PersistVariant models_variant(int groups, int stages, bool tab) {
  if (groups == 1) return tab ? mvariant_for_stages<1, true>(stages) : mvariant_for_stages<1, false>(stages);
  return tab ? mvariant_for_stages<2, true>(stages) : mvariant_for_stages<2, false>(stages);
}

// Model-id batches against slot s (caller holds c->mu and has checked s.models_valid).
int launch_models(lig_ctx* c, const Slot& s, uint64_t seed, uint64_t first_index,
                  const uint32_t* const* ids, int R, lig_mpick* const* outs, int n_batches,
                  cudaStream_t st, bool allow_persistent) {
  if (R == 0 || n_batches == 0) return 0;
  const uint4* cls = reinterpret_cast<const uint4*>(s.d_cls);
  const uint16_t* lists = s.d_lists;
  int A = s.A;
  bool aligned = (R % 4) == 0;
  for (int b = 0; b < n_batches; ++b)
    if ((reinterpret_cast<uintptr_t>(ids[b]) | reinterpret_cast<uintptr_t>(outs[b])) & 15u) aligned = false;
  if (!allow_persistent || !aligned || c->pick_kernel == 2) {
    // plain kernel, one launch per batch (host-mapped buffers, odd sizes or alignments)
    const unsigned char* mtab = s.d_mtab;
    for (int b = 0; b < n_batches; ++b) {
      lig_pick_models_stream_kernel<<<(R + kTile - 1) / kTile, kGroupThreads, 0, st>>>(
          ids[b], reinterpret_cast<uint32_t*>(outs[b]), R, cls, lists, A, mtab, s.n_models,
          seed + (uint64_t)b, first_index, nullptr);
      CUDA_TRY(cudaGetLastError());
      c->launches++;
      c->last_pick = lig_launch_info{LIG_KERNEL_MODELS_PLAIN, 0, 0, 0, 0, 0};
    }
    return 0;
  }
  const bool tab = tables_fit_smem(c, s, true);
  const int tpb = (R + kTile - 1) / kTile;
  int per_launch = (1 << 30) / tpb;
  if (per_launch > kMaxInlineMItems) per_launch = kMaxInlineMItems;   // longer queues: several launches
  for (int lo = 0; lo < n_batches; lo += per_launch) {
    const int n = (n_batches - lo) < per_launch ? (n_batches - lo) : per_launch;
    MQueueParams qp;
    qp.n_batches = n;
    qp.R = R;
    qp.tiles_per_batch = tpb;
    qp.total_tiles = n * tpb;
    qp.dev_items = nullptr;
    for (int b = 0; b < n; ++b)
      qp.items[b] = MQueueItem{ids[lo + b], reinterpret_cast<uint32_t*>(outs[lo + b]), seed + (uint64_t)(lo + b), first_index};
    const unsigned char* ctab = s.d_ctab;
    uint32_t ctab_bytes = tab ? s.h_hdr->bytes : 0u;
    const unsigned char* mtab = s.d_mtab;
    uint32_t mtab_bytes = s.mtab_bytes, n_models = s.n_models;
    TileClaim tc{};
    void* args[10] = {&qp, &cls, &lists, &A, &ctab, &ctab_bytes, &mtab, &mtab_bytes, &n_models, &tc};
    const PersistVariant v = models_variant(c->models_groups, c->models_stages, tab);
    const int cap = c->models_grid[tab ? 1 : 0];
    const int grid = qp.total_tiles < cap ? qp.total_tiles : cap;
    if (int rc = launch_claimed(c, v, grid, qp.total_tiles, args, &tc, st)) return rc;
    c->launches++;
    c->last_pick = lig_launch_info{LIG_KERNEL_MODELS, c->models_groups, c->models_stages, 0, tab ? 1 : 0, 0};
  }
  return 0;
}

// The launch shape of the per-request walks (the direct scan and the retry walk) over R >= 1
// requests of slot s: one warp per request, the pod columns staged in shared memory when they fit.
struct ScanShape {
  bool staged;
  size_t smem;
  int grid;
};

static ScanShape scan_shape(const lig_ctx* c, const Slot& s, int R) {
  ScanShape sh;
  sh.staged = s.P > 0 && staged_fits(c, s.W);
  sh.smem = scratch_bytes(s.W > 0 ? s.W : 1) + (sh.staged ? staged_bytes(s.W) : 0);
  const int ctas_per_sm = sh.staged ? (sh.smem > 110 * 1024 ? 1 : 2) : 4;
  const int ctas_needed = (R + kWarpsPerCta - 1) / kWarpsPerCta;
  sh.grid = ctas_needed < c->sm_count * ctas_per_sm ? ctas_needed : c->sm_count * ctas_per_sm;
  return sh;
}

int launch_scan(lig_ctx* c, const Slot& s, uint64_t seed, const lig_req* d_reqs, int R,
                lig_pick* d_out, uint32_t* d_masks, cudaStream_t stream) {
  if (R == 0) return 0;
  const SnapView v = view_of(s);
  const ScanShape sh = scan_shape(c, s, R);
  if (sh.staged) {
    lig_scan_kernel<true><<<sh.grid, kCtaThreads, sh.smem, stream>>>(
        v, thr_of(c), reinterpret_cast<const int4*>(d_reqs), reinterpret_cast<int2*>(d_out), R,
        d_masks, seed);
  } else {
    lig_scan_kernel<false><<<sh.grid, kCtaThreads, sh.smem, stream>>>(
        v, thr_of(c), reinterpret_cast<const int4*>(d_reqs), reinterpret_cast<int2*>(d_out), R,
        d_masks, seed);
  }
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  return 0;
}

// Pick the slot a new epoch overwrites: the one already holding that epoch, else an empty one,
// else the older of the two.
Slot& victim_slot(lig_ctx* c, uint64_t epoch) {
  if (Slot* s = find_slot(c, epoch)) return *s;
  if (!c->slot[0].valid) return c->slot[0];
  if (!c->slot[1].valid) return c->slot[1];
  return c->slot[0].stamp <= c->slot[1].stamp ? c->slot[0] : c->slot[1];
}

int check_shape(const lig_ctx* c, int P, int A) {
  if (P < 0 || P > c->max_pods)
    return fail(LIG_ERR_INVALID, "P=%d outside [0, max_pods=%d]", P, c->max_pods);
  if (A < 0 || A > c->max_adapters)
    return fail(LIG_ERR_INVALID, "A=%d outside [0, max_adapters=%d]", A, c->max_adapters);
  return 0;
}

// Scoped "allocate on the GPU's NUMA node" memory policy for the calling thread.
struct NumaBind {
  bool active = false;
  int old_mode = 0;
  unsigned long old_mask[16] = {0};
  NumaBind() {
    const char* env = getenv("LIG_NUMA");
    if (env && atoi(env) == 0) return;
    int dev = 0;
    char bus[32] = "";
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetPCIBusId(bus, sizeof(bus), dev) != cudaSuccess) {
      cudaGetLastError();
      return;
    }
    for (char* q = bus; *q; ++q) *q = (char)tolower((unsigned char)*q);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0 || node >= 1024) return;
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    // the calling thread's own policy (numactl, an embedding runtime) is put back afterwards
    if (syscall(SYS_get_mempolicy, &old_mode, old_mask, sizeof(old_mask) * 8, nullptr, 0) != 0) return;
    // MPOL_PREFERRED = 1: fall back to other nodes rather than fail when the node is full
    active = syscall(SYS_set_mempolicy, 1, mask, sizeof(mask) * 8) == 0;
  }
  ~NumaBind() {
    if (!active) return;
    if (old_mode == 0)
      syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
    else
      syscall(SYS_set_mempolicy, old_mode, old_mask, sizeof(old_mask) * 8);
  }
};

// Ranges handed out by lig_host_alloc (and the ctx's own staging buffers): known to be pinned and
// device-mapped, so the per-call driver query below can be skipped for them.
struct PinnedRange { const char* base; size_t bytes; char* dev; };
std::mutex g_pinned_mu;
std::vector<PinnedRange> g_pinned;

void register_pinned(void* host, size_t bytes) {
  void* dev = nullptr;
  if (cudaHostGetDevicePointer(&dev, host, 0) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  std::lock_guard<std::mutex> lk(g_pinned_mu);
  g_pinned.push_back(PinnedRange{static_cast<const char*>(host), bytes, static_cast<char*>(dev)});
}

void unregister_pinned(void* host) {
  std::lock_guard<std::mutex> lk(g_pinned_mu);
  for (size_t i = 0; i < g_pinned.size(); ++i)
    if (g_pinned[i].base == host) {
      g_pinned.erase(g_pinned.begin() + (long)i);
      return;
    }
}

// Device-visible alias of a page-locked host pointer (identical under UVA), or nullptr when p is
// ordinary pageable memory.
template <typename T>
T* mapped_device_pointer(T* p) {
  {
    const char* q = reinterpret_cast<const char*>(p);
    std::lock_guard<std::mutex> lk(g_pinned_mu);
    for (const PinnedRange& r : g_pinned)
      if (q >= r.base && q < r.base + r.bytes)
        return reinterpret_cast<T*>(r.dev + (q - r.base));
  }
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (at.type != cudaMemoryTypeHost || !at.devicePointer) return nullptr;
  return reinterpret_cast<T*>(at.devicePointer);
}

// Every pick kernel reads a request with one 16-byte load (the TMA ring in 16-byte aligned tiles),
// but lig_req itself is only 8-byte aligned: a host request array at an odd 8 bytes is staged
// through the ctx's aligned bounce buffer (lig_schedule_batch) or refused (the async form).
bool req_aligned(const lig_req* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Enqueue one host-buffer batch (device-visible pointers) on a lane and hand back a ticket.
// Caller holds c->mu.
int submit_mapped(lig_ctx* c, Slot* s, uint64_t seed, const lig_req* dev_in, int R, lig_pick* dev_out,
                  int* ticket) {
  if (c->free_tickets.empty())
    return fail(LIG_ERR_BUSY, "all %d tickets are in flight: call lig_schedule_wait first", LIG_MAX_TICKETS);
  const int lane = c->next_lane;
  c->next_lane = (lane + 1) % kLanes;
  cudaStream_t st = c->s_lane[lane];
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  if (c->host_tma) {
    if (int rc = launch_persistent(c, *s, seed, &dev_in, R, &dev_out, 1, st)) return rc;
  } else {
    if (int rc = launch_pick(c, *s, seed, dev_in, R, dev_out, st)) return rc;
  }
  if (int rc = note_reader(*s, st)) return rc;
  const int t = c->free_tickets.back();
  CUDA_TRY(cudaEventRecord(c->ticket_ev[t], st));
  c->free_tickets.pop_back();
  *ticket = t;
  return 0;
}

// n_active of a pod record: len(ActiveModels) <= LIG_MAX_ADAPTERS (a uint16 can hold 65535, which
// beside a saturated MaxActiveModels of 65535 would read as "no room").
int check_n_active(const uint16_t* na, int n) {
  for (int i = 0; i < n; ++i)
    if (na[i] > LIG_MAX_ADAPTERS)
      return fail(LIG_ERR_RANGE, "pod record %d: n_active %u outside [0, %d]", i, (unsigned)na[i], LIG_MAX_ADAPTERS);
  return 0;
}

// The host arrays of a snapshot pack.  Host uploads call this before begin_write, so a refused
// upload evicts no resident epoch and no model table.
int check_snapshot_arrays(int P, int A, const double* kv, const int32_t* q, const uint16_t* na,
                          const uint16_t* ma, const uint32_t* bitmap) {
  if (P < 0 || A < 0) return fail(LIG_ERR_INVALID, "snapshot shape P=%d A=%d", P, A);
  if (P > 0 && (!kv || !q || !na || !ma)) return fail(LIG_ERR_INVALID, "null pod column");
  if (A > 0 && P > 0 && !bitmap) return fail(LIG_ERR_INVALID, "null bitmap");
  return check_n_active(na, P);
}

// Lay checked host arrays out as the packed blob (lig.h).
void pack_blob(void* blob, int P, int A, const double* kv, const int32_t* q, const uint16_t* na,
               const uint16_t* ma, const uint32_t* bitmap) {
  const Layout l = layout_for(P, A);
  unsigned char* b = static_cast<unsigned char*>(blob);
  if (P == 0) {
    memset(b, 0, l.total);
    return;
  }
  // copy the P real pods and zero only the padding pods of each column (no full-blob memset)
  const size_t pad = (size_t)words_for(P) * 32 - (size_t)P;
  memcpy(b + l.kv, kv, (size_t)P * sizeof(double));
  memset(b + l.kv + (size_t)P * sizeof(double), 0, pad * sizeof(double));
  memcpy(b + l.q, q, (size_t)P * sizeof(int32_t));
  memset(b + l.q + (size_t)P * sizeof(int32_t), 0, pad * sizeof(int32_t));
  memcpy(b + l.na, na, (size_t)P * sizeof(uint16_t));
  memset(b + l.na + (size_t)P * sizeof(uint16_t), 0, pad * sizeof(uint16_t));
  memcpy(b + l.ma, ma, (size_t)P * sizeof(uint16_t));
  memset(b + l.ma + (size_t)P * sizeof(uint16_t), 0, pad * sizeof(uint16_t));
  const size_t bm_bytes = (size_t)A * words_for(P) * sizeof(uint32_t);
  if (A > 0) memcpy(b + l.bitmap, bitmap, bm_bytes);
  memset(b + l.bitmap + bm_bytes, 0, l.total - l.bitmap - bm_bytes);
  // bits of padding pods must be clear in the last word of every row
  const int W = words_for(P), rem = P & 31;
  if (rem) {
    uint32_t* bm = reinterpret_cast<uint32_t*>(b + l.bitmap);
    const uint32_t keep = (1u << rem) - 1u;
    for (int a = 0; a < A; ++a) bm[(size_t)a * W + (W - 1)] &= keep;
  }
}

}  // namespace

// ---- snapshot-writer protocol (lig_internal.hpp) ----------------------------------------------------
namespace ligi {

int device_of(const lig_ctx* c) { return c->device; }
int max_batch_of(const lig_ctx* c) { return c->max_batch; }
void*& comm_of(lig_ctx* c) { return c->comm; }
static void (*g_comm_destructor)(void*) = nullptr;
void set_comm_destructor(void (*fn)(void*)) { g_comm_destructor = fn; }
static allreduce_fn g_allreduce = nullptr;
void set_allreduce(allreduce_fn fn) { g_allreduce = fn; }

int check_filter_tree(const lig_filter_node* nodes, int n_nodes) {
  if (!nodes && n_nodes == 0) return 0;   // back to the built-in tree
  if (!nodes || n_nodes < 1 || n_nodes > LIG_MAX_FILTER_NODES)
    return fail(LIG_ERR_INVALID, "filter tree: %d nodes (1..%d, or NULL and 0 for the built-in tree)",
                n_nodes, LIG_MAX_FILTER_NODES);
  for (int i = 0; i < n_nodes; ++i) {
    const lig_filter_node& nd = nodes[i];
    if (nd.kind < LIG_F_CRITICAL_REQUEST || nd.kind > LIG_F_DROP)
      return fail(LIG_ERR_INVALID, "filter tree: node %d has unknown kind %d", i, nd.kind);
    const int32_t next[3] = {nd.next_on_success, nd.next_on_failure, nd.next_on_success_or_failure};
    for (int32_t j : next)
      if (j != -1 && (j <= i || j >= n_nodes))
        return fail(LIG_ERR_INVALID, "filter tree: node %d links to %d (successors are -1 or in (%d, %d))",
                    i, j, i, n_nodes);
  }
  return 0;
}

int begin_write(lig_ctx* c, uint64_t epoch, int P, int A, cudaStream_t stream, bool own_stream,
                SnapshotWrite* w) {
  if (int rc = check_shape(c, P, A)) return rc;
  c->upload_mu.lock();
  cudaError_t e = cudaSetDevice(c->device);
  if (e != cudaSuccess) {
    c->upload_mu.unlock();
    return fail(LIG_ERR_CUDA, "cudaSetDevice(%d) failed: %s", c->device, cudaGetErrorString(e));
  }
  cudaStream_t st = own_stream ? c->s_up : stream;
  int rc = 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot& s = victim_slot(c, epoch);
    s.valid = false;                       // evicted: schedule calls on its old epoch now get STALE_EPOCH
    s.models_valid = false;                // the model table is interned against the old snapshot
    s.keys_valid = false;                  // and the pod keys name the old snapshot's pods
    s.n_ejected = 0;                       // full uploads start with every pod; lig_update_snapshot and
                                           // lig_eject_pods set the set after begin_write
    rc = wait_readers(s, st);              // batches still reading the old content
    if (!rc && cudaStreamWaitEvent(st, s.ready, 0) != cudaSuccess)   // an earlier device-side upload of this slot
      rc = fail(LIG_ERR_CUDA, "cudaStreamWaitEvent failed");
    s.P = P;
    s.A = A;
    s.W = words_for(P);
    w->slot = &s;
    w->d_blob = s.d_blob;
    w->h_blob = s.h_blob;
  }
  if (!rc && own_stream) {
    // Host-staged writers fill the slot's pinned blob next: an earlier _async upload of this slot
    // (two epochs ago) may still be copying out of it.  Waiting for the slot's `ready` is a no-op
    // when that upload completed long ago (the normal case); the ctx lock is not held here.
    cudaError_t e = cudaEventSynchronize(static_cast<Slot*>(w->slot)->ready);
    if (e != cudaSuccess) rc = fail(LIG_ERR_CUDA, "an earlier upload of this slot failed: %s", cudaGetErrorString(e));
  }
  if (rc) {
    c->upload_mu.unlock();
    return rc;
  }
  w->bytes = layout_for(P, A).total;
  w->P = P;
  w->A = A;
  w->epoch = epoch;
  w->stream = st;
  return 0;
}

int enqueue_build(lig_ctx* c, SnapshotWrite* w) {
  Slot& s = *static_cast<Slot*>(w->slot);
  CUDA_TRY(cudaSetDevice(c->device));
  if (int rc = launch_class_build(c, s, w->stream, c->has_tree ? &c->tree : nullptr)) return rc;
  CUDA_TRY(cudaEventRecord(s.ready, w->stream));
  return 0;
}

int finish_write(lig_ctx* c, SnapshotWrite* w, bool synchronise) {
  Slot& s = *static_cast<Slot*>(w->slot);
  int rc = 0;
  if (synchronise) {
    cudaSetDevice(c->device);
    cudaError_t e = cudaStreamSynchronize(w->stream);
    if (e != cudaSuccess) rc = fail(LIG_ERR_CUDA, "snapshot upload failed: %s", cudaGetErrorString(e));
  }
  if (!rc) {
    std::lock_guard<std::mutex> lk(c->mu);
    s.epoch = w->epoch;
    s.stamp = ++c->stamp;
    s.valid = true;
  }
  c->upload_mu.unlock();
  return rc;
}

void abort_write(lig_ctx* c, SnapshotWrite*) { c->upload_mu.unlock(); }

}  // namespace ligi

// The dynamic shared-memory limit of every form of the retry kernel: form I has kModels = bit 0,
// kStaged = bit 1, kTree = bit 2, kPool = bit 3, kRows = bit 4, kCount = bit 5.
template <size_t... I>
static int set_excluding_smem(int bytes, std::index_sequence<I...>) {
  const void* forms[] = {(const void*)lig_schedule_excluding_kernel<(I & 1) != 0, (I & 2) != 0, (I & 4) != 0,
                                                                    (I & 8) != 0, (I & 16) != 0, (I & 32) != 0>...};
  for (const void* fn : forms) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return 0;
}

extern "C" {

const char* lig_last_error(void) { return g_err; }
const char* lig_version(void) { return "lig-b200 0.2 (sm_90a)"; }
int lig_abi_version(void) { return LIG_ABI_VERSION; }

int lig_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

size_t lig_snapshot_bytes(int P, int A) {
  if (P < 0 || A < 0) return 0;
  return layout_for(P, A).total;
}

int lig_pack_pods(int P, const int64_t* q, const int64_t* na, const int64_t* ma, int32_t* q_out,
                  uint16_t* na_out, uint16_t* ma_out) {
  if (P < 0 || (P > 0 && (!q || !na || !ma || !q_out || !na_out || !ma_out)))
    return fail(LIG_ERR_INVALID, "lig_pack_pods: null array");
  for (int i = 0; i < P; ++i) {
    if (q[i] < INT32_MIN || q[i] > INT32_MAX)
      return fail(LIG_ERR_RANGE, "pod %d: WaitingQueueSize %lld does not fit int32", i,
                  (long long)q[i]);
    if (na[i] < 0 || na[i] > LIG_MAX_ADAPTERS)
      return fail(LIG_ERR_RANGE, "pod %d: len(ActiveModels) %lld outside [0, %d]", i,
                  (long long)na[i], LIG_MAX_ADAPTERS);
    q_out[i] = (int32_t)q[i];
    na_out[i] = (uint16_t)na[i];
    ma_out[i] = (uint16_t)(ma[i] < 0 ? 0 : (ma[i] > 65535 ? 65535 : ma[i]));
  }
  return 0;
}

int lig_pack_snapshot(void* blob, int P, int A, const double* kv, const int32_t* q,
                      const uint16_t* na, const uint16_t* ma, const uint32_t* bitmap) {
  if (!blob) return fail(LIG_ERR_INVALID, "lig_pack_snapshot: null blob");
  if (int rc = check_snapshot_arrays(P, A, kv, q, na, ma, bitmap)) return rc;
  pack_blob(blob, P, A, kv, q, na, ma, bitmap);
  return 0;
}

// HBM + pinned memory + events of one snapshot slot (the two resident epochs and, lazily, the
// private scratch copy of the load-feedback mode).
static int alloc_slot(lig_ctx* c, Slot& s) {
  const Layout l = layout_for(c->max_pods, c->max_adapters);
  const size_t n_classes = 2 * ((size_t)c->max_adapters + 1);
  CUDA_TRY(cudaMalloc(&s.d_blob, l.total));
  CUDA_TRY(cudaMalloc(&s.d_cls, n_classes * sizeof(ClassEntry)));
  CUDA_TRY(cudaMalloc(&s.d_lists, list_pool_entries(n_classes, (size_t)c->max_pods) * sizeof(uint16_t)));
  {
    // the compact pool holds the two default lists plus up to 2 M more entries (4 MB); a
    // snapshot whose lists do not fit keeps the strided tables only
    size_t cap = list_pool_entries(n_classes, (size_t)c->max_pods);
    const size_t bound = 2 * (size_t)c->max_pods + 16 + ((size_t)2 << 20);
    if (cap > bound) cap = bound;
    s.ctab_pool_capacity = (uint32_t)cap;
    CUDA_TRY(cudaMalloc(&s.d_ctab, sizeof(CompactHeader) + n_classes * sizeof(ClassEntry) + cap * sizeof(uint16_t) + 16));
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&s.h_hdr), sizeof(CompactHeader), cudaHostAllocMapped));
    memset(s.h_hdr, 0, sizeof(CompactHeader));
    CUDA_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(&s.d_hdr_alias), s.h_hdr, 0));
    CUDA_TRY(cudaMalloc(&s.d_counters, 2 * sizeof(uint32_t)));
    CUDA_TRY(cudaMemset(s.d_counters, 0, 2 * sizeof(uint32_t)));
  }
  CUDA_TRY(cudaMalloc(&s.d_pool, (size_t)(words_for(c->max_pods) > 0 ? words_for(c->max_pods) : 1) * sizeof(uint32_t)));
  CUDA_TRY(cudaHostAlloc(&s.h_blob, l.total, cudaHostAllocDefault));
  CUDA_TRY(cudaEventCreateWithFlags(&s.ready, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&s.models_ready, cudaEventDisableTiming));
  CUDA_TRY(cudaMalloc(&s.d_podkeys, (size_t)c->max_pods * sizeof(uint64_t)));
  CUDA_TRY(cudaHostAlloc(&s.h_podkeys, (size_t)c->max_pods * sizeof(uint64_t), cudaHostAllocDefault));
  CUDA_TRY(cudaEventCreateWithFlags(&s.keys_ready, cudaEventDisableTiming));
  for (auto& ev : s.readers) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  return 0;
}

static void free_slot(Slot& s) {
  cudaFree(s.d_blob);
  cudaFree(s.d_cls);
  cudaFree(s.d_lists);
  cudaFree(s.d_ctab);
  cudaFree(s.d_counters);
  cudaFree(s.d_pool);
  cudaFree(s.d_mtab);
  if (s.h_mtab) cudaFreeHost(s.h_mtab);
  if (s.models_ready) cudaEventDestroy(s.models_ready);
  cudaFree(s.d_podkeys);
  if (s.h_podkeys) cudaFreeHost(s.h_podkeys);
  if (s.keys_ready) cudaEventDestroy(s.keys_ready);
  if (s.h_hdr) cudaFreeHost(s.h_hdr);
  cudaFreeHost(s.h_blob);
  if (s.ready) cudaEventDestroy(s.ready);
  for (auto& ev : s.readers)
    if (ev) cudaEventDestroy(ev);
  s = Slot();
}

static int create_impl(lig_ctx* c, int device, int max_pods, int max_adapters, int max_batch) {
  CUDA_TRY(cudaSetDevice(device));
  c->device = device;
  c->max_pods = max_pods;
  c->max_adapters = max_adapters;
  c->max_batch = max_batch;
  int v = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device));
  c->sm_count = v;
  CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  c->smem_optin = (size_t)v;
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_kernel<true>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_kernel<false>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_fast_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_tree_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_tree_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  // the pool forms (epochs derived by lig_eject_pods)
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_fast_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_tree_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_class_build_tree_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_scan_kernel<true>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  CUDA_TRY(cudaFuncSetAttribute(lig_scan_kernel<false>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, v));
  if (int rc = set_excluding_smem(v, std::make_index_sequence<64>{})) return rc;
  const size_t need = scratch_bytes(words_for(max_pods)) > build_fixed_bytes(words_for(max_pods))
                          ? scratch_bytes(words_for(max_pods)) : build_fixed_bytes(words_for(max_pods));
  if (need > c->smem_optin)
    return fail(LIG_ERR_INVALID, "max_pods=%d needs %zu B of per-CTA scratch, device allows %zu",
                max_pods, need, c->smem_optin);
  for (auto& s : c->slot)
    if (int rc = alloc_slot(c, s)) return rc;
  if (const char* e = getenv("LIG_PICK_PER_THREAD")) {
    int v2 = atoi(e);
    if (v2 == 1 || v2 == 2 || v2 == 4 || v2 == 8 || v2 == 16) c->pick_per_thread = v2;
  }
  if (const char* e = getenv("LIG_PICK_KERNEL")) {
    if (!strcmp(e, "loop")) c->pick_kernel = 1;
    else if (!strcmp(e, "merged")) c->pick_kernel = 2;
    else c->pick_kernel = 0;
  }
  if (const char* e = getenv("LIG_HOST_TMA")) c->host_tma = atoi(e) != 0;
  if (const char* e = getenv("LIG_TMA_GROUPS")) {
    int v2 = atoi(e);
    if (v2 >= 1 && v2 <= 3) c->tma_groups = v2;
  }
  if (const char* e = getenv("LIG_TMA_STAGES")) {
    int v2 = atoi(e);
    if (v2 == 2 || v2 == 3 || v2 == 4 || v2 == 6) c->tma_stages = v2;
  }
  if (const char* e = getenv("LIG_TMA_BULK_STORE")) c->tma_bulk_store = atoi(e) != 0;
  if (const char* e = getenv("LIG_TAB_SMEM")) c->tab_smem = atoi(e) != 0;
  if (const char* e = getenv("LIG_FAST_BUILD")) c->fast_build = atoi(e) != 0;
  if (const char* e = getenv("LIG_MODELS_GROUPS")) {
    int v2 = atoi(e);
    if (v2 == 1 || v2 == 2) c->models_groups = v2;
  }
  if (const char* e = getenv("LIG_MODELS_STAGES")) {
    int v2 = atoi(e);
    if (v2 == 2 || v2 == 4 || v2 == 8) c->models_stages = v2;
  }
  // A consumer group may only wait on a ring stage whose previous phase it consumed itself (an
  // mbarrier parity wait cannot tell "two phases ahead" from "done"): the stage count must be a
  // multiple of the group count, so that a group always returns to the same stages.
  if (c->tma_stages % c->tma_groups != 0) {
    static const int ok[4][4] = {{0, 0, 0, 0}, {2, 3, 4, 6}, {2, 4, 4, 6}, {3, 3, 6, 6}};
    const int idx = c->tma_stages == 2 ? 0 : c->tma_stages == 3 ? 1 : c->tma_stages == 4 ? 2 : 3;
    c->tma_stages = ok[c->tma_groups][idx];
  }
  if (const char* e = getenv("LIG_PERSIST_CTAS")) c->persist_ctas_req = atoi(e);
  if (const char* e = getenv("LIG_MERGE_MAX")) c->merge_max_requests = atoi(e);
  if (const char* e = getenv("LIG_QUEUE_STREAMS")) {
    int v2 = atoi(e);
    if (v2 >= 1 && v2 <= kLanes) c->queue_streams = v2;
  }
  for (int bulk = 0; bulk < 2; ++bulk)
    for (int tab = 0; tab < 2; ++tab) {
      const PersistVariant pv = persist_variant(c->tma_groups, c->tma_stages, bulk != 0, tab != 0);
      CUDA_TRY(cudaFuncSetAttribute(pv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pv.smem));
      int per_sm = 0;
      CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pv.fn, pv.threads, pv.smem));
      if (per_sm < 1) return fail(LIG_ERR_CUDA, "the persistent pick kernel does not fit on this device");
      if (c->persist_ctas_req > 0 && c->persist_ctas_req < per_sm) per_sm = c->persist_ctas_req;
      c->persist_grid[bulk][tab] = per_sm * c->sm_count;
    }
  for (int tab = 0; tab < 2; ++tab) {
    const PersistVariant pv = models_variant(c->models_groups, c->models_stages, tab != 0);
    CUDA_TRY(cudaFuncSetAttribute(pv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pv.smem));
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pv.fn, pv.threads, pv.smem));
    if (per_sm < 1) return fail(LIG_ERR_CUDA, "the model-request kernel does not fit on this device");
    if (c->persist_ctas_req > 0 && c->persist_ctas_req < per_sm) per_sm = c->persist_ctas_req;
    c->models_grid[tab] = per_sm * c->sm_count;
  }
  for (int tab = 0; tab < 2; ++tab) {
    const PersistVariant pv = loop_variant(tab != 0);
    CUDA_TRY(cudaFuncSetAttribute(pv.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(pv.smem ? pv.smem : 16)));
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pv.fn, pv.threads, pv.smem));
    if (per_sm < 1) per_sm = 1;
    if (c->persist_ctas_req > 0 && c->persist_ctas_req < per_sm) per_sm = c->persist_ctas_req;
    c->loop_grid[tab] = per_sm * c->sm_count;
  }
  for (int i = 0; i < lig_ctx::kItemSlots; ++i) {
    CUDA_TRY(cudaMalloc(&c->d_items[i], sizeof(QueueItem) * lig_ctx::kMaxItems));
    CUDA_TRY(cudaHostAlloc(&c->h_items[i], sizeof(QueueItem) * lig_ctx::kMaxItems, cudaHostAllocDefault));
    CUDA_TRY(cudaEventCreateWithFlags(&c->items_free[i], cudaEventDisableTiming));
  }
  for (auto& ev : c->claim_free) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&c->fork, cudaEventDisableTiming));
  for (auto& ev : c->join) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CUDA_TRY(cudaStreamCreateWithFlags(&c->s_up, cudaStreamNonBlocking));
  CUDA_TRY(cudaMalloc(&c->d_claims, sizeof(uint32_t) * lig_ctx::kClaimSlots));
  CUDA_TRY(cudaMemsetAsync(c->d_claims, 0, sizeof(uint32_t) * lig_ctx::kClaimSlots, c->s_up));
  CUDA_TRY(cudaStreamSynchronize(c->s_up));   // the counters are zero before any launch reads one
  for (auto& s : c->s_lane) CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  c->free_tickets.reserve(LIG_MAX_TICKETS);
  for (int i = LIG_MAX_TICKETS - 1; i >= 0; --i) {
    CUDA_TRY(cudaEventCreateWithFlags(&c->ticket_ev[i], cudaEventDisableTiming));
    c->free_tickets.push_back(i);
  }
  CUDA_TRY(cudaMalloc(&c->d_reqs, (size_t)max_batch * sizeof(lig_req)));
  CUDA_TRY(cudaMalloc(&c->d_out, (size_t)max_batch * sizeof(lig_pick)));
  CUDA_TRY(cudaHostAlloc(&c->h_reqs, (size_t)max_batch * sizeof(lig_req), cudaHostAllocMapped | cudaHostAllocPortable));
  CUDA_TRY(cudaHostAlloc(&c->h_out, (size_t)max_batch * sizeof(lig_pick), cudaHostAllocMapped | cudaHostAllocPortable));
  register_pinned(c->h_reqs, (size_t)max_batch * sizeof(lig_req));
  register_pinned(c->h_out, (size_t)max_batch * sizeof(lig_pick));
  // Nothing on the serving path may allocate or load code: a cudaMalloc in a refresh tick, or the
  // lazy load of a kernel at its first launch, stalls every concurrent launch of the process for
  // a millisecond or more (seen as the once-per-run latency outlier of the streaming config).
  // (a) delta staging for a quarter of the pods with 64 adapters each; larger deltas still grow it
  {
    const size_t cap = std::max<size_t>((size_t)64 << 10, (size_t)max_pods / 4 * (24 + 64 * 4) + 4096);
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&c->h_delta), cap, cudaHostAllocDefault));
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&c->d_delta), cap));
    c->delta_capacity = cap;
  }
  // (b) every kernel a tick or a batch can launch is loaded now; a lazy load while the resident
  // doorbell kernel runs can wait for that kernel, which waits for the host: a hang
  {
    cudaFuncAttributes fa;
    const void* fns[] = {
        (const void*)lig_pick_stream_kernel<1>,  (const void*)lig_pick_stream_kernel<2>,
        (const void*)lig_pick_stream_kernel<4>,  (const void*)lig_pick_stream_kernel<8>,
        (const void*)lig_pick_stream_kernel<16>, (const void*)lig_pick_queue_kernel<1>,
        (const void*)lig_pick_queue_kernel<2>,   (const void*)lig_pick_queue_kernel<4>,
        (const void*)lig_pick_queue_kernel<8>,   (const void*)lig_pick_queue_kernel<16>,
        (const void*)lig_pick_models_stream_kernel, (const void*)lig_apply_delta_kernel,
        (const void*)lig_pick_count_kernel,      (const void*)lig_apply_feedback_kernel,
        (const void*)lig_feedback_loads_kernel,  (const void*)lig_pick_models_count_kernel,
        (const void*)lig_pick_fallback_kernel<false, false>, (const void*)lig_pick_fallback_kernel<true, false>,
        (const void*)lig_pick_fallback_kernel<false, true>, (const void*)lig_pick_fallback_kernel<true, true>,
        (const void*)lig_filter_kernel<false>,   (const void*)lig_filter_kernel<true>,
        (const void*)lig_pick_affinity_kernel<false, false>, (const void*)lig_pick_affinity_kernel<true, false>,
        (const void*)lig_pick_affinity_kernel<false, true>, (const void*)lig_pick_affinity_kernel<true, true>,
    };
    for (const void* fn : fns) CUDA_TRY(cudaFuncGetAttributes(&fa, fn));
  }
  return 0;
}

int lig_create(lig_ctx** out, int device, int max_pods, int max_adapters, int max_batch) {
  if (!out) return fail(LIG_ERR_INVALID, "lig_create: out is null");
  *out = nullptr;
  if (max_pods < 1 || max_pods > LIG_MAX_PODS)
    return fail(LIG_ERR_INVALID, "max_pods=%d outside [1, %d]", max_pods, LIG_MAX_PODS);
  if (max_adapters < 0 || max_adapters > LIG_MAX_ADAPTERS)
    return fail(LIG_ERR_INVALID, "max_adapters=%d outside [0, %d]", max_adapters, LIG_MAX_ADAPTERS);
  if (max_batch < 1) return fail(LIG_ERR_INVALID, "max_batch=%d must be >= 1", max_batch);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(LIG_ERR_CUDA, "no CUDA device available (%s); this library has no CPU path",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  }
  if (device < 0 || device >= ndev)
    return fail(LIG_ERR_INVALID, "device %d outside [0, %d)", device, ndev);
  lig_ctx* c = new lig_ctx();
  if (int rc = create_impl(c, device, max_pods, max_adapters, max_batch)) {
    char keep[sizeof(g_err)];
    memcpy(keep, g_err, sizeof(keep));
    lig_destroy(c);
    memcpy(g_err, keep, sizeof(keep));
    return rc;
  }
  *out = c;
  return 0;
}

void lig_destroy(lig_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  lig_stream_close(c);   // a resident doorbell kernel would make the synchronize below wait forever
  cudaDeviceSynchronize();
  if (c->comm && ligi::g_comm_destructor) ligi::g_comm_destructor(c->comm);
  for (auto& s : c->slot) free_slot(s);
  if (c->h_delta) cudaFreeHost(c->h_delta);
  cudaFree(c->d_delta);
  if (c->fb_scratch.d_blob) free_slot(c->fb_scratch);
  cudaFree(c->d_fb_hist);
  cudaFree(c->d_fb_total);
  if (c->h_fb_loads) cudaFreeHost(c->h_fb_loads);
  if (c->h_fb_rows) cudaFreeHost(c->h_fb_rows);
  if (c->s_fb) cudaStreamDestroy(c->s_fb);
  if (c->fb_free) cudaEventDestroy(c->fb_free);
  if (c->mailbox) cudaFreeHost(c->mailbox);
  if (c->s_doorbell) cudaStreamDestroy(c->s_doorbell);
  for (int i = 0; i < lig_ctx::kItemSlots; ++i) {
    cudaFree(c->d_items[i]);
    cudaFreeHost(c->h_items[i]);
    if (c->items_free[i]) cudaEventDestroy(c->items_free[i]);
  }
  cudaFree(c->d_claims);
  for (auto& ev : c->claim_free)
    if (ev) cudaEventDestroy(ev);
  for (auto& ev : c->ticket_ev)
    if (ev) cudaEventDestroy(ev);
  if (c->fork) cudaEventDestroy(c->fork);
  for (auto& ev : c->join)
    if (ev) cudaEventDestroy(ev);
  if (c->s_up) cudaStreamDestroy(c->s_up);
  for (auto& s : c->s_lane)
    if (s) cudaStreamDestroy(s);
  cudaFree(c->d_reqs);
  cudaFree(c->d_out);
  cudaFree(c->d_masks);
  if (c->h_reqs) unregister_pinned(c->h_reqs);
  if (c->h_out) unregister_pinned(c->h_out);
  cudaFreeHost(c->h_reqs);
  cudaFreeHost(c->h_out);
  delete c;
}

int lig_set_thresholds(lig_ctx* c, const lig_thresholds* t) {
  if (!c || !t) return fail(LIG_ERR_INVALID, "lig_set_thresholds: null argument");
  std::lock_guard<std::mutex> uk(c->upload_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->thr = *t;
    // resident class tables built by the built-in tree used the old thresholds: rebuild them
    // (tables of a caller tree do not depend on them)
    for (auto& s : c->slot) {
      if (!s.valid || s.caller_tree) continue;
      if (int rc = wait_readers(s, c->s_up)) return rc;
      CUDA_TRY(cudaStreamWaitEvent(c->s_up, s.ready, 0));
      if (int rc = launch_class_build(c, s, c->s_up, nullptr)) return rc;
      CUDA_TRY(cudaEventRecord(s.ready, c->s_up));
    }
  }
  CUDA_TRY(cudaStreamSynchronize(c->s_up));
  return 0;
}

int lig_set_filter_tree(lig_ctx* c, const lig_filter_node* nodes, int n_nodes) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_set_filter_tree: null ctx");
  if (int rc = ligi::check_filter_tree(nodes, n_nodes)) return rc;
  std::lock_guard<std::mutex> uk(c->upload_mu);
  if (nodes) {
    c->tree = FilterTree{};
    memcpy(c->tree.nodes, nodes, (size_t)n_nodes * sizeof(lig_filter_node));
    c->tree.n_nodes = n_nodes;
  }
  c->has_tree = nodes != nullptr;
  return 0;
}

int lig_get_thresholds(const lig_ctx* c, lig_thresholds* t) {
  if (!c || !t) return fail(LIG_ERR_INVALID, "lig_get_thresholds: null argument");
  *t = c->thr;
  return 0;
}

static int upload_snapshot_impl(lig_ctx* c, uint64_t epoch, int P, int A, const double* kv,
                                const int32_t* q, const uint16_t* na, const uint16_t* ma,
                                const uint32_t* bitmap, bool synchronise) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_upload_snapshot: ctx is null");
  // begin_write evicts the slot the epoch replaces: refuse bad arrays before it
  if (int rc = check_snapshot_arrays(P, A, kv, q, na, ma, bitmap)) return rc;
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, epoch, P, A, nullptr, true, &w)) return rc;
  // The ctx lock is NOT held from here to the publish: batches against the other resident epoch
  // keep flowing while this one is packed, copied and its tables are built.  The slot's pinned
  // staging blob is free: begin_write waited for the slot's previous upload.
  pack_blob(w.h_blob, P, A, kv, q, na, ma, bitmap);
  int rc = 0;
  if (cudaMemcpyAsync(w.d_blob, w.h_blob, w.bytes, cudaMemcpyHostToDevice, w.stream) != cudaSuccess)
    rc = fail(LIG_ERR_CUDA, "snapshot H2D copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (!rc) rc = ligi::enqueue_build(c, &w);
  if (rc) {
    ligi::abort_write(c, &w);
    return rc;
  }
  return ligi::finish_write(c, &w, synchronise);
}

int lig_upload_snapshot(lig_ctx* c, uint64_t epoch, int P, int A, const double* kv, const int32_t* q,
                        const uint16_t* na, const uint16_t* ma, const uint32_t* bitmap) {
  return upload_snapshot_impl(c, epoch, P, A, kv, q, na, ma, bitmap, true);
}

int lig_upload_snapshot_async(lig_ctx* c, uint64_t epoch, int P, int A, const double* kv, const int32_t* q,
                              const uint16_t* na, const uint16_t* ma, const uint32_t* bitmap) {
  return upload_snapshot_impl(c, epoch, P, A, kv, q, na, ma, bitmap, false);
}

int lig_update_snapshot(lig_ctx* c, uint64_t new_epoch, uint64_t base_epoch, int n_dirty,
                        const int32_t* pod_idx, const double* kv, const int32_t* q, const uint16_t* na,
                        const uint16_t* ma, const int32_t* a_off, const int32_t* a_ids) {
  if (!c || n_dirty < 0 || (n_dirty > 0 && (!pod_idx || !kv || !q || !na || !ma || !a_off)))
    return fail(LIG_ERR_INVALID, "lig_update_snapshot: bad argument");
  if (new_epoch == base_epoch) return fail(LIG_ERR_INVALID, "lig_update_snapshot: new_epoch == base_epoch");
  const int n_ids = n_dirty ? a_off[n_dirty] : 0;
  if (n_ids < 0 || (n_ids > 0 && !a_ids)) return fail(LIG_ERR_INVALID, "lig_update_snapshot: bad adapter arrays");
  int P = 0, A = 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* b = nullptr;
    if (int rc = resolve_slot(c, base_epoch, &b)) return rc;
    P = b->P;
    A = b->A;
    // the slot the new epoch will overwrite must not be the base
    if (&victim_slot(c, new_epoch) == b)
      return fail(LIG_ERR_INVALID, "base epoch %llu is the slot epoch %llu would overwrite: use lig_upload_snapshot",
                  (unsigned long long)base_epoch, (unsigned long long)new_epoch);
  }
  // The delta kernel gives every entry its own warp, so a pod listed twice would be patched by two
  // racing warps, and every adapter id is read between the offsets: reject such input here, before
  // the writer lock, so a refused call leaves both resident epochs untouched.
  if (n_dirty > 0) {
    std::vector<unsigned char> seen((size_t)P, 0);
    for (int i = 0; i < n_dirty; ++i) {
      if (pod_idx[i] < 0 || pod_idx[i] >= P) return fail(LIG_ERR_INVALID, "dirty pod index %d outside [0, %d)", pod_idx[i], P);
      if (seen[pod_idx[i]]) return fail(LIG_ERR_INVALID, "dirty pod index %d listed twice", pod_idx[i]);
      seen[pod_idx[i]] = 1;
    }
    if (a_off[0] != 0) return fail(LIG_ERR_INVALID, "adapter_offsets[0] is %d, not 0", a_off[0]);
    for (int i = 0; i < n_dirty; ++i)
      if (a_off[i + 1] < a_off[i])
        return fail(LIG_ERR_INVALID, "adapter_offsets decrease at entry %d (%d -> %d)", i + 1, a_off[i], a_off[i + 1]);
    for (int k = 0; k < n_ids; ++k)
      if (a_ids[k] < 0 || a_ids[k] >= A) return fail(LIG_ERR_INVALID, "adapter id %d outside [0, %d)", a_ids[k], A);
    if (int rc = check_n_active(na, n_dirty)) return rc;
  }
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, new_epoch, P, A, nullptr, true, &w)) return rc;
  // from here on failures must release the writer lock
  auto bail = [&](int rc) { ligi::abort_write(c, &w); return rc; };
  // layout of the staged delta: pod_idx | q | a_off | a_ids | kv | n_active | max_active
  const size_t o_idx = 0, o_q = o_idx + (size_t)n_dirty * 4, o_off = o_q + (size_t)n_dirty * 4,
               o_ids = o_off + ((size_t)n_dirty + 1) * 4, o_kv = (o_ids + (size_t)n_ids * 4 + 7) & ~(size_t)7,
               o_na = o_kv + (size_t)n_dirty * 8, o_ma = o_na + (size_t)n_dirty * 2,
               total = (o_ma + (size_t)n_dirty * 2 + 15) & ~(size_t)15;
  if (total > c->delta_capacity) {
    if (c->stream_open) return bail(fail(LIG_ERR_INVALID, "cannot grow the delta staging while a doorbell stream is open"));
    if (cudaStreamSynchronize(w.stream) != cudaSuccess) return bail(fail(LIG_ERR_CUDA, "stream synchronise failed"));
    if (c->h_delta) cudaFreeHost(c->h_delta);
    cudaFree(c->d_delta);
    c->h_delta = nullptr;
    c->d_delta = nullptr;
    c->delta_capacity = 0;
    const size_t cap = total * 2 + 4096;
    if (cudaHostAlloc(reinterpret_cast<void**>(&c->h_delta), cap, cudaHostAllocDefault) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&c->d_delta), cap) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "delta staging allocation failed"));
    c->delta_capacity = cap;
  }
  Slot* base = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (int rc = resolve_slot(c, base_epoch, &base)) return bail(rc);
    if (base == static_cast<Slot*>(w.slot)) return bail(fail(LIG_ERR_INVALID, "base epoch was evicted meanwhile"));
    if (cudaStreamWaitEvent(w.stream, base->ready, 0) != cudaSuccess) return bail(fail(LIG_ERR_CUDA, "cudaStreamWaitEvent failed"));
    if (cudaMemcpyAsync(w.d_blob, base->d_blob, w.bytes, cudaMemcpyDeviceToDevice, w.stream) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "base snapshot copy failed"));
    if (int rc = note_reader(*base, w.stream)) return bail(rc);     // a later overwrite of the base waits for this copy
    Slot& ns = *static_cast<Slot*>(w.slot);
    ns.n_ejected = base->n_ejected;                                   // the delta keeps base's ejected pods
    if (base->n_ejected > 0 &&
        cudaMemcpyAsync(ns.d_pool, base->d_pool, (size_t)ns.W * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                        w.stream) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "base pool copy failed"));
  }
  if (n_dirty > 0) {
    unsigned char* h = c->h_delta;     // the previous delta upload synchronised before returning
    memcpy(h + o_idx, pod_idx, (size_t)n_dirty * 4);
    memcpy(h + o_q, q, (size_t)n_dirty * 4);
    memcpy(h + o_off, a_off, ((size_t)n_dirty + 1) * 4);
    if (n_ids) memcpy(h + o_ids, a_ids, (size_t)n_ids * 4);
    memcpy(h + o_kv, kv, (size_t)n_dirty * 8);
    memcpy(h + o_na, na, (size_t)n_dirty * 2);
    memcpy(h + o_ma, ma, (size_t)n_dirty * 2);
    if (cudaMemcpyAsync(c->d_delta, h, total, cudaMemcpyHostToDevice, w.stream) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "delta H2D copy failed"));
    const unsigned char* dd = c->d_delta;
    DeltaView dv{reinterpret_cast<const int*>(dd + o_idx), reinterpret_cast<const double*>(dd + o_kv),
                 reinterpret_cast<const int*>(dd + o_q), reinterpret_cast<const uint16_t*>(dd + o_na),
                 reinterpret_cast<const uint16_t*>(dd + o_ma), reinterpret_cast<const int*>(dd + o_off),
                 reinterpret_cast<const int*>(dd + o_ids), n_dirty};
    const Layout l = layout_for(P, A);
    lig_apply_delta_kernel<<<(n_dirty * 32 + 255) / 256, 256, 0, w.stream>>>(
        dv, reinterpret_cast<double*>(w.d_blob + l.kv), reinterpret_cast<int*>(w.d_blob + l.q),
        reinterpret_cast<uint16_t*>(w.d_blob + l.na), reinterpret_cast<uint16_t*>(w.d_blob + l.ma),
        reinterpret_cast<uint32_t*>(w.d_blob + l.bitmap), P, A, words_for(P));
    if (cudaGetLastError() != cudaSuccess) return bail(fail(LIG_ERR_CUDA, "delta kernel launch failed"));
    c->launches++;
  }
  if (int rc = ligi::enqueue_build(c, &w)) return bail(rc);
  return ligi::finish_write(c, &w, true);
}

int lig_eject_pods(lig_ctx* c, uint64_t new_epoch, uint64_t base_epoch, const int32_t* pod_idx, int n) {
  if (!c || n < 0 || (n > 0 && !pod_idx)) return fail(LIG_ERR_INVALID, "lig_eject_pods: bad argument");
  if (new_epoch == base_epoch) return fail(LIG_ERR_INVALID, "lig_eject_pods: new_epoch == base_epoch");
  int P = 0, A = 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* b = nullptr;
    if (int rc = resolve_slot(c, base_epoch, &b)) return rc;
    P = b->P;
    A = b->A;
    if (&victim_slot(c, new_epoch) == b)   // the rule of lig_update_snapshot
      return fail(LIG_ERR_INVALID, "base epoch %llu is the slot epoch %llu would overwrite",
                  (unsigned long long)base_epoch, (unsigned long long)new_epoch);
  }
  if (n > P) return fail(LIG_ERR_INVALID, "lig_eject_pods: n=%d exceeds P=%d", n, P);
  // the pool: every pod of [0, P) but the listed ones; refused before the writer lock, so a refused
  // call leaves both resident epochs untouched
  const int W = words_for(P);
  std::vector<uint32_t> pool((size_t)W, 0u);
  for (int w = 0; w < W; ++w) {
    const int rem = P - w * 32;
    pool[(size_t)w] = rem >= 32 ? 0xffffffffu : ((1u << rem) - 1u);
  }
  for (int i = 0; i < n; ++i) {
    const int p = pod_idx[i];
    if (p < 0 || p >= P) return fail(LIG_ERR_INVALID, "ejected pod index %d outside [0, %d)", p, P);
    const uint32_t bit = 1u << (p & 31);
    if (!(pool[(size_t)(p >> 5)] & bit)) return fail(LIG_ERR_INVALID, "ejected pod index %d listed twice", p);
    pool[(size_t)(p >> 5)] &= ~bit;
  }
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, new_epoch, P, A, nullptr, true, &w)) return rc;
  auto bail = [&](int rc) { ligi::abort_write(c, &w); return rc; };
  Slot& ns = *static_cast<Slot*>(w.slot);
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* base = nullptr;
    if (int rc = resolve_slot(c, base_epoch, &base)) return bail(rc);
    if (base == &ns) return bail(fail(LIG_ERR_INVALID, "base epoch was evicted meanwhile"));
    if (cudaStreamWaitEvent(w.stream, base->ready, 0) != cudaSuccess) return bail(fail(LIG_ERR_CUDA, "cudaStreamWaitEvent failed"));
    if (cudaMemcpyAsync(w.d_blob, base->d_blob, w.bytes, cudaMemcpyDeviceToDevice, w.stream) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "base snapshot copy failed"));
    if (int rc = note_reader(*base, w.stream)) return bail(rc);     // a later overwrite of the base waits for this copy
  }
  // the pool mask (W words, not the blob) crosses PCIe through the slot's pinned staging, which
  // begin_write found free
  ns.n_ejected = n;
  if (n > 0) {
    memcpy(w.h_blob, pool.data(), (size_t)W * sizeof(uint32_t));
    if (cudaMemcpyAsync(ns.d_pool, w.h_blob, (size_t)W * sizeof(uint32_t), cudaMemcpyHostToDevice, w.stream) != cudaSuccess)
      return bail(fail(LIG_ERR_CUDA, "pool mask copy failed"));
  }
  if (int rc = ligi::enqueue_build(c, &w)) return bail(rc);
  return ligi::finish_write(c, &w, true);
}

int lig_upload_snapshot_device(lig_ctx* c, uint64_t epoch, int P, int A, const void* d_blob,
                               void* stream) {
  if (!c || !d_blob) return fail(LIG_ERR_INVALID, "lig_upload_snapshot_device: null argument");
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, epoch, P, A, static_cast<cudaStream_t>(stream), false, &w)) return rc;
  int rc = 0;
  if (cudaMemcpyAsync(w.d_blob, d_blob, w.bytes, cudaMemcpyDeviceToDevice, w.stream) != cudaSuccess)
    rc = fail(LIG_ERR_CUDA, "snapshot D2D copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (!rc) rc = ligi::enqueue_build(c, &w);
  if (rc) {
    ligi::abort_write(c, &w);
    return rc;
  }
  return ligi::finish_write(c, &w, false);
}

int lig_schedule_batch_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                              int R, lig_pick* d_out, void* stream) {
  if (!c || R < 0 || (R > 0 && (!d_reqs || !d_out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_batch_device: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  if (R == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  if (c->pick_kernel != 2) {
    if (int rc = launch_persistent(c, *s, seed, &d_reqs, R, &d_out, 1, st)) return rc;
  } else {
    if (int rc = launch_pick(c, *s, seed, d_reqs, R, d_out, st)) return rc;
  }
  return note_reader(*s, st);
}

int lig_schedule_batches_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                const lig_req* const* d_reqs, int R, lig_pick* const* d_out,
                                int n_batches, void* stream) {
  if (!c || R < 0 || n_batches < 0 || (n_batches > 0 && (!d_reqs || !d_out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_batches_device: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  if (n_batches == 0 || R == 0) return 0;
  for (int b = 0; b < n_batches; ++b)
    if (!d_reqs[b] || !d_out[b])
      return fail(LIG_ERR_INVALID, "lig_schedule_batches_device: null buffer in batch %d", b);
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  if (c->pick_kernel != 2) {
    // default: ONE launch of resident CTAs walks every tile of every batch of the queue
    if (int rc = launch_persistent(c, *s, seed, d_reqs, R, d_out, n_batches, st)) return rc;
    return note_reader(*s, st);
  }
  const uint4* cls = reinterpret_cast<const uint4*>(s->d_cls);
  if (n_batches >= 2 && R <= c->merge_max_requests) {
    // round-1 default: one launch, one short-lived CTA per 1024 requests, blockIdx.y = batch
    const int per_cta = kPickThreads * c->pick_per_thread;
    for (int lo = 0; lo < n_batches; lo += lig_ctx::kMaxItems) {
      const int n = (n_batches - lo) < lig_ctx::kMaxItems ? (n_batches - lo) : lig_ctx::kMaxItems;
      const int slot = c->item_slot;
      c->item_slot = (slot + 1) % lig_ctx::kItemSlots;
      CUDA_TRY(cudaEventSynchronize(c->items_free[slot]));   // the kernel of 4 queues ago is done
      for (int b = 0; b < n; ++b)
        c->h_items[slot][b] = QueueItem{reinterpret_cast<const int4*>(d_reqs[lo + b]),
                                        reinterpret_cast<int2*>(d_out[lo + b]), seed + (uint64_t)(lo + b)};
      CUDA_TRY(cudaMemcpyAsync(c->d_items[slot], c->h_items[slot], sizeof(QueueItem) * (size_t)n,
                               cudaMemcpyHostToDevice, st));
      const dim3 grid((unsigned)((R + per_cta - 1) / per_cta), (unsigned)n);
      LIG_DISPATCH_PPT(c->pick_per_thread,
                       (lig_pick_queue_kernel<kPpt><<<grid, kPickThreads, 0, st>>>(
                           c->d_items[slot], R, cls, s->d_lists, s->A)));
      CUDA_TRY(cudaGetLastError());
      c->launches++;
      c->last_pick = lig_launch_info{LIG_KERNEL_QUEUE, 0, 0, 0, 0, c->pick_per_thread};
      CUDA_TRY(cudaEventRecord(c->items_free[slot], st));    // after the kernel that reads the table
    }
    return note_reader(*s, st);
  }
  // one kernel per batch, forked round-robin over the ctx's streams and joined back
  const int ns = (n_batches > 1) ? c->queue_streams : 1;
  if (ns == 1) {
    for (int b = 0; b < n_batches; ++b)
      if (int rc = launch_pick(c, *s, seed + (uint64_t)b, d_reqs[b], R, d_out[b], st)) return rc;
  } else {
    CUDA_TRY(cudaEventRecord(c->fork, st));
    for (int k = 0; k < ns; ++k) CUDA_TRY(cudaStreamWaitEvent(c->s_lane[k], c->fork, 0));
    for (int b = 0; b < n_batches; ++b)
      if (int rc = launch_pick(c, *s, seed + (uint64_t)b, d_reqs[b], R, d_out[b], c->s_lane[b % ns]))
        return rc;
    for (int k = 0; k < ns; ++k) {
      CUDA_TRY(cudaEventRecord(c->join[k], c->s_lane[k]));
      CUDA_TRY(cudaStreamWaitEvent(st, c->join[k], 0));
    }
  }
  return note_reader(*s, st);
}

int lig_schedule_scan_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                             int R, lig_pick* d_out, uint32_t* d_masks, void* stream) {
  if (!c || R < 0 || (R > 0 && (!d_reqs || !d_out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_scan_device: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  if (int rc = check_scannable(*s, epoch)) return rc;
  if (R == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  if (int rc = launch_scan(c, *s, seed, d_reqs, R, d_out, d_masks, st)) return rc;
  return note_reader(*s, st);
}

int lig_schedule_batch_async(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                             lig_pick* out, int* ticket) {
  if (!c || !ticket || R < 1 || !reqs || !out)
    return fail(LIG_ERR_INVALID, "lig_schedule_batch_async: bad argument (R must be >= 1)");
  const lig_req* dev_in = mapped_device_pointer(reqs);
  lig_pick* dev_out = mapped_device_pointer(out);
  if (!dev_in || !dev_out)
    return fail(LIG_ERR_INVALID, "lig_schedule_batch_async needs page-locked buffers (lig_host_alloc)");
  if (!req_aligned(dev_in))
    return fail(LIG_ERR_INVALID, "lig_schedule_batch_async needs a 16-byte aligned request array");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  CUDA_TRY(cudaSetDevice(c->device));
  return submit_mapped(c, s, seed, dev_in, R, dev_out, ticket);
}

int lig_schedule_wait(lig_ctx* c, int ticket) {
  if (!c || ticket < 0 || ticket >= LIG_MAX_TICKETS)
    return fail(LIG_ERR_INVALID, "lig_schedule_wait: bad ticket %d", ticket);
  cudaError_t e = cudaEventSynchronize(c->ticket_ev[ticket]);   // no ctx lock while waiting
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->free_tickets.push_back(ticket);
  }
  if (e != cudaSuccess)
    return fail(LIG_ERR_CUDA, "batch failed on the device: %s", cudaGetErrorString(e));
  return 0;
}

int lig_schedule_batch(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                       lig_pick* out) {
  if (!c || R < 0 || (R > 0 && (!reqs || !out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_batch: bad argument");
  if (R > c->max_batch)
    return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, c->max_batch);
  // Host buffers are not staged through HBM: the pick kernel reads the descriptors from, and
  // writes the picks to, page-locked host memory directly over PCIe (16 B in / 8 B out per
  // request, both directions in flight at once, one launch, no copy-engine hop).  Pinned caller
  // buffers (lig_host_alloc, cudaHostAlloc, cudaHostRegister) are used in place; pageable ones
  // bounce through the ctx's pinned buffers.
  const lig_req* dev_in = R ? mapped_device_pointer(reqs) : nullptr;
  lig_pick* dev_out = R ? mapped_device_pointer(out) : nullptr;
  const bool bounce = R > 0 && !(dev_in && dev_out && req_aligned(dev_in));
  std::unique_lock<std::mutex> bk(c->bounce_mu, std::defer_lock);
  if (bounce) {
    bk.lock();
    dev_in = mapped_device_pointer(c->h_reqs);
    dev_out = mapped_device_pointer(c->h_out);
    if (!dev_in || !dev_out)
      return fail(LIG_ERR_CUDA, "pinned staging buffers are not device-mapped on this platform");
    memcpy(c->h_reqs, reqs, (size_t)R * sizeof(lig_req));
  }
  int ticket = -1;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = resolve_slot(c, epoch, &s)) return rc;
    if (R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = submit_mapped(c, s, seed, dev_in, R, dev_out, &ticket)) return rc;
  }
  if (int rc = lig_schedule_wait(c, ticket)) return rc;
  if (bounce) memcpy(out, c->h_out, (size_t)R * sizeof(lig_pick));
  return 0;
}

int lig_schedule_scan(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                      lig_pick* out, uint32_t* masks) {
  if (!c || R < 0 || (R > 0 && (!reqs || !out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_scan: bad argument");
  if (R > c->max_batch)
    return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, c->max_batch);
  // test hook: serialised by the bounce lock (it uses the ctx's device staging buffers)
  std::lock_guard<std::mutex> bk(c->bounce_mu);
  cudaStream_t st = c->s_lane[0];
  size_t mask_bytes = 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = resolve_slot(c, epoch, &s)) return rc;
    if (int rc = check_scannable(*s, epoch)) return rc;
    if (R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    mask_bytes = masks ? (size_t)R * (s->W > 0 ? s->W : 1) * sizeof(uint32_t) : 0;
    if (mask_bytes > c->d_masks_bytes) {
      if (c->stream_open)
        return fail(LIG_ERR_INVALID, "lig_schedule_scan: cannot grow the mask buffer while a stream is open "
                                     "(cudaFree would wait for the resident doorbell kernel)");
      CUDA_TRY(cudaStreamSynchronize(st));
      cudaFree(c->d_masks);
      c->d_masks = nullptr;
      c->d_masks_bytes = 0;
      CUDA_TRY(cudaMalloc(&c->d_masks, mask_bytes));
      c->d_masks_bytes = mask_bytes;
    }
    CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
    CUDA_TRY(cudaMemcpyAsync(c->d_reqs, reqs, (size_t)R * sizeof(lig_req), cudaMemcpyHostToDevice, st));
    if (int rc = launch_scan(c, *s, seed, c->d_reqs, R, c->d_out, masks ? c->d_masks : nullptr, st))
      return rc;
    CUDA_TRY(cudaMemcpyAsync(out, c->d_out, (size_t)R * sizeof(lig_pick), cudaMemcpyDeviceToHost, st));
    if (masks && s->W > 0)
      CUDA_TRY(cudaMemcpyAsync(masks, c->d_masks, mask_bytes, cudaMemcpyDeviceToHost, st));
    if (int rc = note_reader(*s, st)) return rc;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// Launch the resident doorbell kernel on a fresh mailbox (tickets restart at 1).  Called with mu held.
static int doorbell_launch(lig_ctx* c) {
  memset(c->mailbox, 0, offsetof(Mailbox, reqs));
  c->next_ticket = 1;
  std::atomic_thread_fence(std::memory_order_seq_cst);
  lig_doorbell_kernel<<<1, kPickThreads, 0, c->s_doorbell>>>(c->d_mailbox);
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  c->stream_open = true;
  return 0;
}

// Make the resident doorbell kernel leave and wait for it.  Called with mu held.
static int doorbell_stop(lig_ctx* c) {
  reinterpret_cast<std::atomic<uint32_t>*>(&c->mailbox->ticket)->store(kMailboxQuit, std::memory_order_release);
  CUDA_TRY(cudaStreamSynchronize(c->s_doorbell));
  c->stream_open = false;
  return 0;
}

static int upload_models_impl(lig_ctx* c, uint64_t epoch, int n_models, const int32_t* off,
                              const int32_t* tgt_ids, const int32_t* tgt_w, const uint8_t* critical,
                              const int32_t* self_ids, const uint8_t* present, bool synchronise) {
  if (!c || n_models < 0 || (n_models > 0 && (!off || !critical || !self_ids)))
    return fail(LIG_ERR_INVALID, "lig_upload_models: bad argument");
  const int n_rec_in = n_models ? off[n_models] : 0;
  if (n_rec_in < 0 || (n_rec_in > 0 && (!tgt_ids || !tgt_w)))
    return fail(LIG_ERR_INVALID, "lig_upload_models: bad target arrays");
  // build the blob on the host (see lig_device.cuh: ModelHeader)
  std::vector<uint32_t> entries((size_t)n_models * 4);
  std::vector<uint32_t> targets;
  for (int m = 0; m < n_models; ++m) {
    const int lo = off[m], hi = off[m + 1];
    if (lo < 0 || hi < lo || hi > n_rec_in) return fail(LIG_ERR_INVALID, "model %d: bad target_offsets", m);
    const int nt = hi - lo;
    if (nt > 255) return fail(LIG_ERR_RANGE, "model %d has %d target models (at most 255)", m, nt);
    int64_t total = 0;
    for (int k = lo; k < hi; ++k) {
      if (tgt_w[k] < 0) return fail(LIG_ERR_RANGE, "model %d: negative weight %d", m, tgt_w[k]);
      total += tgt_w[k];
    }
    if (nt > 0 && (total < 1 || total > 0x7fffffffLL))
      return fail(LIG_ERR_RANGE, "model %d: weights sum to %lld (Go's Int31n needs [1, 2^31-1])", m, (long long)total);
    uint32_t info = (uint32_t)nt | (critical[m] ? kModelCritical : 0u) | ((!present || present[m]) ? kModelPresent : 0u);
    uint32_t magic = 0, w = (uint32_t)self_ids[m];
    if (nt == 1) w = (uint32_t)tgt_ids[lo];
    if (nt >= 2) {
      const uint32_t n = (uint32_t)total;
      if (n >= 2) {
        uint32_t l = 0;
        while ((1ull << l) < n) ++l;                                   // ceil(log2 n)
        const uint32_t shift = l - 1;
        magic = (uint32_t)((((unsigned long long)1 << (32u + shift)) + n - 1u) / n);
        info |= shift << 12;
      }
      w = (uint32_t)(targets.size() / 2);
      uint32_t cum = 0;
      for (int k = lo; k < hi; ++k) {
        cum += (uint32_t)tgt_w[k];
        targets.push_back((uint32_t)tgt_ids[k]);
        targets.push_back(cum);
      }
    }
    entries[(size_t)m * 4 + 0] = info;
    entries[(size_t)m * 4 + 1] = magic;
    entries[(size_t)m * 4 + 2] = (uint32_t)total;
    entries[(size_t)m * 4 + 3] = w;
  }
  const size_t bytes = (sizeof(ModelHeader) + entries.size() * 4 + targets.size() * 4 + 15) & ~(size_t)15;
  std::lock_guard<std::mutex> uk(c->upload_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  Slot* s = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (int rc = resolve_slot(c, epoch, &s)) return rc;
    s->models_valid = false;
    if (int rc = wait_readers(*s, c->s_up)) return rc;      // batches still reading the old table
  }
  if (bytes > s->mtab_capacity) {
    // cudaFree waits for every kernel on the device, the resident doorbell kernel included.  No
    // doorbell round trip is in flight (submits hold upload_mu too), so an open stream is stopped
    // around the reallocation and relaunched: to its callers it stays open.  mu keeps
    // lig_stream_open / lig_stream_close out meanwhile.
    std::lock_guard<std::mutex> lk(c->mu);
    const bool restart = c->stream_open;
    if (restart)
      if (int rc = doorbell_stop(c)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->s_up));                 // the readers are done: safe to free
    cudaFree(s->d_mtab);
    if (s->h_mtab) cudaFreeHost(s->h_mtab);
    s->d_mtab = nullptr;
    s->h_mtab = nullptr;
    s->mtab_capacity = 0;
    const size_t cap = bytes * 2;
    CUDA_TRY(cudaMalloc(&s->d_mtab, cap));
    CUDA_TRY(cudaHostAlloc(&s->h_mtab, cap, cudaHostAllocDefault));
    s->mtab_capacity = cap;
    if (restart)
      if (int rc = doorbell_launch(c)) return rc;
  }
  CUDA_TRY(cudaEventSynchronize(s->models_ready));   // an earlier _async upload may still read the staging copy
  memset(s->h_mtab, 0, bytes);
  ModelHeader* h = reinterpret_cast<ModelHeader*>(s->h_mtab);
  h->bytes = (uint32_t)bytes;
  h->n_models = (uint32_t)n_models;
  h->n_target_records = (uint32_t)(targets.size() / 2);
  if (!entries.empty()) memcpy(s->h_mtab + sizeof(ModelHeader), entries.data(), entries.size() * 4);
  if (!targets.empty()) memcpy(s->h_mtab + sizeof(ModelHeader) + entries.size() * 4, targets.data(), targets.size() * 4);
  CUDA_TRY(cudaMemcpyAsync(s->d_mtab, s->h_mtab, bytes, cudaMemcpyHostToDevice, c->s_up));
  CUDA_TRY(cudaEventRecord(s->models_ready, c->s_up));
  if (synchronise) CUDA_TRY(cudaStreamSynchronize(c->s_up));
  {
    std::lock_guard<std::mutex> lk(c->mu);
    s->mtab_bytes = (uint32_t)bytes;
    s->n_models = (uint32_t)n_models;
    s->models_valid = s->valid && s->epoch == epoch;
  }
  return 0;
}

int lig_upload_models(lig_ctx* c, uint64_t epoch, int n_models, const int32_t* off, const int32_t* tgt_ids,
                      const int32_t* tgt_w, const uint8_t* critical, const int32_t* self_ids,
                      const uint8_t* present) {
  return upload_models_impl(c, epoch, n_models, off, tgt_ids, tgt_w, critical, self_ids, present, true);
}

int lig_upload_models_async(lig_ctx* c, uint64_t epoch, int n_models, const int32_t* off, const int32_t* tgt_ids,
                            const int32_t* tgt_w, const uint8_t* critical, const int32_t* self_ids,
                            const uint8_t* present) {
  return upload_models_impl(c, epoch, n_models, off, tgt_ids, tgt_w, critical, self_ids, present, false);
}

static int resolve_models_slot(lig_ctx* c, uint64_t epoch, Slot** out) {
  if (int rc = resolve_slot(c, epoch, out)) return rc;
  if (!(*out)->models_valid)
    return fail(LIG_ERR_NO_SNAPSHOT, "no model table uploaded for epoch %llu (lig_upload_models)",
                (unsigned long long)epoch);
  return 0;
}

int lig_upload_pod_keys(lig_ctx* c, uint64_t epoch, int P, const uint64_t* keys) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_upload_pod_keys: bad argument");
  std::lock_guard<std::mutex> uk(c->upload_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  Slot* s = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (int rc = resolve_slot(c, epoch, &s)) return rc;
    if (P != s->P)
      return fail(LIG_ERR_INVALID, "lig_upload_pod_keys: P=%d, epoch %llu has P=%d", P, (unsigned long long)epoch,
                  s->P);
    if (P > 0 && !keys) return fail(LIG_ERR_INVALID, "lig_upload_pod_keys: keys is null with P=%d", P);
    s->keys_valid = false;
    if (int rc = wait_readers(*s, c->s_up)) return rc;      // batches still reading the old keys
  }
  CUDA_TRY(cudaEventSynchronize(s->keys_ready));   // an earlier upload may still read the staging copy
  for (int p = 0; p < P; ++p) {
    uint64_t z = keys[p];
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    s->h_podkeys[p] = z ^ (z >> 31);
  }
  if (P > 0)
    CUDA_TRY(cudaMemcpyAsync(s->d_podkeys, s->h_podkeys, (size_t)P * sizeof(uint64_t), cudaMemcpyHostToDevice, c->s_up));
  CUDA_TRY(cudaEventRecord(s->keys_ready, c->s_up));
  {
    std::lock_guard<std::mutex> lk(c->mu);
    s->keys_valid = s->valid && s->epoch == epoch;
  }
  return 0;
}

int lig_schedule_models_batches_device(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                       const uint32_t* const* d_ids, int R, lig_mpick* const* d_out,
                                       int n_batches, void* stream) {
  if (!c || R < 0 || n_batches < 0 || (n_batches > 0 && (!d_ids || !d_out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_models_batches_device: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_models_slot(c, epoch, &s)) return rc;
  if (n_batches == 0 || R == 0) return 0;
  for (int b = 0; b < n_batches; ++b)
    if (!d_ids[b] || !d_out[b])
      return fail(LIG_ERR_INVALID, "lig_schedule_models_batches_device: null buffer in batch %d", b);
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  CUDA_TRY(cudaStreamWaitEvent(st, s->models_ready, 0));
  if (int rc = launch_models(c, *s, seed, first_index, d_ids, R, d_out, n_batches, st, true)) return rc;
  return note_reader(*s, st);
}

int lig_schedule_models_batch(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                              const uint32_t* ids, int R, lig_mpick* out) {
  if (!c || R < 0 || (R > 0 && (!ids || !out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_models_batch: bad argument");
  if (R > c->max_batch) return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, c->max_batch);
  const uint32_t* dev_in = R ? mapped_device_pointer(ids) : nullptr;
  lig_mpick* dev_out = R ? mapped_device_pointer(out) : nullptr;
  const bool bounce = R > 0 && !(dev_in && dev_out);
  std::unique_lock<std::mutex> bk(c->bounce_mu, std::defer_lock);
  if (bounce) {   // the 16 B / 8 B bounce buffers of the descriptor path are large enough
    bk.lock();
    dev_in = reinterpret_cast<const uint32_t*>(mapped_device_pointer(c->h_reqs));
    dev_out = reinterpret_cast<lig_mpick*>(mapped_device_pointer(c->h_out));
    if (!dev_in || !dev_out)
      return fail(LIG_ERR_CUDA, "pinned staging buffers are not device-mapped on this platform");
    memcpy(c->h_reqs, ids, (size_t)R * sizeof(uint32_t));
  }
  int ticket = -1;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = resolve_models_slot(c, epoch, &s)) return rc;
    if (R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    if (c->free_tickets.empty())
      return fail(LIG_ERR_BUSY, "all %d tickets are in flight: call lig_schedule_wait first", LIG_MAX_TICKETS);
    const int lane = c->next_lane;
    c->next_lane = (lane + 1) % kLanes;
    cudaStream_t st = c->s_lane[lane];
    CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
    CUDA_TRY(cudaStreamWaitEvent(st, s->models_ready, 0));
    if (int rc = launch_models(c, *s, seed, first_index, &dev_in, R, &dev_out, 1, st, false)) return rc;
    if (int rc = note_reader(*s, st)) return rc;
    ticket = c->free_tickets.back();
    CUDA_TRY(cudaEventRecord(c->ticket_ev[ticket], st));
    c->free_tickets.pop_back();
  }
  if (int rc = lig_schedule_wait(c, ticket)) return rc;
  if (bounce) memcpy(out, c->h_out, (size_t)R * sizeof(lig_mpick));
  return 0;
}

int lig_resolve_models(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                       const uint32_t* ids, int R, lig_req* reqs_out, lig_mpick* out) {
  if (!c || R < 0 || (R > 0 && (!ids || !reqs_out || !out)))
    return fail(LIG_ERR_INVALID, "lig_resolve_models: bad argument");
  if (R > c->max_batch) return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, c->max_batch);
  std::lock_guard<std::mutex> bk(c->bounce_mu);   // test hook: uses the ctx's staging buffers
  cudaStream_t st = c->s_lane[0];
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = resolve_models_slot(c, epoch, &s)) return rc;
    if (R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    CUDA_TRY(cudaStreamWaitEvent(st, s->models_ready, 0));
    uint32_t* d_ids = reinterpret_cast<uint32_t*>(c->d_out);     // R x 8 B staging holds R ids + R results
    uint32_t* d_res = d_ids + R;
    CUDA_TRY(cudaMemcpyAsync(d_ids, ids, (size_t)R * 4, cudaMemcpyHostToDevice, st));
    lig_pick_models_stream_kernel<<<(R + kTile - 1) / kTile, kGroupThreads, 0, st>>>(
        d_ids, d_res, R, reinterpret_cast<const uint4*>(s->d_cls), s->d_lists, s->A, s->d_mtab, s->n_models,
        seed, first_index, reinterpret_cast<int4*>(c->d_reqs));
    CUDA_TRY(cudaGetLastError());
    c->launches++;
    CUDA_TRY(cudaMemcpyAsync(reqs_out, c->d_reqs, (size_t)R * sizeof(lig_req), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out, d_res, (size_t)R * 4, cudaMemcpyDeviceToHost, st));
    if (int rc = note_reader(*s, st)) return rc;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// ---- survivor lists of a batch (lig_filter_batch, lig_filter_models_batch) -------------------------
// One filter call: descriptors (models = false) or model ids, and the four output buffers.
struct FilterCall {
  bool models;
  uint64_t seed, first_index;
  const void* in;
  int R;
  void* out;
  int64_t* offsets;
  uint16_t* pods;
  int64_t capacity;
  size_t in_bytes() const { return models ? sizeof(uint32_t) : sizeof(lig_req); }
  size_t out_bytes() const { return models ? sizeof(lig_mpick) : sizeof(lig_pick); }
};

static int filter_check(const lig_ctx* c, const char* fn, const FilterCall& f) {
  if (!c || f.R < 0 || f.capacity < 0 || !f.offsets || (f.R > 0 && (!f.in || !f.out)) ||
      (f.capacity > 0 && !f.pods))
    return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  return 0;
}

// Enqueue the filter kernel for f (R >= 1, device-visible pointers) against slot s on st, behind the
// slot's tables, and register st as a reader of the slot.  The look-back state is stream-ordered
// scratch: allocated, zeroed and freed on st.  Caller holds c->mu.
static int enqueue_filter(lig_ctx* c, Slot& s, const FilterCall& f, cudaStream_t st) {
  CUDA_TRY(cudaStreamWaitEvent(st, s.ready, 0));
  if (f.models) CUDA_TRY(cudaStreamWaitEvent(st, s.models_ready, 0));
  const int tiles = (f.R + kFilterTile - 1) / kFilterTile;
  const size_t bytes = (size_t)tiles * sizeof(unsigned long long) + 16;
  void* scratch = nullptr;
  CUDA_TRY(cudaMallocAsync(&scratch, bytes, st));
  cudaError_t e = cudaMemsetAsync(scratch, 0, bytes, st);
  if (e == cudaSuccess) {
    FilterOut fo;
    fo.out = f.out;
    fo.offsets = reinterpret_cast<long long*>(f.offsets);
    fo.pods = f.pods;
    fo.capacity = f.capacity;
    fo.tiles = static_cast<unsigned long long*>(scratch);
    fo.tile_counter = reinterpret_cast<uint32_t*>(fo.tiles + tiles);
    const uint4* cls = reinterpret_cast<const uint4*>(s.d_cls);
    if (f.models)
      lig_filter_kernel<true><<<tiles, kFilterThreads, 0, st>>>(f.in, f.R, cls, s.d_lists, s.A, s.d_ctab, s.d_mtab,
                                                                s.n_models, f.seed, f.first_index, fo);
    else
      lig_filter_kernel<false><<<tiles, kFilterThreads, 0, st>>>(f.in, f.R, cls, s.d_lists, s.A, s.d_ctab, nullptr,
                                                                 0u, f.seed, 0, fo);
    e = cudaGetLastError();
  }
  cudaFreeAsync(scratch, st);
  if (e != cudaSuccess)
    return fail(LIG_ERR_CUDA, "survivor-list kernel: %s", cudaGetErrorString(e));
  c->launches++;
  return note_reader(s, st);
}

static int filter_device(lig_ctx* c, const char* fn, uint64_t epoch, const FilterCall& f, void* stream) {
  if (int rc = filter_check(c, fn, f)) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = f.models ? resolve_models_slot(c, epoch, &s) : resolve_slot(c, epoch, &s)) return rc;
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (f.R == 0) {
    CUDA_TRY(cudaMemsetAsync(f.offsets, 0, sizeof(int64_t), st));
    return 0;
  }
  return enqueue_filter(c, *s, f, st);
}

// Host buffers: page-locked ones are read and written by the kernel in place; the others are
// staged in stream-ordered HBM and copied on the call's lane.  Blocks until everything is back.
static int filter_host(lig_ctx* c, const char* fn, uint64_t epoch, const FilterCall& f) {
  if (int rc = filter_check(c, fn, f)) return rc;
  if (f.R > c->max_batch) return fail(LIG_ERR_INVALID, "%s: R=%d exceeds max_batch=%d", fn, f.R, c->max_batch);
  FilterCall d = f;    // the same call with device-visible pointers
  const size_t in_b = (size_t)f.R * f.in_bytes(), out_b = (size_t)f.R * f.out_bytes();
  const size_t off_b = ((size_t)f.R + 1) * sizeof(int64_t);
  d.in = f.R ? mapped_device_pointer(f.in) : nullptr;
  d.out = f.R ? mapped_device_pointer(f.out) : nullptr;
  d.offsets = f.R ? mapped_device_pointer(f.offsets) : nullptr;
  d.pods = f.R && f.capacity > 0 ? mapped_device_pointer(f.pods) : nullptr;
  // requests that are not aligned to their element (a lig_req array at an odd 8 bytes) are staged
  // as well: the kernel reads a descriptor with one 16-byte load
  const bool st_in = f.R && (!d.in || (reinterpret_cast<uintptr_t>(d.in) & (f.in_bytes() - 1)));
  const bool st_out = f.R && !d.out, st_off = f.R && !d.offsets;
  const bool st_pods = f.R && f.capacity > 0 && !d.pods;
  cudaStream_t st = nullptr;
  unsigned char* stage = nullptr;
  size_t pods_entries = 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = f.models ? resolve_models_slot(c, epoch, &s) : resolve_slot(c, epoch, &s)) return rc;
    if (f.R == 0) {
      f.offsets[0] = 0;
      return 0;
    }
    CUDA_TRY(cudaSetDevice(c->device));
    st = c->s_lane[c->next_lane];
    c->next_lane = (c->next_lane + 1) % kLanes;
    // a list has at most P entries, so R * P bounds what a staged pod buffer can receive
    if (st_pods) pods_entries = (size_t)std::min<int64_t>(f.capacity, (int64_t)f.R * (s->P > 0 ? s->P : 1));
    size_t at = 0, o_in = 0, o_out = 0, o_off = 0, o_pods = 0;
    auto take = [&](bool on, size_t bytes, size_t* o) { if (on) { *o = at; at = (at + bytes + 255) & ~(size_t)255; } };
    take(st_in, in_b, &o_in);
    take(st_out, out_b, &o_out);
    take(st_off, off_b, &o_off);
    take(st_pods, pods_entries * sizeof(uint16_t), &o_pods);
    if (at) {
      CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&stage), at, st));
      if (st_in) d.in = stage + o_in;
      if (st_out) d.out = stage + o_out;
      if (st_off) d.offsets = reinterpret_cast<int64_t*>(stage + o_off);
      if (st_pods) d.pods = reinterpret_cast<uint16_t*>(stage + o_pods);
    }
    int rc = 0;
    if (st_in && cudaMemcpyAsync(const_cast<void*>(d.in), f.in, in_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the requests failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc) rc = enqueue_filter(c, *s, d, st);
    if (rc) {
      if (stage) cudaFreeAsync(stage, st);
      return rc;
    }
  }
  // the copies back wait for the kernel on the lane; they may block, so not under c->mu
  cudaError_t e = cudaSuccess;
  if (st_out && e == cudaSuccess) e = cudaMemcpyAsync(f.out, d.out, out_b, cudaMemcpyDeviceToHost, st);
  if (st_off && e == cudaSuccess) e = cudaMemcpyAsync(f.offsets, d.offsets, off_b, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  const int64_t total = e == cudaSuccess ? f.offsets[f.R] : 0;
  if (st_pods && e == cudaSuccess) {
    const size_t n = (size_t)std::min<int64_t>(total, f.capacity);
    if (n) e = cudaMemcpyAsync(f.pods, d.pods, n * sizeof(uint16_t), cudaMemcpyDeviceToHost, st);
  }
  if (stage) cudaFreeAsync(stage, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(LIG_ERR_CUDA, "%s failed on the device: %s", fn, cudaGetErrorString(e));
  if (total > f.capacity)
    return fail(LIG_ERR_INVALID, "%s: the survivor lists need %lld entries, capacity is %lld (out and offsets "
                                 "are complete)", fn, (long long)total, (long long)f.capacity);
  return 0;
}

int lig_filter_batch(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R, lig_pick* out,
                     int64_t* offsets, uint16_t* pods, int64_t capacity) {
  return filter_host(c, "lig_filter_batch", epoch,
                     FilterCall{false, seed, 0, reqs, R, out, offsets, pods, capacity});
}

int lig_filter_batch_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs, int R,
                            lig_pick* d_out, int64_t* d_offsets, uint16_t* d_pods, int64_t capacity,
                            void* stream) {
  return filter_device(c, "lig_filter_batch_device", epoch,
                       FilterCall{false, seed, 0, d_reqs, R, d_out, d_offsets, d_pods, capacity}, stream);
}

int lig_filter_models_batch(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                            const uint32_t* model_ids, int R, lig_mpick* out, int64_t* offsets,
                            uint16_t* pods, int64_t capacity) {
  return filter_host(c, "lig_filter_models_batch", epoch,
                     FilterCall{true, seed, first_index, model_ids, R, out, offsets, pods, capacity});
}

int lig_filter_models_batch_device(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                   const uint32_t* d_model_ids, int R, lig_mpick* d_out, int64_t* d_offsets,
                                   uint16_t* d_pods, int64_t capacity, void* stream) {
  return filter_device(c, "lig_filter_models_batch_device", epoch,
                       FilterCall{true, seed, first_index, d_model_ids, R, d_out, d_offsets, d_pods, capacity},
                       stream);
}

// ---- fallback endpoints (lig_schedule_batch_fallbacks, lig_schedule_models_batch_fallbacks) ----------
// and the session-affinity calls (lig_schedule_[models_]batch_affinity), which share their staging.
struct FallbackCall {
  bool models;
  uint64_t seed, first_index;
  const void* in;
  int R;
  void* out;
  int n_fallbacks;
  int16_t* fallbacks;
  // affinity: no seed, no first_index; keys (model ids only) are the requests' affinity keys, and
  // n_fallbacks = 0 means no row (fallbacks may then be null)
  bool affinity = false;
  const uint64_t* keys = nullptr;
  size_t in_bytes() const { return models ? sizeof(uint32_t) : sizeof(lig_req); }
  size_t out_bytes() const { return models ? sizeof(lig_mpick) : sizeof(lig_pick); }
  size_t row_bytes() const { return (size_t)n_fallbacks * sizeof(int16_t); }
  bool has_keys() const { return affinity && models; }
  bool has_rows() const { return n_fallbacks > 0; }
};

static int fallback_check(const lig_ctx* c, const char* fn, const FallbackCall& f) {
  if (!c || f.R < 0 ||
      (f.R > 0 && (!f.in || !f.out || (!f.fallbacks && (!f.affinity || f.has_rows())) || (f.has_keys() && !f.keys))))
    return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  const int lo = f.affinity ? 0 : 1;
  if (f.n_fallbacks < lo || f.n_fallbacks > LIG_MAX_FALLBACKS)
    return fail(LIG_ERR_INVALID, "%s: n_fallbacks=%d outside [%d, %d]", fn, f.n_fallbacks, lo, LIG_MAX_FALLBACKS);
  return 0;
}

// The slot a fallback or affinity call reads: the model forms need the epoch's model table, the
// affinity forms its pod keys.  Caller holds c->mu.
static int fallback_slot(lig_ctx* c, uint64_t epoch, const FallbackCall& f, Slot** s) {
  if (int rc = f.models ? resolve_models_slot(c, epoch, s) : resolve_slot(c, epoch, s)) return rc;
  if (f.affinity && !(*s)->keys_valid)
    return fail(LIG_ERR_NO_SNAPSHOT, "no pod keys uploaded for epoch %llu (lig_upload_pod_keys)",
                (unsigned long long)epoch);
  return 0;
}

static bool misaligned(const void* p, size_t align) { return (reinterpret_cast<uintptr_t>(p) & (align - 1)) != 0; }

// Enqueue the fallback kernel for f (R >= 1, device-visible, aligned pointers) against slot s on st,
// behind the slot's tables, and register st as a reader of the slot.  Caller holds c->mu.
static int enqueue_fallbacks(lig_ctx* c, Slot& s, const FallbackCall& f, cudaStream_t st) {
  CUDA_TRY(cudaStreamWaitEvent(st, s.ready, 0));
  if (f.models) CUDA_TRY(cudaStreamWaitEvent(st, s.models_ready, 0));
  const int blocks = (f.R + kFallbackThreads - 1) / kFallbackThreads;
  const uint4* cls = reinterpret_cast<const uint4*>(s.d_cls);
  if (f.affinity) {
    CUDA_TRY(cudaStreamWaitEvent(st, s.keys_ready, 0));
    if (f.models)
      lig_pick_affinity_kernel<true, false><<<blocks, kFallbackThreads, 0, st>>>(
          f.in, f.keys, f.out, f.fallbacks, f.R, f.n_fallbacks, cls, s.d_lists, s.A, s.d_ctab, s.d_mtab, s.n_models,
          s.d_podkeys, nullptr);
    else
      lig_pick_affinity_kernel<false, false><<<blocks, kFallbackThreads, 0, st>>>(
          f.in, nullptr, f.out, f.fallbacks, f.R, f.n_fallbacks, cls, s.d_lists, s.A, s.d_ctab, nullptr, 0u,
          s.d_podkeys, nullptr);
  } else if (f.models)
    lig_pick_fallback_kernel<true, false><<<blocks, kFallbackThreads, 0, st>>>(
        f.in, f.out, f.fallbacks, f.R, f.n_fallbacks, cls, s.d_lists, s.A, s.d_ctab, s.d_mtab, s.n_models, f.seed,
        f.first_index, nullptr);
  else
    lig_pick_fallback_kernel<false, false><<<blocks, kFallbackThreads, 0, st>>>(
        f.in, f.out, f.fallbacks, f.R, f.n_fallbacks, cls, s.d_lists, s.A, s.d_ctab, nullptr, 0u, f.seed, 0, nullptr);
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  return note_reader(s, st);
}

static int fallback_device(lig_ctx* c, const char* fn, uint64_t epoch, const FallbackCall& f, void* stream) {
  if (int rc = fallback_check(c, fn, f)) return rc;
  if (f.R > 0 && (misaligned(f.in, f.in_bytes()) || misaligned(f.out, f.out_bytes()) ||
                  misaligned(f.fallbacks, sizeof(int16_t)) || misaligned(f.keys, sizeof(uint64_t))))
    return fail(LIG_ERR_INVALID, "%s: a device buffer is not aligned to its element", fn);
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = fallback_slot(c, epoch, f, &s)) return rc;
  if (f.R == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  return enqueue_fallbacks(c, *s, f, static_cast<cudaStream_t>(stream));
}

// Host buffers: page-locked, aligned ones are read and written by the kernel in place; the others
// are staged in stream-ordered HBM and copied on the call's lane.  Blocks until everything is back.
static int fallback_host(lig_ctx* c, const char* fn, uint64_t epoch, const FallbackCall& f) {
  if (int rc = fallback_check(c, fn, f)) return rc;
  if (f.R > c->max_batch) return fail(LIG_ERR_INVALID, "%s: R=%d exceeds max_batch=%d", fn, f.R, c->max_batch);
  FallbackCall d = f;    // the same call with device-visible pointers
  const size_t in_b = (size_t)f.R * f.in_bytes(), out_b = (size_t)f.R * f.out_bytes();
  const size_t rows_b = (size_t)f.R * f.row_bytes(), keys_b = (size_t)f.R * sizeof(uint64_t);
  d.in = f.R ? mapped_device_pointer(f.in) : nullptr;
  d.out = f.R ? mapped_device_pointer(f.out) : nullptr;
  d.fallbacks = f.R && f.has_rows() ? mapped_device_pointer(f.fallbacks) : nullptr;
  d.keys = f.R && f.has_keys() ? mapped_device_pointer(f.keys) : nullptr;
  // the kernel reads a descriptor with one 16-byte load and stores every element whole
  const bool st_in = f.R && (!d.in || misaligned(d.in, f.in_bytes()));
  const bool st_out = f.R && (!d.out || misaligned(d.out, f.out_bytes()));
  const bool st_rows = f.R && f.has_rows() && (!d.fallbacks || misaligned(d.fallbacks, sizeof(int16_t)));
  const bool st_keys = f.R && f.has_keys() && (!d.keys || misaligned(d.keys, sizeof(uint64_t)));
  cudaStream_t st = nullptr;
  unsigned char* stage = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = fallback_slot(c, epoch, f, &s)) return rc;
    if (f.R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    st = c->s_lane[c->next_lane];
    c->next_lane = (c->next_lane + 1) % kLanes;
    size_t at = 0, o_in = 0, o_out = 0, o_rows = 0, o_keys = 0;
    auto take = [&](bool on, size_t bytes, size_t* o) { if (on) { *o = at; at = (at + bytes + 255) & ~(size_t)255; } };
    take(st_in, in_b, &o_in);
    take(st_out, out_b, &o_out);
    take(st_rows, rows_b, &o_rows);
    take(st_keys, keys_b, &o_keys);
    if (at) {
      CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&stage), at, st));
      if (st_in) d.in = stage + o_in;
      if (st_out) d.out = stage + o_out;
      if (st_rows) d.fallbacks = reinterpret_cast<int16_t*>(stage + o_rows);
      if (st_keys) d.keys = reinterpret_cast<const uint64_t*>(stage + o_keys);
    }
    int rc = 0;
    if (st_in && cudaMemcpyAsync(const_cast<void*>(d.in), f.in, in_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the requests failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc && st_keys &&
        cudaMemcpyAsync(const_cast<uint64_t*>(d.keys), f.keys, keys_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the keys failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc) rc = enqueue_fallbacks(c, *s, d, st);
    if (rc) {
      if (stage) cudaFreeAsync(stage, st);
      return rc;
    }
  }
  // the copies back wait for the kernel on the lane; they may block, so not under c->mu
  cudaError_t e = cudaSuccess;
  if (st_out) e = cudaMemcpyAsync(f.out, d.out, out_b, cudaMemcpyDeviceToHost, st);
  if (st_rows && e == cudaSuccess) e = cudaMemcpyAsync(f.fallbacks, d.fallbacks, rows_b, cudaMemcpyDeviceToHost, st);
  if (stage) cudaFreeAsync(stage, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(LIG_ERR_CUDA, "%s failed on the device: %s", fn, cudaGetErrorString(e));
  return 0;
}

int lig_schedule_batch_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                 lig_pick* out, int n_fallbacks, int16_t* fallbacks) {
  return fallback_host(c, "lig_schedule_batch_fallbacks", epoch,
                       FallbackCall{false, seed, 0, reqs, R, out, n_fallbacks, fallbacks});
}

int lig_schedule_batch_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs, int R,
                                        lig_pick* d_out, int n_fallbacks, int16_t* d_fallbacks, void* stream) {
  return fallback_device(c, "lig_schedule_batch_fallbacks_device", epoch,
                         FallbackCall{false, seed, 0, d_reqs, R, d_out, n_fallbacks, d_fallbacks}, stream);
}

int lig_schedule_models_batch_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                        const uint32_t* model_ids, int R, lig_mpick* out, int n_fallbacks,
                                        int16_t* fallbacks) {
  return fallback_host(c, "lig_schedule_models_batch_fallbacks", epoch,
                       FallbackCall{true, seed, first_index, model_ids, R, out, n_fallbacks, fallbacks});
}

int lig_schedule_models_batch_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                               const uint32_t* d_model_ids, int R, lig_mpick* d_out,
                                               int n_fallbacks, int16_t* d_fallbacks, void* stream) {
  return fallback_device(c, "lig_schedule_models_batch_fallbacks_device", epoch,
                         FallbackCall{true, seed, first_index, d_model_ids, R, d_out, n_fallbacks, d_fallbacks},
                         stream);
}

int lig_schedule_batch_affinity(lig_ctx* c, uint64_t epoch, const lig_req* reqs, int R, lig_pick* out,
                                int n_fallbacks, int16_t* fallbacks) {
  FallbackCall f{false, 0, 0, reqs, R, out, n_fallbacks, fallbacks};
  f.affinity = true;
  return fallback_host(c, "lig_schedule_batch_affinity", epoch, f);
}

int lig_schedule_batch_affinity_device(lig_ctx* c, uint64_t epoch, const lig_req* d_reqs, int R, lig_pick* d_out,
                                       int n_fallbacks, int16_t* d_fallbacks, void* stream) {
  FallbackCall f{false, 0, 0, d_reqs, R, d_out, n_fallbacks, d_fallbacks};
  f.affinity = true;
  return fallback_device(c, "lig_schedule_batch_affinity_device", epoch, f, stream);
}

int lig_schedule_models_batch_affinity(lig_ctx* c, uint64_t epoch, const uint32_t* model_ids, const uint64_t* keys,
                                       int R, lig_mpick* out, int n_fallbacks, int16_t* fallbacks) {
  FallbackCall f{true, 0, 0, model_ids, R, out, n_fallbacks, fallbacks};
  f.affinity = true;
  f.keys = keys;
  return fallback_host(c, "lig_schedule_models_batch_affinity", epoch, f);
}

int lig_schedule_models_batch_affinity_device(lig_ctx* c, uint64_t epoch, const uint32_t* d_model_ids,
                                              const uint64_t* d_keys, int R, lig_mpick* d_out, int n_fallbacks,
                                              int16_t* d_fallbacks, void* stream) {
  FallbackCall f{true, 0, 0, d_model_ids, R, d_out, n_fallbacks, d_fallbacks};
  f.affinity = true;
  f.keys = d_keys;
  return fallback_device(c, "lig_schedule_models_batch_affinity_device", epoch, f, stream);
}

// ---- retry scheduling (lig_schedule_[models_]batch_excluding[_fallbacks]) -----------------------------
// One retry call: descriptors in, lig_pick out; or (models) model ids in at the fixed targets
// targets[i], lig_mpick out, request i with rand_key = first_index + i, resolved against the model
// table mtab of n_models entries (set where the call is enqueued).  With n_fallbacks > 0, a row of
// n_fallbacks int16 per request as well; every retry rule applies.
struct ExcludingCall {
  uint64_t seed;
  const void* in;                        // lig_req[R] or uint32_t[R]
  int R;
  void* out;                             // lig_pick[R] or lig_mpick[R]
  int n_excluded;
  const int16_t* excluded;
  int n_fallbacks = 0;                   // 0: no rows
  int16_t* fallbacks = nullptr;
  bool models = false;
  uint64_t first_index = 0;
  const uint8_t* targets = nullptr;
  const unsigned char* mtab = nullptr;
  uint32_t n_models = 0;
  size_t in_bytes() const { return models ? sizeof(uint32_t) : sizeof(lig_req); }
  size_t out_bytes() const { return models ? sizeof(lig_mpick) : sizeof(lig_pick); }
  size_t row_bytes() const { return (size_t)n_excluded * sizeof(int16_t); }
};

static ExcludingCall model_retry(uint64_t seed, uint64_t first_index, const uint32_t* ids, const uint8_t* targets,
                                 int R, const int16_t* excluded, int n_excluded, lig_mpick* out,
                                 int n_fallbacks = 0, int16_t* fallbacks = nullptr) {
  ExcludingCall x{seed, ids, R, out, n_excluded, excluded, n_fallbacks, fallbacks};
  x.models = true;
  x.first_index = first_index;
  x.targets = targets;
  return x;
}

// `rows`: the entry point takes fallback rows, so x.n_fallbacks must be in [1, LIG_MAX_FALLBACKS].
static int excluding_check(const lig_ctx* c, const char* fn, const ExcludingCall& x, bool rows) {
  if (!c || x.R < 0 || (x.R > 0 && (!x.in || !x.out || !x.excluded || (x.models && !x.targets))))
    return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  if (x.n_excluded < 1 || x.n_excluded > LIG_MAX_EXCLUDED)
    return fail(LIG_ERR_INVALID, "%s: n_excluded=%d outside [1, %d]", fn, x.n_excluded, LIG_MAX_EXCLUDED);
  if (rows && x.R > 0 && !x.fallbacks) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  if (rows && (x.n_fallbacks < 1 || x.n_fallbacks > LIG_MAX_FALLBACKS))
    return fail(LIG_ERR_INVALID, "%s: n_fallbacks=%d outside [1, %d]", fn, x.n_fallbacks, LIG_MAX_FALLBACKS);
  return 0;
}

static int excluding_slot(lig_ctx* c, const ExcludingCall& x, uint64_t epoch, Slot** s) {
  return x.models ? resolve_models_slot(c, epoch, s) : resolve_slot(c, epoch, s);
}

// Launch the retry kernel for x (R >= 1, device-visible, aligned pointers, x.mtab set for model ids)
// over slot s on st, with the scan's launch shape: `tree` (null = the built-in tree with `thr`); the
// pool of an ejected epoch; a row per request when x.n_fallbacks > 0; `hist` non-null counts each
// LIG_OK pick into it (the feedback chain's segment).  The caller checks the launch.
static void launch_excluding(const lig_ctx* c, const Slot& s, const Thr& thr, const FilterTree* tree,
                             const ExcludingCall& x, int* hist, cudaStream_t st) {
  static const FilterTree kNoTree{};
  const ScanShape sh = scan_shape(c, s, x.R);
  const SnapView v = view_of(s);
  const FilterTree& t = tree ? *tree : kNoTree;
  const uint32_t* pool = s.n_ejected > 0 ? s.d_pool : nullptr;
  auto launch = [&](auto... form) {
    lig_schedule_excluding_kernel<decltype(form)::value...><<<sh.grid, kCtaThreads, sh.smem, st>>>(
        v, thr, t, x.in, x.targets, x.excluded, x.n_excluded, x.out, x.R, x.seed, x.first_index, x.mtab, x.n_models,
        x.n_fallbacks, x.fallbacks, hist, pool);
  };
  using Y = std::true_type;
  using N = std::false_type;
  auto with_count = [&](auto... f) { if (hist) launch(f..., Y{}); else launch(f..., N{}); };
  auto with_rows = [&](auto... f) { if (x.n_fallbacks > 0) with_count(f..., Y{}); else with_count(f..., N{}); };
  auto with_pool = [&](auto... f) { if (pool) with_rows(f..., Y{}); else with_rows(f..., N{}); };
  auto with_tree = [&](auto... f) { if (tree) with_pool(f..., Y{}); else with_pool(f..., N{}); };
  auto with_staged = [&](auto... f) { if (sh.staged) with_tree(f..., Y{}); else with_tree(f..., N{}); };
  if (x.models) with_staged(Y{});
  else with_staged(N{});
}

// Enqueue the retry kernel for x (R >= 1, device-visible, aligned pointers) against slot s on st,
// behind the slot's tables (and model table), and register st as a reader of the slot.  The walk is
// the tree that built the slot's tables.  Caller holds c->mu.
static int enqueue_excluding(lig_ctx* c, Slot& s, const ExcludingCall& x, cudaStream_t st) {
  CUDA_TRY(cudaStreamWaitEvent(st, s.ready, 0));
  ExcludingCall m = x;
  if (x.models) {
    CUDA_TRY(cudaStreamWaitEvent(st, s.models_ready, 0));
    m.mtab = s.d_mtab;
    m.n_models = s.n_models;
  }
  launch_excluding(c, s, thr_of(c), s.caller_tree ? &s.tree : nullptr, m, nullptr, st);
  CUDA_TRY(cudaGetLastError());
  c->launches++;
  return note_reader(s, st);
}

static int excluding_device(lig_ctx* c, const char* fn, uint64_t epoch, const ExcludingCall& x, bool rows,
                            void* stream) {
  if (int rc = excluding_check(c, fn, x, rows)) return rc;
  if (x.R > 0 && (misaligned(x.in, x.in_bytes()) || misaligned(x.out, x.out_bytes()) ||
                  misaligned(x.excluded, sizeof(int16_t)) || (rows && misaligned(x.fallbacks, sizeof(int16_t)))))
    return fail(LIG_ERR_INVALID, "%s: a device buffer is not aligned to its element", fn);
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = excluding_slot(c, x, epoch, &s)) return rc;
  if (x.R == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  return enqueue_excluding(c, *s, x, static_cast<cudaStream_t>(stream));
}

int lig_schedule_batch_excluding_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs, int R,
                                        const int16_t* d_excluded, int n_excluded, lig_pick* d_out, void* stream) {
  return excluding_device(c, "lig_schedule_batch_excluding_device", epoch,
                          ExcludingCall{seed, d_reqs, R, d_out, n_excluded, d_excluded}, false, stream);
}

int lig_schedule_models_batch_excluding_device(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                               const uint32_t* d_model_ids, const uint8_t* d_targets, int R,
                                               const int16_t* d_excluded, int n_excluded, lig_mpick* d_out,
                                               void* stream) {
  return excluding_device(c, "lig_schedule_models_batch_excluding_device", epoch,
                          model_retry(seed, first_index, d_model_ids, d_targets, R, d_excluded, n_excluded, d_out),
                          false, stream);
}

int lig_schedule_batch_excluding_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                                  int R, const int16_t* d_excluded, int n_excluded, lig_pick* d_out,
                                                  int n_fallbacks, int16_t* d_fallbacks, void* stream) {
  return excluding_device(c, "lig_schedule_batch_excluding_fallbacks_device", epoch,
                          ExcludingCall{seed, d_reqs, R, d_out, n_excluded, d_excluded, n_fallbacks, d_fallbacks},
                          true, stream);
}

int lig_schedule_models_batch_excluding_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                         uint64_t first_index, const uint32_t* d_model_ids,
                                                         const uint8_t* d_targets, int R, const int16_t* d_excluded,
                                                         int n_excluded, lig_mpick* d_out, int n_fallbacks,
                                                         int16_t* d_fallbacks, void* stream) {
  return excluding_device(c, "lig_schedule_models_batch_excluding_fallbacks_device", epoch,
                          model_retry(seed, first_index, d_model_ids, d_targets, R, d_excluded, n_excluded, d_out,
                                      n_fallbacks, d_fallbacks),
                          true, stream);
}

// The host buffers of a retry call (with rows when x.n_fallbacks > 0): page-locked, aligned ones are
// read and written by the kernel in place; the others are staged in stream-ordered HBM and copied on
// the call's lane.  Blocks until the picks (and rows) are back.
static int excluding_host(lig_ctx* c, const char* fn, uint64_t epoch, const ExcludingCall& x, bool rows) {
  if (int rc = excluding_check(c, fn, x, rows)) return rc;
  const int R = x.R;
  if (R > c->max_batch) return fail(LIG_ERR_INVALID, "%s: R=%d exceeds max_batch=%d", fn, R, c->max_batch);
  ExcludingCall d = x;    // the same call with device-visible pointers
  const size_t in_b = (size_t)R * x.in_bytes(), out_b = (size_t)R * x.out_bytes();
  const size_t rows_b = (size_t)R * x.row_bytes(), fb_b = (size_t)R * (size_t)x.n_fallbacks * sizeof(int16_t);
  const size_t tg_b = x.models ? (size_t)R : 0;
  d.in = R ? mapped_device_pointer(x.in) : nullptr;
  d.out = R ? mapped_device_pointer(x.out) : nullptr;
  d.excluded = R ? mapped_device_pointer(x.excluded) : nullptr;
  d.targets = R && x.models ? mapped_device_pointer(x.targets) : nullptr;
  d.fallbacks = R && x.n_fallbacks ? mapped_device_pointer(x.fallbacks) : nullptr;
  // the kernels read a descriptor with one 16-byte load and store every pick whole
  const bool st_in = R && (!d.in || misaligned(d.in, x.in_bytes()));
  const bool st_out = R && (!d.out || misaligned(d.out, x.out_bytes()));
  const bool st_rows = R && (!d.excluded || misaligned(d.excluded, sizeof(int16_t)));
  const bool st_tg = R && x.models && !d.targets;
  const bool st_fb = R && x.n_fallbacks && (!d.fallbacks || misaligned(d.fallbacks, sizeof(int16_t)));
  cudaStream_t st = nullptr;
  unsigned char* stage = nullptr;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = excluding_slot(c, x, epoch, &s)) return rc;
    if (R == 0) return 0;
    CUDA_TRY(cudaSetDevice(c->device));
    st = c->s_lane[c->next_lane];
    c->next_lane = (c->next_lane + 1) % kLanes;
    size_t at = 0, o_in = 0, o_out = 0, o_rows = 0, o_tg = 0, o_fb = 0;
    auto take = [&](bool on, size_t bytes, size_t* o) { if (on) { *o = at; at = (at + bytes + 255) & ~(size_t)255; } };
    take(st_in, in_b, &o_in);
    take(st_out, out_b, &o_out);
    take(st_rows, rows_b, &o_rows);
    take(st_tg, tg_b, &o_tg);
    take(st_fb, fb_b, &o_fb);
    if (at) {
      CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&stage), at, st));
      if (st_in) d.in = stage + o_in;
      if (st_out) d.out = stage + o_out;
      if (st_rows) d.excluded = reinterpret_cast<const int16_t*>(stage + o_rows);
      if (st_tg) d.targets = stage + o_tg;
      if (st_fb) d.fallbacks = reinterpret_cast<int16_t*>(stage + o_fb);
    }
    int rc = 0;
    if (st_in && cudaMemcpyAsync(const_cast<void*>(d.in), x.in, in_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the requests failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc && st_rows &&
        cudaMemcpyAsync(const_cast<int16_t*>(d.excluded), x.excluded, rows_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the rows failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc && st_tg &&
        cudaMemcpyAsync(const_cast<uint8_t*>(d.targets), x.targets, tg_b, cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "%s: staging the targets failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
    if (!rc) rc = enqueue_excluding(c, *s, d, st);
    if (rc) {
      if (stage) cudaFreeAsync(stage, st);
      return rc;
    }
  }
  // the copies back wait for the kernel on the lane; they may block, so not under c->mu
  cudaError_t e = cudaSuccess;
  if (st_out) e = cudaMemcpyAsync(x.out, d.out, out_b, cudaMemcpyDeviceToHost, st);
  if (st_fb && e == cudaSuccess) e = cudaMemcpyAsync(x.fallbacks, d.fallbacks, fb_b, cudaMemcpyDeviceToHost, st);
  if (stage) cudaFreeAsync(stage, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(LIG_ERR_CUDA, "%s failed on the device: %s", fn, cudaGetErrorString(e));
  return 0;
}

int lig_schedule_batch_excluding(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                 const int16_t* excluded, int n_excluded, lig_pick* out) {
  return excluding_host(c, "lig_schedule_batch_excluding", epoch,
                        ExcludingCall{seed, reqs, R, out, n_excluded, excluded}, false);
}

int lig_schedule_models_batch_excluding(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                        const uint32_t* model_ids, const uint8_t* targets, int R,
                                        const int16_t* excluded, int n_excluded, lig_mpick* out) {
  return excluding_host(c, "lig_schedule_models_batch_excluding", epoch,
                        model_retry(seed, first_index, model_ids, targets, R, excluded, n_excluded, out), false);
}

int lig_schedule_batch_excluding_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                           const int16_t* excluded, int n_excluded, lig_pick* out,
                                           int n_fallbacks, int16_t* fallbacks) {
  return excluding_host(c, "lig_schedule_batch_excluding_fallbacks", epoch,
                        ExcludingCall{seed, reqs, R, out, n_excluded, excluded, n_fallbacks, fallbacks}, true);
}

int lig_schedule_models_batch_excluding_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                                  const uint32_t* model_ids, const uint8_t* targets, int R,
                                                  const int16_t* excluded, int n_excluded, lig_mpick* out,
                                                  int n_fallbacks, int16_t* fallbacks) {
  return excluding_host(c, "lig_schedule_models_batch_excluding_fallbacks", epoch,
                        model_retry(seed, first_index, model_ids, targets, R, excluded, n_excluded, out, n_fallbacks,
                                    fallbacks),
                        true);
}

int lig_pick_kernel_info(lig_ctx* c, uint64_t epoch, char* name, int name_len, int* grid, int* threads,
                         int* table_bytes, int* tables_in_smem) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_pick_kernel_info: ctx is null");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaEventSynchronize(s->ready));
  const bool tab = tables_fit_smem(c, *s, false);
  const char* nm = "lig_pick_queue_kernel";
  int g = 0, t = kPickThreads;
  if (c->pick_kernel == 0) {
    nm = "lig_pick_persistent_kernel";
    g = c->persist_grid[0][tab ? 1 : 0];
    t = persist_threads(c->tma_groups);
  } else if (c->pick_kernel == 1) {
    nm = "lig_pick_loop_kernel";
    g = c->loop_grid[tab ? 1 : 0];
    t = kLoopThreads;
  }
  if (name && name_len > 0) snprintf(name, (size_t)name_len, "%s", nm);
  if (grid) *grid = g;
  if (threads) *threads = t;
  if (table_bytes) *table_bytes = (int)s->h_hdr->bytes;
  if (tables_in_smem) *tables_in_smem = tab ? 1 : 0;
  return 0;
}

// ---- load feedback: the private scratch copy, its window loop, the in-batch call and the chain ----
// Both entry points schedule against fb_scratch, count the open window's picks in d_fb_hist and
// close a window by adding it to the scratch's WaitingQueueSize column; the in-batch call is a
// chain that starts and ends inside one call.  Everything below runs under c->fb_mu.
struct FbRun {
  int window = 1;                 // W
  int filled = 0;                 // requests in the open window
  bool stale = true;              // the scratch's tables predate the last closed window
  const FilterTree* tree = nullptr;
  Thr thr{};
  int32_t* d_total = nullptr;     // += every closed window (nullable)
  long long closed = 0;           // windows closed
};

static int fb_alloc_scratch(lig_ctx* c) {
  if (c->fb_scratch.d_blob) return 0;
  if (c->stream_open) return fail(LIG_ERR_INVALID, "cannot allocate the feedback scratch while a doorbell stream is open");
  if (int rc = alloc_slot(c, c->fb_scratch)) return rc;
  CUDA_TRY(cudaMalloc(&c->d_fb_hist, (size_t)c->max_pods * sizeof(int32_t)));
  CUDA_TRY(cudaMalloc(&c->d_fb_total, (size_t)c->max_pods * sizeof(int32_t)));
  CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&c->h_fb_loads), (size_t)c->max_pods * sizeof(int32_t),
                         cudaHostAllocMapped));
  CUDA_TRY(cudaStreamCreateWithFlags(&c->s_fb, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&c->fb_free, cudaEventDisableTiming));
  return 0;
}

// Copy resident slot s into the scratch on `st` (after the previous feedback call) and zero the
// open window.  Caller holds c->mu.
static int fb_copy_epoch(lig_ctx* c, Slot* s, cudaStream_t st) {
  Slot& fs = c->fb_scratch;
  CUDA_TRY(cudaStreamWaitEvent(st, c->fb_free, 0));         // an earlier feedback call on another stream
  CUDA_TRY(cudaStreamWaitEvent(st, s->ready, 0));
  fs.P = s->P;
  fs.A = s->A;
  fs.W = s->W;
  fs.n_ejected = s->n_ejected;                              // the private copy carries the pool
  CUDA_TRY(cudaMemcpyAsync(fs.d_blob, s->d_blob, layout_for(s->P, s->A).total, cudaMemcpyDeviceToDevice, st));
  if (s->n_ejected > 0)
    CUDA_TRY(cudaMemcpyAsync(fs.d_pool, s->d_pool, (size_t)s->W * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
  if (fs.P > 0) CUDA_TRY(cudaMemsetAsync(c->d_fb_hist, 0, (size_t)fs.P * sizeof(int32_t), st));
  return note_reader(*s, st);
}

// Close the open window: sum it over the ranks (communicator ctxs), add it to WaitingQueueSize
// (saturating) and to run.d_total, zero it.
static int fb_close_window(lig_ctx* c, FbRun& run, cudaStream_t st) {
  Slot& fs = c->fb_scratch;
  const int P = fs.P;
  if (P > 0) {
    if (c->comm && ligi::g_allreduce)                        // picks of this window on every rank
      if (int rc = ligi::g_allreduce(c, c->d_fb_hist, P, st)) return rc;
    int* q = reinterpret_cast<int*>(fs.d_blob + layout_for(fs.P, fs.A).q);
    lig_apply_feedback_kernel<<<(P + 255) / 256, 256, 0, st>>>(q, c->d_fb_hist, run.d_total, P);
    CUDA_TRY(cudaGetLastError());
    c->launches++;
  }
  run.filled = 0;
  run.stale = true;
  run.closed++;
  return 0;
}

// The requests of one feedback call (device-visible pointers): 16-byte descriptors in, lig_pick
// out; or 4-byte model ids in, lig_mpick out, request i with rand_key = first_index + i, resolved
// against a resident epoch's model table.
struct FbReqs {
  const void* in = nullptr;              // lig_req[R] or uint32_t[R]
  void* out = nullptr;                   // lig_pick[R] or lig_mpick[R]
  bool models = false;
  uint64_t first_index = 0;              // model ids: rand_key of request 0
  const unsigned char* mtab = nullptr;   // model ids: the model table (set by chain_call)
  uint32_t n_models = 0;
  bool rows = false;                     // a chain fallback call: request i's row is at
  int16_t* fallbacks = nullptr;          //   fallbacks + i * n_fallbacks
  int n_fallbacks = 0;
  bool retry = false;                    // a chain retry call: request i excludes the pods of
  const int16_t* excluded = nullptr;     //   excluded + i * n_excluded (with rows: a chain retry
  int n_excluded = 0;                    //   call with fallback rows)
  const uint8_t* targets = nullptr;      // a model-id retry call: request i's fixed target
  bool affinity = false;                 // a chain affinity call: no seed, no first_index; rows as
  const uint64_t* keys = nullptr;        //   above when n_fallbacks > 0; model ids: request i's key
  const uint64_t* hkeys = nullptr;       //   E's pod keys (set by chain_call)
  size_t in_bytes() const { return models ? sizeof(uint32_t) : sizeof(lig_req); }
  size_t out_bytes() const { return models ? sizeof(lig_mpick) : sizeof(lig_pick); }
};

// Schedule R requests through the window sequence: each segment is the rest of the open window or
// of the call, whichever is shorter; one fused pick + count launch per segment (pick + row + count
// when the call asked for rows, the affinity ranking + row + count for an affinity call); a filled
// window is closed at once, its tables are rebuilt only when the next segment needs them.  A retry
// segment (with or without rows) walks the tree over the scratch's pod columns and reads no class
// table: it leaves them stale, so a later table-reading segment rebuilds once.
static int fb_schedule(lig_ctx* c, FbRun& run, uint64_t seed, const FbReqs& rq, int R, cudaStream_t st) {
  Slot& fs = c->fb_scratch;
  for (int pos = 0; pos < R;) {
    const int n = (R - pos) < (run.window - run.filled) ? (R - pos) : (run.window - run.filled);
    if (!rq.retry) {
      std::lock_guard<std::mutex> lk(c->mu);                 // launch counters, build debug stamps
      if (run.stale) {
        if (int rc = launch_class_build(c, fs, st, run.tree, &run.thr)) return rc;
        run.stale = false;
      }
    }
    // the scratch's tables change every window: always the strided tables through L1 (no host
    // round trip for the compact header)
    const void* in = static_cast<const unsigned char*>(rq.in) + (size_t)pos * rq.in_bytes();
    void* out = static_cast<unsigned char*>(rq.out) + (size_t)pos * rq.out_bytes();
    const int grid = (n + kPickThreads * kCountPerThread - 1) / (kPickThreads * kCountPerThread);
    const uint4* fcls = reinterpret_cast<const uint4*>(fs.d_cls);
    if (rq.retry) {
      ExcludingCall x{seed, in, n, out, rq.n_excluded, rq.excluded + (size_t)pos * (size_t)rq.n_excluded};
      if (rq.rows) {
        x.n_fallbacks = rq.n_fallbacks;
        x.fallbacks = rq.fallbacks + (size_t)pos * (size_t)rq.n_fallbacks;
      }
      if (rq.models) {
        x.models = true;
        x.first_index = rq.first_index + (uint64_t)pos;
        x.targets = rq.targets + pos;
        x.mtab = rq.mtab;
        x.n_models = rq.n_models;
      }
      launch_excluding(c, fs, run.thr, run.tree, x, c->d_fb_hist, st);
    } else if (rq.affinity) {
      int16_t* rows = rq.rows ? rq.fallbacks + (size_t)pos * (size_t)rq.n_fallbacks : nullptr;
      const int blocks = (n + kFallbackThreads - 1) / kFallbackThreads;
      if (rq.models)
        lig_pick_affinity_kernel<true, true><<<blocks, kFallbackThreads, 0, st>>>(
            in, rq.keys + pos, out, rows, n, rq.n_fallbacks, fcls, fs.d_lists, fs.A, nullptr, rq.mtab, rq.n_models,
            rq.hkeys, c->d_fb_hist);
      else
        lig_pick_affinity_kernel<false, true><<<blocks, kFallbackThreads, 0, st>>>(
            in, nullptr, out, rows, n, rq.n_fallbacks, fcls, fs.d_lists, fs.A, nullptr, nullptr, 0u, rq.hkeys,
            c->d_fb_hist);
    } else if (rq.rows) {
      int16_t* rows = rq.fallbacks + (size_t)pos * (size_t)rq.n_fallbacks;
      const int blocks = (n + kFallbackThreads - 1) / kFallbackThreads;
      if (rq.models)
        lig_pick_fallback_kernel<true, true><<<blocks, kFallbackThreads, 0, st>>>(
            in, out, rows, n, rq.n_fallbacks, fcls, fs.d_lists, fs.A, nullptr, rq.mtab, rq.n_models, seed,
            rq.first_index + (uint64_t)pos, c->d_fb_hist);
      else
        lig_pick_fallback_kernel<false, true><<<blocks, kFallbackThreads, 0, st>>>(
            in, out, rows, n, rq.n_fallbacks, fcls, fs.d_lists, fs.A, nullptr, nullptr, 0u, seed, 0, c->d_fb_hist);
    } else if (rq.models)
      lig_pick_models_count_kernel<<<grid, kPickThreads, 0, st>>>(
          static_cast<const uint32_t*>(in), static_cast<uint32_t*>(out), n, reinterpret_cast<const uint4*>(fs.d_cls),
          fs.d_lists, fs.A, rq.mtab, rq.n_models, seed, rq.first_index + (uint64_t)pos, c->d_fb_hist);
    else
      lig_pick_count_kernel<<<grid, kPickThreads, 0, st>>>(
          static_cast<const int4*>(in), static_cast<int2*>(out), n, reinterpret_cast<const uint4*>(fs.d_cls),
          fs.d_lists, fs.A, seed, c->d_fb_hist);
    CUDA_TRY(cudaGetLastError());
    c->launches++;
    pos += n;
    run.filled += n;
    if (run.filled == run.window)
      if (int rc = fb_close_window(c, run, st)) return rc;
  }
  return 0;
}

int lig_schedule_batch_feedback_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                       int R, lig_pick* d_out, int sub_batch, int n_windows,
                                       int32_t* d_hist, void* stream) {
  if (!c || R < 0 || sub_batch < 1 || (R > 0 && (!d_reqs || !d_out)))
    return fail(LIG_ERR_INVALID, "lig_schedule_batch_feedback_device: bad argument");
  if (n_windows <= 0) n_windows = (R + sub_batch - 1) / sub_batch;
  if ((long long)n_windows * sub_batch < R)
    return fail(LIG_ERR_INVALID, "n_windows=%d x sub_batch=%d does not cover R=%d", n_windows, sub_batch, R);
  // the tree and thresholds in force when the call starts rebuild every window's tables
  FbRun run;
  FilterTree tree;
  {
    std::lock_guard<std::mutex> uk(c->upload_mu);
    if (c->has_tree) {
      tree = c->tree;
      run.tree = &tree;
    }
    run.thr = thr_of(c);
  }
  run.window = sub_batch;
  run.d_total = d_hist;
  std::lock_guard<std::mutex> fk(c->fb_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = fb_alloc_scratch(c)) return rc;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    Slot* s = nullptr;
    if (int rc = resolve_slot(c, epoch, &s)) return rc;
    c->chain_live = false;                                    // the scratch is reused: any chain ends
    if (int rc = fb_copy_epoch(c, s, st)) return rc;
  }
  const int P = c->fb_scratch.P;
  if (d_hist && P > 0) CUDA_TRY(cudaMemsetAsync(d_hist, 0, (size_t)P * sizeof(int32_t), st));
  FbReqs rq;
  rq.in = d_reqs;
  rq.out = d_out;
  if (int rc = fb_schedule(c, run, seed, rq, R, st)) return rc;
  // the last, partial window, then the trailing empty ones (their all-reduce still carries the
  // picks of the other ranks)
  if (run.filled > 0)
    if (int rc = fb_close_window(c, run, st)) return rc;
  while (run.closed < n_windows)
    if (int rc = fb_close_window(c, run, st)) return rc;
  CUDA_TRY(cudaEventRecord(c->fb_free, st));
  return 0;
}

// One chain call (device-visible buffers, enqueued on `st`).  `d_loads` (nullable) receives the
// chain's loads on the device.  Caller holds c->fb_mu, so no other call changes the chain meanwhile.
// Model ids are resolved against E's resident model table, which the chain never copies: a model
// upload does not restart the chain.  The call holds upload_mu until it is enqueued, so that no
// upload replaces the table between the resolve and the last launch, and registers as a reader of
// E's slot, so that a later upload waits for the launches before it overwrites the table.  An
// affinity call reads E's pod keys the same way: a pod-key upload does not restart the chain either.
static int chain_call(lig_ctx* c, uint64_t epoch, uint64_t seed, FbReqs rq, int R, int window, int32_t* d_loads,
                      cudaStream_t st) {
  std::unique_lock<std::mutex> held(c->upload_mu, std::defer_lock);
  const bool reads_slot = rq.models || rq.affinity;             // E's model table or pod keys
  if (reads_slot) held.lock();
  // A chain (re)starts when it is not live, on another epoch or another upload of it (the next
  // scrape supersedes the estimate), or with another window size.  The tree and thresholds in
  // force at the start rebuild every window of the chain.  The tree is read under upload_mu, which
  // is taken before mu: a start reads it first, then checks that the upload it copies is still the
  // one it read the tree for.
  FilterTree tree;
  bool has_tree = false, have_tree = false;
  Thr thr{};
  uint64_t tree_stamp = 0;
  Slot* s = nullptr;
  for (;;) {
    uint64_t stamp = 0;
    {
      std::lock_guard<std::mutex> lk(c->mu);
      // refused (stale epoch, no model table, no pod keys): the chain is untouched
      if (int rc = rq.models ? resolve_models_slot(c, epoch, &s) : resolve_slot(c, epoch, &s)) return rc;
      if (rq.affinity && !s->keys_valid)
        return fail(LIG_ERR_NO_SNAPSHOT, "no pod keys uploaded for epoch %llu (lig_upload_pod_keys)",
                    (unsigned long long)epoch);
      const bool restart = !c->chain_live || c->chain_epoch != epoch || c->chain_stamp != s->stamp ||
                           c->chain_window != window;
      if (!restart) {
        c->chain_live = false;                                // until this call is enqueued
        CUDA_TRY(cudaStreamWaitEvent(st, c->fb_free, 0));     // the chain's previous call, any stream
        break;
      }
      if (have_tree && tree_stamp == s->stamp) {
        c->chain_live = false;
        c->chain_has_tree = has_tree;
        if (has_tree) c->chain_tree = tree;
        c->chain_thr = thr;
        c->chain_epoch = epoch;
        c->chain_stamp = s->stamp;
        c->chain_window = window;
        c->chain_filled = 0;
        c->chain_stale = true;
        if (int rc = fb_copy_epoch(c, s, st)) return rc;
        if (s->P > 0) CUDA_TRY(cudaMemsetAsync(c->d_fb_total, 0, (size_t)s->P * sizeof(int32_t), st));
        break;
      }
      stamp = s->stamp;
    }
    {
      std::unique_lock<std::mutex> uk(c->upload_mu, std::defer_lock);
      if (!held) uk.lock();
      has_tree = c->has_tree;
      if (has_tree) tree = c->tree;
      thr = thr_of(c);
    }
    have_tree = true;
    tree_stamp = stamp;
  }
  if (reads_slot) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (rq.models) {
      CUDA_TRY(cudaStreamWaitEvent(st, s->models_ready, 0));
      rq.mtab = s->d_mtab;
      rq.n_models = s->n_models;
    }
    if (rq.affinity) {
      CUDA_TRY(cudaStreamWaitEvent(st, s->keys_ready, 0));
      rq.hkeys = s->d_podkeys;
    }
  }
  FbRun run;
  run.window = window;
  run.filled = c->chain_filled;
  run.stale = c->chain_stale;
  run.tree = c->chain_has_tree ? &c->chain_tree : nullptr;
  run.thr = c->chain_thr;
  run.d_total = c->d_fb_total;
  if (int rc = fb_schedule(c, run, seed, rq, R, st)) return rc;
  if (reads_slot) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (int rc = note_reader(*s, st)) return rc;
  }
  const int P = c->fb_scratch.P;
  if (d_loads && P > 0) {
    lig_feedback_loads_kernel<<<(P + 255) / 256, 256, 0, st>>>(c->d_fb_total, c->d_fb_hist, d_loads, P);
    CUDA_TRY(cudaGetLastError());
    c->launches++;
  }
  CUDA_TRY(cudaEventRecord(c->fb_free, st));
  c->chain_filled = run.filled;
  c->chain_stale = run.stale;
  c->chain_live = true;
  return 0;
}

// Checks shared by both chain forms, before anything is touched.  Caller holds c->fb_mu.
static int chain_admit(lig_ctx* c, const char* fn) {
  if (c->comm)
    return fail(LIG_ERR_INVALID, "%s: a ctx with a communicator has no feedback chain (per-rank micro-batch "
                                 "streams share no window boundaries)", fn);
  return fb_alloc_scratch(c);
}

// The row arguments of a chain fallback or retry call, both sets for a retry call with fallback rows,
// and the rows and keys of a chain affinity call; 0 for a plain chain call.
static int chain_rows_check(const char* fn, const FbReqs& rq, int R) {
  if (rq.retry) {
    if (rq.n_excluded < 1 || rq.n_excluded > LIG_MAX_EXCLUDED)
      return fail(LIG_ERR_INVALID, "%s: n_excluded=%d outside [1, %d]", fn, rq.n_excluded, LIG_MAX_EXCLUDED);
    if (R > 0 && (!rq.excluded || (rq.models && !rq.targets))) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  }
  if (rq.affinity) {                                          // n_fallbacks = 0: no row
    if (rq.n_fallbacks < 0 || rq.n_fallbacks > LIG_MAX_FALLBACKS)
      return fail(LIG_ERR_INVALID, "%s: n_fallbacks=%d outside [0, %d]", fn, rq.n_fallbacks, LIG_MAX_FALLBACKS);
    if (R > 0 && rq.models && !rq.keys) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  }
  if (!rq.rows) return 0;
  if (rq.n_fallbacks < 1 || rq.n_fallbacks > LIG_MAX_FALLBACKS)
    return fail(LIG_ERR_INVALID, "%s: n_fallbacks=%d outside [1, %d]", fn, rq.n_fallbacks, LIG_MAX_FALLBACKS);
  if (R > 0 && !rq.fallbacks) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  return 0;
}

// The device form of every chain call.
static int chain_device(lig_ctx* c, const char* fn, uint64_t epoch, uint64_t seed, const FbReqs& rq, int R,
                        int window, int32_t* d_loads, void* stream) {
  if (!c || R < 0 || window < 1 || (R > 0 && (!rq.in || !rq.out))) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  if (int rc = chain_rows_check(fn, rq, R)) return rc;
  if (R > 0 && rq.rows && misaligned(rq.fallbacks, sizeof(int16_t)))
    return fail(LIG_ERR_INVALID, "%s: the row buffer is not 2-byte aligned", fn);
  if (R > 0 && (rq.retry || rq.affinity) &&
      (misaligned(rq.in, rq.in_bytes()) || misaligned(rq.out, rq.out_bytes()) ||
       misaligned(rq.excluded, sizeof(int16_t)) || misaligned(rq.keys, sizeof(uint64_t))))
    return fail(LIG_ERR_INVALID, "%s: a device buffer is not aligned to its element", fn);
  std::lock_guard<std::mutex> fk(c->fb_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  if (int rc = chain_admit(c, fn)) return rc;
  return chain_call(c, epoch, seed, rq, R, window, d_loads, static_cast<cudaStream_t>(stream));
}

// The host form of both chain calls (rq holds the caller's host buffers); blocks.
static int chain_host(lig_ctx* c, const char* fn, uint64_t epoch, uint64_t seed, FbReqs rq, int R, int window,
                      int32_t* loads) {
  if (!c || R < 0 || window < 1 || (R > 0 && (!rq.in || !rq.out))) return fail(LIG_ERR_INVALID, "%s: bad argument", fn);
  if (int rc = chain_rows_check(fn, rq, R)) return rc;
  if (R > c->max_batch) return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, c->max_batch);
  // as lig_schedule_batch: page-locked buffers are read and written in place, pageable ones (and
  // inputs not aligned to their element) bounce (4-byte model ids and picks fit the 16-byte /
  // 8-byte bounce buffers)
  const void* in = rq.in;
  void* out = rq.out;
  rq.in = R ? mapped_device_pointer(in) : nullptr;
  rq.out = R ? mapped_device_pointer(out) : nullptr;
  const bool bounce = R > 0 && !(rq.in && rq.out && !(reinterpret_cast<uintptr_t>(rq.in) & (rq.in_bytes() - 1)) &&
                                 !((rq.retry || rq.affinity) && misaligned(rq.out, rq.out_bytes())));
  std::unique_lock<std::mutex> bk(c->bounce_mu, std::defer_lock);
  if (bounce) {
    bk.lock();
    rq.in = mapped_device_pointer(c->h_reqs);
    rq.out = mapped_device_pointer(c->h_out);
    if (!rq.in || !rq.out)
      return fail(LIG_ERR_CUDA, "pinned staging buffers are not device-mapped on this platform");
    memcpy(c->h_reqs, in, (size_t)R * rq.in_bytes());
  }
  // rows: page-locked, 2-byte aligned ones are written in place, the others staged in h_fb_rows
  int16_t* rows_back = nullptr;                               // the caller's rows, when staged
  if (R > 0 && rq.rows) {
    int16_t* rows = rq.fallbacks;
    rq.fallbacks = mapped_device_pointer(rows);
    if (!rq.fallbacks || misaligned(rq.fallbacks, sizeof(int16_t))) {
      if (!bk.owns_lock()) bk.lock();
      if (!c->h_fb_rows) {
        CUDA_TRY(cudaSetDevice(c->device));
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&c->h_fb_rows),
                               (size_t)c->max_batch * LIG_MAX_FALLBACKS * sizeof(int16_t), cudaHostAllocMapped));
      }
      if (!(rq.fallbacks = mapped_device_pointer(c->h_fb_rows)))
        return fail(LIG_ERR_CUDA, "pinned staging buffers are not device-mapped on this platform");
      rows_back = rows;
    }
  }
  std::lock_guard<std::mutex> fk(c->fb_mu);
  CUDA_TRY(cudaSetDevice(c->device));
  if (int rc = chain_admit(c, fn)) return rc;
  int32_t* dev_loads = loads ? mapped_device_pointer(loads) : nullptr;
  const bool loads_bounce = loads && !dev_loads;
  if (loads_bounce && !(dev_loads = mapped_device_pointer(c->h_fb_loads)))
    return fail(LIG_ERR_CUDA, "pinned staging buffers are not device-mapped on this platform");
  // retry rows: page-locked, 2-byte aligned ones are read in place, the others staged in
  // stream-ordered HBM (as lig_schedule_batch_excluding does); so are the targets of a model-id retry
  int16_t* stage = nullptr;
  if (R > 0 && rq.retry) {
    const int16_t* rows = rq.excluded;
    rq.excluded = mapped_device_pointer(rows);
    if (!rq.excluded || misaligned(rq.excluded, sizeof(int16_t))) {
      const size_t rows_b = (size_t)R * (size_t)rq.n_excluded * sizeof(int16_t);
      CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&stage), rows_b, c->s_fb));
      if (cudaMemcpyAsync(stage, rows, rows_b, cudaMemcpyHostToDevice, c->s_fb) != cudaSuccess) {
        cudaFreeAsync(stage, c->s_fb);
        return fail(LIG_ERR_CUDA, "%s: staging the rows failed: %s", fn, cudaGetErrorString(cudaGetLastError()));
      }
      rq.excluded = stage;
    }
  }
  uint8_t* stage_tg = nullptr;
  if (R > 0 && rq.retry && rq.models) {
    const uint8_t* tg = rq.targets;
    if (!(rq.targets = mapped_device_pointer(tg))) {
      cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&stage_tg), (size_t)R, c->s_fb);
      if (e == cudaSuccess) e = cudaMemcpyAsync(stage_tg, tg, (size_t)R, cudaMemcpyHostToDevice, c->s_fb);
      if (e != cudaSuccess) {
        if (stage_tg) cudaFreeAsync(stage_tg, c->s_fb);
        if (stage) cudaFreeAsync(stage, c->s_fb);
        return fail(LIG_ERR_CUDA, "%s: staging the targets failed: %s", fn, cudaGetErrorString(e));
      }
      rq.targets = stage_tg;
    }
  }
  // affinity keys of model ids: page-locked, 8-byte aligned ones are read in place, the others staged
  // in stream-ordered HBM like the retry rows
  uint64_t* stage_keys = nullptr;
  if (R > 0 && rq.affinity && rq.models) {
    const uint64_t* keys = rq.keys;
    rq.keys = mapped_device_pointer(keys);
    if (!rq.keys || misaligned(rq.keys, sizeof(uint64_t))) {
      const size_t keys_b = (size_t)R * sizeof(uint64_t);
      cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&stage_keys), keys_b, c->s_fb);
      if (e == cudaSuccess) e = cudaMemcpyAsync(stage_keys, keys, keys_b, cudaMemcpyHostToDevice, c->s_fb);
      if (e != cudaSuccess) {
        if (stage_keys) cudaFreeAsync(stage_keys, c->s_fb);
        return fail(LIG_ERR_CUDA, "%s: staging the keys failed: %s", fn, cudaGetErrorString(e));
      }
      rq.keys = stage_keys;
    }
  }
  const int rc = chain_call(c, epoch, seed, rq, R, window, dev_loads, c->s_fb);
  if (stage) cudaFreeAsync(stage, c->s_fb);
  if (stage_tg) cudaFreeAsync(stage_tg, c->s_fb);
  if (stage_keys) cudaFreeAsync(stage_keys, c->s_fb);
  if (rc) return rc;
  const cudaError_t e = cudaStreamSynchronize(c->s_fb);
  if (e != cudaSuccess) {
    c->chain_live = false;
    return fail(LIG_ERR_CUDA, "feedback chain call failed on the device: %s", cudaGetErrorString(e));
  }
  if (bounce) memcpy(out, c->h_out, (size_t)R * rq.out_bytes());
  if (rows_back) memcpy(rows_back, c->h_fb_rows, (size_t)R * (size_t)rq.n_fallbacks * sizeof(int16_t));
  if (loads_bounce && c->fb_scratch.P > 0)
    memcpy(loads, c->h_fb_loads, (size_t)c->fb_scratch.P * sizeof(int32_t));
  return 0;
}

static FbReqs descriptor_reqs(const lig_req* in, lig_pick* out) {
  FbReqs rq;
  rq.in = in;
  rq.out = out;
  return rq;
}

static FbReqs model_reqs(const uint32_t* ids, lig_mpick* out, uint64_t first_index) {
  FbReqs rq;
  rq.in = ids;
  rq.out = out;
  rq.models = true;
  rq.first_index = first_index;
  return rq;
}

static FbReqs with_rows(FbReqs rq, int n_fallbacks, int16_t* fallbacks) {
  rq.rows = true;
  rq.n_fallbacks = n_fallbacks;
  rq.fallbacks = fallbacks;
  return rq;
}

int lig_schedule_batch_feedback_chain_device(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* d_reqs,
                                             int R, lig_pick* d_out, int window, int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_batch_feedback_chain_device", epoch, seed, descriptor_reqs(d_reqs, d_out), R,
                      window, d_loads, stream);
}

int lig_schedule_batch_feedback_chain(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                                      lig_pick* out, int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_batch_feedback_chain", epoch, seed, descriptor_reqs(reqs, out), R, window,
                    loads);
}

int lig_schedule_models_batch_feedback_chain_device(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                                    const uint32_t* d_ids, int R, lig_mpick* d_out, int window,
                                                    int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_models_batch_feedback_chain_device", epoch, seed,
                      model_reqs(d_ids, d_out, first_index), R, window, d_loads, stream);
}

int lig_schedule_models_batch_feedback_chain(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                                             const uint32_t* ids, int R, lig_mpick* out, int window,
                                             int32_t* loads) {
  return chain_host(c, "lig_schedule_models_batch_feedback_chain", epoch, seed, model_reqs(ids, out, first_index), R,
                    window, loads);
}

int lig_schedule_batch_feedback_chain_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                                                int R, lig_pick* out, int n_fallbacks, int16_t* fallbacks,
                                                int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_batch_feedback_chain_fallbacks", epoch, seed,
                    with_rows(descriptor_reqs(reqs, out), n_fallbacks, fallbacks), R, window, loads);
}

int lig_schedule_batch_feedback_chain_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                       const lig_req* d_reqs, int R, lig_pick* d_out,
                                                       int n_fallbacks, int16_t* d_fallbacks, int window,
                                                       int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_batch_feedback_chain_fallbacks_device", epoch, seed,
                      with_rows(descriptor_reqs(d_reqs, d_out), n_fallbacks, d_fallbacks), R, window, d_loads,
                      stream);
}

int lig_schedule_models_batch_feedback_chain_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                       uint64_t first_index, const uint32_t* ids, int R,
                                                       lig_mpick* out, int n_fallbacks, int16_t* fallbacks,
                                                       int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_models_batch_feedback_chain_fallbacks", epoch, seed,
                    with_rows(model_reqs(ids, out, first_index), n_fallbacks, fallbacks), R, window, loads);
}

int lig_schedule_models_batch_feedback_chain_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                              uint64_t first_index, const uint32_t* d_ids, int R,
                                                              lig_mpick* d_out, int n_fallbacks,
                                                              int16_t* d_fallbacks, int window, int32_t* d_loads,
                                                              void* stream) {
  return chain_device(c, "lig_schedule_models_batch_feedback_chain_fallbacks_device", epoch, seed,
                      with_rows(model_reqs(d_ids, d_out, first_index), n_fallbacks, d_fallbacks), R, window,
                      d_loads, stream);
}

// n_fallbacks outside [0, LIG_MAX_FALLBACKS] is refused by chain_rows_check
static FbReqs with_affinity(FbReqs rq, const uint64_t* keys, int n_fallbacks, int16_t* fallbacks) {
  if (n_fallbacks != 0) rq = with_rows(rq, n_fallbacks, fallbacks);
  rq.n_fallbacks = n_fallbacks;
  rq.affinity = true;
  rq.keys = keys;
  return rq;
}

int lig_schedule_batch_feedback_chain_affinity(lig_ctx* c, uint64_t epoch, const lig_req* reqs, int R, lig_pick* out,
                                               int n_fallbacks, int16_t* fallbacks, int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_batch_feedback_chain_affinity", epoch, 0,
                    with_affinity(descriptor_reqs(reqs, out), nullptr, n_fallbacks, fallbacks), R, window, loads);
}

int lig_schedule_batch_feedback_chain_affinity_device(lig_ctx* c, uint64_t epoch, const lig_req* d_reqs, int R,
                                                      lig_pick* d_out, int n_fallbacks, int16_t* d_fallbacks,
                                                      int window, int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_batch_feedback_chain_affinity_device", epoch, 0,
                      with_affinity(descriptor_reqs(d_reqs, d_out), nullptr, n_fallbacks, d_fallbacks), R, window,
                      d_loads, stream);
}

int lig_schedule_models_batch_feedback_chain_affinity(lig_ctx* c, uint64_t epoch, const uint32_t* model_ids,
                                                      const uint64_t* keys, int R, lig_mpick* out, int n_fallbacks,
                                                      int16_t* fallbacks, int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_models_batch_feedback_chain_affinity", epoch, 0,
                    with_affinity(model_reqs(model_ids, out, 0), keys, n_fallbacks, fallbacks), R, window, loads);
}

int lig_schedule_models_batch_feedback_chain_affinity_device(lig_ctx* c, uint64_t epoch, const uint32_t* d_model_ids,
                                                             const uint64_t* d_keys, int R, lig_mpick* d_out,
                                                             int n_fallbacks, int16_t* d_fallbacks, int window,
                                                             int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_models_batch_feedback_chain_affinity_device", epoch, 0,
                      with_affinity(model_reqs(d_model_ids, d_out, 0), d_keys, n_fallbacks, d_fallbacks), R, window,
                      d_loads, stream);
}

static FbReqs with_excluded(FbReqs rq, const int16_t* excluded, int n_excluded) {
  rq.retry = true;
  rq.excluded = excluded;
  rq.n_excluded = n_excluded;
  return rq;
}

int lig_schedule_batch_feedback_chain_excluding(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs,
                                                int R, const int16_t* excluded, int n_excluded, lig_pick* out,
                                                int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_batch_feedback_chain_excluding", epoch, seed,
                    with_excluded(descriptor_reqs(reqs, out), excluded, n_excluded), R, window, loads);
}

int lig_schedule_batch_feedback_chain_excluding_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                       const lig_req* d_reqs, int R, const int16_t* d_excluded,
                                                       int n_excluded, lig_pick* d_out, int window,
                                                       int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_batch_feedback_chain_excluding_device", epoch, seed,
                      with_excluded(descriptor_reqs(d_reqs, d_out), d_excluded, n_excluded), R, window, d_loads,
                      stream);
}

int lig_schedule_batch_feedback_chain_excluding_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                          const lig_req* reqs, int R, const int16_t* excluded,
                                                          int n_excluded, lig_pick* out, int n_fallbacks,
                                                          int16_t* fallbacks, int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_batch_feedback_chain_excluding_fallbacks", epoch, seed,
                    with_rows(with_excluded(descriptor_reqs(reqs, out), excluded, n_excluded), n_fallbacks, fallbacks),
                    R, window, loads);
}

int lig_schedule_batch_feedback_chain_excluding_fallbacks_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                                 const lig_req* d_reqs, int R,
                                                                 const int16_t* d_excluded, int n_excluded,
                                                                 lig_pick* d_out, int n_fallbacks,
                                                                 int16_t* d_fallbacks, int window,
                                                                 int32_t* d_loads, void* stream) {
  return chain_device(c, "lig_schedule_batch_feedback_chain_excluding_fallbacks_device", epoch, seed,
                      with_rows(with_excluded(descriptor_reqs(d_reqs, d_out), d_excluded, n_excluded), n_fallbacks,
                                d_fallbacks),
                      R, window, d_loads, stream);
}

static FbReqs with_targets(FbReqs rq, const uint8_t* targets) {
  rq.targets = targets;
  return rq;
}

int lig_schedule_models_batch_feedback_chain_excluding(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                       uint64_t first_index, const uint32_t* model_ids,
                                                       const uint8_t* targets, int R, const int16_t* excluded,
                                                       int n_excluded, lig_mpick* out, int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_models_batch_feedback_chain_excluding", epoch, seed,
                    with_targets(with_excluded(model_reqs(model_ids, out, first_index), excluded, n_excluded), targets),
                    R, window, loads);
}

int lig_schedule_models_batch_feedback_chain_excluding_device(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                              uint64_t first_index, const uint32_t* d_model_ids,
                                                              const uint8_t* d_targets, int R,
                                                              const int16_t* d_excluded, int n_excluded,
                                                              lig_mpick* d_out, int window, int32_t* d_loads,
                                                              void* stream) {
  return chain_device(c, "lig_schedule_models_batch_feedback_chain_excluding_device", epoch, seed,
                      with_targets(with_excluded(model_reqs(d_model_ids, d_out, first_index), d_excluded, n_excluded),
                                   d_targets),
                      R, window, d_loads, stream);
}

int lig_schedule_models_batch_feedback_chain_excluding_fallbacks(lig_ctx* c, uint64_t epoch, uint64_t seed,
                                                                 uint64_t first_index, const uint32_t* model_ids,
                                                                 const uint8_t* targets, int R,
                                                                 const int16_t* excluded, int n_excluded,
                                                                 lig_mpick* out, int n_fallbacks, int16_t* fallbacks,
                                                                 int window, int32_t* loads) {
  return chain_host(c, "lig_schedule_models_batch_feedback_chain_excluding_fallbacks", epoch, seed,
                    with_rows(with_targets(with_excluded(model_reqs(model_ids, out, first_index), excluded, n_excluded),
                                           targets),
                              n_fallbacks, fallbacks),
                    R, window, loads);
}

int lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device(
    lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index, const uint32_t* d_model_ids,
    const uint8_t* d_targets, int R, const int16_t* d_excluded, int n_excluded, lig_mpick* d_out, int n_fallbacks,
    int16_t* d_fallbacks, int window, int32_t* d_loads, void* stream) {
  return chain_device(
      c, "lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device", epoch, seed,
      with_rows(with_targets(with_excluded(model_reqs(d_model_ids, d_out, first_index), d_excluded, n_excluded),
                             d_targets),
                n_fallbacks, d_fallbacks),
      R, window, d_loads, stream);
}

int lig_feedback_chain_reset(lig_ctx* c) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_feedback_chain_reset: ctx is null");
  std::lock_guard<std::mutex> fk(c->fb_mu);
  c->chain_live = false;
  return 0;
}

int lig_read_class(lig_ctx* c, uint64_t epoch, int critical, int adapter_id, int* status,
                   int* n_survivors, uint16_t* list) {
  if (!c || !status || !n_survivors) return fail(LIG_ERR_INVALID, "lig_read_class: null argument");
  std::lock_guard<std::mutex> lk(c->mu);
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaEventSynchronize(s->ready));
  const int a = (adapter_id >= 0 && adapter_id < s->A) ? adapter_id : s->A;
  const int cls = (critical ? 1 : 0) * (s->A + 1) + a;
  ClassEntry e;
  CUDA_TRY(cudaMemcpy(&e, s->d_cls + cls, sizeof(e), cudaMemcpyDeviceToHost));
  *n_survivors = (int)entry_n(e.info);
  *status = (int)entry_status(e.info);
  if (list && *n_survivors > 0)
    CUDA_TRY(cudaMemcpy(list, s->d_lists + e.list_off, (size_t)*n_survivors * sizeof(uint16_t),
                        cudaMemcpyDeviceToHost));
  return 0;
}

void* lig_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  // Place the pages on the NUMA node the current CUDA device hangs off: the pick kernel reads and
  // writes these buffers over PCIe in place, and a remote node adds an inter-socket hop to every
  // transaction.  Best effort (a sandbox may refuse set_mempolicy): LIG_NUMA=0 turns it off.
  NumaBind bind;
  cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable);
  if (e != cudaSuccess) {
    cudaGetLastError();
    fail(LIG_ERR_CUDA, "cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return nullptr;
  }
  register_pinned(p, bytes);
  return p;
}

void lig_host_free(void* p) {
  if (!p) return;
  unregister_pinned(p);
  cudaFreeHost(p);
}

int lig_stream_capacity(void) { return kMailboxCapacity; }

int lig_stream_open(lig_ctx* c) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_stream_open: ctx is null");
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->stream_open) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  if (!c->mailbox) {
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&c->mailbox), sizeof(Mailbox), cudaHostAllocMapped));
    CUDA_TRY(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->d_mailbox), c->mailbox, 0));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->s_doorbell, cudaStreamNonBlocking));
  }
  return doorbell_launch(c);
}

int lig_stream_close(lig_ctx* c) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_stream_close: ctx is null");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->stream_open) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  return doorbell_stop(c);
}

// Ring the doorbell for the micro-batch the caller wrote into the mailbox and spin until the
// resident kernel has answered.  Called with upload_mu and mu held.
static int doorbell_round_trip(lig_ctx* c) {
  Mailbox* mb = c->mailbox;
  const uint32_t ticket = c->next_ticket++;
  reinterpret_cast<std::atomic<uint32_t>*>(&mb->ticket)->store(ticket, std::memory_order_release);
  auto* done = reinterpret_cast<std::atomic<uint32_t>*>(&mb->done);
  uint64_t spins = 0;
  while (done->load(std::memory_order_acquire) != ticket) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
    if ((++spins & 0xfffff) == 0 && cudaStreamQuery(c->s_doorbell) != cudaErrorNotReady) {
      c->stream_open = false;   // the resident kernel is gone (error or device reset)
      return fail(LIG_ERR_CUDA, "doorbell kernel is not running: %s", cudaGetErrorString(cudaGetLastError()));
    }
  }
  return 0;
}

int lig_stream_submit(lig_ctx* c, uint64_t epoch, uint64_t seed, const lig_req* reqs, int n,
                      lig_pick* out) {
  if (!c || n < 0 || (n > 0 && (!reqs || !out)))
    return fail(LIG_ERR_INVALID, "lig_stream_submit: bad argument");
  if (n > kMailboxCapacity)
    return fail(LIG_ERR_INVALID, "n=%d exceeds the doorbell capacity %d", n, kMailboxCapacity);
  // one doorbell round trip at a time: the single mailbox is the resource, and a snapshot upload
  // must not overwrite the slot while the resident kernel reads it (it is not in any reader ring)
  std::lock_guard<std::mutex> uk(c->upload_mu);
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->stream_open) return fail(LIG_ERR_INVALID, "lig_stream_submit: call lig_stream_open first");
  Slot* s = nullptr;
  if (int rc = resolve_slot(c, epoch, &s)) return rc;
  if (n == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  // the tables of this slot must be complete before the resident kernel reads them; uploads
  // through the host API have already synchronised, device-side uploads are waited for here
  CUDA_TRY(cudaEventSynchronize(s->ready));
  Mailbox* mb = c->mailbox;
  memcpy(mb->reqs, reqs, (size_t)n * sizeof(lig_req));
  mb->count = (uint32_t)n;
  mb->A = (uint32_t)s->A;
  mb->mode = kMailboxDescriptors;
  mb->seed = seed;
  mb->cls = reinterpret_cast<const uint4*>(s->d_cls);
  mb->lists = s->d_lists;
  if (int rc = doorbell_round_trip(c)) return rc;
  memcpy(out, mb->picks, (size_t)n * sizeof(lig_pick));
  return 0;
}

int lig_stream_submit_models(lig_ctx* c, uint64_t epoch, uint64_t seed, uint64_t first_index,
                             const uint32_t* ids, int n, lig_mpick* out) {
  if (!c || n < 0 || (n > 0 && (!ids || !out)))
    return fail(LIG_ERR_INVALID, "lig_stream_submit_models: bad argument");
  if (n > kMailboxCapacity)
    return fail(LIG_ERR_INVALID, "n=%d exceeds the doorbell capacity %d", n, kMailboxCapacity);
  // upload_mu for the whole round trip, as above: lig_upload_models takes it too, so the model
  // table cannot be rewritten while the resident kernel reads it
  std::lock_guard<std::mutex> uk(c->upload_mu);
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->stream_open) return fail(LIG_ERR_INVALID, "lig_stream_submit_models: call lig_stream_open first");
  Slot* s = nullptr;
  if (int rc = resolve_models_slot(c, epoch, &s)) return rc;
  if (n == 0) return 0;
  CUDA_TRY(cudaSetDevice(c->device));
  CUDA_TRY(cudaEventSynchronize(s->ready));
  CUDA_TRY(cudaEventSynchronize(s->models_ready));   // an _async model upload may still be in flight
  Mailbox* mb = c->mailbox;
  memcpy(mb->reqs, ids, (size_t)n * sizeof(uint32_t));
  mb->count = (uint32_t)n;
  mb->A = (uint32_t)s->A;
  mb->mode = kMailboxModels;
  mb->seed = seed;
  mb->cls = reinterpret_cast<const uint4*>(s->d_cls);
  mb->lists = s->d_lists;
  mb->mtab = s->d_mtab;
  mb->first_index = first_index;
  mb->n_models = s->n_models;
  if (int rc = doorbell_round_trip(c)) return rc;
  memcpy(out, mb->picks, (size_t)n * sizeof(lig_mpick));
  return 0;
}

uint64_t lig_kernel_launches(const lig_ctx* c) { return c ? c->launches.load() : 0; }

int lig_last_pick_launch(lig_ctx* c, lig_launch_info* info) {
  if (!c || !info) return fail(LIG_ERR_INVALID, "lig_last_pick_launch: null argument");
  std::lock_guard<std::mutex> lk(c->mu);
  *info = c->last_pick;
  return 0;
}
int lig_sm_count(const lig_ctx* c) { return c ? c->sm_count : 0; }

}  // extern "C"
