// lig_multi.cpp — several GPUs behind the C ABI: lig_group_* (one process owns all devices, the
// reference's wiring: ONE scheduler per ext-proc process, pkg/ext-proc/main.go:137) and lig_comm_*
// (one process per GPU, torchrun-style).
//
// The path shards BY REQUEST: decisions are independent given a frozen snapshot (Schedule never
// mutates pod metrics, pkg/ext-proc/scheduling/scheduler.go:113-122).  The only exchange step is
// the replication of the packed snapshot once per refresh tick: one ncclBroadcast over
// NVLink/NVSwitch whose receive buffer IS each member's resident snapshot slot, so the class-table
// build consumes it in place on the same stream.  Picks need no collective.
//
// NCCL is bound at run time (dlopen "libnccl.so.2"): when the host process already carries an
// NCCL (e.g. the one bundled with PyTorch) that copy is reused, otherwise the system library is
// loaded.  A single-GPU deployment needs no NCCL at all.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

#include "lig_internal.hpp"

using ligi::fail;

namespace {

struct NcclApi {
  bool ok = false;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi g_nccl;
std::once_flag g_nccl_once;
char g_nccl_why[256] = "";

void load_nccl() {
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) {
    snprintf(g_nccl_why, sizeof(g_nccl_why), "dlopen(libnccl.so.2) failed: %s", dlerror());
    return;
  }
  auto sym = [&](const char* name) -> void* {
    void* p = dlsym(h, name);
    if (!p && !g_nccl_why[0]) snprintf(g_nccl_why, sizeof(g_nccl_why), "libnccl has no %s", name);
    return p;
  };
  g_nccl.GetUniqueId = reinterpret_cast<decltype(g_nccl.GetUniqueId)>(sym("ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<decltype(g_nccl.CommInitRank)>(sym("ncclCommInitRank"));
  g_nccl.CommInitAll = reinterpret_cast<decltype(g_nccl.CommInitAll)>(sym("ncclCommInitAll"));
  g_nccl.CommDestroy = reinterpret_cast<decltype(g_nccl.CommDestroy)>(sym("ncclCommDestroy"));
  g_nccl.Broadcast = reinterpret_cast<decltype(g_nccl.Broadcast)>(sym("ncclBroadcast"));
  g_nccl.AllReduce = reinterpret_cast<decltype(g_nccl.AllReduce)>(sym("ncclAllReduce"));
  g_nccl.GroupStart = reinterpret_cast<decltype(g_nccl.GroupStart)>(sym("ncclGroupStart"));
  g_nccl.GroupEnd = reinterpret_cast<decltype(g_nccl.GroupEnd)>(sym("ncclGroupEnd"));
  g_nccl.GetErrorString = reinterpret_cast<decltype(g_nccl.GetErrorString)>(sym("ncclGetErrorString"));
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommInitAll && g_nccl.CommDestroy &&
              g_nccl.Broadcast && g_nccl.AllReduce && g_nccl.GroupStart && g_nccl.GroupEnd &&
              g_nccl.GetErrorString;
}

// What a ctx's communicator slot (ligi::comm_of) points to.
struct CommState {
  ncclComm_t comm = nullptr;
  int rank = 0, n_ranks = 1;
};

void destroy_comm(void* p) {
  CommState* cs = static_cast<CommState*>(p);
  if (!cs) return;
  if (cs->comm && g_nccl.ok) g_nccl.CommDestroy(cs->comm);
  delete cs;
}

CommState* comm_state(lig_ctx* c) { return static_cast<CommState*>(ligi::comm_of(c)); }

int allreduce_i32(lig_ctx* c, int32_t* d_values, int n, cudaStream_t stream) {
  CommState* cs = comm_state(c);
  if (!cs || cs->n_ranks <= 1 || n == 0) return 0;
  ncclResult_t r = g_nccl.AllReduce(d_values, d_values, (size_t)n, ncclInt32, ncclSum, cs->comm, stream);
  if (r != ncclSuccess) return fail(LIG_ERR_NCCL, "ncclAllReduce failed: %s", g_nccl.GetErrorString(r));
  return 0;
}

int need_nccl() {
  std::call_once(g_nccl_once, [] {
    load_nccl();
    ligi::set_comm_destructor(&destroy_comm);
    ligi::set_allreduce(&allreduce_i32);
  });
  if (!g_nccl.ok) return fail(LIG_ERR_NCCL, "NCCL is not available: %s", g_nccl_why);
  return 0;
}

#define NCCL_TRY(expr)                                                                     \
  do {                                                                                     \
    ncclResult_t r__ = (expr);                                                             \
    if (r__ != ncclSuccess)                                                                \
      return fail(LIG_ERR_NCCL, "%s failed: %s", #expr, g_nccl.GetErrorString(r__));       \
  } while (0)

}  // namespace

struct lig_group {
  std::vector<lig_ctx*> ctx;
  std::mutex mu;                 // one group-level call at a time
  unsigned char* h_blob = nullptr;   // page-locked, portable: the one packed copy of a tick
  size_t h_blob_bytes = 0;
  lig_req* h_reqs = nullptr;     // portable pinned bounce buffers for pageable callers
  lig_pick* h_out = nullptr;
  int max_batch = 0;
};

extern "C" {

// ---------------------------------------------------------------------------------------------------
int lig_group_create(lig_group** out, const int* devices, int n, int max_pods, int max_adapters,
                     int max_batch) {
  if (!out || !devices || n < 1) return fail(LIG_ERR_INVALID, "lig_group_create: bad argument");
  *out = nullptr;
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j)
      if (devices[i] == devices[j]) return fail(LIG_ERR_INVALID, "device %d listed twice", devices[i]);
  if (n > 1)
    if (int rc = need_nccl()) return rc;
  lig_group* g = new lig_group();
  g->max_batch = max_batch;
  // every member can take a whole batch (ragged shards, and a group of one)
  for (int i = 0; i < n; ++i) {
    lig_ctx* c = nullptr;
    if (int rc = lig_create(&c, devices[i], max_pods, max_adapters, max_batch)) {
      lig_group_destroy(g);
      return rc;
    }
    g->ctx.push_back(c);
  }
  if (n > 1) {
    std::vector<ncclComm_t> comms((size_t)n);
    ncclResult_t r = g_nccl.CommInitAll(comms.data(), n, devices);
    if (r != ncclSuccess) {
      lig_group_destroy(g);
      return fail(LIG_ERR_NCCL, "ncclCommInitAll over %d devices failed: %s", n, g_nccl.GetErrorString(r));
    }
    for (int i = 0; i < n; ++i) ligi::comm_of(g->ctx[(size_t)i]) = new CommState{comms[(size_t)i], i, n};
  }
  g->h_blob_bytes = lig_snapshot_bytes(max_pods, max_adapters);
  cudaSetDevice(devices[0]);
  if (cudaHostAlloc(reinterpret_cast<void**>(&g->h_blob), g->h_blob_bytes, cudaHostAllocPortable) != cudaSuccess) {
    lig_group_destroy(g);
    return fail(LIG_ERR_CUDA, "cudaHostAlloc of the group staging blob failed");
  }
  g->h_reqs = static_cast<lig_req*>(lig_host_alloc((size_t)max_batch * sizeof(lig_req)));
  g->h_out = static_cast<lig_pick*>(lig_host_alloc((size_t)max_batch * sizeof(lig_pick)));
  if (!g->h_reqs || !g->h_out) {
    lig_group_destroy(g);
    return LIG_ERR_CUDA;
  }
  *out = g;
  return 0;
}

void lig_group_destroy(lig_group* g) {
  if (!g) return;
  for (lig_ctx* c : g->ctx) lig_destroy(c);   // destroys the member's communicator too
  if (g->h_blob) cudaFreeHost(g->h_blob);
  if (g->h_reqs) lig_host_free(g->h_reqs);
  if (g->h_out) lig_host_free(g->h_out);
  delete g;
}

int lig_group_size(const lig_group* g) { return g ? (int)g->ctx.size() : 0; }

lig_ctx* lig_group_ctx(lig_group* g, int member) {
  if (!g || member < 0 || member >= (int)g->ctx.size()) return nullptr;
  return g->ctx[(size_t)member];
}

int lig_group_set_thresholds(lig_group* g, const lig_thresholds* t) {
  if (!g || !t) return fail(LIG_ERR_INVALID, "lig_group_set_thresholds: null argument");
  std::lock_guard<std::mutex> lk(g->mu);
  for (lig_ctx* c : g->ctx)
    if (int rc = lig_set_thresholds(c, t)) return rc;
  return 0;
}

int lig_group_set_filter_tree(lig_group* g, const lig_filter_node* nodes, int n_nodes) {
  if (!g) return fail(LIG_ERR_INVALID, "lig_group_set_filter_tree: group is null");
  if (int rc = ligi::check_filter_tree(nodes, n_nodes)) return rc;   // all members or none
  std::lock_guard<std::mutex> lk(g->mu);
  for (lig_ctx* c : g->ctx)
    if (int rc = lig_set_filter_tree(c, nodes, n_nodes)) return rc;
  return 0;
}

int lig_group_upload_snapshot(lig_group* g, uint64_t epoch, int P, int A, const double* kv,
                              const int32_t* q, const uint16_t* na, const uint16_t* ma,
                              const uint32_t* bitmap) {
  if (!g) return fail(LIG_ERR_INVALID, "lig_group_upload_snapshot: group is null");
  std::lock_guard<std::mutex> lk(g->mu);
  const int n = (int)g->ctx.size();
  if (n == 1) return lig_upload_snapshot(g->ctx[0], epoch, P, A, kv, q, na, ma, bitmap);
  if (lig_snapshot_bytes(P, A) > g->h_blob_bytes)
    return fail(LIG_ERR_INVALID, "P=%d, A=%d exceed the group's capacity", P, A);
  if (int rc = lig_pack_snapshot(g->h_blob, P, A, kv, q, na, ma, bitmap)) return rc;   // ONE pack
  std::vector<ligi::SnapshotWrite> w((size_t)n);
  int begun = 0, rc = 0;
  for (; begun < n && !rc; ++begun)
    rc = ligi::begin_write(g->ctx[(size_t)begun], epoch, P, A, nullptr, true, &w[(size_t)begun]);
  if (rc) --begun;   // the failing member holds no lock
  if (!rc) {
    // ONE H2D copy (member 0), then ONE broadcast over NVLink, received in every member's slot
    cudaSetDevice(ligi::device_of(g->ctx[0]));
    if (cudaMemcpyAsync(w[0].d_blob, g->h_blob, w[0].bytes, cudaMemcpyHostToDevice, w[0].stream) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "snapshot H2D copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (!rc) {
    ncclResult_t r = g_nccl.GroupStart();
    for (int i = 0; i < n && r == ncclSuccess; ++i) {
      cudaSetDevice(ligi::device_of(g->ctx[(size_t)i]));
      r = g_nccl.Broadcast(w[(size_t)i].d_blob, w[(size_t)i].d_blob, w[(size_t)i].bytes, ncclUint8, 0,
                           comm_state(g->ctx[(size_t)i])->comm, w[(size_t)i].stream);
    }
    ncclResult_t r2 = g_nccl.GroupEnd();
    if (r == ncclSuccess) r = r2;
    if (r != ncclSuccess) rc = fail(LIG_ERR_NCCL, "ncclBroadcast of the snapshot failed: %s", g_nccl.GetErrorString(r));
  }
  for (int i = 0; i < n && !rc; ++i) rc = ligi::enqueue_build(g->ctx[(size_t)i], &w[(size_t)i]);
  for (int i = 0; i < begun; ++i) {
    if (rc) {
      ligi::abort_write(g->ctx[(size_t)i], &w[(size_t)i]);
    } else {
      const int rc_i = ligi::finish_write(g->ctx[(size_t)i], &w[(size_t)i], true);
      if (rc_i && !rc) {
        rc = rc_i;
        for (int j = i + 1; j < begun; ++j) ligi::abort_write(g->ctx[(size_t)j], &w[(size_t)j]);
        break;
      }
    }
  }
  return rc;
}

int lig_group_schedule_batch(lig_group* g, uint64_t epoch, uint64_t seed, const lig_req* reqs, int R,
                             lig_pick* out) {
  if (!g || R < 0 || (R > 0 && (!reqs || !out)))
    return fail(LIG_ERR_INVALID, "lig_group_schedule_batch: bad argument");
  if (R > g->max_batch) return fail(LIG_ERR_INVALID, "R=%d exceeds max_batch=%d", R, g->max_batch);
  const int n = (int)g->ctx.size();
  if (R == 0) return lig_schedule_batch(g->ctx[0], epoch, seed, reqs, 0, out);
  // contiguous shards [R*i/n, R*(i+1)/n): result order == request order, no collective
  std::vector<int> ticket((size_t)n, -1);
  std::unique_lock<std::mutex> lk(g->mu, std::defer_lock);
  const lig_req* in = reqs;
  lig_pick* res = out;
  int rc = 0, submitted = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
    rc = 0;
    submitted = 0;
    for (int i = 0; i < n && !rc; ++i) {
      const long long lo = (long long)R * i / n, hi = (long long)R * (i + 1) / n;
      if (hi == lo) continue;
      rc = lig_schedule_batch_async(g->ctx[(size_t)i], epoch, seed, in + lo, (int)(hi - lo), res + lo,
                                    &ticket[(size_t)i]);
      if (!rc) ++submitted;
    }
    if (rc == LIG_ERR_INVALID && attempt == 0 && submitted == 0 && in == reqs) {
      // pageable caller buffers: bounce through the group's portable pinned buffers
      lk.lock();
      memcpy(g->h_reqs, reqs, (size_t)R * sizeof(lig_req));
      in = g->h_reqs;
      res = g->h_out;
      continue;
    }
    break;
  }
  for (int i = 0; i < n; ++i)
    if (ticket[(size_t)i] >= 0) {
      const int rc_i = lig_schedule_wait(g->ctx[(size_t)i], ticket[(size_t)i]);
      if (rc_i && !rc) rc = rc_i;
    }
  if (!rc && res != out) memcpy(out, g->h_out, (size_t)R * sizeof(lig_pick));
  return rc;
}

// ---------------------------------------------------------------------------------------------------
int lig_comm_unique_id(void* id) {
  if (!id) return fail(LIG_ERR_INVALID, "lig_comm_unique_id: null argument");
  if (int rc = need_nccl()) return rc;
  static_assert(sizeof(ncclUniqueId) == LIG_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId u;
  NCCL_TRY(g_nccl.GetUniqueId(&u));
  memcpy(id, &u, sizeof(u));
  return 0;
}

int lig_comm_init_rank(lig_ctx* c, int n_ranks, int rank, const void* id) {
  if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks)
    return fail(LIG_ERR_INVALID, "lig_comm_init_rank: bad argument");
  if (int rc = need_nccl()) return rc;
  if (ligi::comm_of(c)) return fail(LIG_ERR_INVALID, "this ctx already has a communicator");
  if (cudaSetDevice(ligi::device_of(c)) != cudaSuccess) return fail(LIG_ERR_CUDA, "cudaSetDevice failed");
  ncclUniqueId u;
  memcpy(&u, id, sizeof(u));
  ncclComm_t comm = nullptr;
  NCCL_TRY(g_nccl.CommInitRank(&comm, n_ranks, u, rank));
  ligi::comm_of(c) = new CommState{comm, rank, n_ranks};
  return 0;
}

int lig_comm_upload_snapshot_device(lig_ctx* c, uint64_t epoch, int P, int A, const void* d_blob,
                                    int root, void* stream) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_comm_upload_snapshot_device: ctx is null");
  if (int rc = need_nccl()) return rc;
  CommState* cs = comm_state(c);
  if (!cs) return fail(LIG_ERR_INVALID, "call lig_comm_init_rank first");
  if (root < 0 || root >= cs->n_ranks) return fail(LIG_ERR_INVALID, "root %d outside [0, %d)", root, cs->n_ranks);
  if (cs->rank == root && !d_blob) return fail(LIG_ERR_INVALID, "the root rank must pass the packed blob");
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, epoch, P, A, static_cast<cudaStream_t>(stream), false, &w)) return rc;
  // the root sends from the caller's blob, everybody receives straight into the resident slot
  const void* send = cs->rank == root ? d_blob : w.d_blob;
  ncclResult_t r = g_nccl.Broadcast(send, w.d_blob, w.bytes, ncclUint8, root, cs->comm, w.stream);
  int rc = 0;
  if (r != ncclSuccess) rc = fail(LIG_ERR_NCCL, "ncclBroadcast of the snapshot failed: %s", g_nccl.GetErrorString(r));
  if (!rc) rc = ligi::enqueue_build(c, &w);
  if (rc) {
    ligi::abort_write(c, &w);
    return rc;
  }
  return ligi::finish_write(c, &w, false);
}

int lig_comm_upload_snapshot(lig_ctx* c, uint64_t epoch, int P, int A, const double* kv,
                             const int32_t* q, const uint16_t* na, const uint16_t* ma,
                             const uint32_t* bitmap, int root) {
  if (!c) return fail(LIG_ERR_INVALID, "lig_comm_upload_snapshot: ctx is null");
  if (int rc = need_nccl()) return rc;
  CommState* cs = comm_state(c);
  if (!cs) return fail(LIG_ERR_INVALID, "call lig_comm_init_rank first");
  if (root < 0 || root >= cs->n_ranks) return fail(LIG_ERR_INVALID, "root %d outside [0, %d)", root, cs->n_ranks);
  ligi::SnapshotWrite w;
  if (int rc = ligi::begin_write(c, epoch, P, A, nullptr, true, &w)) return rc;
  int rc = 0;
  if (cs->rank == root) {   // the arrays are read on the root only
    rc = lig_pack_snapshot(w.h_blob, P, A, kv, q, na, ma, bitmap);
    if (!rc && cudaMemcpyAsync(w.d_blob, w.h_blob, w.bytes, cudaMemcpyHostToDevice, w.stream) != cudaSuccess)
      rc = fail(LIG_ERR_CUDA, "snapshot H2D copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  if (!rc) {
    ncclResult_t r = g_nccl.Broadcast(w.d_blob, w.d_blob, w.bytes, ncclUint8, root, cs->comm, w.stream);
    if (r != ncclSuccess) rc = fail(LIG_ERR_NCCL, "ncclBroadcast of the snapshot failed: %s", g_nccl.GetErrorString(r));
  }
  if (!rc) rc = ligi::enqueue_build(c, &w);
  if (rc) {
    ligi::abort_write(c, &w);
    return rc;
  }
  return ligi::finish_write(c, &w, true);
}

int lig_comm_allreduce_i32(lig_ctx* c, int32_t* d_values, int n, void* stream) {
  if (!c || n < 0 || (n > 0 && !d_values)) return fail(LIG_ERR_INVALID, "lig_comm_allreduce_i32: bad argument");
  if (int rc = need_nccl()) return rc;
  CommState* cs = comm_state(c);
  if (!cs) return fail(LIG_ERR_INVALID, "call lig_comm_init_rank first");
  if (n == 0) return 0;
  if (cudaSetDevice(ligi::device_of(c)) != cudaSuccess) return fail(LIG_ERR_CUDA, "cudaSetDevice failed");
  NCCL_TRY(g_nccl.AllReduce(d_values, d_values, (size_t)n, ncclInt32, ncclSum, cs->comm,
                            static_cast<cudaStream_t>(stream)));
  return 0;
}

}  // extern "C"
