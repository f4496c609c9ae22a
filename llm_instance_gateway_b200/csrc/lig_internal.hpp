// lig_internal.hpp — what lig_multi.cpp (device groups, NCCL) needs from lig.cu besides the public
// C ABI: a snapshot-writer protocol that lets a collective deliver the packed blob straight into a
// ctx's resident snapshot slot.  Not installed, not part of the ABI.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/lig.h"

namespace ligi {

int fail(int code, const char* fmt, ...);

// One snapshot write in progress on a ctx.  begin_write() picks the slot the new epoch replaces,
// evicts it, makes `stream` wait for every batch still reading it and keeps the ctx's writer lock
// until finish_write()/abort_write(); nothing is synchronised with the host in between.
struct SnapshotWrite {
  void* slot = nullptr;            // opaque
  unsigned char* d_blob = nullptr; // the slot's packed blob in HBM (lig_snapshot_bytes(P, A) bytes)
  unsigned char* h_blob = nullptr; // the slot's page-locked staging copy
  size_t bytes = 0;
  int P = 0, A = 0;
  uint64_t epoch = 0;
  cudaStream_t stream = nullptr;   // where the blob is produced and the tables are built
};

// own_stream: use the ctx's own upload stream (then `stream` is ignored); otherwise `stream` is
// the caller's stream (nullptr = the legacy default stream).
int begin_write(lig_ctx* c, uint64_t epoch, int P, int A, cudaStream_t stream, bool own_stream,
                SnapshotWrite* w);
// Class-table build + "ready" event on w->stream (after the producer of d_blob on that stream).
int enqueue_build(lig_ctx* c, SnapshotWrite* w);
// Publish the epoch (schedule calls resolve it from now on) and release the writer lock.
// synchronise: wait for w->stream first (blocking uploads); otherwise readers order themselves
// behind the "ready" event.
int finish_write(lig_ctx* c, SnapshotWrite* w, bool synchronise);
void abort_write(lig_ctx* c, SnapshotWrite* w);

// Validate a caller filter tree table (see lig_set_filter_tree); 0 or LIG_ERR_INVALID.
int check_filter_tree(const lig_filter_node* nodes, int n_nodes);

int device_of(const lig_ctx* c);
int max_batch_of(const lig_ctx* c);

// NCCL communicator slot of a ctx (owned by lig_multi.cpp; destroyed through the hook at
// lig_destroy).
void*& comm_of(lig_ctx* c);
void set_comm_destructor(void (*fn)(void*));
// In-place int32 sum over the ranks of the ctx's communicator (set by lig_multi.cpp once NCCL is
// loaded); lig.cu calls it between the windows of the load-feedback mode.
typedef int (*allreduce_fn)(lig_ctx* c, int32_t* d_values, int n, cudaStream_t stream);
void set_allreduce(allreduce_fn fn);

}  // namespace ligi
