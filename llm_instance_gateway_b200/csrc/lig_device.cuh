// lig_device.cuh — sm_90a (H100) device code of the endpoint picker.
//
// Three kernels, all integer / FP64-compare work (no tensor cores; HBM + issue bound):
//   lig_class_build_kernel  per snapshot: the adapter-independent stages of the reference's filter
//                           tree once per CTA, then one warp per request class (critical?,
//                           adapter) finishes the walk and writes the class's survivor list.
//   lig_pick_stream_kernel  one thread per request: 16 B descriptor in, class lookup, Go Int31n
//                           draw, one 2 B gather from the class list, 8 B result out.  The
//                           bandwidth-bound stream the roofline is quoted on.
//   lig_scan_kernel         one warp per request: the same tree walk done per request with no
//                           class tables (the direct formulation; also returns survivor masks).
//
// The tree walked by tree_eval_warp() is the reference's defaultFilter, flattened:
//   pkg/ext-proc/scheduling/scheduler.go:26-91 (tree), filter.go:44-73 (success/failure routing),
//   filter.go:79-93 (predicate nodes), :102-122 (least queuing), :134-154 (least KV cache),
//   :124-126, :163-187 (predicates).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/lig.h"

namespace lig {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWarpsPerCta = 8;
constexpr int kCtaThreads = kWarpsPerCta * 32;

// Device view of one resident snapshot (pointers into the packed blob, see include/lig.h).
struct SnapView {
  const double* kv;
  const int* q;
  const uint16_t* n_active;
  const uint16_t* max_active;
  const uint32_t* bitmap;  // [A][W]
  int P, A, W;
};

struct Thr {
  double kv_thr;      // kvCacheThreshold        scheduler.go:17
  long long q_crit;   // queueThresholdCritical  scheduler.go:19
  long long q_lora;   // queueingThresholdLoRA   scheduler.go:23
};

// One entry per request class c = critical * (A + 1) + min(adapter, A); 16 bytes (one LDG.128).
// Classes whose survivor set does not depend on the adapter share one of two default lists; the
// others own row c.  Adapter id A has no bitmap row, so the built-in builds always give the classes
// (sheddable, A) and (critical, A) the default lists, which therefore live in those classes' own
// rows A and 2A+1.  The sentinel follows the 2(A+1) rows.  List offsets are in list entries and
// fit 32 bits: 2 * 65535 rows x 32768 entries + 1 = 2^32 - 65535.
//
//   info    : bits 0-2 status | 4-8 shift | 16-31 n   (bit 2 only for LIG_NO_PODS_LEFT, which only
//             caller filter trees produce)
//             (info & 0xffff0007 is the second word of lig_pick as is: status | n_survivors << 16)
//   magic   : M = ceil(2^(32+shift) / n), shift = ceil(log2 n) - 1, so that for every v < 2^31
//             floor(v / n) == umulhi(v, M) >> shift   (Granlund-Montgomery, N = 31 bits; n >= 2)
//   q_limit : floor(2^31 / n).  With q = floor(v / n), Go's Int31n is k = v - q * n, resampling
//             while v > 2^31-1-(2^31 % n), i.e. while q >= floor(2^31 / n) (never for a power of
//             two, where v < 2^31 already implies q < 2^31 / n).
//   list_off: first entry of the class's survivor list in the list pool.  A class without
//             survivors points at the pool's sentinel entry 0xffff, which sign-extends to
//             pod_idx = -1: the pick needs no branch on n.
struct ClassEntry {
  uint32_t info;
  uint32_t magic;
  uint32_t q_limit;
  uint32_t list_off;
};

__host__ __device__ inline uint32_t entry_n(uint32_t info) { return info >> 16; }
__host__ __device__ inline uint32_t entry_status(uint32_t info) { return info & 7u; }
// Entries of the list pool: one row per class, then the sentinel.
__host__ __device__ inline size_t list_pool_entries(size_t n_classes, size_t stride) {
  return n_classes * stride + 8;
}

// Pod metric columns as the tree walk reads them: either the snapshot in global memory (read
// through the read-only path) or a copy the CTA staged into shared memory.
struct Fields {
  const double* kv;
  const int* q;
  const uint16_t* na;
  const uint16_t* ma;
};

template <bool kStaged>
__device__ __forceinline__ double ld_kv(const Fields& f, int p) {
  if constexpr (kStaged) return f.kv[p]; else return __ldg(f.kv + p);
}
template <bool kStaged>
__device__ __forceinline__ int ld_q(const Fields& f, int p) {
  if constexpr (kStaged) return f.q[p]; else return __ldg(f.q + p);
}
template <bool kStaged>
__device__ __forceinline__ bool has_room(const Fields& f, int p) {
  // canAcceptNewLoraPredicate: len(ActiveModels) < MaxActiveModels          filter.go:175-177
  if constexpr (kStaged) return f.na[p] < f.ma[p];
  else return __ldg(f.na + p) < __ldg(f.ma + p);
}

__device__ __forceinline__ int4 ld_stream_int4(const int4* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_int2(int2* p, int2 v) {
  asm volatile("st.global.L1::no_allocate.v2.s32 [%0], {%1, %2};" :: "l"(p), "r"(v.x), "r"(v.y)
               : "memory");
}

// ---- the request's private random stream (include/lig.h) ---------------------------------------
__device__ __forceinline__ uint32_t splitmix_int31(uint64_t& state) {
  state += 0x9E3779B97F4A7C15ull;
  uint64_t z = state;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)(z >> 33);  // Int31() = Int63() >> 32 = next() >> 33
}

__device__ __forceinline__ uint32_t max_accept_for(uint32_t n) {
  return (n & (n - 1)) == 0 ? 0xffffffffu : 0x7fffffffu - (0x80000000u % n);
}

// rand.Intn(n) for 0 < n <= 2^31-1  ->  Int31n(n)          scheduler.go:120, math/rand Go 1.22
// (plain form, used by the direct-scan kernel)
__device__ __forceinline__ uint32_t int31n(uint64_t state, uint32_t n, uint32_t max_accept) {
  uint32_t v = splitmix_int31(state);
  if (max_accept == 0xffffffffu) return v & (n - 1);
  while (v > max_accept) v = splitmix_int31(state);
  return v % n;
}

// The same draw with the class entry's precomputed magic and rejection limit (no integer division
// and no branch on n on the hot path).  n <= 1: magic 0 gives q = 0 < q_limit, k = 0.
// int31n_entry_next leaves `state` after the last value the draw took (the fallback kernel
// continues the stream from there); int31n_entry is the same draw on a copy.
__device__ __forceinline__ uint32_t int31n_entry_next(uint64_t& state, const uint4 e) {
  const uint32_t n = e.x >> 16;
  const uint32_t shift = (e.x >> 4) & 31u;
  uint32_t v = splitmix_int31(state);
  uint32_t q = __umulhi(v, e.y) >> shift;
  while (q >= e.z) {   // probability < n / 2^31 per draw
    v = splitmix_int31(state);
    q = __umulhi(v, e.y) >> shift;
  }
  return n > 1u ? v - q * n : 0u;
}
__device__ __forceinline__ uint32_t int31n_entry(uint64_t state, const uint4 e) {
  return int31n_entry_next(state, e);
}

// ---- one pass helpers; X is a per-warp mask of W words in shared memory -----------------------
// "member" = bit `lane` of word w.  Every lane reads the same word (broadcast), evaluates its own
// pod, and the ballot is the new word: survivor order is pod order by construction.

// leastQueuingFilterFunc                                                    filter.go:102-122
template <bool kStaged>
__device__ __forceinline__ uint32_t stage_least_queuing(const Fields& f, uint32_t* X, int W,
                                                         int lane, uint32_t n) {
  if (n == 0) return 0;  // empty in => empty out, no division                filter_test.go:226-231
  int mn = 0x7fffffff;   // math.MaxInt: lowered by the first member           filter.go:103
  int mx = 0;            // max starts at 0, not MinInt                        filter.go:104
  for (int w = 0; w < W; ++w) {
    uint32_t word = X[w];
    if (word == 0) continue;
    if ((word >> lane) & 1u) {
      int v = ld_q<kStaged>(f, w * 32 + lane);
      mn = min(mn, v);
      mx = max(mx, v);
    }
  }
  mn = __reduce_min_sync(kFull, mn);
  mx = __reduce_max_sync(kFull, mx);
  // min + (max-min)/len(pods), Go int64 truncated division.  mx >= mn always (mx >= every
  // member, or 0 >= all-negative members), so the range is a non-negative value < 2^32.
  uint32_t range = (uint32_t)mx - (uint32_t)mn;
  long long thr = (long long)mn + (long long)(range / n);
  uint32_t cnt = 0;
  for (int w = 0; w < W; ++w) {
    uint32_t word = X[w];
    if (word == 0) continue;
    bool keep = false;
    if ((word >> lane) & 1u) {
      long long v = ld_q<kStaged>(f, w * 32 + lane);
      keep = v >= (long long)mn && v <= thr;                                 // filter.go:117
    }
    uint32_t nw = __ballot_sync(kFull, keep);
    __syncwarp();  // every lane's read of X[w] is ordered before lane 0 overwrites it
    if (lane == 0) X[w] = nw;
    cnt += __popc(nw);
  }
  __syncwarp();
  return cnt;
}

// leastKVCacheFilterFunc                                                    filter.go:134-154
template <bool kStaged>
__device__ __forceinline__ uint32_t stage_least_kv(const Fields& f, uint32_t* X, int W, int lane,
                                                   uint32_t n) {
  if (n == 0) return 0;                                                      // filter_test.go:265-270
  double mn = 1.7976931348623157e308;  // math.MaxFloat64                     filter.go:135
  double mx = 0.0;                     //                                      filter.go:136
  for (int w = 0; w < W; ++w) {
    uint32_t word = X[w];
    if (word == 0) continue;
    if ((word >> lane) & 1u) {
      double v = ld_kv<kStaged>(f, w * 32 + lane);
      if (v <= mn) mn = v;  // NaN compares false: never updates, as in Go    filter.go:140-145
      if (v >= mx) mx = v;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {  // mn/mx are never NaN here
    double o = __shfl_xor_sync(kFull, mn, off);
    if (o < mn) mn = o;
    o = __shfl_xor_sync(kFull, mx, off);
    if (o > mx) mx = o;
  }
  // min + (max-min)/float64(len(pods)): three separately rounded binary64 ops, no FMA.
  double thr = __dadd_rn(mn, __ddiv_rn(__dsub_rn(mx, mn), (double)n));       // filter.go:149
  uint32_t cnt = 0;
  for (int w = 0; w < W; ++w) {
    uint32_t word = X[w];
    if (word == 0) continue;
    bool keep = false;
    if ((word >> lane) & 1u) {
      double v = ld_kv<kStaged>(f, w * 32 + lane);
      keep = v >= mn && v <= thr;
    }
    uint32_t nw = __ballot_sync(kFull, keep);
    __syncwarp();  // every lane's read of X[w] is ordered before lane 0 overwrites it
    if (lane == 0) X[w] = nw;
    cnt += __popc(nw);
  }
  __syncwarp();
  return cnt;
}

struct EvalResult {
  uint32_t* mask;   // X or T: the W survivor words (shared memory, per warp)
  uint32_t n;
  uint32_t status;  // LIG_OK / LIG_DROP / LIG_EMPTY
};

// Walk defaultFilter for one (critical, adapter row) over all P pods, one warp.
//   X, T : per-warp scratch masks (W words each);  H : the adapter's bitmap row staged in shared
//   memory (W words), or nullptr when the adapter is in no pod's ActiveModels.
// kRootMask: the root's input is not every pod but the n_root pods of the mask the caller left in T
// (a request's pool without its excluded pods, lig_schedule_batch_excluding).
template <bool kStaged, bool kRootMask = false>
__device__ __forceinline__ EvalResult tree_eval_warp(const Fields& f, const uint32_t* H,
                                                     bool critical, const Thr thr, int P, int W,
                                                     uint32_t* X, uint32_t* T, int lane,
                                                     uint32_t n_root = 0) {
  uint32_t n = 0;
  // criticalRequestPredicate keeps every pod or none; with an empty pool the predicate node yields
  // "no pods left" and the sheddable branch runs.            scheduler.go:26-31, filter.go:179-181
  if (critical && (kRootMask ? n_root > 0 : P > 0)) {
    // "low queueing filter": q < queueingThresholdLoRA        scheduler.go:58-60, filter.go:124-126
    for (int w = 0; w < W; ++w) {
      int p = w * 32 + lane;
      bool in_pool;
      if constexpr (kRootMask) in_pool = (T[w] >> lane) & 1u; else in_pool = p < P;
      bool keep = in_pool && (long long)ld_q<kStaged>(f, p) < thr.q_lora;
      uint32_t nw = __ballot_sync(kFull, keep);
      if (lane == 0) X[w] = nw;
      n += __popc(nw);
    }
    __syncwarp();
    if (n > 0) {
      // "affinity LoRA": ResolvedTargetModel in ActiveModels   scheduler.go:61-64, filter.go:169-172
      uint32_t nb = 0;
      for (int w = lane; w < W; w += 32) {
        uint32_t t = H ? (X[w] & H[w]) : 0u;
        T[w] = t;
        nb += __popc(t);
      }
      nb = __reduce_add_sync(kFull, nb);
      __syncwarp();
      if (nb > 0) {
        uint32_t* s = X; X = T; T = s;
        n = nb;
      } else {
        // "can accept LoRA Adapter"                            scheduler.go:65-69, filter.go:175-177
        uint32_t nc = 0;
        for (int w = 0; w < W; ++w) {
          uint32_t word = X[w];
          bool keep = ((word >> lane) & 1u) && has_room<kStaged>(f, w * 32 + lane);
          uint32_t nw = __ballot_sync(kFull, keep);
          if (lane == 0) T[w] = nw;
          nc += __popc(nw);
        }
        __syncwarp();
        if (nc > 0) {  // on failure the node's INPUT (the low-queue set) is forwarded  filter.go:71
          uint32_t* s = X; X = T; T = s;
          n = nc;
        }
      }
      // queueAndKVCacheFilter                                   scheduler.go:49-56
      n = stage_least_queuing<kStaged>(f, X, W, lane, n);
      n = stage_least_kv<kStaged>(f, X, W, lane, n);
      return {X, n, n ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY};
    }
    // low-queueing failed: its input (all pods) goes to queueLoRAAndKVCacheFilter   scheduler.go:71
    if constexpr (kRootMask) {
      uint32_t* s = X; X = T; T = s;
      n = n_root;
    } else {
      for (int w = lane; w < W; w += 32) {
        int rem = P - w * 32;
        X[w] = rem >= 32 ? 0xffffffffu : ((1u << rem) - 1u);
      }
      __syncwarp();
      n = (uint32_t)P;
    }
  } else {
    // "has capacity for sheddable requests"                     scheduler.go:74-79, filter.go:183-187
    for (int w = 0; w < W; ++w) {
      int p = w * 32 + lane;
      bool keep = false;
      bool in_pool;
      if constexpr (kRootMask) in_pool = (T[w] >> lane) & 1u; else in_pool = p < P;
      if (in_pool) {
        keep = (long long)ld_q<kStaged>(f, p) <= thr.q_crit && ld_kv<kStaged>(f, p) <= thr.kv_thr;
      }
      uint32_t nw = __ballot_sync(kFull, keep);
      if (lane == 0) X[w] = nw;
      n += __popc(nw);
    }
    __syncwarp();
    if (n == 0) return {X, 0u, (uint32_t)LIG_DROP};              // "drop request"  scheduler.go:83-89
  }
  // queueLoRAAndKVCacheFilter: least queuing -> low cost LoRA -> least KV    scheduler.go:35-46
  n = stage_least_queuing<kStaged>(f, X, W, lane, n);
  uint32_t nz = 0;
  for (int w = 0; w < W; ++w) {
    uint32_t word = X[w];
    if (word == 0) { if (lane == 0) T[w] = 0; continue; }
    uint32_t hw = H ? H[w] : 0u;
    // lowLoRACostPredicate: affinity OR room                               filter.go:163-166
    bool keep = ((word >> lane) & 1u) && (((hw >> lane) & 1u) || has_room<kStaged>(f, w * 32 + lane));
    uint32_t nw = __ballot_sync(kFull, keep);
    if (lane == 0) T[w] = nw;
    nz += __popc(nw);
  }
  __syncwarp();
  if (nz > 0) {
    uint32_t* s = X; X = T; T = s;
    n = nz;
  }
  n = stage_least_kv<kStaged>(f, X, W, lane, n);
  return {X, n, n ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY};
}

// Shared memory carve-up common to the two tree-walking kernels:
//   [ per-warp scratch: kWarpsPerCta x 3 x W words ][ staged pod columns (kStaged only) ]
__host__ __device__ inline size_t scratch_bytes(int W) {
  return (size_t)kWarpsPerCta * 3u * (size_t)W * sizeof(uint32_t);
}
__host__ __device__ inline size_t staged_bytes(int W) {  // kv f64 + q i32 + na u16 + ma u16 = 16 B/pod
  return (size_t)W * 32u * 16u;
}

// Coalesced 16-byte copies of the four pod columns into shared memory (every column of the
// packed blob is 16-byte aligned and padded to 32 pods).
__device__ __forceinline__ Fields stage_fields(const SnapView& s, unsigned char* smem) {
  const int Ppad = s.W * 32;
  double* kv = reinterpret_cast<double*>(smem);
  int* q = reinterpret_cast<int*>(kv + Ppad);
  uint16_t* na = reinterpret_cast<uint16_t*>(q + Ppad);
  uint16_t* ma = na + Ppad;
  const int4* src_kv = reinterpret_cast<const int4*>(s.kv);
  const int4* src_q = reinterpret_cast<const int4*>(s.q);
  const int4* src_na = reinterpret_cast<const int4*>(s.n_active);
  const int4* src_ma = reinterpret_cast<const int4*>(s.max_active);
  int4* dkv = reinterpret_cast<int4*>(kv);
  int4* dq = reinterpret_cast<int4*>(q);
  int4* dna = reinterpret_cast<int4*>(na);
  int4* dma = reinterpret_cast<int4*>(ma);
  for (int i = threadIdx.x; i < Ppad / 2; i += blockDim.x) dkv[i] = __ldg(src_kv + i);
  for (int i = threadIdx.x; i < Ppad / 4; i += blockDim.x) dq[i] = __ldg(src_q + i);
  for (int i = threadIdx.x; i < Ppad / 8; i += blockDim.x) {
    dna[i] = __ldg(src_na + i);
    dma[i] = __ldg(src_ma + i);
  }
  return Fields{kv, q, na, ma};
}

// Stage one adapter's bitmap row through shared memory; nullptr for an adapter outside [0, A).
__device__ __forceinline__ const uint32_t* stage_adapter_row(const SnapView& s, int adapter,
                                                             uint32_t* H, int lane) {
  if (adapter < 0 || adapter >= s.A) return nullptr;  // Go map miss on every pod  filter.go:170
  const uint32_t* row = s.bitmap + (size_t)adapter * s.W;
  for (int w = lane; w < s.W; w += 32) H[w] = __ldg(row + w);
  __syncwarp();
  return H;
}

// ---- K2a: class tables ---------------------------------------------------------------------------
// Class c = critical * (A + 1) + a, a in [0, A] (a == A: adapter active nowhere).
//
// Most of the tree does not depend on the adapter (SURVEY.md A.2/A.4): the low-queue set, the
// "has room" set, the sheddable-capacity set and the least-queuing stage that follows them are
// the same for every class.  Each CTA therefore first walks those shared stages once with all its
// warps (dense, pod-parallel, ballot words), and a class then only costs one AND of its bitmap
// row with a shared mask; only classes whose adapter actually intersects the mask run their own
// range filters, on the (sparse) set bits.  Classes that do not intersect share one of two
// default survivor lists.  lig_scan_kernel keeps the plain per-request walk (tree_eval_warp), so
// the GPU holds two independent formulations of the tree (the parity tests check both).

constexpr int kBuildWarps = 16;   // the class build runs 512-thread CTAs, at most one per SM
constexpr int kBuildThreads = kBuildWarps * 32;

struct BuildShared {        // block-wide scalars of the shared stages (shared memory)
  uint32_t n_shed;          // |S|, S = {q <= q_crit && kv <= kv_thr}              scheduler.go:74-79
  uint32_t crit_mode;       // 0: low-queue set non-empty; 1: empty (all pods go to queueLoRAAndKV)
  uint32_t rc_n, rc_status; // default result of critical classes
  uint32_t rs_n, rs_status; // default result of sheddable classes
  uint32_t red_u[kBuildWarps];
  int red_i[2 * kBuildWarps];
  double red_d[2 * kBuildWarps];
};

__device__ __forceinline__ uint32_t blk_sum(uint32_t warp_value, BuildShared* sh, int warp, int lane) {
  __syncthreads();
  if (lane == 0) sh->red_u[warp] = warp_value;
  __syncthreads();
  uint32_t t = 0;
#pragma unroll
  for (int i = 0; i < kBuildWarps; ++i) t += sh->red_u[i];
  return t;
}

// out[w] = ballot(member(in, w) && pred(p)) for all words, block-wide; returns the block count.
template <class Pred>
__device__ __forceinline__ uint32_t blk_pred_pass(uint32_t* out, const uint32_t* in, int P, int W,
                                                  BuildShared* sh, int warp, int lane, Pred pred) {
  uint32_t cnt = 0;
  for (int w = warp; w < W; w += kBuildWarps) {
    const int p = w * 32 + lane;
    const bool member = in ? ((in[w] >> lane) & 1u) : (p < P);
    const bool keep = member && pred(p);
    const uint32_t nw = __ballot_sync(kFull, keep);
    if (lane == 0) out[w] = nw;
    cnt += __popc(nw);
  }
  return blk_sum(cnt, sh, warp, lane);
}

// leastQueuingFilterFunc over mask X (in place), block-wide.                 filter.go:102-122
template <bool kStaged>
__device__ __forceinline__ uint32_t blk_least_queuing(const Fields& f, uint32_t* X, int W, uint32_t n,
                                                      BuildShared* sh, int warp, int lane) {
  if (n == 0) return 0;
  int mn = 0x7fffffff, mx = 0;
  for (int w = warp; w < W; w += kBuildWarps) {
    if ((X[w] >> lane) & 1u) {
      const int v = ld_q<kStaged>(f, w * 32 + lane);
      mn = min(mn, v);
      mx = max(mx, v);
    }
  }
  mn = __reduce_min_sync(kFull, mn);
  mx = __reduce_max_sync(kFull, mx);
  __syncthreads();
  if (lane == 0) { sh->red_i[warp] = mn; sh->red_i[kBuildWarps + warp] = mx; }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kBuildWarps; ++i) {
    mn = min(mn, sh->red_i[i]);
    mx = max(mx, sh->red_i[kBuildWarps + i]);
  }
  const uint32_t range = (uint32_t)mx - (uint32_t)mn;   // see stage_least_queuing
  const long long thr = (long long)mn + (long long)(range / n);
  uint32_t cnt = 0;
  for (int w = warp; w < W; w += kBuildWarps) {
    const uint32_t word = X[w];
    bool keep = false;
    if ((word >> lane) & 1u) {
      const long long v = ld_q<kStaged>(f, w * 32 + lane);
      keep = v >= (long long)mn && v <= thr;
    }
    const uint32_t nw = __ballot_sync(kFull, keep);
    __syncwarp();  // every lane's read of X[w] is ordered before lane 0 overwrites it
    if (lane == 0) X[w] = nw;
    cnt += __popc(nw);
  }
  return blk_sum(cnt, sh, warp, lane);
}

// leastKVCacheFilterFunc over mask X (in place), block-wide.                 filter.go:134-154
template <bool kStaged>
__device__ __forceinline__ uint32_t blk_least_kv(const Fields& f, uint32_t* X, int W, uint32_t n,
                                                 BuildShared* sh, int warp, int lane) {
  if (n == 0) return 0;
  double mn = 1.7976931348623157e308, mx = 0.0;
  for (int w = warp; w < W; w += kBuildWarps) {
    if ((X[w] >> lane) & 1u) {
      const double v = ld_kv<kStaged>(f, w * 32 + lane);
      if (v <= mn) mn = v;
      if (v >= mx) mx = v;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    double o = __shfl_xor_sync(kFull, mn, off);
    if (o < mn) mn = o;
    o = __shfl_xor_sync(kFull, mx, off);
    if (o > mx) mx = o;
  }
  __syncthreads();
  if (lane == 0) { sh->red_d[warp] = mn; sh->red_d[kBuildWarps + warp] = mx; }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kBuildWarps; ++i) {
    const double a = sh->red_d[i], b = sh->red_d[kBuildWarps + i];
    if (a < mn) mn = a;
    if (b > mx) mx = b;
  }
  const double thr = __dadd_rn(mn, __ddiv_rn(__dsub_rn(mx, mn), (double)n));
  uint32_t cnt = 0;
  for (int w = warp; w < W; w += kBuildWarps) {
    const uint32_t word = X[w];
    bool keep = false;
    if ((word >> lane) & 1u) {
      const double v = ld_kv<kStaged>(f, w * 32 + lane);
      keep = v >= mn && v <= thr;
    }
    const uint32_t nw = __ballot_sync(kFull, keep);
    __syncwarp();  // every lane's read of X[w] is ordered before lane 0 overwrites it
    if (lane == 0) X[w] = nw;
    cnt += __popc(nw);
  }
  return blk_sum(cnt, sh, warp, lane);
}

// The same two range filters for ONE warp on a sparse mask: lane l owns words l, l+32, ... and
// walks their set bits.
template <bool kStaged>
__device__ __forceinline__ uint32_t sparse_least_queuing(const Fields& f, uint32_t* X, int W, int lane,
                                                         uint32_t n) {
  if (n == 0) return 0;
  int mn = 0x7fffffff, mx = 0;
  for (int w = lane; w < W; w += 32) {
    uint32_t bits = X[w];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const int v = ld_q<kStaged>(f, w * 32 + b);
      mn = min(mn, v);
      mx = max(mx, v);
    }
  }
  mn = __reduce_min_sync(kFull, mn);
  mx = __reduce_max_sync(kFull, mx);
  const uint32_t range = (uint32_t)mx - (uint32_t)mn;
  const long long thr = (long long)mn + (long long)(range / n);
  uint32_t cnt = 0;
  for (int w = lane; w < W; w += 32) {
    uint32_t bits = X[w], nw = 0;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const long long v = ld_q<kStaged>(f, w * 32 + b);
      if (v >= (long long)mn && v <= thr) nw |= 1u << b;
    }
    X[w] = nw;
    cnt += __popc(nw);
  }
  cnt = __reduce_add_sync(kFull, cnt);
  __syncwarp();
  return cnt;
}

template <bool kStaged>
__device__ __forceinline__ uint32_t sparse_least_kv(const Fields& f, uint32_t* X, int W, int lane,
                                                    uint32_t n) {
  if (n == 0) return 0;
  double mn = 1.7976931348623157e308, mx = 0.0;
  for (int w = lane; w < W; w += 32) {
    uint32_t bits = X[w];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const double v = ld_kv<kStaged>(f, w * 32 + b);
      if (v <= mn) mn = v;
      if (v >= mx) mx = v;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    double o = __shfl_xor_sync(kFull, mn, off);
    if (o < mn) mn = o;
    o = __shfl_xor_sync(kFull, mx, off);
    if (o > mx) mx = o;
  }
  const double thr = __dadd_rn(mn, __ddiv_rn(__dsub_rn(mx, mn), (double)n));
  uint32_t cnt = 0;
  for (int w = lane; w < W; w += 32) {
    uint32_t bits = X[w], nw = 0;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const double v = ld_kv<kStaged>(f, w * 32 + b);
      if (v >= mn && v <= thr) nw |= 1u << b;
    }
    X[w] = nw;
    cnt += __popc(nw);
  }
  cnt = __reduce_add_sync(kFull, cnt);
  __syncwarp();
  return cnt;
}

// Write the set bits of X, ascending, to list[0..n): lane-strided words, warp prefix per 32 words.
__device__ __forceinline__ void compact_mask_to_list(const uint32_t* X, int W, int lane,
                                                     uint16_t* __restrict__ list) {
  uint32_t base = 0;
  for (int w0 = 0; w0 < W; w0 += 32) {
    const int w = w0 + lane;
    uint32_t bits = w < W ? X[w] : 0u;
    const uint32_t c = __popc(bits);
    uint32_t incl = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t o = __shfl_up_sync(kFull, incl, off);
      if (lane >= off) incl += o;
    }
    uint32_t pos = base + incl - c;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      list[pos++] = (uint16_t)(w * 32 + b);
    }
    base += __shfl_sync(kFull, incl, 31);
  }
}

// Shared-memory carve-up of the class build:
//   [ BuildShared ][ 7 block masks x W ][ per-warp scratch kBuildWarps x W ][ staged columns ]
__host__ __device__ inline size_t build_fixed_bytes(int W) {
  const size_t b = ((sizeof(BuildShared) + 15) & ~(size_t)15) +
                   (size_t)(7 + kBuildWarps) * (size_t)W * sizeof(uint32_t);
  return (b + 15) & ~(size_t)15;   // the staged columns behind it are written with 16-byte stores
}

__device__ __forceinline__ ClassEntry make_entry(uint32_t n, uint32_t status, uint32_t list_off) {
  ClassEntry e;
  // n <= 1: magic 0 gives q = 0 for every draw and the limit 1 accepts the first one: k = 0.
  uint32_t shift = 0, magic = 0, q_limit = 1;
  if (n >= 2) {
    const uint32_t l = 32u - (uint32_t)__clz(n - 1u);          // ceil(log2 n), 1..15
    shift = l - 1u;
    // ceil(2^(32+shift) / n) < 2^32 because n > 2^(l-1)
    magic = (uint32_t)((((unsigned long long)1 << (32u + shift)) + n - 1u) / n);
    q_limit = 0x80000000u / n;
  }
  e.info = status | (shift << 4) | (n << 16);
  e.magic = magic;
  e.q_limit = q_limit;
  e.list_off = list_off;
  return e;
}

// ---- compact tables -----------------------------------------------------------------------------
// The survivor lists are tiny in practice (a handful of pods per class after the least-KV stage).
// Besides the strided rows (one row of P entries per class: every warp works alone, and
// lig_read_class can address a class directly) the build packs them behind a copy of the class
// entries into ONE contiguous blob that the persistent pick kernels pull into shared memory with a
// single TMA bulk copy:
//
//   [ header 16 B ][ entries: n_classes x 16 B, list_off relative to the pool ][ pool: u16[] ]
//
// pool[0] is the 0xffff sentinel (pod_idx -1) every class without survivors points at, then the
// two default lists (stored once), then the own lists in the order their warps finished (pool
// space is handed out by an atomic cursor).  If the pool does not fit `pool_capacity` entries the
// header says so (bytes = 0) and the pick kernels keep to the strided tables in global memory.
struct CompactHeader {
  uint32_t bytes;         // header + entries + pool, rounded up to 16; 0 = not available
  uint32_t n_classes;
  uint32_t pool_entries;
  uint32_t reserved;
};
struct CompactOut {       // where the build writes the blob; counters[0] = pool cursor of the own
  unsigned char* blob;    // lists, counters[1] = finished CTAs (zero at allocation, reset by the sealing CTA)
  uint32_t* counters;
  uint32_t pool_capacity;
  CompactHeader* host_hdr;   // page-locked, device-mapped copy of the header for the host's launch
                             // decision: written by the sealing thread, no D2H copy on the stream
  unsigned long long* dbg;   // LIG_BUILD_DEBUG: clock64() stamps of CTA 0 / thread 0 (nullable)
};
#define LIG_STAMP(k) do { if (co.dbg && blockIdx.x == 0 && threadIdx.x == 0) co.dbg[k] = clock64(); } while (0)

// The last CTA of a build to finish seals the compact blob: total size, or 0 when the pool
// overflowed (the pick kernels then keep to the strided tables).  Called by every thread.
__device__ __forceinline__ void seal_compact(const CompactOut& co, int n_classes, uint32_t fixed_entries) {
  CompactHeader* chdr = reinterpret_cast<CompactHeader*>(co.blob);
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(co.counters + 1, 1u) == gridDim.x - 1) {
      __threadfence();
      const uint32_t total = fixed_entries + *reinterpret_cast<volatile uint32_t*>(co.counters);
      chdr->n_classes = (uint32_t)n_classes;
      chdr->pool_entries = total;
      chdr->reserved = 0;
      chdr->bytes = total <= co.pool_capacity
                        ? (uint32_t)((sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry) +
                                      (size_t)total * sizeof(uint16_t) + 15) & ~(size_t)15) : 0u;
      if (co.host_hdr) {
        co.host_hdr->n_classes = chdr->n_classes;
        co.host_hdr->pool_entries = total;
        co.host_hdr->reserved = 0;
        co.host_hdr->bytes = chdr->bytes;
      }
      co.counters[0] = 0;   // ready for the next build of this slot
      co.counters[1] = 0;
    }
  }
}

// kPool (an epoch derived by lig_eject_pods): the tree's input is not every pod but the n_pool pods
// set in `pool` (W words, global memory); an ejected pod is treated like a padding pod.
template <bool kStaged, bool kPool = false>
__global__ void __launch_bounds__(kBuildThreads)
lig_class_build_kernel(SnapView s, Thr thr, ClassEntry* __restrict__ cls,
                       uint16_t* __restrict__ lists, int list_stride, CompactOut co,
                       const uint32_t* __restrict__ pool = nullptr, int n_pool = 0) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int P = s.P, W = s.W, A = s.A;
  BuildShared* sh = reinterpret_cast<BuildShared*>(smem);
  uint32_t* masks = reinterpret_cast<uint32_t*>(smem + ((sizeof(BuildShared) + 15) & ~(size_t)15));
  uint32_t* M_room = masks;            // n_active < max_active                       filter.go:175-177
  uint32_t* CB = masks + 1 * W;        // critical: mask the adapter row is ANDed with
  uint32_t* CZ = masks + 2 * W;        // critical mode 1: (least-queuing set) & room
  uint32_t* SB = masks + 3 * W;        // sheddable: (least-queuing set of S) & ~room
  uint32_t* SZ = masks + 4 * W;        // sheddable: (least-queuing set of S) & room
  uint32_t* TMP = masks + 5 * W;
  uint32_t* SHED = masks + 6 * W;      // q <= q_crit && kv <= kv_thr                 filter.go:183-187
  uint32_t* X = masks + (size_t)(7 + warp) * W;   // per-warp scratch
  Fields f{s.kv, s.q, s.n_active, s.max_active};
  if constexpr (kStaged) {
    f = stage_fields(s, smem + build_fixed_bytes(W));
  }
  __syncthreads();
  const int n_classes = 2 * (A + 1);
  const uint32_t rc_row = (uint32_t)(2 * A + 1) * (uint32_t)list_stride;     // default lists: the rows of
  const uint32_t rs_row = (uint32_t)A * (uint32_t)list_stride;               // (critical, A), (sheddable, A)
  const uint32_t none = (uint32_t)n_classes * (uint32_t)list_stride;         // sentinel entry
  if (blockIdx.x == 0 && threadIdx.x == 0) lists[none] = 0xffffu;             // reads back as pod_idx -1
  uint4* centries = reinterpret_cast<uint4*>(co.blob + sizeof(CompactHeader));
  uint16_t* cpool = reinterpret_cast<uint16_t*>(co.blob + sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry));
  // the last CTA to finish seals the blob: total size, or 0 when the pool overflowed
  auto seal = [&](uint32_t fixed_entries) { seal_compact(co, n_classes, fixed_entries); };

  if (kPool ? n_pool == 0 : P == 0) {   // critical: predicate node errs on an empty pool -> sheddable branch -> drop
    for (int c = blockIdx.x * kBuildThreads + threadIdx.x; c < n_classes; c += gridDim.x * kBuildThreads) {
      const ClassEntry e = make_entry(0u, (uint32_t)LIG_DROP, none);
      cls[c] = e;
      centries[c] = make_uint4(e.info, e.magic, e.q_limit, 0u);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) cpool[0] = 0xffffu;
    seal(1u);
    return;
  }

  // ---- shared stages (every CTA, all its warps) -----------------------------------------------
  auto ldq = [&](int p) { return (long long)ld_q<kStaged>(f, p); };
  // one pass over the pods for the three request-independent predicate sets
  uint32_t n_low = 0, n_shed_w = 0;
  for (int w = warp; w < W; w += kBuildWarps) {
    const int p = w * 32 + lane;
    bool room = false, low = false, shed = false;
    if (kPool ? ((pool[w] >> lane) & 1u) != 0 : p < P) {
      const long long qq = ldq(p);
      room = has_room<kStaged>(f, p);                                     // filter.go:175-177
      low = qq < thr.q_lora;                                              // scheduler.go:58-60
      shed = qq <= thr.q_crit && ld_kv<kStaged>(f, p) <= thr.kv_thr;      // scheduler.go:74-79
    }
    const uint32_t wr = __ballot_sync(kFull, room), wl = __ballot_sync(kFull, low),
                   ws = __ballot_sync(kFull, shed);
    if (lane == 0) { M_room[w] = wr; CB[w] = wl; SHED[w] = ws; }
    n_low += __popc(wl);
    n_shed_w += __popc(ws);
  }
  n_low = blk_sum(n_low, sh, warp, lane);
  const uint32_t n_shed = blk_sum(n_shed_w, sh, warp, lane);
  uint32_t rc_n, rc_status;
  if (n_low > 0) {
    // default (adapter active in none of the low-queue pods): "can accept LoRA Adapter" on the
    // low-queue set, falling back to that set, then queueAndKVCacheFilter   scheduler.go:65-69,49-56
    uint32_t nc = 0;
    for (int w = warp; w < W; w += kBuildWarps) {
      const uint32_t t = CB[w] & M_room[w];
      if (lane == 0) TMP[w] = t;
      nc += __popc(t);
    }
    nc = blk_sum(nc, sh, warp, lane);
    if (nc == 0) {
      for (int w = threadIdx.x; w < W; w += kBuildThreads) TMP[w] = CB[w];
      nc = n_low;
    }
    __syncthreads();
    nc = blk_least_queuing<kStaged>(f, TMP, W, nc, sh, warp, lane);
    rc_n = blk_least_kv<kStaged>(f, TMP, W, nc, sh, warp, lane);
    rc_status = rc_n ? LIG_OK : LIG_EMPTY;
    if (blockIdx.x == 0 && warp == 0 && rc_n) {
      compact_mask_to_list(TMP, W, lane, lists + rc_row);
      compact_mask_to_list(TMP, W, lane, cpool + 1);
    }
    __syncthreads();
  } else {
    // low-queue filter failed: all pods -> least queuing -> low cost LoRA -> least KV  scheduler.go:71,35-46
    uint32_t ny = blk_pred_pass(TMP, kPool ? pool : nullptr, P, W, sh, warp, lane, [&](int) { return true; });
    ny = blk_least_queuing<kStaged>(f, TMP, W, ny, sh, warp, lane);
    uint32_t nz = 0;
    for (int w = warp; w < W; w += kBuildWarps) {
      const uint32_t y = TMP[w], r = M_room[w];
      if (lane == 0) { CZ[w] = y & r; CB[w] = y & ~r; }
      nz += __popc(y & r);
    }
    nz = blk_sum(nz, sh, warp, lane);
    if (nz > 0) {
      for (int w = threadIdx.x; w < W; w += kBuildThreads) TMP[w] = CZ[w];
      ny = nz;
    }
    __syncthreads();
    rc_n = blk_least_kv<kStaged>(f, TMP, W, ny, sh, warp, lane);
    rc_status = rc_n ? LIG_OK : LIG_EMPTY;
    if (blockIdx.x == 0 && warp == 0 && rc_n) {
      compact_mask_to_list(TMP, W, lane, lists + rc_row);
      compact_mask_to_list(TMP, W, lane, cpool + 1);
    }
    __syncthreads();
  }
  // sheddable side: "has capacity for sheddable requests"                 scheduler.go:74-79
  uint32_t rs_n = 0, rs_status = LIG_DROP;
  for (int w = threadIdx.x; w < W; w += kBuildThreads) TMP[w] = SHED[w];
  __syncthreads();
  if (n_shed > 0) {
    uint32_t ny = blk_least_queuing<kStaged>(f, TMP, W, n_shed, sh, warp, lane);
    uint32_t nz = 0;
    for (int w = warp; w < W; w += kBuildWarps) {
      const uint32_t y = TMP[w], r = M_room[w];
      if (lane == 0) { SZ[w] = y & r; SB[w] = y & ~r; }
      nz += __popc(y & r);
    }
    nz = blk_sum(nz, sh, warp, lane);
    if (nz > 0) {
      for (int w = threadIdx.x; w < W; w += kBuildThreads) TMP[w] = SZ[w];
      ny = nz;
    }
    __syncthreads();
    rs_n = blk_least_kv<kStaged>(f, TMP, W, ny, sh, warp, lane);
    rs_status = rs_n ? LIG_OK : LIG_EMPTY;
    if (blockIdx.x == 0 && warp == 0 && rs_n) {
      compact_mask_to_list(TMP, W, lane, lists + rs_row);
      compact_mask_to_list(TMP, W, lane, cpool + 1 + rc_n);
    }
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) cpool[0] = 0xffffu;
  const uint32_t fixed_entries = 1u + rc_n + rs_n;   // sentinel + the two default lists

  // ---- per class (one warp each): AND the adapter row with the shared mask --------------------
  for (int c = blockIdx.x * kBuildWarps + warp; c < n_classes; c += gridDim.x * kBuildWarps) {
    const bool critical = c >= A + 1;
    const int a = critical ? c - (A + 1) : c;
    const uint32_t* row = a < A ? s.bitmap + (size_t)a * W : nullptr;
    ClassEntry e;
    uint32_t coff = 0;                   // the class's list in the compact pool (0 = the sentinel)
    if (!critical && n_shed == 0) {
      e = make_entry(0u, (uint32_t)LIG_DROP, none);                        // scheduler.go:83-89
    } else {
      const uint32_t* Bm = critical ? CB : SB;
      const uint32_t* Zm = critical ? (n_low > 0 ? nullptr : CZ) : SZ;
      uint32_t hit = 0;
      if (row) {
        for (int w = lane; w < W; w += 32) {
          const uint32_t t = Bm[w] & __ldg(row + w);
          X[w] = t;
          hit += __popc(t);
        }
        hit = __reduce_add_sync(kFull, hit);
      }
      if (hit == 0) {
        e = critical ? make_entry(rc_n, rc_status, rc_n ? rc_row : none)
                     : make_entry(rs_n, rs_status, rs_n ? rs_row : none);
        coff = critical ? (rc_n ? 1u : 0u) : (rs_n ? 1u + rc_n : 0u);
      } else {
        uint32_t n = hit;
        if (Zm) {   // low cost LoRA: (affinity | room) on the least-queuing set     filter.go:163-166
          n = 0;
          for (int w = lane; w < W; w += 32) {
            const uint32_t t = X[w] | Zm[w];
            X[w] = t;
            n += __popc(t);
          }
          n = __reduce_add_sync(kFull, n);
        }
        __syncwarp();
        if (critical && n_low > 0)      // "affinity LoRA" succeeded -> queueAndKVCacheFilter
          n = sparse_least_queuing<kStaged>(f, X, W, lane, n);
        n = sparse_least_kv<kStaged>(f, X, W, lane, n);
        const uint32_t off = (uint32_t)c * (uint32_t)list_stride;
        if (n) {
          compact_mask_to_list(X, W, lane, lists + off);
          uint32_t at = 0;
          if (lane == 0) at = atomicAdd(co.counters, n);           // pool space for this list
          at = __shfl_sync(kFull, at, 0) + fixed_entries;
          if (at + n <= co.pool_capacity) compact_mask_to_list(X, W, lane, cpool + at);
          coff = at;
        }
        e = make_entry(n, n ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY, n ? off : none);
      }
    }
    if (lane == 0) {
      *reinterpret_cast<uint4*>(cls + c) = make_uint4(e.info, e.magic, e.q_limit, e.list_off);
      centries[c] = make_uint4(e.info, e.magic, e.q_limit, coff);
    }
    __syncwarp();
  }
  seal(fixed_entries);
}

// ---- K2a (fast form): pools of up to 4096 pods ------------------------------------------------------
// Same tables, bit for bit, as lig_class_build_kernel; the differences are all about latency (the
// build is a chain of a dozen tiny block-wide stages, so it is bound by synchronisation and
// dependent shared-memory round trips, not by work):
//   * the shared stages keep each thread's 8 pods (word warp + 16 j, bit lane) in REGISTERS, sets
//     are 8-bit masks per thread, a stage is a few compares + one warp reduction + ONE
//     __syncthreads (double-buffered scratch) instead of ballot passes over shared-memory masks;
//   * one class per warp (twice the CTAs, up to one per SM), its bitmap row requested from HBM/L2
//     before the shared stages start, pool space reserved (atomic) before the compaction, one
//     compaction pass that writes the strided row and the pool entry together, lanes owning
//     contiguous words.  From 8 * SMs adapters on (2(A+1) > 16 * SMs classes), each warp takes
//     several classes round-robin (c, c + 16 * gridDim.x, ...) and fetches each later one's row
//     when it gets to it.
constexpr int kOwn = 8;                                 // words per warp: W <= kBuildWarps * kOwn
constexpr int kFastMaxWords = kBuildWarps * kOwn;       // 128 words = 4096 pods

struct FastShared {          // double-buffered scratch of the block-wide stages
  uint32_t red_u[2][4][kBuildWarps];
  int red_i[2][4][kBuildWarps];
  double red_d[2][4][kBuildWarps];
};

__host__ __device__ inline size_t fast_fixed_bytes(int W) {
  const size_t b = ((sizeof(FastShared) + 15) & ~(size_t)15) + (size_t)(7 + kBuildWarps) * (size_t)W * sizeof(uint32_t);
  return (b + 15) & ~(size_t)15;
}

// Set bits of X (ascending) -> out_a[0..n) and out_b[0..n); lane l owns the contiguous words
// [l * per, (l + 1) * per): one warp scan for the whole mask.
__device__ __forceinline__ void compact_mask_to_two_lists(const uint32_t* X, int W, int lane,
                                                          uint16_t* __restrict__ out_a,
                                                          uint16_t* __restrict__ out_b, bool write_b) {
  const int per = (W + 31) / 32;
  const int w0 = lane * per;
  uint32_t c = 0;
  for (int i = 0; i < per; ++i) c += (w0 + i < W) ? __popc(X[w0 + i]) : 0;
  uint32_t incl = c;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t o = __shfl_up_sync(kFull, incl, off);
    if (lane >= off) incl += o;
  }
  uint32_t pos = incl - c;
  for (int i = 0; i < per; ++i) {
    if (w0 + i >= W) break;
    uint32_t bits = X[w0 + i];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const uint16_t pod = (uint16_t)((w0 + i) * 32 + b);
      out_a[pos] = pod;
      if (write_b) out_b[pos] = pod;
      ++pos;
    }
  }
}

// kPool: as in lig_class_build_kernel, for a non-empty pool (an empty one takes the general build's
// early path).
template <bool kPool = false>
__global__ void __launch_bounds__(kBuildThreads)
lig_class_build_fast_kernel(SnapView s, Thr thr, ClassEntry* __restrict__ cls, uint16_t* __restrict__ lists,
                            int list_stride, CompactOut co, const uint32_t* __restrict__ pool = nullptr,
                            int n_pool = 0) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int P = s.P, W = s.W, A = s.A;
  FastShared* sh = reinterpret_cast<FastShared*>(smem);
  uint32_t* masks = reinterpret_cast<uint32_t*>(smem + ((sizeof(FastShared) + 15) & ~(size_t)15));
  uint32_t* M_room = masks;            // n_active < max_active                       filter.go:175-177
  uint32_t* CB = masks + 1 * W;        // critical: mask the adapter row is ANDed with
  uint32_t* CZ = masks + 2 * W;        // critical mode 1: (least-queuing set) & room
  uint32_t* SB = masks + 3 * W;        // sheddable: (least-queuing set of S) & ~room
  uint32_t* SZ = masks + 4 * W;        // sheddable: (least-queuing set of S) & room
  uint32_t* TMPC = masks + 5 * W;      // the default critical survivor set on its way to a list
  uint32_t* TMPS = masks + 6 * W;      // the default sheddable one
  uint32_t* X = masks + (size_t)(7 + warp) * W;   // per-warp scratch
  const int n_classes = 2 * (A + 1);
  const uint32_t rc_row = (uint32_t)(2 * A + 1) * (uint32_t)list_stride;     // as in lig_class_build_kernel
  const uint32_t rs_row = (uint32_t)A * (uint32_t)list_stride;
  const uint32_t none = (uint32_t)n_classes * (uint32_t)list_stride;
  uint4* centries = reinterpret_cast<uint4*>(co.blob + sizeof(CompactHeader));
  uint16_t* cpool = reinterpret_cast<uint16_t*>(co.blob + sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry));

  // this warp's first class: ask for its bitmap row now, use it after the shared stages
  // classes are dealt to the CTAs round-robin: the popular adapters (low ids, long sparse walks)
  // end up on different SMs instead of sharing one
  const int c0 = warp * (int)gridDim.x + (int)blockIdx.x;
  uint32_t rowreg[kFastMaxWords / 32] = {0, 0, 0, 0};
  {
    const int a0 = c0 >= A + 1 ? c0 - (A + 1) : c0;
    if (c0 < n_classes && a0 < A) {
      const uint32_t* row = s.bitmap + (size_t)a0 * W;
#pragma unroll
      for (int i = 0; i < kFastMaxWords / 32; ++i)
        if (lane + 32 * i < W) rowreg[i] = __ldg(row + lane + 32 * i);
    }
  }
  LIG_STAMP(0);
  const Fields f = stage_fields(s, smem + fast_fixed_bytes(W));
  __syncthreads();
  LIG_STAMP(1);

  // ---- this thread's pods ----
  int q[kOwn];
  double kv[kOwn];
  uint32_t valid = 0, room = 0, low = 0, shed = 0;
#pragma unroll
  for (int j = 0; j < kOwn; ++j) {
    const int w = warp + kBuildWarps * j;
    const int p = w * 32 + lane;
    q[j] = 0;
    kv[j] = 0.0;
    if (w < W && (kPool ? ((pool[w] >> lane) & 1u) != 0 : p < P)) {
      q[j] = f.q[p];
      kv[j] = f.kv[p];
      valid |= 1u << j;
      if (f.na[p] < f.ma[p]) room |= 1u << j;                                       // filter.go:175-177
      if ((long long)q[j] < thr.q_lora) low |= 1u << j;                             // scheduler.go:58-60
      if ((long long)q[j] <= thr.q_crit && kv[j] <= thr.kv_thr) shed |= 1u << j;    // scheduler.go:74-79
    }
  }
  int rb = 0;   // which half of the reduction scratch the next block-wide stage uses
  // Block-wide stages.  The critical and the sheddable side of the tree are independent, so every
  // stage reduces BOTH at once: 5 barriers for the whole shared part of the tree.
  auto sum4 = [&](uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t* out) {
    a = __reduce_add_sync(kFull, a);
    b = __reduce_add_sync(kFull, b);
    c = __reduce_add_sync(kFull, c);
    d = __reduce_add_sync(kFull, d);
    if (lane == 0) { sh->red_u[rb][0][warp] = a; sh->red_u[rb][1][warp] = b; sh->red_u[rb][2][warp] = c; sh->red_u[rb][3][warp] = d; }
    __syncthreads();
    out[0] = out[1] = out[2] = out[3] = 0;
#pragma unroll
    for (int i = 0; i < kBuildWarps; ++i) {
      out[0] += sh->red_u[rb][0][i]; out[1] += sh->red_u[rb][1][i];
      out[2] += sh->red_u[rb][2][i]; out[3] += sh->red_u[rb][3][i];
    }
    rb ^= 1;
  };
  auto seal = [&](uint32_t fixed_entries) { seal_compact(co, n_classes, fixed_entries); };

  // ---- shared stages ----
  LIG_STAMP(2);
  uint32_t cnt[4];
  sum4(__popc(low), __popc(shed), __popc(low & room), 0u, cnt);                       // barrier 1
  const uint32_t n_low = cnt[0], n_shed = cnt[1], n_low_room = cnt[2];
  LIG_STAMP(3);
  // critical side, start set:  low-queue pods that can accept the adapter, else all low-queue pods
  // (scheduler.go:58-69); no low-queue pod at all: every pod (scheduler.go:71)
  uint32_t tc = n_low > 0 ? (n_low_room > 0 ? (low & room) : low) : valid;
  uint32_t n_tc = n_low > 0 ? (n_low_room > 0 ? n_low_room : n_low) : (uint32_t)(kPool ? n_pool : P);
  // sheddable side, start set: pods with capacity (scheduler.go:74-79); empty -> drop
  uint32_t ts = shed;
  uint32_t n_ts = n_shed;
  // leastQueuingFilterFunc on both                                             filter.go:102-122
  {
    int mnc = 0x7fffffff, mxc = 0, mns = 0x7fffffff, mxs = 0;
#pragma unroll
    for (int j = 0; j < kOwn; ++j) {
      if ((tc >> j) & 1u) { mnc = min(mnc, q[j]); mxc = max(mxc, q[j]); }
      if ((ts >> j) & 1u) { mns = min(mns, q[j]); mxs = max(mxs, q[j]); }
    }
    mnc = __reduce_min_sync(kFull, mnc); mxc = __reduce_max_sync(kFull, mxc);
    mns = __reduce_min_sync(kFull, mns); mxs = __reduce_max_sync(kFull, mxs);
    if (lane == 0) { sh->red_i[rb][0][warp] = mnc; sh->red_i[rb][1][warp] = mxc; sh->red_i[rb][2][warp] = mns; sh->red_i[rb][3][warp] = mxs; }
    __syncthreads();                                                                  // barrier 2
#pragma unroll
    for (int i = 0; i < kBuildWarps; ++i) {
      mnc = min(mnc, sh->red_i[rb][0][i]); mxc = max(mxc, sh->red_i[rb][1][i]);
      mns = min(mns, sh->red_i[rb][2][i]); mxs = max(mxs, sh->red_i[rb][3][i]);
    }
    rb ^= 1;
    // min + (max - min) / len, Go int64 truncated division (see stage_least_queuing)
    const long long thc = (long long)mnc + (long long)(((uint32_t)mxc - (uint32_t)mnc) / (n_tc ? n_tc : 1u));
    const long long ths = (long long)mns + (long long)(((uint32_t)mxs - (uint32_t)mns) / (n_ts ? n_ts : 1u));
    uint32_t kc = 0, ks = 0;
#pragma unroll
    for (int j = 0; j < kOwn; ++j) {
      if (((tc >> j) & 1u) && (long long)q[j] >= (long long)mnc && (long long)q[j] <= thc) kc |= 1u << j;
      if (((ts >> j) & 1u) && (long long)q[j] >= (long long)mns && (long long)q[j] <= ths) ks |= 1u << j;
    }
    tc = n_tc ? kc : 0u;
    ts = n_ts ? ks : 0u;
  }
  sum4(__popc(tc), __popc(ts), __popc(tc & room), __popc(ts & room), cnt);            // barrier 3
  n_tc = cnt[0];
  n_ts = cnt[1];
  // "low cost LoRA" on the least-queuing set: (affinity | room); for the default lists (no
  // affinity) that is the room part, falling back to the whole set           scheduler.go:35-46
  uint32_t cb_set, cz_set = 0, sb_set = 0, sz_set = 0;
  if (n_low > 0) {
    cb_set = low;                      // rows are ANDed with the low-queue set ("affinity LoRA")
  } else {
    cz_set = tc & room;
    cb_set = tc & ~room;
    if (cnt[2] > 0) { tc = cz_set; n_tc = cnt[2]; }
  }
  if (n_shed > 0) {
    sz_set = ts & room;
    sb_set = ts & ~room;
    if (cnt[3] > 0) { ts = sz_set; n_ts = cnt[3]; }
  }
  // leastKVCacheFilterFunc on both                                             filter.go:134-154
  {
    double mnc = 1.7976931348623157e308, mxc = 0.0, mns = 1.7976931348623157e308, mxs = 0.0;
#pragma unroll
    for (int j = 0; j < kOwn; ++j) {
      if ((tc >> j) & 1u) { if (kv[j] <= mnc) mnc = kv[j]; if (kv[j] >= mxc) mxc = kv[j]; }
      if ((ts >> j) & 1u) { if (kv[j] <= mns) mns = kv[j]; if (kv[j] >= mxs) mxs = kv[j]; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      double o = __shfl_xor_sync(kFull, mnc, off); if (o < mnc) mnc = o;
      o = __shfl_xor_sync(kFull, mxc, off);        if (o > mxc) mxc = o;
      o = __shfl_xor_sync(kFull, mns, off);        if (o < mns) mns = o;
      o = __shfl_xor_sync(kFull, mxs, off);        if (o > mxs) mxs = o;
    }
    if (lane == 0) { sh->red_d[rb][0][warp] = mnc; sh->red_d[rb][1][warp] = mxc; sh->red_d[rb][2][warp] = mns; sh->red_d[rb][3][warp] = mxs; }
    __syncthreads();                                                                  // barrier 4
#pragma unroll
    for (int i = 0; i < kBuildWarps; ++i) {
      double v = sh->red_d[rb][0][i]; if (v < mnc) mnc = v;
      v = sh->red_d[rb][1][i];        if (v > mxc) mxc = v;
      v = sh->red_d[rb][2][i];        if (v < mns) mns = v;
      v = sh->red_d[rb][3][i];        if (v > mxs) mxs = v;
    }
    rb ^= 1;
    const double thc = __dadd_rn(mnc, __ddiv_rn(__dsub_rn(mxc, mnc), (double)(n_tc ? n_tc : 1u)));
    const double ths = __dadd_rn(mns, __ddiv_rn(__dsub_rn(mxs, mns), (double)(n_ts ? n_ts : 1u)));
    uint32_t kc = 0, ks = 0;
#pragma unroll
    for (int j = 0; j < kOwn; ++j) {
      if (((tc >> j) & 1u) && kv[j] >= mnc && kv[j] <= thc) kc |= 1u << j;
      if (((ts >> j) & 1u) && kv[j] >= mns && kv[j] <= ths) ks |= 1u << j;
    }
    tc = n_tc ? kc : 0u;
    ts = n_ts ? ks : 0u;
  }
  sum4(__popc(tc), __popc(ts), 0u, 0u, cnt);                                          // barrier 5
  const uint32_t rc_n = cnt[0], rs_n = cnt[1];
  const uint32_t rc_status = rc_n ? LIG_OK : LIG_EMPTY;
  const uint32_t rs_status = n_shed == 0 ? (uint32_t)LIG_DROP : (rs_n ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY);
  LIG_STAMP(4);
  // sets -> mask words in shared memory (what the per-class part ANDs the bitmap rows with)
#pragma unroll
  for (int j = 0; j < kOwn; ++j) {
    const int w = warp + kBuildWarps * j;
    const uint32_t w_room = __ballot_sync(kFull, (room >> j) & 1u), w_cb = __ballot_sync(kFull, (cb_set >> j) & 1u),
                   w_cz = __ballot_sync(kFull, (cz_set >> j) & 1u), w_sb = __ballot_sync(kFull, (sb_set >> j) & 1u),
                   w_sz = __ballot_sync(kFull, (sz_set >> j) & 1u), w_tc = __ballot_sync(kFull, (tc >> j) & 1u),
                   w_ts = __ballot_sync(kFull, (ts >> j) & 1u);
    if (lane == 0 && w < W) {
      M_room[w] = w_room; CB[w] = w_cb; CZ[w] = w_cz; SB[w] = w_sb; SZ[w] = w_sz; TMPC[w] = w_tc; TMPS[w] = w_ts;
    }
  }
  __syncthreads();
  // the two default lists, by the last two warps of CTA 0 (its first warps hold the most popular adapters)
  if (blockIdx.x == 0 && warp == kBuildWarps - 1 && rc_n) compact_mask_to_two_lists(TMPC, W, lane, lists + rc_row, cpool + 1, true);
  if (blockIdx.x == 0 && warp == kBuildWarps - 2 && rs_n)
    compact_mask_to_two_lists(TMPS, W, lane, lists + rs_row, cpool + 1 + rc_n, true);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    cpool[0] = 0xffffu;
    lists[none] = 0xffffu;
  }
  const uint32_t fixed_entries = 1u + rc_n + rs_n;
  LIG_STAMP(5);

  // ---- per class (one warp each) ----
  for (int c = c0; c < n_classes; c += gridDim.x * kBuildWarps) {
    const bool critical = c >= A + 1;
    const int a = critical ? c - (A + 1) : c;
    ClassEntry e;
    uint32_t coff = 0;
    if (!critical && n_shed == 0) {
      e = make_entry(0u, (uint32_t)LIG_DROP, none);                        // scheduler.go:83-89
    } else {
      const uint32_t* Bm = critical ? CB : SB;
      const uint32_t* Zm = critical ? (n_low > 0 ? nullptr : CZ) : SZ;
      uint32_t hit = 0;
      if (a < A) {
        if (c != c0) {   // later classes of this warp (A >= 8 * SMs): fetch the row now
          const uint32_t* row = s.bitmap + (size_t)a * W;
#pragma unroll
          for (int i = 0; i < kFastMaxWords / 32; ++i) rowreg[i] = (lane + 32 * i < W) ? __ldg(row + lane + 32 * i) : 0u;
        }
#pragma unroll
        for (int i = 0; i < kFastMaxWords / 32; ++i) {
          const int w = lane + 32 * i;
          if (w < W) {
            const uint32_t t = Bm[w] & rowreg[i];
            X[w] = t;
            hit += __popc(t);
          }
        }
        hit = __reduce_add_sync(kFull, hit);
      }
      if (hit == 0) {
        e = critical ? make_entry(rc_n, rc_status, rc_n ? rc_row : none)
                     : make_entry(rs_n, rs_status, rs_n ? rs_row : none);
        coff = critical ? (rc_n ? 1u : 0u) : (rs_n ? 1u + rc_n : 0u);
      } else {
        uint32_t n = hit;
        if (Zm) {   // low cost LoRA: (affinity | room) on the least-queuing set     filter.go:163-166
          n = 0;
          for (int w = lane; w < W; w += 32) {
            const uint32_t t = X[w] | Zm[w];
            X[w] = t;
            n += __popc(t);
          }
          n = __reduce_add_sync(kFull, n);
        }
        __syncwarp();
        if (critical && n_low > 0)      // "affinity LoRA" succeeded -> queueAndKVCacheFilter
          n = sparse_least_queuing<true>(f, X, W, lane, n);
        n = sparse_least_kv<true>(f, X, W, lane, n);
        const uint32_t off = (uint32_t)c * (uint32_t)list_stride;
        if (n) {
          uint32_t at = 0;
          if (lane == 0) at = atomicAdd(co.counters, n);           // pool space for this list
          at = __shfl_sync(kFull, at, 0) + fixed_entries;
          compact_mask_to_two_lists(X, W, lane, lists + off, cpool + at, at + n <= co.pool_capacity);
          coff = at;
        }
        e = make_entry(n, n ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY, n ? off : none);
      }
    }
    if (lane == 0) {
      *reinterpret_cast<uint4*>(cls + c) = make_uint4(e.info, e.magic, e.q_limit, e.list_off);
      centries[c] = make_uint4(e.info, e.magic, e.q_limit, coff);
    }
    __syncwarp();
  }
  LIG_STAMP(6);
  seal(fixed_entries);
  LIG_STAMP(7);
}

// ---- K2a (caller filter trees): any chart of the reference's filter nodes ---------------------------
// lig_set_filter_tree.  Only the class-table build knows the tree: every node kind depends on the
// request only through (Critical, ResolvedTargetModel), so a caller tree still has one survivor set
// per class and every pick kernel consumes its tables unchanged.
//
// One warp per class walks the table (filter.go:44-73) over all P pods with two W-word masks: `in`
// is the node's input, `res` its result.  A failing node forwards its input (`in` stays), a
// succeeding one its result (the masks swap), so the walk needs no stack; successors only point
// forward, so it visits at most LIG_MAX_FILTER_NODES nodes.  Every class owns its strided row (no
// shared default rows); the compact blob is packed and sealed as by the built-in builds.
struct FilterTree {                      // passed by value: a __grid_constant__ kernel parameter
  lig_filter_node nodes[LIG_MAX_FILTER_NODES];
  int n_nodes;
};
constexpr size_t kTreeNodeBytes = sizeof(lig_filter_node) * LIG_MAX_FILTER_NODES;   // 1 KB
static_assert(sizeof(lig_filter_node) == 32 && kTreeNodeBytes % 16 == 0, "node table layout");

// Shared-memory carve-up of the tree build:
//   [ node table ][ per-warp scratch: kWarpsPerCta x 3 x W words (H, in, res) ][ staged columns ]
__host__ __device__ inline size_t tree_fixed_bytes(int W) { return kTreeNodeBytes + scratch_bytes(W); }

// Does the predicate node `nd` keep pod w * 32 + lane?                          filter.go:163-187
template <bool kStaged>
__device__ __forceinline__ bool node_keeps(const lig_filter_node& nd, const Fields& f, const uint32_t* H,
                                           bool critical, int w, int lane) {
  const int p = w * 32 + lane;
  switch (nd.kind) {
    case LIG_F_CRITICAL_REQUEST: return critical;                                   // filter.go:179-181
    case LIG_F_LOW_QUEUEING: return (long long)ld_q<kStaged>(f, p) < nd.queue_threshold;   // :124-126
    case LIG_F_LORA_AFFINITY: return H && ((H[w] >> lane) & 1u);                     // filter.go:169-172
    case LIG_F_CAN_ACCEPT_NEW_LORA: return has_room<kStaged>(f, p);                  // filter.go:175-177
    case LIG_F_LOW_LORA_COST:                                                        // filter.go:163-166
      return (H && ((H[w] >> lane) & 1u)) || has_room<kStaged>(f, p);
    default:                             // LIG_F_NO_QUEUE_AND_LOW_KV                  filter.go:183-187
      return (long long)ld_q<kStaged>(f, p) <= nd.queue_threshold && ld_kv<kStaged>(f, p) <= nd.kv_threshold;
  }
}

// Walk the caller's tree for one (critical, adapter row), one warp.  H: the adapter's bitmap row in
// shared memory, or nullptr for an adapter in no pod's ActiveModels (a Go map miss on every pod).
// kRootMask: the root's input is the n_root pods of the mask the caller left in `in`, not every pod.
template <bool kStaged, bool kRootMask = false>
__device__ __forceinline__ EvalResult tree_walk_warp(const Fields& f, const lig_filter_node* nodes,
                                                     const uint32_t* H, bool critical, int P, int W,
                                                     uint32_t* in, uint32_t* res, int lane,
                                                     uint32_t n_root = 0) {
  if constexpr (!kRootMask) {
    for (int w = lane; w < W; w += 32) {   // the root's input: AllPodMetrics()    scheduler.go:115
      const int rem = P - w * 32;
      in[w] = rem >= 32 ? kFull : ((1u << rem) - 1u);
    }
    __syncwarp();
  }
  uint32_t n = kRootMask ? n_root : (uint32_t)P;
  int i = 0;
  for (;;) {
    const lig_filter_node nd = nodes[i];
    uint32_t nr = 0, err = LIG_OK;
    if (nd.kind == LIG_F_LEAST_QUEUING || nd.kind == LIG_F_LEAST_KV_CACHE) {
      // the range filters work in place and a failure forwards the input: filter a copy
      for (int w = lane; w < W; w += 32) res[w] = in[w];
      __syncwarp();
      nr = nd.kind == LIG_F_LEAST_QUEUING ? stage_least_queuing<kStaged>(f, res, W, lane, n)
                                          : stage_least_kv<kStaged>(f, res, W, lane, n);
    } else if (nd.kind == LIG_F_DROP) {
      err = LIG_DROP;                    // ([], ResourceExhausted)                   scheduler.go:83-89
    } else {                             // toFilterFunc(predicate)                    filter.go:79-93
      for (int w = 0; w < W; ++w) {
        const uint32_t word = in[w];
        uint32_t nw = 0;
        if (word != 0) nw = __ballot_sync(kFull, ((word >> lane) & 1u) && node_keeps<kStaged>(nd, f, H, critical, w, lane));
        if (lane == 0) res[w] = nw;
        nr += __popc(nw);
      }
      __syncwarp();
      if (nr == 0) err = LIG_NO_PODS_LEFT;   // fmt.Errorf("no pods left")            filter.go:88-90
    }
    const bool ok = err == LIG_OK && nr > 0;                                        // filter.go:50
    const int next = ok ? (nd.next_on_success >= 0 ? nd.next_on_success : nd.next_on_success_or_failure)
                        : (nd.next_on_failure >= 0 ? nd.next_on_failure : nd.next_on_success_or_failure);
    if (next < 0)                        // no successor: the node's own (filtered, err)  filter.go:52-54, 62-64
      return {res, nr, err != LIG_OK ? err : (nr ? (uint32_t)LIG_OK : (uint32_t)LIG_EMPTY)};
    if (ok) {                            // success passes the result on, failure the input  filter.go:60, 71
      uint32_t* t = in; in = res; res = t;
      n = nr;
    }
    i = next;
  }
}

// kPool: the root's input is the n_pool pods set in `pool` (as in lig_class_build_kernel).
template <bool kStaged, bool kPool = false>
__global__ void __launch_bounds__(kCtaThreads)
lig_class_build_tree_kernel(SnapView s, const __grid_constant__ FilterTree tree, ClassEntry* __restrict__ cls,
                            uint16_t* __restrict__ lists, int list_stride, CompactOut co,
                            const uint32_t* __restrict__ pool = nullptr, int n_pool = 0) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int P = s.P, W = s.W, A = s.A;
  lig_filter_node* nodes = reinterpret_cast<lig_filter_node*>(smem);
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(tree.nodes);
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem);
    const int words = tree.n_nodes * (int)(sizeof(lig_filter_node) / sizeof(uint32_t));
    for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  }
  uint32_t* H = reinterpret_cast<uint32_t*>(smem + kTreeNodeBytes) + (size_t)warp * 3 * W;
  uint32_t* M0 = H + W;
  uint32_t* M1 = H + 2 * W;
  Fields f{s.kv, s.q, s.n_active, s.max_active};
  if constexpr (kStaged) {
    f = stage_fields(s, smem + tree_fixed_bytes(W));
  }
  __syncthreads();
  const int n_classes = 2 * (A + 1);
  const uint32_t none = (uint32_t)n_classes * (uint32_t)list_stride;   // sentinel, as in the other builds
  uint4* centries = reinterpret_cast<uint4*>(co.blob + sizeof(CompactHeader));
  uint16_t* cpool = reinterpret_cast<uint16_t*>(co.blob + sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry));
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    lists[none] = 0xffffu;               // reads back as pod_idx -1
    cpool[0] = 0xffffu;
  }
  for (int c = blockIdx.x * kWarpsPerCta + warp; c < n_classes; c += gridDim.x * kWarpsPerCta) {
    const bool critical = c >= A + 1;
    const int a = critical ? c - (A + 1) : c;
    const uint32_t* Hrow = stage_adapter_row(s, a, H, lane);     // nullptr for a == A
    EvalResult r;
    if constexpr (kPool) {
      for (int w = lane; w < W; w += 32) M0[w] = __ldg(pool + w);
      __syncwarp();
      r = tree_walk_warp<kStaged, true>(f, nodes, Hrow, critical, P, W, M0, M1, lane, (uint32_t)n_pool);
    } else {
      r = tree_walk_warp<kStaged>(f, nodes, Hrow, critical, P, W, M0, M1, lane);
    }
    const uint32_t off = (uint32_t)c * (uint32_t)list_stride;
    uint32_t coff = 0;                   // the class's list in the compact pool (0 = the sentinel)
    if (r.n) {
      compact_mask_to_list(r.mask, W, lane, lists + off);
      uint32_t at = 0;
      if (lane == 0) at = atomicAdd(co.counters, r.n);             // pool space for this list
      at = __shfl_sync(kFull, at, 0) + 1u;                          // behind the sentinel
      if (at + r.n <= co.pool_capacity) compact_mask_to_list(r.mask, W, lane, cpool + at);
      coff = at;
    }
    const ClassEntry e = make_entry(r.n, r.status, r.n ? off : none);
    if (lane == 0) {
      *reinterpret_cast<uint4*>(cls + c) = make_uint4(e.info, e.magic, e.q_limit, e.list_off);
      centries[c] = make_uint4(e.info, e.magic, e.q_limit, coff);
    }
    __syncwarp();
  }
  seal_compact(co, n_classes, 1u);
}

// ---- snapshot delta ---------------------------------------------------------------------------------
// One warp per dirty pod: overwrite its four column values, clear its bit in every adapter row,
// set it again in the rows of its new ActiveModels.  Different pods may share a bitmap word, hence
// the atomics; a pod appears at most once in a delta.
struct DeltaView {
  const int* pod_idx;
  const double* kv;
  const int* q;
  const uint16_t* n_active;
  const uint16_t* max_active;
  const int* adapter_offsets;   // n_dirty + 1
  const int* adapter_ids;
  int n_dirty;
};

__global__ void lig_apply_delta_kernel(DeltaView d, double* __restrict__ kv, int* __restrict__ q,
                                       uint16_t* __restrict__ n_active, uint16_t* __restrict__ max_active,
                                       uint32_t* __restrict__ bitmap, int P, int A, int W) {
  const int lane = threadIdx.x & 31;
  const int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (i >= d.n_dirty) return;
  const int p = d.pod_idx[i];
  if (p < 0 || p >= P) return;
  if (lane == 0) {
    kv[p] = d.kv[i];
    q[p] = d.q[i];
    n_active[p] = d.n_active[i];
    max_active[p] = d.max_active[i];
  }
  const uint32_t bit = 1u << (p & 31);
  uint32_t* col = bitmap + (p >> 5);
  for (int a = lane; a < A; a += 32)
    if (col[(size_t)a * W] & bit) atomicAnd(col + (size_t)a * W, ~bit);
  __syncwarp();
  for (int k = d.adapter_offsets[i] + lane; k < d.adapter_offsets[i + 1]; k += 32) {
    const int a = d.adapter_ids[k];
    if (a >= 0 && a < A) atomicOr(col + (size_t)a * W, bit);
  }
}

// ---- K2b: the streaming pick -----------------------------------------------------------------------
// kPerThread requests per thread, strided by the CTA size so that every warp-level load is 512
// contiguous bytes and every store 256.  All loads of a thread are issued before the first use.
constexpr int kPickThreads = 256;

// The class entry {info, magic, q_limit, list_off} of descriptor r (the pick's class lookup).
__device__ __forceinline__ uint4 class_entry(const int4 r, const uint4* __restrict__ cls, uint32_t A) {
  const uint32_t critical = (uint32_t)r.y & LIG_REQ_CRITICAL;
  const uint32_t a = min((uint32_t)r.x, A);          // ids outside [0, A) (negative too) -> A
  const uint32_t c = critical * (A + 1u) + a;
  return __ldg(cls + c);
}

// `entry` (nullable) receives the class entry the pick used: the survivor-list kernel copies the
// class's list from it.  Every other caller passes nothing and compiles as without it.
__device__ __forceinline__ int2 pick_one(const int4 r, const uint4* __restrict__ cls,
                                         const uint16_t* __restrict__ lists, uint32_t A,
                                         uint64_t seed, uint4* entry = nullptr) {
  const uint4 e = class_entry(r, cls, A);
  const uint64_t key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
  if (entry) *entry = e;
  const uint32_t k = int31n_entry(seed ^ key, e);
  // n == 0: list_off is the pool's 0xffff sentinel -> -1
  const int pod = (int)(short)__ldg(lists + (e.w + k));
  return make_int2(pod, (int)(e.x & 0xffff0007u));   // {pod_idx, status | n_survivors << 16}
}

// The same pick against the compact tables in shared memory (entries + pool, see CompactHeader).
__device__ __forceinline__ int2 pick_one_smem(const int4 r, const uint4* tab, const uint16_t* pool,
                                              uint32_t A, uint64_t seed) {
  const uint32_t critical = (uint32_t)r.y & LIG_REQ_CRITICAL;
  const uint64_t key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
  const uint32_t a = min((uint32_t)r.x, A);
  const uint32_t c = critical * (A + 1u) + a;
  const uint4 e = tab[c];
  const uint32_t k = int31n_entry(seed ^ key, e);
  const int pod = (int)(short)pool[e.w + k];
  return make_int2(pod, (int)(e.x & 0xffff0007u));
}

// One CTA's share of one batch: kPerThread requests per thread.
template <int kPerThread>
__device__ __forceinline__ void pick_cta(const int4* __restrict__ reqs, int2* __restrict__ out, int R,
                                         int cta, const uint4* __restrict__ cls,
                                         const uint16_t* __restrict__ lists, int A, uint64_t seed) {
  constexpr int kPerCta = kPickThreads * kPerThread;
  const int first = cta * kPerCta;
  const int4* src = reqs + first + threadIdx.x;
  int2* dst = out + first + threadIdx.x;
  if constexpr (kPerThread > 4) {
    // Software-pipelined form: kPerThread = kIter x kWidth; the loads of iteration i+1 are in
    // flight while iteration i is being scheduled, so one batch needs only R / kPerThread
    // threads and two consecutive batches of a queue are co-resident on the SMs.
    constexpr int kWidth = kPerThread / 4;
    constexpr int kIter = 4;
    if (first + kPerCta <= R) {
      int4 cur[kWidth], nxt[kWidth];
#pragma unroll
      for (int j = 0; j < kWidth; ++j) cur[j] = ld_stream_int4(src + j * kPickThreads);
#pragma unroll
      for (int it = 0; it < kIter; ++it) {
        if (it + 1 < kIter) {
#pragma unroll
          for (int j = 0; j < kWidth; ++j)
            nxt[j] = ld_stream_int4(src + ((it + 1) * kWidth + j) * kPickThreads);
        }
#pragma unroll
        for (int j = 0; j < kWidth; ++j)
          st_stream_int2(dst + (it * kWidth + j) * kPickThreads,
                         pick_one(cur[j], cls, lists, (uint32_t)A, seed));
#pragma unroll
        for (int j = 0; j < kWidth; ++j) cur[j] = nxt[j];
      }
      return;
    }
#pragma unroll 1
    for (int j = 0; j < kPerThread; ++j) {   // ragged tail CTA
      const int i = first + threadIdx.x + j * kPickThreads;
      if (i < R)
        st_stream_int2(dst + j * kPickThreads,
                       pick_one(ld_stream_int4(src + j * kPickThreads), cls, lists,
                                (uint32_t)A, seed));
    }
    return;
  }
  int4 r[kPerThread > 4 ? 1 : kPerThread];
  if (first + kPerCta <= R) {              // full CTA: no per-request bounds checks
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) r[j] = ld_stream_int4(src + j * kPickThreads);
#pragma unroll
    for (int j = 0; j < kPerThread; ++j)
      st_stream_int2(dst + j * kPickThreads,
                     pick_one(r[j], cls, lists, (uint32_t)A, seed));
  } else {                                 // ragged tail CTA
#pragma unroll
    for (int j = 0; j < kPerThread; ++j) {
      const int i = first + threadIdx.x + j * kPickThreads;
      if (i < R)
        st_stream_int2(dst + j * kPickThreads,
                       pick_one(ld_stream_int4(src + j * kPickThreads), cls, lists,
                                (uint32_t)A, seed));
    }
  }
}

// One batch, one short-lived CTA per kPickThreads * kPerThread requests.  This is the kernel of the
// host-buffer path: `reqs` / `out` may be page-locked host memory, read and written over PCIe in
// place.  8 CTAs/SM (<= 32 registers).
template <int kPerThread>
__global__ void __launch_bounds__(kPickThreads, kPerThread <= 8 ? 8 : 6)
lig_pick_stream_kernel(const int4* __restrict__ reqs, int2* __restrict__ out, int R,
                       const uint4* __restrict__ cls, const uint16_t* __restrict__ lists,
                       int A, uint64_t seed) {
  pick_cta<kPerThread>(reqs, out, R, blockIdx.x, cls, lists, A, seed);
}

// A whole queue of batches in one launch: blockIdx.y selects the batch.  A batch of a few thousand
// requests is far below one kernel launch's worth of work (C2: 1024 requests = one CTA), and even
// at 2^20 requests per batch one launch per batch only matches the merged launch on an otherwise
// idle host (see lig_ctx::merge_max_requests).
struct QueueItem {
  const int4* reqs;
  int2* out;
  uint64_t seed;
};

template <int kPerThread>
__global__ void __launch_bounds__(kPickThreads, kPerThread <= 8 ? 8 : 6)
lig_pick_queue_kernel(const QueueItem* __restrict__ items, int R, const uint4* __restrict__ cls,
                      const uint16_t* __restrict__ lists, int A) {
  const QueueItem* it = items + blockIdx.y;
  const int4* reqs = reinterpret_cast<const int4*>(__ldg(reinterpret_cast<const unsigned long long*>(&it->reqs)));
  int2* out = reinterpret_cast<int2*>(__ldg(reinterpret_cast<const unsigned long long*>(&it->out)));
  const uint64_t seed = __ldg(reinterpret_cast<const unsigned long long*>(&it->seed));
  pick_cta<kPerThread>(reqs, out, R, blockIdx.x, cls, lists, A, seed);
}

// ---- K2c: the persistent, TMA-pipelined pick (default for HBM-resident batches) -----------------
// One launch serves a whole queue of batches with a FIXED grid of resident CTAs.  The CTAs claim
// the queue's 1024-request tiles from a shared counter (see produce_claimed_tiles):
//   * a producer warp streams each tile's 16 KB of descriptors global -> shared with one TMA bulk
//     copy (cp.async.bulk, SASS UBLKCP.S.G) into a kStages-deep ring, completion signalled on an
//     mbarrier (expect_tx), so HBM reads never wait for the compute of an earlier tile;
//   * kGroups consumer groups of 8 warps take the CTA's tiles in turn (group g: ring positions g,
//     g + kGroups, ...).  A group waits for its tile, takes 4 descriptors per thread out of shared
//     memory (conflict-free LDS.128) and hands the stage straight back (mbarrier arrive): the ring
//     only holds bytes in flight, never bytes being worked on, so a few 16 KB stages feed many
//     warps.  kStages must be a multiple of kGroups: a group then always returns to the stages
//     whose previous phase it consumed itself, which is what makes the parity wait unambiguous.  Then class lookup + Int31n + list gather from the L1-resident tables;
//   * picks leave either as plain coalesced 8-byte stores or (kBulkStore) staged in shared memory
//     and written with one TMA bulk store per tile (UBLKCP.G.S), tracked by bulk async-groups.
// The CTAs live for the whole queue, so L1 keeps the class tables across tiles and across
// batches (L1 is invalidated at launch boundaries only) and there is no per-CTA launch/drain.
constexpr int kTile = 1024;                     // requests per tile: 16 KB in, 8 KB out
constexpr int kGroupThreads = 256;              // one consumer group: 8 warps x 4 requests per thread
constexpr int kMaxInlineItems = 96;             // queue items carried in kernel parameters

struct QueueParams {
  int n_batches;
  int R;                    // requests per batch
  int tiles_per_batch;      // ceil(R / kTile)
  int total_tiles;          // n_batches * tiles_per_batch (< 2^31, the host splits longer queues)
  const QueueItem* dev_items;             // used when n_batches > kMaxInlineItems
  QueueItem items[kMaxInlineItems];       // else: the per-batch pointers and seeds, inline
};

// Shared-memory budget of the compact tables (CompactHeader blob) inside the persistent kernels:
// 72 KB hold C4's 2050 class entries (32 KB), its 5.5 K list entries (11 KB) and a ~1100-model
// table (18 KB) of the model-request kernels.
constexpr uint32_t kTabBudget = 72 * 1024;

__host__ __device__ constexpr int persist_threads(int groups) { return groups * kGroupThreads + 32; }
// Ring, [bulk-store staging,] full[] and empty[] barriers, then 64 bytes for the table barrier and
// tile_of[stages] (8 + 4 * 8 bytes at most: both kernels have <= 8 stages).
__host__ __device__ constexpr size_t persist_smem_bytes(int groups, int stages, bool bulk_store, bool tab_smem) {
  return (tab_smem ? (size_t)kTabBudget : 0) + (size_t)stages * kTile * 16 +
         (bulk_store ? (size_t)groups * kTile * 8 : 0) + 2u * (size_t)stages * 8 + 64;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = smem_addr(bar);
  uint32_t done;
  do {   // try_wait suspends the thread in hardware up to a time limit; loop until the phase flips
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(a), "r"(parity) : "memory");
  } while (!done);
}
// TMA bulk copy global -> shared, completing `bytes` transaction bytes on `bar` (16 B granular).
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_addr(dst_smem)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
// TMA bulk copy shared -> global, tracked by the issuing thread's bulk async-group.
__device__ __forceinline__ void bulk_store(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(dst), "r"(smem_addr(src_smem)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_store_wait_read_all() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void group_barrier(int group) {   // named barrier 1 + group: that group's 8 warps
  asm volatile("bar.sync %0, %1;" :: "r"(group + 1), "n"(kGroupThreads) : "memory");
}

__device__ __forceinline__ QueueItem queue_item(const QueueParams& qp, int b) {
  if (qp.n_batches <= kMaxInlineItems) return qp.items[b];
  QueueItem it;
  it.reqs = reinterpret_cast<const int4*>(__ldg(reinterpret_cast<const unsigned long long*>(&qp.dev_items[b].reqs)));
  it.out = reinterpret_cast<int2*>(__ldg(reinterpret_cast<const unsigned long long*>(&qp.dev_items[b].out)));
  it.seed = __ldg(reinterpret_cast<const unsigned long long*>(&qp.dev_items[b].seed));
  return it;
}

// ---- dynamic tile claiming (both persistent kernels) ----------------------------------------------
// The producer lane of every CTA claims the launch's tiles one at a time, in global tile order, from
// one counter, so a CTA whose tiles land early takes more of them and all CTAs finish within about a
// tile of each other.  (With a fixed split every group owned ~39 tiles at C4, K = 20, and the launch
// waited for the slowest group while the others sat idle and HBM ran below bandwidth.)  Which CTA
// computes a tile does not change its picks: they depend on (batch, tile, seed) only.
//
// The counter is never reset: the host passes its value before the launch as `base` and then
// advances its copy by total_tiles + gridDim.x, the exact number of claims of a launch (every
// producer claims until its first failed claim, and fails exactly once).  Unsigned 32-bit
// arithmetic, so wrapping is harmless (total_tiles + gridDim.x < 2^31).
struct TileClaim {
  uint32_t* counter;
  uint32_t base;
};

__device__ __forceinline__ uint32_t claim_tile(const TileClaim& tc) {
  return atomicAdd(tc.counter, 1u) - tc.base;
}

// The producer lane: ring position p (stage p % kStages) goes to consumer group p % kGroups, as with
// a fixed split; what is dynamic is which tile a position carries.  For every claimed tile g it
// finds the tile's source and byte count (src_of(g, &bytes)), waits for the stage to be free,
// writes g into tile_of[stage], arrives on full[stage] with expect_tx and starts the bulk copy.
// The next claim and the source lookup go out before that wait, so neither the atomic's round trip
// nor the lookup delays the copy once the stage frees: in steady state the ring is HBM-latency
// bound, and every cycle between a stage's release and its next copy is bytes not in flight.
//
// Termination.  After the first failed claim the producer posts the end marker -1, with a plain
// arrive (no transaction bytes, so the phase completes at once), into the next kGroups ring
// positions n .. n + kGroups - 1, where n is the number of tiles it loaded: exactly one position
// of every group, and every earlier position of that group carried a tile.  So each group
// consumes its tiles, then meets one marker and leaves; no group waits on a position nobody
// fills.  The producer's own waits all pass: position p >= kStages waits for position p - kStages
// to be freed, which the same group (kStages is a multiple of kGroups) consumed, and every such
// position carried a tile (p - kStages < n because kGroups <= kStages), so the group freed it
// right after its full wait.  This covers
//   * a CTA whose first claim fails (fewer tiles than CTAs, a queue of one, or a late CTA): n = 0,
//     the markers go into stages 0 .. kGroups - 1 on the first lap, whose empty waits pass at once;
//   * ragged last tiles: only the byte count differs, never the handshake;
//   * the bulk-store path: all 256 threads of a group read the same tile_of word, so they take
//     the same branches to the group's named barriers and leave the loop together;
//   * 1 group (markers: position n) and 3 groups (kStages 3 or 6: positions n, n + 1, n + 2).
template <int kGroups, int kStages, typename TileSrc>
__device__ __forceinline__ void produce_claimed_tiles(const TileClaim& tc, uint32_t total, unsigned char* ring,
                                                      uint32_t stage_bytes, uint64_t* full, uint64_t* empty,
                                                      int* tile_of, TileSrc src_of) {
  int stage = 0;                                     // (the host only launches kStages % kGroups == 0)
  uint32_t phase = 0;
  for (uint32_t g = claim_tile(tc); g < total;) {
    const uint32_t next = claim_tile(tc);
    uint32_t bytes;
    const void* src = src_of((int)g, &bytes);
    mbar_wait(empty + stage, phase ^ 1u);            // free (passes at once on the first lap)
    tile_of[stage] = (int)g;
    mbar_arrive_expect_tx(full + stage, bytes);
    bulk_load(ring + (size_t)stage * stage_bytes, src, bytes, full + stage);
    if (++stage == kStages) { stage = 0; phase ^= 1u; }
    g = next;
  }
  for (int k = 0; k < kGroups; ++k) {
    mbar_wait(empty + stage, phase ^ 1u);
    tile_of[stage] = -1;
    mbar_arrive(full + stage);
    if (++stage == kStages) { stage = 0; phase ^= 1u; }
  }
}

// kTabSmem: the compact tables (ctab, ctab_bytes <= kTabBudget) are pulled into shared memory by
// one TMA bulk copy at CTA start and every lookup is an LDS; otherwise lookups go to the strided
// tables (cls, lists) through L1.  The host picks the variant (see launch_persistent).
template <int kGroups, int kStages, bool kBulkStore, bool kTabSmem>
__global__ void __launch_bounds__(persist_threads(kGroups), (kTabSmem ? 2 : 6) / kGroups > 0 ? (kTabSmem ? 2 : 6) / kGroups : 1)
lig_pick_persistent_kernel(const __grid_constant__ QueueParams qp, const uint4* __restrict__ cls,
                           const uint16_t* __restrict__ lists, int A,
                           const unsigned char* __restrict__ ctab, uint32_t ctab_bytes, TileClaim tc) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned char* base = smem + (kTabSmem ? kTabBudget : 0u);
  int4* in_ring = reinterpret_cast<int4*>(base);                                   // [kStages][kTile]
  int2* out_stage = reinterpret_cast<int2*>(base + (size_t)kStages * kTile * 16);  // [kGroups][kTile] (kBulkStore)
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)kStages * kTile * 16 +
                                               (kBulkStore ? (size_t)kGroups * kTile * 8 : 0));
  uint64_t* empty = full + kStages;
  uint64_t* tab_bar = empty + kStages;
  int* tile_of = reinterpret_cast<int*>(tab_bar + 1);  // [kStages] the tile each stage holds, -1 = end
  const uint4* tab = reinterpret_cast<const uint4*>(smem + sizeof(CompactHeader));
  const uint16_t* pool = reinterpret_cast<const uint16_t*>(smem + sizeof(CompactHeader) +
                                                           (size_t)2 * ((size_t)A + 1) * sizeof(ClassEntry));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, 1);                          // the producer's arrive.expect_tx
      mbar_init(empty + s, kGroupThreads / 32);        // one arrive per warp of the consuming group
    }
    mbar_init(tab_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int tpb = qp.tiles_per_batch, R = qp.R;

  if (warp == kGroups * (kGroupThreads / 32)) {
    // ---- producer: one lane feeds the ring with the tiles it claims ----
    if (lane == 0) {
      if (kTabSmem) {                                  // the tables first: one bulk copy, L2-resident
        mbar_arrive_expect_tx(tab_bar, ctab_bytes);
        bulk_load(smem, ctab, ctab_bytes, tab_bar);
      }
      produce_claimed_tiles<kGroups, kStages>(tc, (uint32_t)qp.total_tiles, base, kTile * 16u, full, empty,
                                              tile_of, [&](int g, uint32_t* bytes) {
        const int b = g / tpb, t = g - b * tpb;
        *bytes = (uint32_t)min(kTile, R - t * kTile) * 16u;
        return static_cast<const void*>(queue_item(qp, b).reqs + (size_t)t * kTile);
      });
    }
    return;
  }

  // ---- consumer group `grp`: ring positions grp, grp + kGroups, ... until the end marker ----
  const int grp = warp / (kGroupThreads / 32);
  const int tid = (int)threadIdx.x - grp * kGroupThreads;
  int stage = grp % kStages;
  uint32_t phase = (uint32_t)(grp / kStages) & 1u;
  bool tab_ready = !kTabSmem;
  for (;;) {
    mbar_wait(full + stage, phase);                    // the tile's bytes (or the end marker) have landed
    const int g = tile_of[stage];
    if (g < 0) break;
    const int b = g / tpb, t = g - b * tpb;
    const QueueItem it = queue_item(qp, b);
    const int n = min(kTile, R - t * kTile);
    const int4* tile = in_ring + (size_t)stage * kTile + tid;
    int4 r[4];
    if (n == kTile) {
#pragma unroll
      for (int j = 0; j < 4; ++j) r[j] = tile[j * kGroupThreads];
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        r[j] = (tid + j * kGroupThreads < n) ? tile[j * kGroupThreads] : make_int4(0, 0, 0, 0);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + stage);         // descriptors are in registers: stage is free
    // this group's next tile is kGroups ring positions further
    stage += kGroups;
    while (stage >= kStages) { stage -= kStages; phase ^= 1u; }
    // the first tile's stage is free before the wait for the tables, so the producer refills the
    // ring while they are still landing
    if (!tab_ready) { mbar_wait(tab_bar, 0); tab_ready = true; }
    int2 p[4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      p[j] = kTabSmem ? pick_one_smem(r[j], tab, pool, (uint32_t)A, it.seed)
                      : pick_one(r[j], cls, lists, (uint32_t)A, it.seed);
    int2* dst = it.out + (size_t)t * kTile + tid;
    if (kBulkStore && n == kTile) {
      int2* ob = out_stage + (size_t)grp * kTile;
      // the group's previous bulk store has finished READING the staging buffer
      if (tid == 0) bulk_store_wait_read_all();
      group_barrier(grp);
#pragma unroll
      for (int j = 0; j < 4; ++j) ob[tid + j * kGroupThreads] = p[j];
      fence_proxy_async_smem();                        // generic-proxy writes -> visible to the TMA
      group_barrier(grp);
      if (tid == 0) bulk_store(it.out + (size_t)t * kTile, ob, kTile * 8u);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (tid + j * kGroupThreads < n) st_stream_int2(dst + j * kGroupThreads, p[j]);
    }
  }
  // shared memory must outlive the bulk copies: the table pull of a CTA that got no tile, the
  // bulk stores' reads
  if (!tab_ready) mbar_wait(tab_bar, 0);
  if (kBulkStore && tid == 0) bulk_store_wait_read_all();
}

// ---- K2d: persistent grid-stride pick with register prefetch (no shared memory) ------------------
// The LDG/STG counterpart of K2c, kept as the A/B reference of the TMA ring: resident CTAs walk
// a tile sequence of their own (2048-request tiles); the 4 descriptors of a thread's NEXT tile are requested (LDG.128) before
// the current tile is computed, so every warp always has one tile's worth of loads in flight.
constexpr int kLoopThreads = 512;   // tile = 2048 requests (4 per thread)
constexpr int kLoopTile = kLoopThreads * 4;

template <bool kTabSmem>
__global__ void __launch_bounds__(kLoopThreads, 3)
lig_pick_loop_kernel(const __grid_constant__ QueueParams qp, const uint4* __restrict__ cls,
                     const uint16_t* __restrict__ lists, int A,
                     const unsigned char* __restrict__ ctab, uint32_t ctab_bytes) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* tab_bar = reinterpret_cast<uint64_t*>(smem + kTabBudget);
  const uint4* tab = reinterpret_cast<const uint4*>(smem + sizeof(CompactHeader));
  const uint16_t* pool = reinterpret_cast<const uint16_t*>(smem + sizeof(CompactHeader) +
                                                           (size_t)2 * ((size_t)A + 1) * sizeof(ClassEntry));
  if (kTabSmem) {
    if (threadIdx.x == 0) {
      mbar_init(tab_bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(tab_bar, ctab_bytes);
      bulk_load(smem, ctab, ctab_bytes, tab_bar);
    }
  }
  const int tpb = qp.tiles_per_batch, total = qp.total_tiles, R = qp.R;
  const int step = (int)gridDim.x;
  int g = (int)blockIdx.x;
  int b = g / tpb;
  int t = g - b * tpb;
  if (g >= total) return;
  QueueItem it = queue_item(qp, b);
  int n = min(kLoopTile, R - t * kLoopTile);
  int4 cur[4];
  {
    const int4* src = it.reqs + (size_t)t * kLoopTile + threadIdx.x;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      cur[j] = ((int)threadIdx.x + j * kLoopThreads < n) ? ld_stream_int4(src + j * kLoopThreads) : make_int4(0, 0, 0, 0);
  }
  if (kTabSmem) mbar_wait(tab_bar, 0);                 // the tables have landed
  for (;;) {
    const int g2 = g + step;
    int b2 = b, t2 = t + step;
    while (t2 >= tpb) { t2 -= tpb; ++b2; }
    QueueItem it2 = it;
    int n2 = 0;
    int4 nxt[4];
    if (g2 < total) {
      it2 = queue_item(qp, b2);
      n2 = min(kLoopTile, R - t2 * kLoopTile);
      const int4* src = it2.reqs + (size_t)t2 * kLoopTile + threadIdx.x;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        nxt[j] = ((int)threadIdx.x + j * kLoopThreads < n2) ? ld_stream_int4(src + j * kLoopThreads) : make_int4(0, 0, 0, 0);
    }
    int2* dst = it.out + (size_t)t * kLoopTile + threadIdx.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int2 p = kTabSmem ? pick_one_smem(cur[j], tab, pool, (uint32_t)A, it.seed)
                              : pick_one(cur[j], cls, lists, (uint32_t)A, it.seed);
      if ((int)threadIdx.x + j * kLoopThreads < n) st_stream_int2(dst + j * kLoopThreads, p);
    }
    if (g2 >= total) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) cur[j] = nxt[j];
    g = g2; b = b2; t = t2; it = it2; n = n2;
  }
}

// ---- K2e: model requests (the step before Schedule, fused into the pick) --------------------------
// Replaces per request handlers/request.go:42-56: FetchModelData (backend/datastore.go:70-76),
// RandomWeightedDraw (datastore.go:78-98), IsCritical (datastore.go:100-105).  A request is one
// 32-bit model id, a result one 32-bit lig_mpick: 8 bytes per decision.
//
// Model blob (global; the persistent kernel appends it to the class tables in shared memory):
//   [ header 16 B ][ entries: n_models x 16 B ][ targets: 8 B each ]
//   entry.x  bits 0-7 n_targets | 8 critical | 9 present | 12-16 shift (Int31n magic of `total`)
//   entry.y  magic (see ClassEntry) of total = sum of weights, when n_targets >= 2
//   entry.z  total
//   entry.w  n_targets >= 2: index of the first target record; == 1: that target's adapter id;
//            == 0: the model's own adapter id (TargetModels empty, request.go:47)
//   target   {adapter_id, inclusive cumulative weight}: the reference's loop "if randomVal <
//            Weight return; randomVal -= Weight" (datastore.go:91-97) picks the first k with
//            randomVal < cum[k] when the weights are non-negative.
struct ModelHeader {
  uint32_t bytes;        // header + entries + targets, multiple of 16
  uint32_t n_models;
  uint32_t n_target_records;
  uint32_t reserved;
};
constexpr uint32_t kModelCritical = 1u << 8, kModelPresent = 1u << 9;

struct ModelTables {         // where a kernel reads the model blob from (shared or global memory)
  const uint4* entries;
  const uint2* targets;
  uint32_t n_models;
};

__device__ __forceinline__ uint32_t pack_mpick(int pod, uint32_t status, uint32_t target) {
  return ((uint32_t)pod & 0xffffu) | (status << 16) | (target << 24);
}

// L2-only loads (ld.global.cg): for a kernel that outlives uploads (the doorbell kernel), whose
// L1 is not coherent with the copies that rewrite the tables it reads.
__device__ __forceinline__ uint4 ld_cg_uint4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_cg_uint2(const uint2* p) {
  uint2 r;
  asm volatile("ld.global.cg.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ld_cg_u16(const uint16_t* p) {
  uint16_t r;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(r) : "l"(p));
  return r;
}

// pick_one with L2-only loads of the class tables (see ld_cg_uint4).
__device__ __forceinline__ int2 doorbell_pick(const int4 r, const uint4* cls, const uint16_t* lists,
                                              uint32_t A, uint64_t seed) {
  const uint32_t critical = (uint32_t)r.y & LIG_REQ_CRITICAL;
  const uint64_t key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
  const uint32_t a = min((uint32_t)r.x, A);
  const uint32_t c = critical * (A + 1u) + a;
  const uint4 e = ld_cg_uint4(cls + c);
  const uint32_t k = int31n_entry(seed ^ key, e);
  const int pod = (int)(short)ld_cg_u16(lists + (e.w + k));
  return make_int2(pod, (int)(e.x & 0xffff0007u));
}

// How the model helpers below load the model table and the class tables: from shared memory
// (the persistent kernel's copies), through the read-only path (__ldg), or L2 only (the doorbell).
enum class Ld { kSmem, kLdg, kL2 };

template <Ld L>
__device__ __forceinline__ uint4 ld_model_entry(const uint4* p) {
  if constexpr (L == Ld::kSmem) return *p;
  else if constexpr (L == Ld::kLdg) return __ldg(p);
  else return ld_cg_uint4(p);
}
template <Ld L>
__device__ __forceinline__ uint2 ld_model_target(const uint2* p) {
  if constexpr (L == Ld::kSmem) return *p;
  else if constexpr (L == Ld::kLdg) return __ldg(p);
  else return ld_cg_uint2(p);
}

// The weighted draw of a model with >= 2 targets (entry e): randomVal = r.Int31n(total), then the
// first k with randomVal < cum[k]                                                datastore.go:81-97
template <Ld L>
__device__ __forceinline__ void draw_target(const uint4 e, const ModelTables& mt, uint64_t seed, uint64_t key,
                                            uint32_t* adapter, uint32_t* target) {
  const uint32_t nt = e.x & 0xffu;
  const uint32_t total = e.z, shift = (e.x >> 12) & 31u;
  const uint32_t q_limit = total > 1u ? 0x80000000u / total : 1u;
  uint64_t state = seed ^ key ^ LIG_DRAW_DOMAIN;
  uint32_t v = splitmix_int31(state);
  uint32_t q = __umulhi(v, e.y) >> shift;
  while (q >= q_limit) {
    v = splitmix_int31(state);
    q = __umulhi(v, e.y) >> shift;
  }
  const uint32_t r = total > 1u ? v - q * total : 0u;
  uint32_t k = 0;
  uint2 tr = ld_model_target<L>(mt.targets + e.w);
  while (k + 1u < nt && r >= tr.y) {   // first k with randomVal < cum[k]       datastore.go:91-97
    ++k;
    tr = ld_model_target<L>(mt.targets + e.w + k);
  }
  *adapter = tr.x;
  *target = k;
}

// resolve: model id -> (adapter, critical, target index); false = LIG_NO_MODEL.
template <Ld L>
__device__ __forceinline__ bool resolve_model(uint32_t m, const ModelTables& mt, uint64_t seed, uint64_t key,
                                              uint32_t* adapter, uint32_t* critical, uint32_t* target) {
  *adapter = 0xffffffffu; *critical = 0; *target = 255u;
  if (m >= mt.n_models) return false;
  const uint4 e = ld_model_entry<L>(mt.entries + m);
  if (!(e.x & kModelPresent)) return false;
  *critical = (e.x >> 8) & 1u;
  const uint32_t nt = e.x & 0xffu;
  if (nt <= 1u) {                      // no TargetModels, or a single one: nothing to draw
    *adapter = e.w;
    *target = nt ? 0u : 255u;
    return true;
  }
  draw_target<L>(e, mt, seed, key, adapter, target);
  return true;
}

// One model request end to end; the class lookup as in pick_one / pick_one_smem / doorbell_pick.
// `entry` (Ld::kLdg only, nullable): the class entry of the pick, untouched for LIG_NO_MODEL.
template <Ld L>
__device__ __forceinline__ uint32_t pick_model(uint32_t m, uint64_t key, const ModelTables& mt,
                                               const uint4* cls, const uint16_t* lists, uint32_t A,
                                               uint64_t seed, uint4* entry = nullptr) {
  uint32_t adapter, critical, target;
  if (!resolve_model<L>(m, mt, seed, key, &adapter, &critical, &target))
    return pack_mpick(-1, (uint32_t)LIG_NO_MODEL, 255u);
  const int4 r = make_int4((int)adapter, (int)critical, (int)(uint32_t)key, (int)(uint32_t)(key >> 32));
  int2 p;
  if constexpr (L == Ld::kSmem) p = pick_one_smem(r, cls, lists, A, seed);
  else if constexpr (L == Ld::kLdg) p = pick_one(r, cls, lists, A, seed, entry);
  else p = doorbell_pick(r, cls, lists, A, seed);
  return pack_mpick(p.x, (uint32_t)p.y & 7u, target);
}

struct MQueueItem {
  const uint32_t* ids;
  uint32_t* out;
  uint64_t seed;
  uint64_t first_index;
};
constexpr int kMaxInlineMItems = 64;
struct MQueueParams {
  int n_batches;
  int R;
  int tiles_per_batch;
  int total_tiles;
  const MQueueItem* dev_items;
  MQueueItem items[kMaxInlineMItems];
};

__device__ __forceinline__ MQueueItem mqueue_item(const MQueueParams& qp, int b) {
  if (qp.n_batches <= kMaxInlineMItems) return qp.items[b];
  MQueueItem it;
  const unsigned long long* p = reinterpret_cast<const unsigned long long*>(qp.dev_items + b);
  it.ids = reinterpret_cast<const uint32_t*>(__ldg(p));
  it.out = reinterpret_cast<uint32_t*>(__ldg(p + 1));
  it.seed = __ldg(p + 2);
  it.first_index = __ldg(p + 3);
  return it;
}

__host__ __device__ constexpr size_t mpersist_smem_bytes(int stages, bool tab_smem) {
  return (tab_smem ? (size_t)kTabBudget : 0) + (size_t)stages * kTile * 4 + 2u * (size_t)stages * 8 + 64;
}

// Persistent kernel for HBM-resident model-id batches: same structure as K2c (TMA ring, consumer
// groups, claimed tiles, tables in shared memory), 4 KB tiles, every thread takes 4 consecutive requests
// (one LDS.128 in, one 16-byte store out).
template <int kGroups, int kStages, bool kTabSmem>
__global__ void __launch_bounds__(persist_threads(kGroups), kGroups == 1 ? 3 : 2)
lig_pick_models_kernel(const __grid_constant__ MQueueParams qp, const uint4* __restrict__ cls,
                       const uint16_t* __restrict__ lists, int A,
                       const unsigned char* __restrict__ ctab, uint32_t ctab_bytes,
                       const unsigned char* __restrict__ mtab, uint32_t mtab_bytes, uint32_t n_models,
                       TileClaim tc) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned char* base = smem + (kTabSmem ? kTabBudget : 0u);
  uint4* in_ring = reinterpret_cast<uint4*>(base);                                  // [kStages][kTile / 4]
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)kStages * kTile * 4);
  uint64_t* empty = full + kStages;
  uint64_t* tab_bar = empty + kStages;
  int* tile_of = reinterpret_cast<int*>(tab_bar + 1);  // [kStages] the tile each stage holds, -1 = end
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty + s, kGroupThreads / 32);
    }
    mbar_init(tab_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int tpb = qp.tiles_per_batch, R = qp.R;

  if (warp == kGroups * (kGroupThreads / 32)) {
    if (lane == 0) {
      if (kTabSmem) {      // class tables, then the model table right behind them
        mbar_arrive_expect_tx(tab_bar, ctab_bytes + mtab_bytes);
        bulk_load(smem, ctab, ctab_bytes, tab_bar);
        bulk_load(smem + ctab_bytes, mtab, mtab_bytes, tab_bar);
      }
      produce_claimed_tiles<kGroups, kStages>(tc, (uint32_t)qp.total_tiles, base, kTile * 4u, full, empty,
                                              tile_of, [&](int g, uint32_t* bytes) {
        const int b = g / tpb, t = g - b * tpb;
        const uint32_t n = (uint32_t)min(kTile, R - t * kTile);
        *bytes = (n * 4u + 15u) & ~15u;   // the buffers are padded to 16 bytes by the ABI
        return static_cast<const void*>(mqueue_item(qp, b).ids + (size_t)t * kTile);
      });
    }
    return;
  }

  const int grp = warp / (kGroupThreads / 32);
  const int tid = (int)threadIdx.x - grp * kGroupThreads;
  int stage = grp % kStages;
  uint32_t phase = (uint32_t)(grp / kStages) & 1u;
  ModelTables mt;
  const uint4* tab = cls;
  const uint16_t* pool = lists;
  if (kTabSmem) {
    tab = reinterpret_cast<const uint4*>(smem + sizeof(CompactHeader));
    pool = reinterpret_cast<const uint16_t*>(smem + sizeof(CompactHeader) + (size_t)2 * ((size_t)A + 1) * sizeof(ClassEntry));
    mt.entries = reinterpret_cast<const uint4*>(smem + ctab_bytes + sizeof(ModelHeader));
  } else {
    mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
  }
  mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
  mt.n_models = n_models;
  bool tab_ready = !kTabSmem;
  for (;;) {
    mbar_wait(full + stage, phase);
    const int g = tile_of[stage];
    if (g < 0) break;
    const int b = g / tpb, t = g - b * tpb;
    const MQueueItem it = mqueue_item(qp, b);
    const int n = min(kTile, R - t * kTile);
    const uint4 ids = in_ring[(size_t)stage * (kTile / 4) + tid];
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + stage);
    stage += kGroups;
    while (stage >= kStages) { stage -= kStages; phase ^= 1u; }
    if (!tab_ready) { mbar_wait(tab_bar, 0); tab_ready = true; }   // after freeing the first stage
    const int i0 = tid * 4;
    const uint64_t key0 = it.first_index + (uint64_t)t * kTile + (uint64_t)i0;
    // The thread's 4 requests in three passes.  (1) entry lookups; models with at most one target
    // are resolved on the spot.  (2) the weighted draws: few requests need one (only models that
    // split traffic), so instead of a divergent branch inside each of the 4 requests every lane
    // works off its OWN pending requests — the warp runs the draw max-over-lanes(pending) times
    // (1-2) rather than 4.  (3) the 4 picks.
    constexpr Ld kMtLd = kTabSmem ? Ld::kSmem : Ld::kLdg;
    const uint32_t m[4] = {ids.x, ids.y, ids.z, ids.w};
    uint32_t adapter[4], tgt[4];
    uint32_t crit = 0, okm = 0, pending = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool in_range = m[j] < mt.n_models;
      const uint4 e = in_range ? ld_model_entry<kMtLd>(mt.entries + m[j]) : make_uint4(0, 0, 0, 0);
      const uint32_t nt = e.x & 0xffu;
      const bool ok = (e.x & kModelPresent) != 0;
      okm |= (ok ? 1u : 0u) << j;
      crit |= ((e.x >> 8) & 1u) << j;
      adapter[j] = e.w;
      tgt[j] = nt ? 0u : 255u;
      pending |= ((ok && nt >= 2u) ? 1u : 0u) << j;
    }
    while (pending) {
      const int j = __ffs((int)pending) - 1;
      pending &= pending - 1u;
      const uint32_t mj = j == 0 ? m[0] : j == 1 ? m[1] : j == 2 ? m[2] : m[3];
      const uint4 e = ld_model_entry<kMtLd>(mt.entries + mj);
      uint32_t a, k;
      draw_target<kMtLd>(e, mt, it.seed, key0 + (uint64_t)j, &a, &k);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
        if (jj == j) { adapter[jj] = a; tgt[jj] = k; }
    }
    uint32_t ov[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint64_t key = key0 + (uint64_t)j;
      const int4 r = make_int4((int)adapter[j], (int)((crit >> j) & 1u), (int)(uint32_t)key, (int)(uint32_t)(key >> 32));
      const int2 p = kTabSmem ? pick_one_smem(r, tab, pool, (uint32_t)A, it.seed) : pick_one(r, tab, pool, (uint32_t)A, it.seed);
      ov[j] = ((okm >> j) & 1u) ? pack_mpick(p.x, (uint32_t)p.y & 7u, tgt[j]) : pack_mpick(-1, (uint32_t)LIG_NO_MODEL, 255u);
    }
    uint4 o = make_uint4(ov[0], ov[1], ov[2], ov[3]);
    uint32_t* dst = it.out + (size_t)t * kTile + i0;
    if (i0 + 4 <= n) {
      asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};"
                   :: "l"(dst), "r"(o.x), "r"(o.y), "r"(o.z), "r"(o.w) : "memory");
    } else {
      if (i0 + 0 < n) dst[0] = o.x;
      if (i0 + 1 < n) dst[1] = o.y;
      if (i0 + 2 < n) dst[2] = o.z;
    }
  }
  if (!tab_ready) mbar_wait(tab_bar, 0);   // a CTA that got no tile: its table pull must land before exit
}

// The plain form: one short-lived CTA per 1024 requests, LDG/STG only.  Host-buffer path (`ids` /
// `out` may be page-locked host memory), unaligned device buffers, and the resolve-only test hook
// (reqs_out != nullptr: also write the 16-byte descriptor built for every request).
__global__ void __launch_bounds__(kGroupThreads)
lig_pick_models_stream_kernel(const uint32_t* __restrict__ ids, uint32_t* __restrict__ out, int R,
                              const uint4* __restrict__ cls, const uint16_t* __restrict__ lists, int A,
                              const unsigned char* __restrict__ mtab, uint32_t n_models, uint64_t seed,
                              uint64_t first_index, int4* __restrict__ reqs_out) {
  ModelTables mt;
  mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
  mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
  mt.n_models = n_models;
  const int first = (int)blockIdx.x * kTile + (int)threadIdx.x;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = first + j * kGroupThreads;
    if (i >= R) break;
    const uint32_t m = __ldg(ids + i);
    const uint64_t key = first_index + (uint64_t)i;
    if (reqs_out) {
      uint32_t adapter, critical, target;
      const bool ok = resolve_model<Ld::kLdg>(m, mt, seed, key, &adapter, &critical, &target);
      reqs_out[i] = make_int4((int)adapter, (int)critical, (int)(uint32_t)key, (int)(uint32_t)(key >> 32));
      out[i] = pack_mpick(-1, ok ? (uint32_t)LIG_OK : (uint32_t)LIG_NO_MODEL, target);
    } else {
      out[i] = pick_model<Ld::kLdg>(m, key, mt, cls, lists, (uint32_t)A, seed);
    }
  }
}

// ---- K2f: load feedback between the windows of a batch or of a chain of calls (opt-in) ------------
// WaitingQueueSize += picks of the window (all ranks); total += window; window = 0.
__global__ void lig_apply_feedback_kernel(int* __restrict__ q, int* __restrict__ hist_window,
                                          int* __restrict__ hist_total, int P) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int h = hist_window[p];
  // saturating: a queue size beyond int32 is not representable in the device record
  const long long nq = (long long)q[p] + h;
  q[p] = nq > 0x7fffffffLL ? 0x7fffffff : (int)nq;
  if (hist_total) hist_total[p] += h;
  hist_window[p] = 0;
}

// Adds one pick per lane to the open window's histogram.  A herd puts most picks of a warp on a
// few pods, so the count is warp-aggregated: lanes that picked the same pod find each other with
// __match_any_sync and the lowest of them adds the group's size with one atomic; pod -1 (DROP,
// EMPTY, NO_MODEL, NO_PODS_LEFT, or a lane past the end) adds nothing.  Every lane of the warp
// must call it.
__device__ __forceinline__ void count_window_picks(int pod, int lane, int* __restrict__ hist) {
  const unsigned same = __match_any_sync(kFull, pod);
  if (pod >= 0 && lane == __ffs(same) - 1) atomicAdd(hist + pod, __popc(same));
}

// The pick of lig_pick_stream_kernel (same pick_one, so the picks are byte-identical) that also
// counts the picks per pod into the open window's histogram, for the load-feedback chain
// (lig_schedule_batch_feedback_chain).  `reqs` / `out` may be mapped host memory.  Every lane of
// a CTA runs every round, ragged ones with pod -1, so the full-warp match is always legal.
constexpr int kCountPerThread = 4;
__global__ void __launch_bounds__(kPickThreads, 8)
lig_pick_count_kernel(const int4* __restrict__ reqs, int2* __restrict__ out, int R,
                      const uint4* __restrict__ cls, const uint16_t* __restrict__ lists, int A,
                      uint64_t seed, int* __restrict__ hist) {
  const int first = blockIdx.x * (kPickThreads * kCountPerThread) + threadIdx.x;
  const int lane = threadIdx.x & 31;
  int4 r[kCountPerThread];
#pragma unroll
  for (int j = 0; j < kCountPerThread; ++j) {      // every load in flight before the first use
    const int i = first + j * kPickThreads;
    r[j] = i < R ? ld_stream_int4(reqs + i) : make_int4(0, 0, 0, 0);
  }
#pragma unroll
  for (int j = 0; j < kCountPerThread; ++j) {
    const int i = first + j * kPickThreads;
    int pod = -1;
    if (i < R) {
      const int2 p = pick_one(r[j], cls, lists, (uint32_t)A, seed);
      st_stream_int2(out + i, p);
      pod = p.x;
    }
    count_window_picks(pod, lane, hist);
  }
}

// The same for model-id requests (lig_schedule_models_batch_feedback_chain): request i has
// rand_key = first_index + i and goes through pick_model<Ld::kLdg>, so the picks are byte-identical
// to lig_pick_models_stream_kernel on the same tables.  `ids` / `out` may be mapped host memory;
// the model table is a resident epoch's, the class tables are the chain's private copy.  The pod
// is the 16-bit field of the packed pick (0xffff = -1: pods stay below LIG_MAX_PODS = 32768).
__global__ void __launch_bounds__(kPickThreads, 8)
lig_pick_models_count_kernel(const uint32_t* __restrict__ ids, uint32_t* __restrict__ out, int R,
                             const uint4* __restrict__ cls, const uint16_t* __restrict__ lists, int A,
                             const unsigned char* __restrict__ mtab, uint32_t n_models, uint64_t seed,
                             uint64_t first_index, int* __restrict__ hist) {
  ModelTables mt;
  mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
  mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
  mt.n_models = n_models;
  const int first = blockIdx.x * (kPickThreads * kCountPerThread) + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint32_t m[kCountPerThread];
#pragma unroll
  for (int j = 0; j < kCountPerThread; ++j) {      // every load in flight before the first use
    const int i = first + j * kPickThreads;
    m[j] = i < R ? __ldg(ids + i) : 0u;
  }
#pragma unroll
  for (int j = 0; j < kCountPerThread; ++j) {
    const int i = first + j * kPickThreads;
    int pod = -1;
    if (i < R) {
      const uint32_t v = pick_model<Ld::kLdg>(m[j], first_index + (uint64_t)i, mt, cls, lists, (uint32_t)A, seed);
      out[i] = v;
      pod = (int)(int16_t)(v & 0xffffu);
    }
    count_window_picks(pod, lane, hist);
  }
}

// ---- K2h: every request's survivor list next to its pick (lig_filter_batch, lig_filter_models_batch)
// One pass over the batch in tiles of kFilterTile requests.  A CTA claims the next tile from a
// counter (so every lower tile has started: the look-back below cannot wait on a CTA that is not
// resident), and then
//   1. picks each request exactly as lig_pick_stream_kernel / lig_pick_models_stream_kernel do
//      (pick_one / pick_model<Ld::kLdg>: same bytes out) and keeps the class entry the pick used;
//      n = the entry's survivor count for LIG_OK, else 0;
//   2. scans the tile's n in shared memory and finds the tile's base offset with a decoupled
//      look-back over the per-tile state words (Merrill & Garland, "Single-pass Parallel Prefix Scan
//      with Decoupled Look-back", 2016);
//   3. writes the tile's int64 offsets, then copies the tile's lists into one contiguous range of
//      `pods`: output entry j of the tile belongs to the last request whose offset is <= j (binary
//      search in shared memory), so consecutive threads store consecutive entries.  Entries at or
//      beyond `capacity` are not written.
// The lists come from the compact pool when the build sealed one (header bytes != 0), else from
// the strided rows: the entries of both carry the same survivor sets.
constexpr int kFilterThreads = 256;
constexpr int kFilterPerThread = 4;
constexpr int kFilterTile = kFilterThreads * kFilterPerThread;
// Tile state: bits 62-63 = flag, bits 0-61 = value (a sum of n stays below 2^31 * 2^15 = 2^46).
constexpr unsigned long long kScanAggregate = 1ull << 62, kScanPrefix = 2ull << 62;
constexpr unsigned long long kScanValue = (1ull << 62) - 1;

struct FilterOut {
  void* out;                      // lig_pick[R] or lig_mpick[R]
  long long* offsets;             // R + 1 entries
  uint16_t* pods;                 // capacity entries (null when capacity is 0)
  long long capacity;
  unsigned long long* tiles;      // one state word per tile, zero before the launch
  uint32_t* tile_counter;         // zero before the launch
};

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
  return *reinterpret_cast<const volatile unsigned long long*>(p);
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long* p, unsigned long long v) {
  *reinterpret_cast<volatile unsigned long long*>(p) = v;
}

// The base of `tile` (the sum of n over all lower tiles), given this tile's own sum.  Warp 0 only.
__device__ __forceinline__ unsigned long long filter_look_back(unsigned long long* tiles, int tile,
                                                               unsigned long long total, int lane) {
  if (tile == 0) {
    if (lane == 0) st_volatile_u64(tiles, kScanPrefix | total);
    return 0;
  }
  if (lane == 0) st_volatile_u64(tiles + tile, kScanAggregate | total);
  unsigned long long base = 0;
  for (int last = tile - 1;; last -= 32) {
    const int t = last - lane;      // lane 0 looks at the nearest predecessor
    unsigned long long s = t >= 0 ? ld_volatile_u64(tiles + t) : kScanPrefix;
    for (;;) {
      const bool ready = (s >> 62) != 0;
      if (__all_sync(kFull, ready)) break;
      if (!ready) s = ld_volatile_u64(tiles + t);
    }
    const unsigned prefix = __ballot_sync(kFull, (s >> 62) == (kScanPrefix >> 62));
    const int stop = prefix ? __ffs(prefix) - 1 : 31;    // nearest tile whose inclusive prefix is known
    unsigned long long v = lane <= stop ? (s & kScanValue) : 0ull;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
    base += v;
    if (prefix) break;
  }
  if (lane == 0) st_volatile_u64(tiles + tile, kScanPrefix | (base + total));
  return base;
}

template <bool kModels>
__global__ void __launch_bounds__(kFilterThreads)
lig_filter_kernel(const void* __restrict__ in, int R, const uint4* __restrict__ cls,
                  const uint16_t* __restrict__ lists, int A, const unsigned char* __restrict__ ctab,
                  const unsigned char* __restrict__ mtab, uint32_t n_models, uint64_t seed,
                  uint64_t first_index, FilterOut fo) {
  __shared__ __align__(16) uint32_t s_excl[kFilterTile + 4];   // tile-local exclusive offsets, [kFilterTile] = sum
  __shared__ uint32_t s_list[kFilterTile];                    // list start of each request
  __shared__ uint32_t s_warp[kFilterThreads / 32];
  __shared__ unsigned long long s_base;
  __shared__ int s_tile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_tile = (int)atomicAdd(fo.tile_counter, 1u);
  // the compact pool when the build sealed one
  const CompactHeader hdr = *reinterpret_cast<const CompactHeader*>(ctab);
  const uint32_t n_classes = 2u * ((uint32_t)A + 1u);
  const uint4* gcls = cls;
  const uint16_t* glists = lists;
  if (hdr.bytes != 0u && hdr.n_classes == n_classes) {
    gcls = reinterpret_cast<const uint4*>(ctab + sizeof(CompactHeader));
    glists = reinterpret_cast<const uint16_t*>(ctab + sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry));
  }
  __syncthreads();
  const int tile = s_tile;
  const int first = tile * kFilterTile;

  // 1. picks and survivor counts
  if constexpr (kModels) {
    ModelTables mt;
    mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
    mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
    mt.n_models = n_models;
    const uint32_t* ids = static_cast<const uint32_t*>(in);
    uint32_t* out = static_cast<uint32_t*>(fo.out);
    uint32_t m[kFilterPerThread];
#pragma unroll
    for (int j = 0; j < kFilterPerThread; ++j) {
      const int i = first + (int)threadIdx.x + j * kFilterThreads;
      m[j] = i < R ? __ldg(ids + i) : 0u;
    }
#pragma unroll
    for (int j = 0; j < kFilterPerThread; ++j) {
      const int local = (int)threadIdx.x + j * kFilterThreads;
      const int i = first + local;
      uint32_t n = 0, off = 0;
      if (i < R) {
        uint4 e = make_uint4(0u, 0u, 0u, 0u);
        const uint32_t v = pick_model<Ld::kLdg>(m[j], first_index + (uint64_t)i, mt, gcls, glists, (uint32_t)A,
                                                seed, &e);
        out[i] = v;
        if (((v >> 16) & 0xffu) == (uint32_t)LIG_OK) { n = e.x >> 16; off = e.w; }
      }
      s_excl[local] = n;
      s_list[local] = off;
    }
  } else {
    const int4* reqs = static_cast<const int4*>(in);
    int2* out = static_cast<int2*>(fo.out);
    int4 r[kFilterPerThread];
#pragma unroll
    for (int j = 0; j < kFilterPerThread; ++j) {
      const int i = first + (int)threadIdx.x + j * kFilterThreads;
      r[j] = i < R ? ld_stream_int4(reqs + i) : make_int4(0, 0, 0, 0);
    }
#pragma unroll
    for (int j = 0; j < kFilterPerThread; ++j) {
      const int local = (int)threadIdx.x + j * kFilterThreads;
      const int i = first + local;
      uint32_t n = 0, off = 0;
      if (i < R) {
        uint4 e;
        const int2 p = pick_one(r[j], gcls, glists, (uint32_t)A, seed, &e);
        st_stream_int2(out + i, p);
        if (((uint32_t)p.y & 7u) == (uint32_t)LIG_OK) { n = e.x >> 16; off = e.w; }
      }
      s_excl[local] = n;
      s_list[local] = off;
    }
  }
  __syncthreads();

  // 2. tile-local exclusive scan (thread t owns requests 4t .. 4t+3), then the look-back
  uint4 v = reinterpret_cast<const uint4*>(s_excl)[threadIdx.x];
  const uint32_t own = v.x + v.y + v.z + v.w;
  uint32_t incl = own;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += y;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kFilterThreads / 32; ++w) {
    before += w < warp ? s_warp[w] : 0u;
    total += s_warp[w];
  }
  uint32_t run = before + incl - own;
  const uint4 ex = make_uint4(run, run + v.x, run + v.x + v.y, run + v.x + v.y + v.z);
  reinterpret_cast<uint4*>(s_excl)[threadIdx.x] = ex;
  if (threadIdx.x == 0) s_excl[kFilterTile] = total;
  if (warp == 0) {
    const unsigned long long base = filter_look_back(fo.tiles, tile, total, lane);
    if (lane == 0) s_base = base;
  }
  __syncthreads();
  const unsigned long long base = s_base;

  // 3. offsets, then the lists
#pragma unroll
  for (int j = 0; j < kFilterPerThread; ++j) {
    const int local = (int)threadIdx.x + j * kFilterThreads;
    if (first + local < R) fo.offsets[first + local] = (long long)(base + s_excl[local]);
  }
  if (threadIdx.x == 0 && R - first <= kFilterTile) fo.offsets[R] = (long long)(base + total);
  const long long room = fo.capacity - (long long)base;
  const uint32_t limit = room <= 0 ? 0u : (room < (long long)total ? (uint32_t)room : total);
  uint16_t* dst = fo.pods + base;
  for (uint32_t j = threadIdx.x; j < limit; j += kFilterThreads) {
    int lo = 0, hi = kFilterTile;   // s_excl[lo] <= j < s_excl[hi]
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (s_excl[mid] <= j) lo = mid; else hi = mid;
    }
    dst[j] = __ldg(glists + s_list[lo] + (j - s_excl[lo]));
  }
}

// ---- K2i: the pick and up to LIG_MAX_FALLBACKS more distinct survivors in retry order
// (lig_schedule_batch_fallbacks, lig_schedule_models_batch_fallbacks; definition in include/lig.h).
// One thread per request with plain loads and stores, like lig_pick_stream_kernel /
// lig_pick_models_stream_kernel, so `in`, `out` and `fallbacks` may be page-locked host memory.
// The pick is pick_one / pick_model<Ld::kLdg> (same bytes out); the stream then continues from the
// state after the pick's draws into a partial Fisher-Yates shuffle of the class's list.  The
// permutation is kept as a record of the (position, value) pairs the swaps wrote: step j reads
// positions j and r_j >= j only, so a record at a position below j is never looked at again, and
// the last step's write is never read: at most LIG_MAX_FALLBACKS records, all in registers.
// Tables: the compact pool when the build sealed one, else the strided rows (as lig_filter_kernel).
constexpr int kFallbackThreads = 256;

// Go 1.22 Int31n(n) for 0 < n < 2^31, continuing `state` (the division is off the pick itself).
__device__ __forceinline__ uint32_t int31n_next(uint64_t& state, uint32_t n) {
  uint32_t v = splitmix_int31(state);
  if ((n & (n - 1)) == 0) return v & (n - 1);
  const uint32_t max_accept = 0x7fffffffu - (0x80000000u % n);
  while (v > max_accept) v = splitmix_int31(state);
  return v % n;
}

// Ranked entries 1 .. m-1 of a request's fallback row, then -1 to the end of the row: `state` is
// the pick's stream (seed ^ rand_key), `e` the class entry the pick used, `ok` whether it is LIG_OK.
__device__ __forceinline__ void write_fallback_row(uint64_t state, const uint4 e, bool ok, int n_fallbacks,
                                                   const uint16_t* __restrict__ glists, int16_t* __restrict__ row) {
  const uint32_t n = ok ? e.x >> 16 : 0u;
  const uint32_t m = min(n, (uint32_t)n_fallbacks + 1u);   // ranked entries, the pick included
  uint32_t pos[LIG_MAX_FALLBACKS], val[LIG_MAX_FALLBACKS];
  if (m >= 2u) {
    pos[0] = int31n_entry_next(state, e);   // step 0: the pick's own draws, perm[r0] = 0
    val[0] = 0u;
  }
  const uint16_t* list = glists + e.w;
#pragma unroll
  for (int j = 1; j <= LIG_MAX_FALLBACKS; ++j) {
    if (j > n_fallbacks) break;
    int16_t pod = -1;
    if ((uint32_t)j < m) {
      const uint32_t rj = (uint32_t)j + int31n_next(state, n - (uint32_t)j);
      uint32_t a = (uint32_t)j, b = rj;   // perm[j], perm[r_j]: the latest record wins
#pragma unroll
      for (int k = 0; k < j; ++k) {
        if (pos[k] == (uint32_t)j) a = val[k];
        if (pos[k] == rj) b = val[k];
      }
      pod = (int16_t)__ldg(list + b);
      if (j < LIG_MAX_FALLBACKS) {
        pos[j] = rj;
        val[j] = a;
      }
    }
    row[j - 1] = pod;
  }
}

// The compact pool when the build sealed one for this epoch's A, else the strided rows as given.
__device__ __forceinline__ void sealed_tables(const unsigned char* __restrict__ ctab, int A, const uint4** gcls,
                                              const uint16_t** glists) {
  const CompactHeader hdr = *reinterpret_cast<const CompactHeader*>(ctab);
  const uint32_t n_classes = 2u * ((uint32_t)A + 1u);
  if (hdr.bytes != 0u && hdr.n_classes == n_classes) {
    *gcls = reinterpret_cast<const uint4*>(ctab + sizeof(CompactHeader));
    *glists = reinterpret_cast<const uint16_t*>(ctab + sizeof(CompactHeader) + (size_t)n_classes * sizeof(ClassEntry));
  }
}

// kCount: the chain segment of lig_schedule_[models_]batch_feedback_chain_fallbacks.  The same pick
// and row on the chain's private tables (always the strided rows, as the count kernels read them),
// and the pick counted into the open window like lig_pick_[models_]count_kernel.  Row entries are
// not counted.  A lane past the end still reaches the full-warp match with pod -1.
template <bool kModels, bool kCount>
__global__ void __launch_bounds__(kFallbackThreads)
lig_pick_fallback_kernel(const void* __restrict__ in, void* __restrict__ out, int16_t* __restrict__ fallbacks,
                         int R, int n_fallbacks, const uint4* __restrict__ cls, const uint16_t* __restrict__ lists,
                         int A, const unsigned char* __restrict__ ctab, const unsigned char* __restrict__ mtab,
                         uint32_t n_models, uint64_t seed, uint64_t first_index, int* __restrict__ hist) {
  const int i = (int)blockIdx.x * kFallbackThreads + (int)threadIdx.x;
  if (!kCount && i >= R) return;
  const uint4* gcls = cls;
  const uint16_t* glists = lists;
  if constexpr (!kCount) sealed_tables(ctab, A, &gcls, &glists);
  int pod = -1;
  if (i < R) {
    uint4 e = make_uint4(0u, 0u, 0u, 0u);
    uint64_t key;
    bool ok;
    if constexpr (kModels) {
      ModelTables mt;
      mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
      mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
      mt.n_models = n_models;
      key = first_index + (uint64_t)i;
      const uint32_t v = pick_model<Ld::kLdg>(__ldg(static_cast<const uint32_t*>(in) + i), key, mt, gcls, glists,
                                              (uint32_t)A, seed, &e);
      static_cast<uint32_t*>(out)[i] = v;
      ok = ((v >> 16) & 0xffu) == (uint32_t)LIG_OK;
      pod = (int)(int16_t)(v & 0xffffu);
    } else {
      const int4 r = ld_stream_int4(static_cast<const int4*>(in) + i);
      key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
      const int2 p = pick_one(r, gcls, glists, (uint32_t)A, seed, &e);
      st_stream_int2(static_cast<int2*>(out) + i, p);
      ok = ((uint32_t)p.y & 7u) == (uint32_t)LIG_OK;
      pod = p.x;
    }
    write_fallback_row(seed ^ key, e, ok, n_fallbacks, glists, fallbacks + (size_t)i * (size_t)n_fallbacks);
  }
  if constexpr (kCount) count_window_picks(pod, (int)threadIdx.x & 31, hist);
}

// ---- K2j: session affinity (lig_schedule_[models_]batch_affinity; definition in include/lig.h) -----
// The class lookup and model resolve of the fallback kernel; only the selection differs.  A survivor
// p of the request's list scores mix(key ^ h[p]), h[p] = mix(pod_key[p]) (the slot's key table), and
// ranked entry j is the (j+1)-th in descending (score, ascending pod) order: pass j takes the largest
// pair below pass j-1's, so a row needs no sort and no per-thread storage.  Lists of up to
// kAffinityShortList pods are scored by their own thread; longer ones (caller trees of predicate
// nodes, KV ties) are found with a ballot and served one at a time by the whole warp, strided scoring
// and a __shfl_xor max-reduce per rank.  One thread per request, plain loads and stores (`in`, `keys`,
// `out` and `fallbacks` may be page-locked host memory); `fallbacks` is null when n_fallbacks = 0.
// kCount: the chain segment of lig_schedule_[models_]batch_feedback_chain_affinity.  The same ranking
// on the chain's private tables (always the strided rows, as the count kernels read them), and the
// pick counted into the open window like lig_pick_[models_]count_kernel; row entries are not counted.
constexpr int kAffinityShortList = 32;

__device__ __forceinline__ uint64_t affinity_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// (s, p) ranks before (bs, bp): a higher score, or an equal score (equal pod keys) and a lower pod.
__device__ __forceinline__ bool ranks_before(uint64_t s, int p, uint64_t bs, int bp) {
  return s > bs || (s == bs && p < bp);
}

template <bool kModels, bool kCount>
__global__ void __launch_bounds__(kFallbackThreads)
lig_pick_affinity_kernel(const void* __restrict__ in, const uint64_t* __restrict__ keys, void* __restrict__ out,
                         int16_t* __restrict__ fallbacks, int R, int n_fallbacks, const uint4* __restrict__ cls,
                         const uint16_t* __restrict__ lists, int A, const unsigned char* __restrict__ ctab,
                         const unsigned char* __restrict__ mtab, uint32_t n_models,
                         const uint64_t* __restrict__ hkeys, int* __restrict__ hist) {
  const int i = (int)blockIdx.x * kFallbackThreads + (int)threadIdx.x;
  const int lane = (int)threadIdx.x & 31;
  const uint4* gcls = cls;
  const uint16_t* glists = lists;
  if constexpr (!kCount) sealed_tables(ctab, A, &gcls, &glists);
  uint4 e = make_uint4(0u, 0u, 0u, 0u);
  uint64_t key = 0;
  bool resolved = false;
  uint32_t target = 255u;
  if (i < R) {
    if constexpr (kModels) {
      ModelTables mt;
      mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
      mt.targets = reinterpret_cast<const uint2*>(mt.entries + n_models);
      mt.n_models = n_models;
      key = keys[i];
      uint32_t adapter, critical;
      // the draw state is seed ^ key ^ LIG_DRAW_DOMAIN with seed 0: key ^ LIG_DRAW_DOMAIN
      resolved = resolve_model<Ld::kLdg>(static_cast<const uint32_t*>(in)[i], mt, 0, key, &adapter, &critical,
                                         &target);
      if (resolved) e = class_entry(make_int4((int)adapter, (int)critical, 0, 0), gcls, (uint32_t)A);
    } else {
      const int4 r = ld_stream_int4(static_cast<const int4*>(in) + i);
      key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
      e = class_entry(r, gcls, (uint32_t)A);
      resolved = true;
    }
  }
  const bool ok = resolved && (e.x & 7u) == (uint32_t)LIG_OK;
  const uint32_t n = ok ? e.x >> 16 : 0u;
  const uint32_t m = min(n, (uint32_t)n_fallbacks + 1u);   // ranked entries, the pick included
  const uint16_t* list = glists + e.w;
  int16_t* row = fallbacks ? fallbacks + (size_t)i * (size_t)n_fallbacks : nullptr;
  int pod = -1;
  if (n <= (uint32_t)kAffinityShortList) {
    uint64_t ps = ~0ull;   // pass j-1's pair; (2^64-1, -1) ranks before every pair
    int pp = -1;
    for (uint32_t j = 0; j < m; ++j) {
      uint64_t bs = 0;
      int bp = 0x7fffffff;   // (0, INT_MAX) ranks after every pair
      for (uint32_t t = 0; t < n; ++t) {
        const int p = (int)__ldg(list + t);
        const uint64_t s = affinity_mix(key ^ __ldg(hkeys + p));
        if (ranks_before(ps, pp, s, p) && ranks_before(s, p, bs, bp)) {
          bs = s;
          bp = p;
        }
      }
      if (j == 0) pod = bp; else row[j - 1] = (int16_t)bp;
      ps = bs;
      pp = bp;
    }
  }
  // long lists: the warp serves each in turn (lanes past R take part with n = 0)
  unsigned pending = __ballot_sync(0xffffffffu, n > (uint32_t)kAffinityShortList);
  while (pending) {
    const int src = __ffs(pending) - 1;
    pending &= pending - 1u;
    const uint64_t k = __shfl_sync(0xffffffffu, key, src);
    const uint32_t off = __shfl_sync(0xffffffffu, e.w, src);
    const uint32_t nn = __shfl_sync(0xffffffffu, n, src);
    const uint32_t mm = __shfl_sync(0xffffffffu, m, src);
    uint64_t ps = ~0ull;
    int pp = -1;
    for (uint32_t j = 0; j < mm; ++j) {
      uint64_t bs = 0;
      int bp = 0x7fffffff;
      for (uint32_t t = (uint32_t)lane; t < nn; t += 32u) {
        const int p = (int)__ldg(glists + off + t);
        const uint64_t s = affinity_mix(k ^ __ldg(hkeys + p));
        if (ranks_before(ps, pp, s, p) && ranks_before(s, p, bs, bp)) {
          bs = s;
          bp = p;
        }
      }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {
        const uint64_t os = __shfl_xor_sync(0xffffffffu, bs, d);
        const int op = __shfl_xor_sync(0xffffffffu, bp, d);
        if (ranks_before(os, op, bs, bp)) {
          bs = os;
          bp = op;
        }
      }
      if (lane == src) {
        if (j == 0) pod = bp; else row[j - 1] = (int16_t)bp;
      }
      ps = bs;
      pp = bp;
    }
  }
  if constexpr (kCount) count_window_picks(pod, lane, hist);   // every lane, pod -1 past R
  if (i >= R) return;
  for (int j = (int)max(m, 1u); j <= n_fallbacks; ++j) row[j - 1] = -1;
  if constexpr (kModels) {
    const uint32_t status = resolved ? e.x & 7u : (uint32_t)LIG_NO_MODEL;
    static_cast<uint32_t*>(out)[i] = pack_mpick(pod, status, resolved ? target : 255u);
  } else {
    st_stream_int2(static_cast<int2*>(out) + i, make_int2(pod, (int)(e.x & 0xffff0007u)));
  }
}

// loads[p] = picks of the closed windows + picks of the open one (the chain's per-pod loads).
__global__ void lig_feedback_loads_kernel(const int* __restrict__ total, const int* __restrict__ window,
                                          int* __restrict__ loads, int P) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < P) loads[p] = total[p] + window[p];
}

// ---- K3: persistent doorbell kernel (streaming micro-batches) ------------------------------------
// One resident CTA polls a mailbox in page-locked host memory.  The host writes the micro-batch
// (header + descriptors), then the ticket; the CTA schedules it with the same pick_one() and
// writes the picks and the completion ticket back to host memory.  No kernel launch and no stream
// synchronisation per micro-batch: the round trip is two PCIe crossings.  Class tables and model
// tables are read with ld.global.cg (L2 only): the kernel outlives snapshot and model uploads, and
// L1 is not coherent.
//
// Model-id mode (mode == kMailboxModels, lig_stream_submit_models): `reqs` holds `count` 4-byte
// model ids and `picks` receives `count` 4-byte lig_mpicks; each thread takes 4 consecutive ids,
// one 16-byte load and one 16-byte store.  The mode's extra header fields (first_index, n_models)
// sit in the last 16 bytes of the header, which the descriptor mode never reads.
constexpr int kMailboxCapacity = 4096;   // requests per doorbell
constexpr uint32_t kMailboxQuit = 0xffffffffu;
constexpr uint32_t kMailboxDescriptors = 0, kMailboxModels = 1;

struct alignas(64) Mailbox {
  // --- written by the host ---
  uint32_t ticket;            // doorbell: last field written (release); kMailboxQuit = leave the kernel
  uint32_t count;
  uint32_t A;
  uint32_t mode;              // kMailboxDescriptors / kMailboxModels
  uint64_t seed;
  const uint4* cls;           // device pointers of the snapshot slot to use
  const uint16_t* lists;
  const unsigned char* mtab;  // model mode: the slot's model blob (ModelHeader first)
  uint64_t first_index;       // model mode: rand_key of the first id
  uint32_t n_models;          // model mode
  uint32_t pad0;
  // --- written by the device ---
  alignas(64) uint32_t done;  // completion ticket (release)
  uint32_t pad1[15];
  alignas(64) lig_req reqs[kMailboxCapacity];
  alignas(64) lig_pick picks[kMailboxCapacity];
};
static_assert(offsetof(Mailbox, done) == 64, "the host-written header is one 64-byte line");
static_assert(offsetof(Mailbox, first_index) == 48, "descriptor mode reads bytes 0-47 of the header only");

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int4 ld_sys_int4(const void* p) {
  int4 r;
  asm volatile("ld.relaxed.sys.global.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__global__ void __launch_bounds__(kPickThreads)
lig_doorbell_kernel(Mailbox* mb) {
  __shared__ uint32_t s_go;
  uint32_t ticket = 1;
  for (;;) {
    if (threadIdx.x == 0) {
      uint32_t go = 1;
      for (;;) {
        const uint32_t t = ld_acquire_sys_u32(&mb->ticket);
        if (t == ticket) break;
        if (t == kMailboxQuit) { go = 0; break; }
      }
      s_go = go;
    }
    __syncthreads();
    if (!s_go) return;
    // One PCIe round trip for everything a small micro-batch needs: the header (same 64-byte
    // line as the ticket) and this thread's first descriptor are requested together, the
    // descriptor speculatively (the mailbox always holds kMailboxCapacity slots).  Every word of
    // h0-h2 is used (mode in h0.w, mtab in h2.zw), so each stays one 16-byte sys load: when only
    // some words were used, ptxas split them into 4- and 8-byte loads, one more PCIe read per
    // round trip, ~10 us on H100 (DESIGN.md section 7).  Keep them whole when editing the header.
    const int4 h0 = ld_sys_int4(&mb->ticket);          // ticket, count, A, mode
    const int4 h1 = ld_sys_int4(&mb->seed);            // seed lo/hi, cls lo/hi
    const int4 h2 = ld_sys_int4(&mb->lists);           // lists lo/hi, mtab lo/hi
    int4 r = ld_sys_int4(&mb->reqs[threadIdx.x]);      // a descriptor, or 4 model ids
    const uint32_t count = (uint32_t)h0.y, A = (uint32_t)h0.z;
    const uint64_t seed = ((uint64_t)(uint32_t)h1.y << 32) | (uint32_t)h1.x;
    const uint4* cls = reinterpret_cast<const uint4*>(((uint64_t)(uint32_t)h1.w << 32) | (uint32_t)h1.z);
    const uint16_t* lists = reinterpret_cast<const uint16_t*>(((uint64_t)(uint32_t)h2.y << 32) | (uint32_t)h2.x);
    if ((uint32_t)h0.w == kMailboxModels) {
      const int4 h3 = ld_sys_int4(&mb->first_index);   // first_index lo/hi, n_models, pad
      const uint64_t first_index = ((uint64_t)(uint32_t)h3.y << 32) | (uint32_t)h3.x;
      const unsigned char* mtab = reinterpret_cast<const unsigned char*>(((uint64_t)(uint32_t)h2.w << 32) | (uint32_t)h2.z);
      ModelTables mt;
      mt.n_models = (uint32_t)h3.z;
      mt.entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
      mt.targets = reinterpret_cast<const uint2*>(mt.entries + mt.n_models);
      uint32_t* out = reinterpret_cast<uint32_t*>(mb->picks);
      for (uint32_t g = threadIdx.x; 4u * g < count; g += kPickThreads) {   // ids 4g .. 4g+3
        if (g != threadIdx.x) r = ld_sys_int4(&mb->reqs[g]);
        const uint32_t m[4] = {(uint32_t)r.x, (uint32_t)r.y, (uint32_t)r.z, (uint32_t)r.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t i = 4u * g + (uint32_t)j;
          o[j] = i < count ? pick_model<Ld::kL2>(m[j], first_index + i, mt, cls, lists, A, seed) : 0u;
        }
        if (4u * g + 4u <= count) {
          asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1, %2, %3, %4};"
                       :: "l"(out + 4u * g), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
        } else {
#pragma unroll
          for (int j = 0; j < 3; ++j)
            if (4u * g + (uint32_t)j < count)
              asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(out + 4u * g + j), "r"(o[j]) : "memory");
        }
      }
    } else {
      for (uint32_t i = threadIdx.x; i < count; i += kPickThreads) {
        if (i != threadIdx.x) r = ld_sys_int4(&mb->reqs[i]);
        const int2 p = doorbell_pick(r, cls, lists, A, seed);
        asm volatile("st.relaxed.sys.global.v2.s32 [%0], {%1, %2};"
                     :: "l"(reinterpret_cast<int2*>(&mb->picks[i])), "r"(p.x), "r"(p.y) : "memory");
      }
    }
    // the barrier orders every thread's pick stores before thread 0's release store (cumulative)
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys_u32(&mb->done, ticket);
    ++ticket;
  }
}

// ---- K1: direct scan -------------------------------------------------------------------------------
template <bool kStaged>
__global__ void __launch_bounds__(kCtaThreads)
lig_scan_kernel(SnapView s, Thr thr, const int4* __restrict__ reqs, int2* __restrict__ out, int R,
                uint32_t* __restrict__ masks, uint64_t seed) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* X = reinterpret_cast<uint32_t*>(smem) + (size_t)warp * 3 * s.W;
  uint32_t* T = X + s.W;
  uint32_t* H = T + s.W;
  Fields f{s.kv, s.q, s.n_active, s.max_active};
  if constexpr (kStaged) {
    f = stage_fields(s, smem + scratch_bytes(s.W));
    __syncthreads();
  }
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < R; i += gridDim.x * kWarpsPerCta) {
    int4 r = __ldg(reqs + i);  // whole warp reads the same 16 bytes (broadcast)
    const bool critical = ((uint32_t)r.y & LIG_REQ_CRITICAL) != 0;
    const uint64_t key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
    const uint32_t* Hrow = stage_adapter_row(s, r.x, H, lane);
    EvalResult e = tree_eval_warp<kStaged>(f, Hrow, critical, thr, s.P, s.W, X, T, lane);
    int pod = -1;
    if (e.n > 0) {
      uint32_t k = int31n(seed ^ key, e.n, max_accept_for(e.n));
      for (int w = 0; w < s.W; ++w) {  // k-th survivor in pod order = pods[k]   scheduler.go:121
        uint32_t word = e.mask[w];
        uint32_t c = __popc(word);
        if (k < c) { pod = w * 32 + (int)__fns(word, 0, (int)k + 1); break; }
        k -= c;
      }
    }
    if (masks) {
      uint32_t* dst = masks + (size_t)i * s.W;
      for (int w = lane; w < s.W; w += 32) dst[w] = e.n ? e.mask[w] : 0u;
    }
    if (lane == 0) out[i] = make_int2(pod, (int)(e.status | (e.n << 16)));
    __syncwarp();
  }
}

// ---- retry scheduling: the tree over each request's pool without the pods it excludes --------------
// The p-th set bit of the W-word survivor mask M (p < the mask's popcount), warp-cooperatively.
// Survivors are counted per group of 32 words: lane g holds the inclusive prefix `incl` of the
// groups' counts (zero past the last group).  A ballot finds the group that holds position p, lane t
// reads word t of that group, and a second prefix and ballot find the word; __fns finds the bit.  The
// result is the same on every lane.
__device__ __forceinline__ int warp_select_survivor(const uint32_t* M, int W, uint32_t incl, uint32_t p, int lane) {
  const int g = __ffs(__ballot_sync(kFull, incl > p)) - 1;
  const uint32_t before = __shfl_sync(kFull, incl, (g + 31) & 31);   // survivors in groups 0 .. g-1
  const uint32_t excl_g = g > 0 ? before : 0u;
  const int w = g * 32 + lane;
  const uint32_t word = w < W ? M[w] : 0u;
  const uint32_t c = __popc(word);
  uint32_t in = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(kFull, in, d);
    if (lane >= d) in += t;
  }
  const uint32_t q = p - excl_g;
  const int t = __ffs(__ballot_sync(kFull, in > q)) - 1;
  int pod = -1;
  if (lane == t) pod = w * 32 + (int)__fns(word, 0, (int)(q - (in - c)) + 1);
  return __shfl_sync(kFull, pod, t);
}

// Every retry call (lig_schedule_[models_]batch[_feedback_chain]_excluding[_fallbacks]), with the
// scan's launch shape: one warp per request, columns staged when they fit (kStaged).
//
// Request i is a lig_req descriptor, or (kModels) model ids[i] at the fixed target targets[i] (the
// target_idx an earlier model call returned) with rand_key = first_index + i.  The warp resolves a
// model id without a draw: one broadcast 16-byte gather of the model entry, plus one target record
// when the model has >= 2 targets.  The request is LIG_NO_MODEL for an id past the table, an absent
// model, a model without TargetModels and t != 255, or a model with TargetModels and t >= their
// count; it writes that result (and a row of -1) and adds no load.  The model table is read through
// the read-only path: every launch is ordered behind the table's upload.
//
// The walk: lanes 0 .. n_excluded-1 each take one entry of the request's row and clear that pod's bit
// in the warp's root mask, which starts from every pod (kPool: the pool words of an epoch derived by
// lig_eject_pods).  A shared-memory atomicAnd, so a duplicate clears nothing twice, and entries
// outside [0, P) clear nothing.  The walk starts from that mask: the built-in tree, or (kTree) the
// caller tree that built the epoch (under the chain, the tree and thresholds the chain started with,
// on its private copy).  Requests and rows are read with plain loads: they may be page-locked host
// memory.
//
// The pick is the k-th survivor in pod order.  kRows adds the fallback row of the reduced survivor
// set: the pick is the same (the same Int31n(n') draws on seed ^ rand_key, continued here rather than
// on a copy), and entries 1 .. m-1 rank that set as write_fallback_row ranks a class's list, with the
// same (position, value) record of the partial Fisher-Yates shuffle.  Entry j is the perm[j]-th set
// bit of the survivor mask, selected by the whole warp (warp_select_survivor).  Lane j-1 keeps entry j
// and the row is stored by lanes 0 .. n_fallbacks-1.  kCount (the chain's segment): lane 0 adds each
// LIG_OK pick to the open window's histogram, one atomic per request (one warp per request: no
// cross-lane match as in count_window_picks); row entries add no load.
template <bool kModels, bool kStaged, bool kTree, bool kPool, bool kRows, bool kCount>
__global__ void __launch_bounds__(kCtaThreads)
lig_schedule_excluding_kernel(SnapView s, Thr thr, const __grid_constant__ FilterTree tree, const void* in,
                              const uint8_t* targets, const int16_t* excluded, int n_excluded, void* out, int R,
                              uint64_t seed, uint64_t first_index, const unsigned char* __restrict__ mtab,
                              uint32_t n_models, int n_fallbacks, int16_t* fallbacks, int* __restrict__ hist,
                              const uint32_t* __restrict__ pool) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* X = reinterpret_cast<uint32_t*>(smem) + (size_t)warp * 3 * s.W;
  uint32_t* T = X + s.W;       // the root mask: the built-in walk's second scratch mask, a tree walk's `in`
  uint32_t* H = T + s.W;
  const uint4* entries = reinterpret_cast<const uint4*>(mtab + sizeof(ModelHeader));
  const uint2* records = reinterpret_cast<const uint2*>(entries + n_models);
  Fields f{s.kv, s.q, s.n_active, s.max_active};
  if constexpr (kStaged) {
    f = stage_fields(s, smem + scratch_bytes(s.W));
    __syncthreads();
  }
  for (int i = blockIdx.x * kWarpsPerCta + warp; i < R; i += gridDim.x * kWarpsPerCta) {
    // ptxas's register allocation depends on the order of the statements below; this one gives the
    // figures of DESIGN §3.
    int4 r;                                    // whole warp reads the same request (broadcast)
    uint32_t m = 0, t = 0;
    if constexpr (kModels) {
      m = static_cast<const uint32_t*>(in)[i];
      t = targets[i];
    } else {
      r = static_cast<const int4*>(in)[i];
    }
    const int ex = lane < n_excluded ? excluded[(size_t)i * n_excluded + lane] : -1;
    uint64_t key;
    bool found = false;
    uint32_t adapter = 0, critical = 0;
    if constexpr (kModels) {
      key = first_index + (uint64_t)i;
      if (m < n_models) {
        const uint4 e = __ldg(entries + m);
        const uint32_t nt = e.x & 0xffu;
        found = (e.x & kModelPresent) && (nt == 0 ? t == 255u : t < nt);
        critical = (e.x >> 8) & 1u;
        adapter = e.w;                         // the own id (nt == 0) or the single target (nt == 1)
        if (found && nt >= 2u) adapter = __ldg(records + e.w + t).x;
      }
      if (!found) {
        if (lane == 0) static_cast<uint32_t*>(out)[i] = pack_mpick(-1, (uint32_t)LIG_NO_MODEL, 255u);
        if (kRows && lane < n_fallbacks) fallbacks[(size_t)i * (size_t)n_fallbacks + lane] = -1;
        __syncwarp();
        continue;
      }
    } else {
      critical = ((uint32_t)r.y & LIG_REQ_CRITICAL) != 0;
      key = ((uint64_t)(uint32_t)r.w << 32) | (uint32_t)r.z;
      adapter = (uint32_t)r.x;
    }
    const uint32_t* Hrow = stage_adapter_row(s, (int)adapter, H, lane);
    for (int w = lane; w < s.W; w += 32) {   // the request's pool: every pod (kPool: of the epoch's pool) ...
      if constexpr (kPool) {
        T[w] = pool[w];
      } else {
        const int rem = s.P - w * 32;
        T[w] = rem >= 32 ? kFull : ((1u << rem) - 1u);
      }
    }
    __syncwarp();
    if (ex >= 0 && ex < s.P) atomicAnd(T + (ex >> 5), ~(1u << (ex & 31)));   // ... but the excluded
    __syncwarp();
    uint32_t n = 0;
    for (int w = lane; w < s.W; w += 32) n += __popc(T[w]);
    n = __reduce_add_sync(kFull, n);
    EvalResult e;
    if constexpr (kTree)
      e = tree_walk_warp<kStaged, true>(f, tree.nodes, Hrow, critical != 0, s.P, s.W, T, X, lane, n);
    else
      e = tree_eval_warp<kStaged, true>(f, Hrow, critical != 0, thr, s.P, s.W, X, T, lane, n);
    int pod = -1;
    int16_t mine = -1;                         // kRows: row entry lane + 1
    if (e.n > 0) {
      if constexpr (kRows) {
        // survivors per group of 32 words: group g's count on lane g, then the inclusive prefix
        uint32_t incl = 0;
        const int groups = (s.W + 31) >> 5;
        for (int g = 0; g < groups; ++g) {
          const int w = g * 32 + lane;
          const uint32_t cg = __reduce_add_sync(kFull, w < s.W ? __popc(e.mask[w]) : 0u);
          if (lane == g) incl = cg;
        }
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t u = __shfl_up_sync(kFull, incl, d);
          if (lane >= d) incl += u;
        }
        uint64_t state = seed ^ key;
        uint32_t pos[LIG_MAX_FALLBACKS], val[LIG_MAX_FALLBACKS];
        pos[0] = int31n_next(state, e.n);     // step 0: the pick's own draws, perm[r0] = 0
        val[0] = 0u;
        pod = warp_select_survivor(e.mask, s.W, incl, pos[0], lane);
        const uint32_t mm = e.status == (uint32_t)LIG_OK ? min(e.n, (uint32_t)n_fallbacks + 1u) : 0u;
#pragma unroll
        for (int j = 1; j <= LIG_MAX_FALLBACKS; ++j) {
          if ((uint32_t)j >= mm) break;
          const uint32_t rj = (uint32_t)j + int31n_next(state, e.n - (uint32_t)j);
          uint32_t a = (uint32_t)j, b = rj;   // perm[j], perm[r_j]: the latest record wins
#pragma unroll
          for (int k = 0; k < j; ++k) {
            if (pos[k] == (uint32_t)j) a = val[k];
            if (pos[k] == rj) b = val[k];
          }
          const int p = warp_select_survivor(e.mask, s.W, incl, b, lane);
          if (lane == j - 1) mine = (int16_t)p;
          if (j < LIG_MAX_FALLBACKS) {
            pos[j] = rj;
            val[j] = a;
          }
        }
      } else {
        uint32_t k = int31n(seed ^ key, e.n, max_accept_for(e.n));
        for (int w = 0; w < s.W; ++w) {        // k-th survivor in pod order = pods[k]   scheduler.go:121
          uint32_t word = e.mask[w];
          uint32_t c = __popc(word);
          if (k < c) { pod = w * 32 + (int)__fns(word, 0, (int)k + 1); break; }
          k -= c;
        }
      }
    }
    if (lane == 0) {
      if constexpr (kModels)
        static_cast<uint32_t*>(out)[i] = pack_mpick(pod, e.status, t);
      else
        static_cast<int2*>(out)[i] = make_int2(pod, (int)(e.status | (e.n << 16)));
      if (kCount && pod >= 0) atomicAdd(hist + pod, 1);   // pod >= 0 only for LIG_OK
    }
    if (kRows && lane < n_fallbacks) fallbacks[(size_t)i * (size_t)n_fallbacks + lane] = mine;
    __syncwarp();
  }
}

}  // namespace lig
