"""Thin object wrapper over the C ABI (one ``lig_ctx`` = one CUDA device)."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import _native as N
from .packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, PackedModels, PackedSnapshot, _ptr


def _node_table(nodes):
    """(pointer, count) of a filter-tree table for lig_set_filter_tree (see Engine.set_filter_tree)."""
    if nodes is None:
        return None, 0
    if hasattr(nodes, "flatten"):
        nodes = nodes.flatten()
    rows = [n if isinstance(n, N.LigFilterNode) else N.LigFilterNode(*n) for n in nodes]
    return (N.LigFilterNode * len(rows))(*rows), len(rows)


class Engine:
    def __init__(self, device: int = 0, max_pods: int = 4096, max_adapters: int = 1024,
                 max_batch: int = 1 << 20, _borrowed_ctx=None):
        self._lib = N.load()
        self._owned = _borrowed_ctx is None
        if self._owned:
            self._ctx = C.c_void_p()
            N.check(self._lib.lig_create(C.byref(self._ctx), device, max_pods, max_adapters, max_batch))
        else:
            self._ctx = C.c_void_p(_borrowed_ctx)      # a member of an EngineGroup
        self.device = device
        self.max_batch = max_batch

    def close(self) -> None:
        if getattr(self, "_ctx", None):
            if self._owned:
                self._lib.lig_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ---- thresholds (scheduler.go:15-24) ----
    def set_thresholds(self, kv_cache_threshold=0.8, queue_threshold_critical=5,
                       queueing_threshold_lora=50) -> None:
        t = N.LigThresholds(kv_cache_threshold, queue_threshold_critical, queueing_threshold_lora)
        N.check(self._lib.lig_set_thresholds(self._ctx, C.byref(t)))

    # ---- caller filter trees ----
    def set_filter_tree(self, nodes) -> None:
        """Build the class tables of later uploads with a caller filter tree: a ``scheduling.Filter``
        chart, a sequence of ``LigFilterNode`` / (kind, next_on_success, next_on_failure,
        next_on_success_or_failure, queue_threshold, kv_threshold) rows (node 0 = root), or None for
        the built-in tree.  Resident epochs keep their tables."""
        N.check(self._lib.lig_set_filter_tree(self._ctx, *_node_table(nodes)))

    # ---- snapshots ----
    def upload_snapshot(self, epoch: int, snap: PackedSnapshot, block: bool = True) -> None:
        """block=False: lig_upload_snapshot_async (staged + enqueued, the device is not waited for)."""
        fn = self._lib.lig_upload_snapshot if block else self._lib.lig_upload_snapshot_async
        N.check(fn(self._ctx, epoch, snap.P, snap.A, _ptr(snap.kv), _ptr(snap.q), _ptr(snap.n_active),
                   _ptr(snap.max_active), _ptr(snap.bitmap)))

    def update_snapshot(self, new_epoch: int, base_epoch: int, pod_idx, kv, q, n_active, max_active,
                        adapter_offsets, adapter_ids) -> None:
        """Delta upload: base_epoch with the listed pods replaced becomes new_epoch."""
        a = [np.ascontiguousarray(pod_idx, dtype=np.int32), np.ascontiguousarray(kv, dtype=np.float64),
             np.ascontiguousarray(q, dtype=np.int32), np.ascontiguousarray(n_active, dtype=np.uint16),
             np.ascontiguousarray(max_active, dtype=np.uint16), np.ascontiguousarray(adapter_offsets, dtype=np.int32),
             np.ascontiguousarray(adapter_ids, dtype=np.int32)]
        N.check(self._lib.lig_update_snapshot(self._ctx, new_epoch, base_epoch, len(a[0]), *[_ptr(x) for x in a]))

    def eject_pods(self, new_epoch: int, base_epoch: int, pod_idx) -> None:
        """lig_eject_pods: new_epoch is base_epoch's snapshot scheduled without the pods `pod_idx` (the
        complete ejected set; empty = every pod back)."""
        idx = np.ascontiguousarray(pod_idx, dtype=np.int32)
        N.check(self._lib.lig_eject_pods(self._ctx, new_epoch, base_epoch, _ptr(idx), len(idx)))

    def upload_snapshot_device(self, epoch: int, P: int, A: int, d_blob: int, stream: int = 0) -> None:
        N.check(self._lib.lig_upload_snapshot_device(self._ctx, epoch, P, A, d_blob, stream or None))

    # ---- host-buffer hot path ----
    def schedule_batch(self, epoch: int, seed: int, reqs: np.ndarray,
                       out: Optional[np.ndarray] = None) -> np.ndarray:
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        if out is None:
            out = np.empty(R, dtype=PICK_DTYPE)
        N.check(self._lib.lig_schedule_batch(self._ctx, epoch, seed, _ptr(reqs), R, _ptr(out)))
        return out

    def schedule_batch_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int) -> None:
        N.check(self._lib.lig_schedule_batch(self._ctx, epoch, seed, h_reqs, R, h_out))

    def schedule_batch_async(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int) -> int:
        """Page-locked buffers only; returns a ticket for schedule_wait."""
        t = C.c_int(-1)
        N.check(self._lib.lig_schedule_batch_async(self._ctx, epoch, seed, h_reqs, R, h_out, C.byref(t)))
        return t.value

    def schedule_wait(self, ticket: int) -> None:
        N.check(self._lib.lig_schedule_wait(self._ctx, ticket))

    # ---- model requests: the resolve step of HandleRequestBody on the device ----
    def upload_models(self, epoch: int, models: PackedModels, block: bool = True) -> None:
        fn = self._lib.lig_upload_models if block else self._lib.lig_upload_models_async
        N.check(fn(self._ctx, epoch, models.n_models, _ptr(models.target_offsets),
                   _ptr(models.target_adapter_ids), _ptr(models.target_weights),
                   _ptr(models.critical), _ptr(models.self_adapter_ids), _ptr(models.present)))

    def schedule_models_batch(self, epoch: int, seed: int, model_ids: np.ndarray, first_index: int = 0,
                              out: Optional[np.ndarray] = None) -> np.ndarray:
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        if out is None:
            out = np.empty(R, dtype=MPICK_DTYPE)
        N.check(self._lib.lig_schedule_models_batch(self._ctx, epoch, seed, first_index, _ptr(model_ids), R, _ptr(out)))
        return out

    def schedule_models_batch_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int, R: int, h_out: int) -> None:
        N.check(self._lib.lig_schedule_models_batch(self._ctx, epoch, seed, first_index, h_ids, R, h_out))

    def schedule_models_batches_device(self, epoch: int, seed: int, first_index: int, d_ids_ptrs, R: int,
                                       d_out_ptrs, stream: int = 0) -> None:
        n = len(d_ids_ptrs)
        a = (C.c_void_p * n)(*d_ids_ptrs)
        b = (C.c_void_p * n)(*d_out_ptrs)
        N.check(self._lib.lig_schedule_models_batches_device(self._ctx, epoch, seed, first_index, a, R, b, n,
                                                             stream or None))

    def resolve_models(self, epoch: int, seed: int, model_ids: np.ndarray, first_index: int = 0):
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        reqs = np.empty(R, dtype=REQ_DTYPE)
        out = np.empty(R, dtype=MPICK_DTYPE)
        N.check(self._lib.lig_resolve_models(self._ctx, epoch, seed, first_index, _ptr(model_ids), R,
                                             _ptr(reqs), _ptr(out)))
        return reqs, out

    def schedule_batch_feedback_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int, sub_batch: int,
                                       n_windows: int = 0, d_hist: int = 0, stream: int = 0) -> None:
        """Opt-in in-batch load feedback: windows of `sub_batch` requests, the picks of each window
        (all ranks) are added to the pods' queue sizes before the next window is scheduled."""
        N.check(self._lib.lig_schedule_batch_feedback_device(self._ctx, epoch, seed, d_reqs, R, d_out, sub_batch,
                                                             n_windows, d_hist or None, stream or None))

    def schedule_batch_feedback_chain(self, epoch: int, seed: int, reqs: np.ndarray, window: int,
                                      loads: Optional[np.ndarray] = None,
                                      out: Optional[np.ndarray] = None) -> np.ndarray:
        """Load feedback carried across calls against one epoch (include/lig.h, the feedback chain):
        windows of `window` requests over the sequence of all chain calls, cut regardless of call
        boundaries.  `loads` (int32[P], optional) receives the picks per pod since the chain began."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        if out is None:
            out = np.empty(R, dtype=PICK_DTYPE)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_batch_feedback_chain(self._ctx, epoch, seed, _ptr(reqs), R, _ptr(out), window,
                                                            _ptr(loads) if loads is not None else None))
        return out

    def schedule_batch_feedback_chain_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int, window: int,
                                          h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_feedback_chain(self._ctx, epoch, seed, h_reqs, R, h_out, window,
                                                            h_loads or None))

    def schedule_batch_feedback_chain_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int,
                                             window: int, d_loads: int = 0, stream: int = 0) -> None:
        """The chain with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_feedback_chain_device(self._ctx, epoch, seed, d_reqs or None, R,
                                                                   d_out or None, window, d_loads or None,
                                                                   stream or None))

    def schedule_models_batch_feedback_chain(self, epoch: int, seed: int, model_ids: np.ndarray, window: int,
                                             first_index: int = 0, loads=False,
                                             out: Optional[np.ndarray] = None):
        """Model-id requests in the feedback chain: one more chain call, in the same sequence and
        windows as schedule_batch_feedback_chain, resolved against the epoch's resident model table
        (rand_key of request i = first_index + i).  `loads` (an int32[P] array, or False) receives
        the picks per pod since the chain began."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        if out is None:
            out = np.empty(R, dtype=MPICK_DTYPE)
        if loads is False or loads is None:
            loads = None
        else:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_models_batch_feedback_chain(self._ctx, epoch, seed, first_index, _ptr(model_ids),
                                                                   R, _ptr(out), window,
                                                                   _ptr(loads) if loads is not None else None))
        return out

    def schedule_models_batch_feedback_chain_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int, R: int,
                                                 h_out: int, window: int, h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_models_batch_feedback_chain(self._ctx, epoch, seed, first_index, h_ids, R,
                                                                   h_out, window, h_loads or None))

    def schedule_models_batch_feedback_chain_device(self, epoch: int, seed: int, first_index: int, d_ids: int, R: int,
                                                    d_out: int, window: int, d_loads: int = 0,
                                                    stream: int = 0) -> None:
        """The model-id chain call with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_device(self._ctx, epoch, seed, first_index,
                                                                          d_ids or None, R, d_out or None, window,
                                                                          d_loads or None, stream or None))

    def feedback_chain_reset(self) -> None:
        """The next feedback-chain call starts a new chain from its epoch's scrape."""
        N.check(self._lib.lig_feedback_chain_reset(self._ctx))

    # ---- survivor lists of a batch: Filter.Filter next to the pick ----
    def _filter(self, fn, args, R: int, out: np.ndarray, capacity: Optional[int]):
        """Call a host filter form with a pod buffer of `capacity` entries (default 4 per request);
        when the lists need more, call once more with exactly what offsets[R] asks for."""
        offsets = np.full(R + 1, -1, dtype=np.int64)
        cap = 4 * R if capacity is None else capacity
        for _ in range(2):
            pods = np.empty(cap, dtype=np.uint16)
            rc = fn(self._ctx, *args, _ptr(out), _ptr(offsets), _ptr(pods), cap)
            if rc == N.LIG_ERR_INVALID and capacity is None and int(offsets[R]) > cap:
                cap = int(offsets[R])
                continue
            break
        N.check(rc)
        return out, offsets, pods[: int(offsets[R])]

    def filter_batch(self, epoch: int, seed: int, reqs: np.ndarray, capacity: Optional[int] = None):
        """lig_filter_batch: (picks, int64 offsets[R + 1], uint16 pods) where request i's survivors are
        pods[offsets[i]:offsets[i + 1]] and picks equal schedule_batch's.  With `capacity` given, the
        pod buffer has that many entries and a larger total raises LigError."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        return self._filter(self._lib.lig_filter_batch, (epoch, seed, _ptr(reqs), R), R,
                            np.empty(R, dtype=PICK_DTYPE), capacity)

    def filter_models_batch(self, epoch: int, seed: int, model_ids: np.ndarray, first_index: int = 0,
                            capacity: Optional[int] = None):
        """lig_filter_models_batch: (picks, offsets, pods) as filter_batch, the picks those of
        schedule_models_batch with the same first_index."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        return self._filter(self._lib.lig_filter_models_batch, (epoch, seed, first_index, _ptr(model_ids), R), R,
                            np.empty(R, dtype=MPICK_DTYPE), capacity)

    def filter_batch_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int, h_offsets: int, h_pods: int,
                         capacity: int) -> None:
        N.check(self._lib.lig_filter_batch(self._ctx, epoch, seed, h_reqs or None, R, h_out or None,
                                           h_offsets or None, h_pods or None, capacity))

    def filter_models_batch_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int, R: int, h_out: int,
                                h_offsets: int, h_pods: int, capacity: int) -> None:
        N.check(self._lib.lig_filter_models_batch(self._ctx, epoch, seed, first_index, h_ids or None, R, h_out or None,
                                                  h_offsets or None, h_pods or None, capacity))

    def filter_batch_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int, d_offsets: int,
                            d_pods: int, capacity: int, stream: int = 0) -> None:
        """lig_filter_batch_device: device pointers, enqueued on `stream` (not synchronised); the
        caller checks offsets[R] against `capacity`."""
        N.check(self._lib.lig_filter_batch_device(self._ctx, epoch, seed, d_reqs or None, R, d_out or None,
                                                  d_offsets or None, d_pods or None, capacity, stream or None))

    def filter_models_batch_device(self, epoch: int, seed: int, first_index: int, d_ids: int, R: int, d_out: int,
                                   d_offsets: int, d_pods: int, capacity: int, stream: int = 0) -> None:
        """lig_filter_models_batch_device: the model-id form of filter_batch_device."""
        N.check(self._lib.lig_filter_models_batch_device(self._ctx, epoch, seed, first_index, d_ids or None, R,
                                                         d_out or None, d_offsets or None, d_pods or None, capacity,
                                                         stream or None))

    # ---- fallback endpoints: the pick and up to LIG_MAX_FALLBACKS more distinct survivors ----
    def schedule_batch_fallbacks(self, epoch: int, seed: int, reqs: np.ndarray, n: int):
        """lig_schedule_batch_fallbacks: (picks, int16 fallbacks of shape (R, n)); the picks equal
        schedule_batch's, row i holds request i's next distinct survivors in retry order, -1 padded."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_batch_fallbacks(self._ctx, epoch, seed, _ptr(reqs), R, _ptr(out), n,
                                                       _ptr(rows)))
        return out, rows

    def schedule_batch_fallbacks_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int, n: int,
                                     h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_batch_fallbacks(self._ctx, epoch, seed, h_reqs or None, R, h_out or None, n,
                                                       h_fallbacks or None))

    def schedule_batch_fallbacks_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int, n: int,
                                        d_fallbacks: int, stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_fallbacks_device(self._ctx, epoch, seed, d_reqs or None, R,
                                                              d_out or None, n, d_fallbacks or None, stream or None))

    # ---- session affinity: rendezvous hashing of a caller key over the survivors ----
    def upload_pod_keys(self, epoch: int, keys) -> None:
        """lig_upload_pod_keys: one stable uint64 identity per pod of `epoch`, in its pod order."""
        k = np.ascontiguousarray(keys, dtype=np.uint64)
        N.check(self._lib.lig_upload_pod_keys(self._ctx, epoch, len(k), _ptr(k)))

    def schedule_batch_affinity(self, epoch: int, reqs: np.ndarray, n: int = 0):
        """lig_schedule_batch_affinity: (picks, int16 fallbacks of shape (R, n)); rand_key is the affinity
        key, status and n_survivors are schedule_batch's, pod_idx the survivor with the highest score."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_batch_affinity(self._ctx, epoch, _ptr(reqs), R, _ptr(out), n,
                                                      _ptr(rows) if n > 0 else None))
        return out, rows

    def schedule_batch_affinity_ptr(self, epoch: int, h_reqs: int, R: int, h_out: int, n: int,
                                    h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_batch_affinity(self._ctx, epoch, h_reqs or None, R, h_out or None, n,
                                                      h_fallbacks or None))

    def schedule_batch_affinity_device(self, epoch: int, d_reqs: int, R: int, d_out: int, n: int,
                                       d_fallbacks: int, stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_affinity_device(self._ctx, epoch, d_reqs or None, R, d_out or None, n,
                                                             d_fallbacks or None, stream or None))

    def schedule_models_batch_affinity(self, epoch: int, model_ids: np.ndarray, keys: np.ndarray, n: int = 0):
        """lig_schedule_models_batch_affinity: (picks, int16 fallbacks (R, n)); request i is model_ids[i]
        with affinity key keys[i], its target drawn on the state keys[i] ^ LIG_DRAW_DOMAIN."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        R = int(model_ids.shape[0])
        assert keys.shape == (R,)
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_models_batch_affinity(self._ctx, epoch, _ptr(model_ids), _ptr(keys), R,
                                                             _ptr(out), n, _ptr(rows) if n > 0 else None))
        return out, rows

    def schedule_models_batch_affinity_ptr(self, epoch: int, h_ids: int, h_keys: int, R: int, h_out: int, n: int,
                                           h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_models_batch_affinity(self._ctx, epoch, h_ids or None, h_keys or None, R,
                                                             h_out or None, n, h_fallbacks or None))

    def schedule_models_batch_affinity_device(self, epoch: int, d_ids: int, d_keys: int, R: int, d_out: int, n: int,
                                              d_fallbacks: int, stream: int = 0) -> None:
        """The model-id form with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_affinity_device(self._ctx, epoch, d_ids or None, d_keys or None,
                                                                    R, d_out or None, n, d_fallbacks or None,
                                                                    stream or None))

    # ---- retry scheduling: the tree again over each request's pool without the pods it excludes ----
    def schedule_batch_excluding(self, epoch: int, seed: int, reqs: np.ndarray, excluded: np.ndarray) -> np.ndarray:
        """lig_schedule_batch_excluding: excluded is an int16 array of shape (R, n_excluded) of pod indices
        (entries outside [0, P) exclude nothing); request i is scheduled over the epoch's pods without
        the pods of row i."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        assert excluded.dtype == np.int16 and excluded.flags.c_contiguous and excluded.ndim == 2
        R = int(reqs.shape[0])
        assert excluded.shape[0] == R
        out = np.empty(R, dtype=PICK_DTYPE)
        N.check(self._lib.lig_schedule_batch_excluding(self._ctx, epoch, seed, _ptr(reqs), R, _ptr(excluded),
                                                       int(excluded.shape[1]), _ptr(out)))
        return out

    def schedule_batch_excluding_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_excluded: int,
                                     n_excluded: int, h_out: int) -> None:
        N.check(self._lib.lig_schedule_batch_excluding(self._ctx, epoch, seed, h_reqs or None, R, h_excluded or None,
                                                       n_excluded, h_out or None))

    def schedule_batch_excluding_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_excluded: int,
                                        n_excluded: int, d_out: int, stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_excluding_device(self._ctx, epoch, seed, d_reqs or None, R,
                                                              d_excluded or None, n_excluded, d_out or None,
                                                              stream or None))

    # ---- retry scheduling with fallback rows: the retry's pick and more survivors of the reduced pool ----
    def schedule_batch_excluding_fallbacks(self, epoch: int, seed: int, reqs: np.ndarray, excluded: np.ndarray,
                                           n: int):
        """lig_schedule_batch_excluding_fallbacks: (picks, int16 fallbacks of shape (R, n)); the picks equal
        schedule_batch_excluding's, row i holds request i's next distinct survivors of its reduced pool in
        retry order, -1 padded."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        assert excluded.dtype == np.int16 and excluded.flags.c_contiguous and excluded.ndim == 2
        R = int(reqs.shape[0])
        assert excluded.shape[0] == R
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_batch_excluding_fallbacks(self._ctx, epoch, seed, _ptr(reqs), R,
                                                                 _ptr(excluded), int(excluded.shape[1]), _ptr(out),
                                                                 n, _ptr(rows)))
        return out, rows

    def schedule_batch_excluding_fallbacks_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_excluded: int,
                                               n_excluded: int, h_out: int, n: int, h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_batch_excluding_fallbacks(self._ctx, epoch, seed, h_reqs or None, R,
                                                                 h_excluded or None, n_excluded, h_out or None, n,
                                                                 h_fallbacks or None))

    def schedule_batch_excluding_fallbacks_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_excluded: int,
                                                  n_excluded: int, d_out: int, n: int, d_fallbacks: int,
                                                  stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_excluding_fallbacks_device(self._ctx, epoch, seed, d_reqs or None, R,
                                                                        d_excluded or None, n_excluded,
                                                                        d_out or None, n, d_fallbacks or None,
                                                                        stream or None))

    # ---- retries under the feedback chain: a chain call whose requests exclude the pods they tried ----
    def schedule_batch_feedback_chain_excluding(self, epoch: int, seed: int, reqs: np.ndarray, excluded: np.ndarray,
                                                window: int, loads: Optional[np.ndarray] = None) -> np.ndarray:
        """lig_schedule_batch_feedback_chain_excluding: request i is scheduled as schedule_batch_excluding
        would on the chain's load-adjusted copy at its position in the chain's sequence, and its pick
        counts toward the open window.  `loads` as schedule_batch_feedback_chain's."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        assert excluded.dtype == np.int16 and excluded.flags.c_contiguous and excluded.ndim == 2
        R = int(reqs.shape[0])
        assert excluded.shape[0] == R
        out = np.empty(R, dtype=PICK_DTYPE)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding(
            self._ctx, epoch, seed, _ptr(reqs), R, _ptr(excluded), int(excluded.shape[1]), _ptr(out), window,
            _ptr(loads) if loads is not None else None))
        return out

    def schedule_batch_feedback_chain_excluding_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_excluded: int,
                                                    n_excluded: int, h_out: int, window: int,
                                                    h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding(self._ctx, epoch, seed, h_reqs or None, R,
                                                                      h_excluded or None, n_excluded, h_out or None,
                                                                      window, h_loads or None))

    def schedule_batch_feedback_chain_excluding_device(self, epoch: int, seed: int, d_reqs: int, R: int,
                                                       d_excluded: int, n_excluded: int, d_out: int, window: int,
                                                       d_loads: int = 0, stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding_device(
            self._ctx, epoch, seed, d_reqs or None, R, d_excluded or None, n_excluded, d_out or None, window,
            d_loads or None, stream or None))

    def schedule_batch_feedback_chain_excluding_fallbacks(self, epoch: int, seed: int, reqs: np.ndarray,
                                                          excluded: np.ndarray, n: int, window: int,
                                                          loads: Optional[np.ndarray] = None):
        """lig_schedule_batch_feedback_chain_excluding_fallbacks: (picks, int16 fallbacks of shape (R, n)); the
        picks and loads are schedule_batch_feedback_chain_excluding's, row i ranks request i's reduced
        survivor set on the chain's copy as schedule_batch_excluding_fallbacks ranks it on the epoch."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        assert excluded.dtype == np.int16 and excluded.flags.c_contiguous and excluded.ndim == 2
        R = int(reqs.shape[0])
        assert excluded.shape[0] == R
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding_fallbacks(
            self._ctx, epoch, seed, _ptr(reqs), R, _ptr(excluded), int(excluded.shape[1]), _ptr(out), n, _ptr(rows),
            window, _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_batch_feedback_chain_excluding_fallbacks_ptr(self, epoch: int, seed: int, h_reqs: int, R: int,
                                                              h_excluded: int, n_excluded: int, h_out: int, n: int,
                                                              h_fallbacks: int, window: int, h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding_fallbacks(
            self._ctx, epoch, seed, h_reqs or None, R, h_excluded or None, n_excluded, h_out or None, n,
            h_fallbacks or None, window, h_loads or None))

    def schedule_batch_feedback_chain_excluding_fallbacks_device(self, epoch: int, seed: int, d_reqs: int, R: int,
                                                                 d_excluded: int, n_excluded: int, d_out: int, n: int,
                                                                 d_fallbacks: int, window: int, d_loads: int = 0,
                                                                 stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_feedback_chain_excluding_fallbacks_device(
            self._ctx, epoch, seed, d_reqs or None, R, d_excluded or None, n_excluded, d_out or None, n,
            d_fallbacks or None, window, d_loads or None, stream or None))

    # ---- model-id retries: keep the drawn target (an earlier model call's target_idx), resolve on the device ----
    @staticmethod
    def _model_retry_args(model_ids: np.ndarray, targets: np.ndarray, excluded: np.ndarray) -> int:
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        assert targets.dtype == np.uint8 and targets.flags.c_contiguous
        assert excluded.dtype == np.int16 and excluded.flags.c_contiguous and excluded.ndim == 2
        R = int(model_ids.shape[0])
        assert targets.shape == (R,) and excluded.shape[0] == R
        return R

    def schedule_models_batch_excluding(self, epoch: int, seed: int, model_ids: np.ndarray, targets: np.ndarray,
                                        excluded: np.ndarray, first_index: int = 0) -> np.ndarray:
        """lig_schedule_models_batch_excluding: request i is model_ids[i] at the fixed target targets[i]
        (uint8, the target_idx an earlier model call returned; 255 = the model's own adapter), resolved
        without a draw and scheduled as schedule_batch_excluding schedules its descriptor, rand_key
        first_index + i."""
        R = self._model_retry_args(model_ids, targets, excluded)
        out = np.empty(R, dtype=MPICK_DTYPE)
        N.check(self._lib.lig_schedule_models_batch_excluding(self._ctx, epoch, seed, first_index, _ptr(model_ids),
                                                              _ptr(targets), R, _ptr(excluded),
                                                              int(excluded.shape[1]), _ptr(out)))
        return out

    def schedule_models_batch_excluding_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int, h_targets: int,
                                            R: int, h_excluded: int, n_excluded: int, h_out: int) -> None:
        N.check(self._lib.lig_schedule_models_batch_excluding(self._ctx, epoch, seed, first_index, h_ids or None,
                                                              h_targets or None, R, h_excluded or None, n_excluded,
                                                              h_out or None))

    def schedule_models_batch_excluding_device(self, epoch: int, seed: int, first_index: int, d_ids: int,
                                               d_targets: int, R: int, d_excluded: int, n_excluded: int, d_out: int,
                                               stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_excluding_device(self._ctx, epoch, seed, first_index,
                                                                     d_ids or None, d_targets or None, R,
                                                                     d_excluded or None, n_excluded, d_out or None,
                                                                     stream or None))

    def schedule_models_batch_excluding_fallbacks(self, epoch: int, seed: int, model_ids: np.ndarray,
                                                  targets: np.ndarray, excluded: np.ndarray, n: int,
                                                  first_index: int = 0):
        """lig_schedule_models_batch_excluding_fallbacks: (picks, int16 fallbacks (R, n)); the picks equal
        schedule_models_batch_excluding's, the rows rank the reduced pool as
        schedule_batch_excluding_fallbacks does."""
        R = self._model_retry_args(model_ids, targets, excluded)
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_models_batch_excluding_fallbacks(
            self._ctx, epoch, seed, first_index, _ptr(model_ids), _ptr(targets), R, _ptr(excluded),
            int(excluded.shape[1]), _ptr(out), n, _ptr(rows)))
        return out, rows

    def schedule_models_batch_excluding_fallbacks_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int,
                                                      h_targets: int, R: int, h_excluded: int, n_excluded: int,
                                                      h_out: int, n: int, h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_models_batch_excluding_fallbacks(
            self._ctx, epoch, seed, first_index, h_ids or None, h_targets or None, R, h_excluded or None, n_excluded,
            h_out or None, n, h_fallbacks or None))

    def schedule_models_batch_excluding_fallbacks_device(self, epoch: int, seed: int, first_index: int, d_ids: int,
                                                         d_targets: int, R: int, d_excluded: int, n_excluded: int,
                                                         d_out: int, n: int, d_fallbacks: int,
                                                         stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_excluding_fallbacks_device(
            self._ctx, epoch, seed, first_index, d_ids or None, d_targets or None, R, d_excluded or None, n_excluded,
            d_out or None, n, d_fallbacks or None, stream or None))

    def schedule_models_batch_feedback_chain_excluding(self, epoch: int, seed: int, model_ids: np.ndarray,
                                                       targets: np.ndarray, excluded: np.ndarray, window: int,
                                                       first_index: int = 0,
                                                       loads: Optional[np.ndarray] = None) -> np.ndarray:
        """lig_schedule_models_batch_feedback_chain_excluding: the model-id retry as a chain call, in the
        chain's sequence and windows, on its load-adjusted copy.  `loads` as schedule_batch_feedback_chain's."""
        R = self._model_retry_args(model_ids, targets, excluded)
        out = np.empty(R, dtype=MPICK_DTYPE)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding(
            self._ctx, epoch, seed, first_index, _ptr(model_ids), _ptr(targets), R, _ptr(excluded),
            int(excluded.shape[1]), _ptr(out), window, _ptr(loads) if loads is not None else None))
        return out

    def schedule_models_batch_feedback_chain_excluding_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int,
                                                           h_targets: int, R: int, h_excluded: int, n_excluded: int,
                                                           h_out: int, window: int, h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding(
            self._ctx, epoch, seed, first_index, h_ids or None, h_targets or None, R, h_excluded or None, n_excluded,
            h_out or None, window, h_loads or None))

    def schedule_models_batch_feedback_chain_excluding_device(self, epoch: int, seed: int, first_index: int,
                                                              d_ids: int, d_targets: int, R: int, d_excluded: int,
                                                              n_excluded: int, d_out: int, window: int,
                                                              d_loads: int = 0, stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding_device(
            self._ctx, epoch, seed, first_index, d_ids or None, d_targets or None, R, d_excluded or None, n_excluded,
            d_out or None, window, d_loads or None, stream or None))

    def schedule_models_batch_feedback_chain_excluding_fallbacks(self, epoch: int, seed: int, model_ids: np.ndarray,
                                                                 targets: np.ndarray, excluded: np.ndarray, n: int,
                                                                 window: int, first_index: int = 0,
                                                                 loads: Optional[np.ndarray] = None):
        """lig_schedule_models_batch_feedback_chain_excluding_fallbacks: (picks, int16 fallbacks (R, n)); the
        picks and loads are schedule_models_batch_feedback_chain_excluding's."""
        R = self._model_retry_args(model_ids, targets, excluded)
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks(
            self._ctx, epoch, seed, first_index, _ptr(model_ids), _ptr(targets), R, _ptr(excluded),
            int(excluded.shape[1]), _ptr(out), n, _ptr(rows), window, _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_models_batch_feedback_chain_excluding_fallbacks_ptr(self, epoch: int, seed: int, first_index: int,
                                                                     h_ids: int, h_targets: int, R: int,
                                                                     h_excluded: int, n_excluded: int, h_out: int,
                                                                     n: int, h_fallbacks: int, window: int,
                                                                     h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks(
            self._ctx, epoch, seed, first_index, h_ids or None, h_targets or None, R, h_excluded or None, n_excluded,
            h_out or None, n, h_fallbacks or None, window, h_loads or None))

    def schedule_models_batch_feedback_chain_excluding_fallbacks_device(self, epoch: int, seed: int,
                                                                        first_index: int, d_ids: int, d_targets: int,
                                                                        R: int, d_excluded: int, n_excluded: int,
                                                                        d_out: int, n: int, d_fallbacks: int,
                                                                        window: int, d_loads: int = 0,
                                                                        stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device(
            self._ctx, epoch, seed, first_index, d_ids or None, d_targets or None, R, d_excluded or None, n_excluded,
            d_out or None, n, d_fallbacks or None, window, d_loads or None, stream or None))

    def schedule_models_batch_fallbacks(self, epoch: int, seed: int, model_ids: np.ndarray, n: int,
                                        first_index: int = 0):
        """lig_schedule_models_batch_fallbacks: (picks, int16 fallbacks (R, n)), the picks those of
        schedule_models_batch with the same first_index."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        N.check(self._lib.lig_schedule_models_batch_fallbacks(self._ctx, epoch, seed, first_index, _ptr(model_ids), R,
                                                              _ptr(out), n, _ptr(rows)))
        return out, rows

    def schedule_models_batch_fallbacks_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int, R: int,
                                            h_out: int, n: int, h_fallbacks: int) -> None:
        N.check(self._lib.lig_schedule_models_batch_fallbacks(self._ctx, epoch, seed, first_index, h_ids or None, R,
                                                              h_out or None, n, h_fallbacks or None))

    def schedule_models_batch_fallbacks_device(self, epoch: int, seed: int, first_index: int, d_ids: int, R: int,
                                               d_out: int, n: int, d_fallbacks: int, stream: int = 0) -> None:
        """The model-id form with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_fallbacks_device(self._ctx, epoch, seed, first_index,
                                                                     d_ids or None, R, d_out or None, n,
                                                                     d_fallbacks or None, stream or None))

    # ---- fallback rows under the feedback chain: a chain call that also returns each request's row ----
    def schedule_batch_feedback_chain_fallbacks(self, epoch: int, seed: int, reqs: np.ndarray, n: int, window: int,
                                                loads: Optional[np.ndarray] = None):
        """lig_schedule_batch_feedback_chain_fallbacks: (picks, int16 fallbacks (R, n)).  The picks and
        `loads` are schedule_batch_feedback_chain's for the same sequence; row i ranks the survivors of
        request i's class in the chain's tables at its position, the list its pick drew from."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_batch_feedback_chain_fallbacks(
            self._ctx, epoch, seed, _ptr(reqs), R, _ptr(out), n, _ptr(rows), window,
            _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_batch_feedback_chain_fallbacks_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int,
                                                    n: int, h_fallbacks: int, window: int, h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_feedback_chain_fallbacks(self._ctx, epoch, seed, h_reqs or None, R,
                                                                      h_out or None, n, h_fallbacks or None, window,
                                                                      h_loads or None))

    def schedule_batch_feedback_chain_fallbacks_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int,
                                                       n: int, d_fallbacks: int, window: int, d_loads: int = 0,
                                                       stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_feedback_chain_fallbacks_device(
            self._ctx, epoch, seed, d_reqs or None, R, d_out or None, n, d_fallbacks or None, window,
            d_loads or None, stream or None))

    def schedule_models_batch_feedback_chain_fallbacks(self, epoch: int, seed: int, model_ids: np.ndarray, n: int,
                                                       window: int, first_index: int = 0,
                                                       loads: Optional[np.ndarray] = None):
        """lig_schedule_models_batch_feedback_chain_fallbacks: (picks, int16 fallbacks (R, n)), the
        picks and `loads` those of schedule_models_batch_feedback_chain with the same first_index."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        R = int(model_ids.shape[0])
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_fallbacks(
            self._ctx, epoch, seed, first_index, _ptr(model_ids), R, _ptr(out), n, _ptr(rows), window,
            _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_models_batch_feedback_chain_fallbacks_ptr(self, epoch: int, seed: int, first_index: int, h_ids: int,
                                                           R: int, h_out: int, n: int, h_fallbacks: int, window: int,
                                                           h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_fallbacks(
            self._ctx, epoch, seed, first_index, h_ids or None, R, h_out or None, n, h_fallbacks or None, window,
            h_loads or None))

    def schedule_models_batch_feedback_chain_fallbacks_device(self, epoch: int, seed: int, first_index: int,
                                                              d_ids: int, R: int, d_out: int, n: int,
                                                              d_fallbacks: int, window: int, d_loads: int = 0,
                                                              stream: int = 0) -> None:
        """The model-id form with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_fallbacks_device(
            self._ctx, epoch, seed, first_index, d_ids or None, R, d_out or None, n, d_fallbacks or None, window,
            d_loads or None, stream or None))

    # ---- session affinity under the feedback chain: the affinity ranking over the chain's tables ----
    def schedule_batch_feedback_chain_affinity(self, epoch: int, reqs: np.ndarray, n: int, window: int,
                                               loads: Optional[np.ndarray] = None):
        """lig_schedule_batch_feedback_chain_affinity: (picks, int16 fallbacks (R, n)).  A chain call whose
        pick and row rank the survivors of request i's class in the chain's tables at its position by
        the affinity key rand_key; only the pick is counted into the chain's windows."""
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        out = np.empty(R, dtype=PICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_batch_feedback_chain_affinity(
            self._ctx, epoch, _ptr(reqs), R, _ptr(out), n, _ptr(rows) if n > 0 else None, window,
            _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_batch_feedback_chain_affinity_ptr(self, epoch: int, h_reqs: int, R: int, h_out: int, n: int,
                                                   h_fallbacks: int, window: int, h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_feedback_chain_affinity(self._ctx, epoch, h_reqs or None, R,
                                                                     h_out or None, n, h_fallbacks or None, window,
                                                                     h_loads or None))

    def schedule_batch_feedback_chain_affinity_device(self, epoch: int, d_reqs: int, R: int, d_out: int, n: int,
                                                      d_fallbacks: int, window: int, d_loads: int = 0,
                                                      stream: int = 0) -> None:
        """Device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_batch_feedback_chain_affinity_device(
            self._ctx, epoch, d_reqs or None, R, d_out or None, n, d_fallbacks or None, window, d_loads or None,
            stream or None))

    def schedule_models_batch_feedback_chain_affinity(self, epoch: int, model_ids: np.ndarray, keys: np.ndarray,
                                                      n: int, window: int, loads: Optional[np.ndarray] = None):
        """lig_schedule_models_batch_feedback_chain_affinity: (picks, int16 fallbacks (R, n)); request i is
        model_ids[i] with affinity key keys[i], resolved as schedule_models_batch_affinity resolves it."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        R = int(model_ids.shape[0])
        assert keys.shape == (R,)
        out = np.empty(R, dtype=MPICK_DTYPE)
        rows = np.empty((R, max(n, 0)), dtype=np.int16)
        if loads is not None:
            assert loads.dtype == np.int32 and loads.flags.c_contiguous
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_affinity(
            self._ctx, epoch, _ptr(model_ids), _ptr(keys), R, _ptr(out), n, _ptr(rows) if n > 0 else None, window,
            _ptr(loads) if loads is not None else None))
        return out, rows

    def schedule_models_batch_feedback_chain_affinity_ptr(self, epoch: int, h_ids: int, h_keys: int, R: int,
                                                          h_out: int, n: int, h_fallbacks: int, window: int,
                                                          h_loads: int = 0) -> None:
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_affinity(
            self._ctx, epoch, h_ids or None, h_keys or None, R, h_out or None, n, h_fallbacks or None, window,
            h_loads or None))

    def schedule_models_batch_feedback_chain_affinity_device(self, epoch: int, d_ids: int, d_keys: int, R: int,
                                                             d_out: int, n: int, d_fallbacks: int, window: int,
                                                             d_loads: int = 0, stream: int = 0) -> None:
        """The model-id form with device pointers, enqueued on `stream` (not synchronised)."""
        N.check(self._lib.lig_schedule_models_batch_feedback_chain_affinity_device(
            self._ctx, epoch, d_ids or None, d_keys or None, R, d_out or None, n, d_fallbacks or None, window,
            d_loads or None, stream or None))

    def pick_kernel_info(self, epoch: int) -> dict:
        name = C.create_string_buffer(64)
        grid, threads, tb, in_smem = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        N.check(self._lib.lig_pick_kernel_info(self._ctx, epoch, name, 64, C.byref(grid), C.byref(threads),
                                               C.byref(tb), C.byref(in_smem)))
        return {"kernel": name.value.decode(), "grid": grid.value, "threads": threads.value,
                "table_bytes": tb.value, "tables_in_smem": bool(in_smem.value)}

    def last_pick_launch(self) -> dict:
        """The pick kernel of the most recent pick launch and its template arguments (lig.h)."""
        info = N.LigLaunchInfo()
        N.check(self._lib.lig_last_pick_launch(self._ctx, C.byref(info)))
        return {f: getattr(info, f) for f, _ in N.LigLaunchInfo._fields_}

    # ---- one process per GPU: NCCL inside the library ----
    def comm_unique_id(self) -> bytes:
        buf = (C.c_char * N.LIG_COMM_ID_BYTES)()
        N.check(self._lib.lig_comm_unique_id(buf))
        return bytes(buf)

    def comm_init_rank(self, n_ranks: int, rank: int, unique_id: bytes) -> None:
        buf = (C.c_char * N.LIG_COMM_ID_BYTES).from_buffer_copy(unique_id)
        N.check(self._lib.lig_comm_init_rank(self._ctx, n_ranks, rank, buf))

    def comm_upload_snapshot_device(self, epoch: int, P: int, A: int, d_blob: int, root: int = 0,
                                    stream: int = 0) -> None:
        N.check(self._lib.lig_comm_upload_snapshot_device(self._ctx, epoch, P, A, d_blob or None, root,
                                                          stream or None))

    def comm_upload_snapshot(self, epoch: int, P: int, A: int, snap: Optional[PackedSnapshot], root: int = 0) -> None:
        if snap is None:
            N.check(self._lib.lig_comm_upload_snapshot(self._ctx, epoch, P, A, None, None, None, None, None, root))
        else:
            N.check(self._lib.lig_comm_upload_snapshot(self._ctx, epoch, P, A, _ptr(snap.kv), _ptr(snap.q),
                                                       _ptr(snap.n_active), _ptr(snap.max_active),
                                                       _ptr(snap.bitmap), root))

    def comm_allreduce_i32(self, d_values: int, n: int, stream: int = 0) -> None:
        N.check(self._lib.lig_comm_allreduce_i32(self._ctx, d_values, n, stream or None))

    def schedule_scan(self, epoch: int, seed: int, reqs: np.ndarray, want_masks: bool = True,
                      W: int = 0) -> Tuple[np.ndarray, Optional[np.ndarray]]:
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        out = np.empty(R, dtype=PICK_DTYPE)
        masks = np.zeros((R, W), dtype=np.uint32) if want_masks else None
        N.check(self._lib.lig_schedule_scan(self._ctx, epoch, seed, _ptr(reqs), R, _ptr(out),
                                            _ptr(masks) if masks is not None else None))
        return out, masks

    # ---- HBM-resident hot path (device pointers, async on `stream`) ----
    def schedule_batch_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int,
                              stream: int = 0) -> None:
        N.check(self._lib.lig_schedule_batch_device(self._ctx, epoch, seed, d_reqs, R, d_out,
                                                    stream or None))

    def schedule_batches_device(self, epoch: int, seed: int, d_reqs_ptrs, R: int, d_out_ptrs,
                                stream: int = 0) -> None:
        """Queue len(d_reqs_ptrs) resident batches back to back (one pass through the ABI)."""
        n = len(d_reqs_ptrs)
        assert n == len(d_out_ptrs)
        a = (C.c_void_p * n)(*d_reqs_ptrs)
        b = (C.c_void_p * n)(*d_out_ptrs)
        N.check(self._lib.lig_schedule_batches_device(self._ctx, epoch, seed, a, R, b, n,
                                                      stream or None))

    def schedule_scan_device(self, epoch: int, seed: int, d_reqs: int, R: int, d_out: int,
                             d_masks: int = 0, stream: int = 0) -> None:
        N.check(self._lib.lig_schedule_scan_device(self._ctx, epoch, seed, d_reqs, R, d_out,
                                                   d_masks or None, stream or None))

    # ---- streaming doorbell (persistent kernel) ----
    def stream_open(self) -> None:
        N.check(self._lib.lig_stream_open(self._ctx))

    def stream_close(self) -> None:
        N.check(self._lib.lig_stream_close(self._ctx))

    def stream_submit(self, epoch: int, seed: int, reqs: np.ndarray) -> np.ndarray:
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        out = np.empty(len(reqs), dtype=PICK_DTYPE)
        N.check(self._lib.lig_stream_submit(self._ctx, epoch, seed, _ptr(reqs), len(reqs), _ptr(out)))
        return out

    def stream_submit_models(self, epoch: int, seed: int, model_ids: np.ndarray, first_index: int = 0) -> np.ndarray:
        """One doorbell round trip for model ids: the picks of schedule_models_batch, without a launch."""
        assert model_ids.dtype == np.uint32 and model_ids.flags.c_contiguous
        out = np.empty(len(model_ids), dtype=MPICK_DTYPE)
        N.check(self._lib.lig_stream_submit_models(self._ctx, epoch, seed, first_index, _ptr(model_ids),
                                                   len(model_ids), _ptr(out)))
        return out

    def read_class(self, epoch: int, critical: bool, adapter_id: int, P: int):
        status, n = C.c_int(), C.c_int()
        lst = np.zeros(max(P, 1), dtype=np.uint16)
        N.check(self._lib.lig_read_class(self._ctx, epoch, int(bool(critical)), adapter_id,
                                         C.byref(status), C.byref(n), _ptr(lst)))
        return status.value, n.value, lst[: n.value].copy()

    @property
    def kernel_launches(self) -> int:
        return int(self._lib.lig_kernel_launches(self._ctx))

    @property
    def sm_count(self) -> int:
        return int(self._lib.lig_sm_count(self._ctx))


class EngineGroup:
    """Several GPUs owned by one process (lig_group_*): the snapshot is replicated with one in-library
    ncclBroadcast per upload, the request batch shards contiguously, results stay in request order."""

    def __init__(self, devices, max_pods: int = 4096, max_adapters: int = 1024, max_batch: int = 1 << 20):
        self._lib = N.load()
        self._g = C.c_void_p()
        arr = (C.c_int * len(devices))(*devices)
        N.check(self._lib.lig_group_create(C.byref(self._g), arr, len(devices), max_pods, max_adapters, max_batch))
        self.devices = list(devices)
        self.max_batch = max_batch

    def close(self) -> None:
        if getattr(self, "_g", None):
            self._lib.lig_group_destroy(self._g)
            self._g = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def size(self) -> int:
        return int(self._lib.lig_group_size(self._g))

    def member(self, i: int) -> Engine:
        ctx = self._lib.lig_group_ctx(self._g, i)
        if not ctx:
            raise IndexError(i)
        return Engine(self.devices[i], max_batch=self.max_batch, _borrowed_ctx=ctx)

    def set_thresholds(self, kv_cache_threshold=0.8, queue_threshold_critical=5, queueing_threshold_lora=50) -> None:
        t = N.LigThresholds(kv_cache_threshold, queue_threshold_critical, queueing_threshold_lora)
        N.check(self._lib.lig_group_set_thresholds(self._g, C.byref(t)))

    def set_filter_tree(self, nodes) -> None:
        """Engine.set_filter_tree on every member (an invalid table changes none)."""
        N.check(self._lib.lig_group_set_filter_tree(self._g, *_node_table(nodes)))

    def upload_snapshot(self, epoch: int, snap: PackedSnapshot) -> None:
        N.check(self._lib.lig_group_upload_snapshot(self._g, epoch, snap.P, snap.A, _ptr(snap.kv), _ptr(snap.q),
                                                    _ptr(snap.n_active), _ptr(snap.max_active), _ptr(snap.bitmap)))

    def schedule_batch(self, epoch: int, seed: int, reqs: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        if out is None:
            out = np.empty(R, dtype=PICK_DTYPE)
        N.check(self._lib.lig_group_schedule_batch(self._g, epoch, seed, _ptr(reqs), R, _ptr(out)))
        return out

    def schedule_batch_ptr(self, epoch: int, seed: int, h_reqs: int, R: int, h_out: int) -> None:
        N.check(self._lib.lig_group_schedule_batch(self._g, epoch, seed, h_reqs, R, h_out))
