"""Outlier ejection (lig_eject_pods, include/lig.h) by its definition (test infrastructure).

An epoch derived from a base with the pods E ejected answers every call as an epoch uploaded from the
literally reduced snapshot would: retry_ref.reduce_snapshot over the kept pods (their columns in
order, the ejected pods' bitmap columns dropped, A unchanged), then every pod index of the results
(pod_idx, survivor lists, fallback rows, loads) mapped back to the base's order.  Each function runs an
existing definition on that reduced snapshot and maps back: retry_ref (a retry row of -1 excludes
nothing, so it is Schedule on the reduced pool, under the built-in tree or a caller tree),
retry_fallbacks_ref and fallback_ref's ranking over those lists, and the chain references.  A retry row
is translated into the reduced pod order first; an entry that names an ejected pod leaves out nothing.
Nothing here masks a full pool, so the reference shares no logic with the kernels.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

import feedback_chain_fallbacks_ref as FCF
import feedback_chain_retry_fallbacks_ref as CRF
import feedback_chain_retry_ref as CR
import retry_fallbacks_ref as RF
import oracle_tree as OT
import retry_ref as RR
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PackedSnapshot
from oracle import binding as B


_memo: dict = {}


def reduced(snap: PackedSnapshot, ejected: Sequence[int]) -> Tuple[PackedSnapshot, np.ndarray]:
    """(the reduced snapshot, kept pods in the base's order), memoised per (snapshot, set): the memo
    holds the snapshot, so its id is not reused while the entry lives."""
    key = (id(snap), tuple(sorted(int(p) for p in ejected)))
    if key not in _memo:
        kept = RR.kept_pods(snap.P, list(ejected))
        _memo[key] = (snap, RR.reduce_snapshot(snap, kept), kept, {})
    return _memo[key][1], _memo[key][2]


def map_back(kept: np.ndarray, idx) -> np.ndarray:
    """Reduced pod indices -> the base's (negative entries stay -1)."""
    idx = np.asarray(idx, dtype=np.int64)
    if not len(kept):
        return np.full(idx.shape, -1, dtype=np.int64)
    return np.where(idx >= 0, kept[np.clip(idx, 0, len(kept) - 1)], -1)


def to_reduced(kept: np.ndarray, P: int, rows) -> np.ndarray:
    """A retry row in the base's order -> the reduced order: ejected and out-of-range entries become -1."""
    where = np.full(P, -1, dtype=np.int64)
    where[kept] = np.arange(len(kept))
    rows = np.asarray(rows, dtype=np.int64)
    ok = (rows >= 0) & (rows < P)
    return np.where(ok, where[np.clip(rows, 0, max(P - 1, 0))] if P else -1, -1).astype(np.int16)


def _picks_back(kept: np.ndarray, picks: np.ndarray) -> np.ndarray:
    out = picks.copy()
    out["pod_idx"] = map_back(kept, picks["pod_idx"])
    return out


def _no_rows(R: int) -> np.ndarray:
    return np.full((R, 1), -1, dtype=np.int16)


def schedule_batch(snap, ejected, reqs: np.ndarray, seed: int, thresholds=(0.8, 5, 50), nodes=None) -> np.ndarray:
    """lig_schedule_batch on the derived epoch."""
    small, kept = reduced(snap, ejected)
    return _picks_back(kept, RR.retry_batch(small, reqs, _no_rows(len(reqs)), seed, thresholds, nodes))


def klass(snap, ejected, critical: bool, adapter: int, thresholds=(0.8, 5, 50), nodes=None) -> Tuple[int, List[int]]:
    """lig_read_class on the derived epoch: (status, survivors in the base's order).  The same as
    retry_ref.survivors on the reduced snapshot with nothing excluded, with that snapshot's class table
    (or caller-tree pool) built once per (snapshot, set, thresholds, tree)."""
    small, kept = reduced(snap, ejected)
    tables = _memo[(id(snap), tuple(sorted(int(p) for p in ejected)))][3]
    tkey = (tuple(thresholds), None if nodes is None else tuple(tuple(n) if isinstance(n, tuple) else
                                                                (n.kind, n.next_on_success, n.next_on_failure,
                                                                 n.next_on_success_or_failure, n.queue_threshold,
                                                                 n.kv_threshold) for n in nodes))
    if nodes is None:
        if tkey not in tables:
            tables[tkey] = B.ClassTable(small.P, small.A, small.kv, small.q, small.n_active, small.max_active,
                                        small.bitmap, thresholds)
        st, _, lst = tables[tkey].klass(critical, adapter if 0 <= adapter < small.A else small.A)
    else:
        if tkey not in tables:
            tables[tkey] = OT.Pool(RR.records(small))
        names = RR.adapter_names(small)
        OT.set_filter_tree(nodes)
        try:
            st, lst = tables[tkey].filter(names[adapter] if 0 <= adapter < small.A else WL.UNKNOWN_MODEL, critical)
        finally:
            OT.set_filter_tree(None)
    return st, [int(kept[p]) for p in lst]


def fallback_batch(snap, ejected, reqs: np.ndarray, seed: int, k: int, thresholds=(0.8, 5, 50), nodes=None):
    """lig_schedule_batch_fallbacks on the derived epoch: (picks, rows (R, k)), fallback_ref's ranking
    of each request's class list on the reduced snapshot (through feedback_chain_fallbacks_ref's
    segment_rows, which also checks that step 0 of each ranking is the pick)."""
    picks = schedule_batch(snap, ejected, reqs, seed, thresholds, nodes)
    rows = FCF.segment_rows(reqs, picks, seed, k, lambda c, a: klass(snap, ejected, c, a, thresholds, nodes), snap.A)
    return picks, rows


def retry_batch(snap, ejected, reqs: np.ndarray, excluded, seed: int, thresholds=(0.8, 5, 50), nodes=None):
    """lig_schedule_batch_excluding on the derived epoch."""
    small, kept = reduced(snap, ejected)
    ex = to_reduced(kept, snap.P, np.asarray(excluded).reshape(len(reqs), -1))
    return _picks_back(kept, RR.retry_batch(small, reqs, ex, seed, thresholds, nodes))


def retry_fallback_batch(snap, ejected, reqs: np.ndarray, excluded, seed: int, k: int, thresholds=(0.8, 5, 50),
                         nodes=None):
    """lig_schedule_batch_excluding_fallbacks on the derived epoch: (picks, rows (R, k))."""
    small, kept = reduced(snap, ejected)
    ex = to_reduced(kept, snap.P, np.asarray(excluded).reshape(len(reqs), -1))
    picks, rows = RF.retry_fallback_batch(small, reqs, ex, seed, k, thresholds, nodes)
    return _picks_back(kept, picks), map_back(kept, rows).astype(np.int16)


def chain(snap, ejected, calls: Sequence, window: int, ks: Optional[Sequence[int]] = None,
          thresholds=(0.8, 5, 50), nodes=None):
    """(picks of every call, rows of every call, loads[P]) of a feedback chain on the derived epoch.
    calls: descriptor calls (reqs, seed) and retry calls (feedback_chain_retry_ref.retry_call) in the
    base's order; ks as in feedback_chain_retry_fallbacks_ref (rows for fallback and retry calls)."""
    small, kept = reduced(snap, ejected)
    red = [(CR.retry_call(c["req"], to_reduced(kept, snap.P, c["excluded"]), s) if CR.is_retry(c) else (c, s))
           for c, s in calls]
    kw = {}
    if nodes is not None:
        kw = dict(nodes=nodes, records=RR.records(small), names=RR.adapter_names(small) + [WL.UNKNOWN_MODEL])
    outs, rows, loads = CRF.run_chain_retry_fallbacks(small, red, window, ks, thresholds=thresholds, **kw)
    full = np.zeros(snap.P, dtype=np.int64)
    full[kept] = loads
    return ([_picks_back(kept, o) for o in outs], [map_back(kept, r).astype(np.int16) for r in rows], full)
