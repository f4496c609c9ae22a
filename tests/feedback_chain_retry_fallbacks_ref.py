"""Sequential definition of retries with fallback rows under the load-feedback chain (include/lig.h,
lig_schedule_batch_feedback_chain_excluding_fallbacks), composed from existing definitions only.

A chain retry call with rows is a chain retry call (feedback_chain_retry_ref.retry_call) given
n_fallbacks k > 0.  It joins run_chain's sequence and windows like any other call; a segment of it is
retry_fallbacks_ref.retry_fallback_batch on the snapshot whose WaitingQueueSize is the chain's current
q, with the chain's tree and thresholds.  run_chain counts its picks like every other segment's; the
row entries add nothing.

Calls may mix all five kinds (plain, model-id, fallback, retry, retry with rows): run_chain_retry_fallbacks
takes the calls and ks of feedback_chain_retry_ref.run_chain_retries, where a retry call with ks[i] > 0
is a retry call with rows.  Such a call is handed to feedback_chain_fallbacks_ref.run_chain_fallbacks
with k = 0 and each request tagged with its position in the sequence, so its segments' rows land in
the right place whatever the window cuts.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

import numpy as np

import feedback_chain_fallbacks_ref as FR
import feedback_chain_retry_ref as CR
import oracle_tree as OT
import retry_fallbacks_ref as RF
from oracle import binding as B

retry_call = CR.retry_call


def _tagged(x: np.ndarray, at: int) -> np.ndarray:
    """The RETRY rows of x plus each request's position in the chain's sequence."""
    t = np.zeros(len(x), dtype=np.dtype([("req", B.REQ_DTYPE), ("excluded", np.int16, (x["excluded"].shape[1],)),
                                         ("at", np.int64)]))
    t["req"] = x["req"]
    t["excluded"] = x["excluded"]
    t["at"] = at + np.arange(len(x), dtype=np.int64)
    return t


def with_retry_fallback_calls(tables_for: FR.TablesFor, snap, rows: np.ndarray, k_at: np.ndarray,
                              thresholds=(0.8, 5, 50), nodes=None) -> FR.TablesFor:
    """tables_for(q) whose schedule() also takes tagged retry-with-rows segments: retry_fallback_batch on
    `snap` with the chain's queue sizes q; the rows go to rows[at] (k_at[at] = the call's k)."""
    def wrapped(q):
        schedule, klass, A = tables_for(q)
        snap_q = dataclasses.replace(snap, q=np.asarray(q, dtype=np.int64).astype(np.int32))

        def run(x, seed):
            if x.dtype.names is None or "at" not in x.dtype.names:
                return schedule(x, seed)
            at = x["at"]
            k = int(k_at[at[0]])                 # run_chain never crosses a call
            out, r = RF.retry_fallback_batch(snap_q, np.ascontiguousarray(x["req"]),
                                             np.ascontiguousarray(x["excluded"]), seed, k, thresholds, nodes)
            if nodes is not None:                # retry_ref clears the tree the chain's other calls walk
                OT.set_filter_tree(nodes)
            rows[at, :k] = r
            return out
        return run, klass, A
    return wrapped


def run_chain_retry_fallbacks(snap, calls: Sequence, window: int, ks: Optional[Sequence[int]] = None,
                              thresholds=(0.8, 5, 50), nodes=None, records: Optional[List[dict]] = None,
                              names: Optional[List[str]] = None):
    """(picks of every call, fallback rows of every call, loads[P]) for a chain over the packed snapshot
    `snap` of plain, model-id, fallback (ks[i] > 0), retry and retry-with-rows (a retry call with
    ks[i] > 0) calls.  nodes: a caller tree (with the oracle records and names of
    feedback_chain_fallbacks_ref.tree_tables), else the built-in tree with thresholds."""
    ks = [0] * len(calls) if ks is None else [int(k) for k in ks]
    bounds = np.cumsum([0] + [len(c) for c, _ in calls])
    with_rows = [CR.is_retry(c) and k > 0 for (c, _), k in zip(calls, ks)]
    rows = np.full((int(bounds[-1]), max([0] + ks)), -1, dtype=np.int16)
    k_at = np.repeat(np.array(ks, dtype=np.int64), np.diff(bounds))
    run_calls = [(_tagged(c, int(bounds[i])), s) if with_rows[i] else (c, s) for i, (c, s) in enumerate(calls)]
    run_ks = [0 if w else k for w, k in zip(with_rows, ks)]
    if nodes is None:
        tf = FR.class_table_tables(snap.P, snap.A, snap.kv, snap.n_active, snap.max_active, snap.bitmap, thresholds)
        tf = with_retry_fallback_calls(CR.with_retry_calls(tf, snap, thresholds), snap, rows, k_at, thresholds)
        outs, call_rows, loads = FR.run_chain_fallbacks(snap.P, snap.q, run_calls, run_ks, window, tf)
    else:
        OT.set_filter_tree(nodes)
        try:
            tf = FR.tree_tables(records, names)
            tf = with_retry_fallback_calls(CR.with_retry_calls(tf, snap, nodes=nodes), snap, rows, k_at, nodes=nodes)
            outs, call_rows, loads = FR.run_chain_fallbacks(snap.P, snap.q, run_calls, run_ks, window, tf)
        finally:
            OT.set_filter_tree(None)
    for i, w in enumerate(with_rows):
        if w:
            call_rows[i] = rows[bounds[i]:bounds[i + 1], :ks[i]].copy()
    return outs, call_rows, loads


def chain_retry_fallbacks(snap, calls: Sequence, window: int, k: int, **kw):
    """(picks of every call, rows of every call, loads[P]) of a chain of retry-with-rows calls, each
    with n_fallbacks = k."""
    return run_chain_retry_fallbacks(snap, calls, window, [k] * len(calls), **kw)
