"""Sequential definition of retries under the load-feedback chain (include/lig.h,
lig_schedule_batch_feedback_chain_excluding), on top of feedback_chain_ref.run_chain.

A chain retry call is one more chain call: its requests join the sequence and the windows of
run_chain like any other.  The call is a structured array of RETRY dtype (the descriptor and its row
of excluded pods), so scheduler_for(q) can tell it from descriptor, model-id (MREQ_DTYPE) and
fallback calls: a retry segment is retry_ref.retry_batch on the snapshot whose WaitingQueueSize is
the chain's current q, with the chain's tree and thresholds.  run_chain counts its picks (pod_idx >= 0
only for LIG_OK) like every other segment's.

Calls may mix all four kinds: run_chain_retries takes feedback_chain_fallbacks_ref's calls and ks (k = 0
for plain, model-id and retry calls) and wraps its tables_for.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

import numpy as np

import feedback_chain_fallbacks_ref as FR
import oracle_tree as OT
import retry_ref as RR
from oracle import binding as B


def retry_dtype(k: int) -> np.dtype:
    return np.dtype([("req", B.REQ_DTYPE), ("excluded", np.int16, (k,))])


def retry_call(reqs: np.ndarray, excluded: np.ndarray, seed: int):
    """A chain retry call for run_chain_retries: (RETRY rows, seed)."""
    excluded = np.asarray(excluded, dtype=np.int16)
    assert excluded.ndim == 2 and len(excluded) == len(reqs)
    x = np.zeros(len(reqs), dtype=retry_dtype(excluded.shape[1]))
    x["req"] = reqs
    x["excluded"] = excluded
    return x, seed


def is_retry(x: np.ndarray) -> bool:
    return x.dtype.names is not None and "excluded" in x.dtype.names


def with_retry_calls(tables_for: FR.TablesFor, snap, thresholds=(0.8, 5, 50), nodes=None) -> FR.TablesFor:
    """tables_for(q) whose schedule() also takes retry segments: retry_ref.retry_batch on `snap` with the
    chain's queue sizes q (nodes: the chain's caller tree, None = the built-in tree with thresholds)."""
    def wrapped(q):
        schedule, klass, A = tables_for(q)
        snap_q = dataclasses.replace(snap, q=np.asarray(q, dtype=np.int64).astype(np.int32))

        def run(x, seed):
            if not is_retry(x):
                return schedule(x, seed)
            out = RR.retry_batch(snap_q, np.ascontiguousarray(x["req"]),
                                 np.ascontiguousarray(x["excluded"]), seed, thresholds, nodes)
            if nodes is not None:          # retry_batch clears the tree the chain's other calls walk
                OT.set_filter_tree(nodes)
            return out
        return run, klass, A
    return wrapped


def run_chain_retries(snap, calls: Sequence, window: int, ks: Optional[Sequence[int]] = None,
                      thresholds=(0.8, 5, 50), nodes=None, records: Optional[List[dict]] = None,
                      names: Optional[List[str]] = None):
    """(picks of every call, fallback rows of every call, loads[P]) for a chain over the packed snapshot
    `snap` of plain, model-id, fallback (ks[i] > 0) and retry calls.  nodes: a caller tree (with the
    oracle records and names of feedback_chain_fallbacks_ref.tree_tables), else the built-in tree."""
    ks = [0] * len(calls) if ks is None else list(ks)
    if nodes is None:
        tf = FR.class_table_tables(snap.P, snap.A, snap.kv, snap.n_active, snap.max_active, snap.bitmap, thresholds)
        return FR.run_chain_fallbacks(snap.P, snap.q, calls, ks, window, with_retry_calls(tf, snap, thresholds))
    OT.set_filter_tree(nodes)
    try:
        tf = FR.tree_tables(records, names)
        return FR.run_chain_fallbacks(snap.P, snap.q, calls, ks, window, with_retry_calls(tf, snap, nodes=nodes))
    finally:
        OT.set_filter_tree(None)


def chain_retry(snap, calls: Sequence, window: int, **kw):
    """(picks of every call, loads[P]) of a chain of retry (and other) calls."""
    outs, _, loads = run_chain_retries(snap, calls, window, **kw)
    return outs, loads
