"""Sequential definition of fallback rows under the load-feedback chain (include/lig.h,
lig_schedule_[models_]batch_feedback_chain_fallbacks), on top of feedback_chain_ref.run_chain.

A chain fallback call is a chain call of its kind plus a row per request.  The window walk, the
picks and the loads are run_chain's, untouched: only picks are counted, row entries add nothing.
The row of a request ranks the survivor list of its class in the tables of the queue sizes at its
position in the sequence (the list its pick drew from) with fallback_ref.fallback_rows.  So each
segment that run_chain schedules also takes its rows from the tables that segment was picked on.

Calls are (reqs, seed) descriptor calls or model_call() rows of models_feedback_chain_ref, each with
its n_fallbacks k (0 = a plain chain call: no rows).  Requests that are not LIG_OK get a row of -1.
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import numpy as np

import models_feedback_chain_ref as MC
from fallback_ref import fallback_rows
from feedback_chain_ref import run_chain
from oracle import binding as B

LIG_OK = 0

# tables_for(q) -> (schedule(reqs, seed) -> picks, klass(critical, adapter) -> (status, survivor list), A)
TablesFor = Callable[[np.ndarray], Tuple[Callable, Callable, int]]


def class_of(reqs: np.ndarray, A: int) -> Tuple[np.ndarray, np.ndarray]:
    """(critical, adapter class) of descriptors: ids outside [0, A) are the class A, as on the device."""
    crit = (reqs["flags"] & 1).astype(np.int64)
    a = np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)
    return crit, a


def segment_rows(reqs: np.ndarray, picks: np.ndarray, seed: int, k: int, klass: Callable, A: int) -> np.ndarray:
    """Rows (R, k) of one segment: the ranking over each request's class list in `klass`."""
    R = len(reqs)
    ok = picks["status"] == LIG_OK
    crit, a = class_of(reqs, A)
    cls = crit * (A + 1) + a
    starts = np.zeros(R, dtype=np.int64)
    counts = np.zeros(R, dtype=np.int64)
    uniq, inv = np.unique(cls[ok], return_inverse=True)
    lists = [np.asarray(klass(bool(c // (A + 1)), int(c % (A + 1)))[1], dtype=np.int64) for c in uniq.tolist()]
    n_of = np.array([len(x) for x in lists], dtype=np.int64)
    first = np.concatenate([[0], np.cumsum(n_of)])[:-1].astype(np.int64)
    starts[ok], counts[ok] = first[inv], n_of[inv]
    pods = np.concatenate(lists) if lists else np.zeros(0, dtype=np.int64)
    rows, r0 = fallback_rows(seed, reqs["rand_key"], ok, starts, counts, pods, k)
    # step 0 of the ranking is the pick the chain made on these tables
    got = np.where(ok, pods[np.where(ok, starts + np.maximum(r0, 0), 0)] if len(pods) else -1, -1)
    assert np.array_equal(got, np.where(ok, picks["pod_idx"].astype(np.int64), -1))
    return rows


def run_chain_fallbacks(P: int, q0, calls: Sequence, ks: Sequence[int], window: int, tables_for: TablesFor):
    """(picks of every call, rows of every call (R, k), loads[P]) for the chain of `calls` with
    n_fallbacks ks[i] per call (0: no rows, an (R, 0) array)."""
    assert len(ks) == len(calls)
    bounds = np.cumsum([0] + [len(c) for c, _ in calls])
    rows: List[np.ndarray] = [np.full((len(c), max(int(k), 0)), -1, dtype=np.int16) for (c, _), k in zip(calls, ks)]
    cursor = [0]

    def scheduler_for(q):
        schedule, klass, A = tables_for(q)

        def run(x, seed):
            pos = cursor[0]
            cursor[0] += len(x)
            ci = int(np.searchsorted(bounds, pos, side="right")) - 1     # run_chain never crosses a call
            off = pos - int(bounds[ci])
            if x.dtype == MC.MREQ_DTYPE:
                out = np.zeros(len(x), dtype=B.PICK_DTYPE)
                out["pod_idx"] = -1
                out["status"] = MC.LIG_NO_MODEL
                ok = x["ok"] == 1
                if ok.any():
                    out[ok] = schedule(np.ascontiguousarray(x["req"][ok]), seed)
                reqs = x["req"]
            else:
                out = schedule(x, seed)
                reqs = x
            if ks[ci] > 0:
                rows[ci][off:off + len(x)] = segment_rows(reqs, out, seed, int(ks[ci]), klass, A)
            return out
        return run

    outs, loads = run_chain(P, q0, calls, window, scheduler_for)
    return MC.finish(outs, calls), rows, loads


def class_table_tables(P: int, A: int, kv, n_active, max_active, bitmap, thresholds=(0.8, 5, 50)) -> TablesFor:
    """The built-in tree: oracle.binding.ClassTable on the current queue sizes."""
    def tables_for(q):
        tab = B.ClassTable(P, A, kv, np.asarray(q).astype(np.int32), n_active, max_active, bitmap, thresholds)
        cache = {}

        def klass(crit, a):
            if (crit, a) not in cache:
                st, _, lst = tab.klass(crit, a)
                cache[(crit, a)] = (st, lst)
            return cache[(crit, a)]
        return tab.schedule_batch, klass, A
    return tables_for


def tree_tables(records: List[dict], names: List[str]) -> TablesFor:
    """A caller filter tree (set with oracle_tree.set_filter_tree by the caller): oracle_tree's port
    over the pool with the current queue sizes (names = adapter names, then the model no pod lists)."""
    import oracle_tree
    A = len(names) - 1

    def tables_for(q):
        pool = oracle_tree.Pool([dict(r, waiting_queue_size=int(q[i])) for i, r in enumerate(records)])
        cache = {}

        def klass(crit, a):
            if (crit, a) not in cache:
                cache[(crit, a)] = pool.filter(names[a], crit)
            return cache[(crit, a)]
        return (lambda reqs, seed: pool.schedule_batch(names[:-1], names[-1], reqs, seed)), klass, A
    return tables_for


def schedule_chain_fallbacks(P, A, kv, q, n_active, max_active, bitmap, calls, ks, window: int,
                             thresholds=(0.8, 5, 50)):
    """The chain with rows on the class-table oracle: (picks, rows, loads)."""
    return run_chain_fallbacks(P, q, calls, ks, window,
                               class_table_tables(P, A, kv, n_active, max_active, bitmap, thresholds))


def schedule_chain_fallbacks_tree(nodes, records: List[dict], names: List[str], calls, ks, window: int):
    """The chain with rows under a caller filter tree: (picks, rows, loads)."""
    import oracle_tree
    q0 = [r["waiting_queue_size"] for r in records]
    oracle_tree.set_filter_tree(nodes)
    try:
        return run_chain_fallbacks(len(records), q0, calls, ks, window, tree_tables(records, names))
    finally:
        oracle_tree.set_filter_tree(None)
