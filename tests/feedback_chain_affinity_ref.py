"""Sequential definition of session affinity under the load-feedback chain (include/lig.h,
lig_schedule_[models_]batch_feedback_chain_affinity), on top of feedback_chain_ref.run_chain.

A chain affinity call is a chain call in every respect except the choice among survivors.  The window
walk and the loads are run_chain's: only picks are counted, row entries add nothing.  Request j of an
affinity call takes its class's survivor list in the tables of the queue sizes at its position in the
sequence (the list a plain chain request there draws from), status and n_survivors from that class
entry, and affinity_ref.ranking over that list by its key: the top is the pick, the next entries its
row.  Model ids resolve on the oracle's datastore with draw state key ^ LIG_DRAW_DOMAIN (seed 0), as
lig_schedule_models_batch_affinity resolves them.

One chain may mix every call kind, descriptor or model id: a call is (x, seed) as for run_chain with a
spec (kind, k): kind "plain" (k = 0), "fallbacks" (k rows of fallback_ref's ranking, as in
feedback_chain_fallbacks_ref) or "affinity" (k rows, 0 = none; x carries the keys as rand_key, and its
seed is ignored).  Each segment run_chain schedules is routed to its call by a cursor over the sequence.
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import numpy as np

import feedback_chain_fallbacks_ref as FF
import models_feedback_chain_ref as MC
from affinity_ref import ranking
from feedback_chain_ref import run_chain
from oracle import binding as B

LIG_OK = 0
M64 = (1 << 64) - 1


def affinity_model_call(models: "B.Models", adapter_id: Callable[[str], int], ids, keys) -> Tuple[np.ndarray, int]:
    """A model-id chain affinity call for run_chain_affinity: (MREQ_DTYPE rows, 0).  Model i resolves on
    the oracle's datastore with seed 0 and key keys[i] (draw state key ^ LIG_DRAW_DOMAIN); the
    descriptor it resolves to carries rand_key = keys[i]."""
    ids = np.asarray(ids, dtype=np.uint32)
    keys = np.asarray(keys, dtype=np.uint64)
    out = np.zeros(len(ids), dtype=MC.MREQ_DTYPE)
    out["target_idx"] = 255
    out["req"]["rand_key"] = keys
    for i, (m, k) in enumerate(zip(ids.tolist(), keys.tolist())):
        if m >= models.n:
            continue
        rc, name, crit, t = models.resolve(m, 0, k)
        if rc != 0:
            continue
        out["req"]["adapter_id"][i] = adapter_id(name)
        out["req"]["flags"][i] = 1 if crit else 0
        out["ok"][i] = 1
        out["target_idx"][i] = t
    return out, 0


def affinity_segment(reqs: np.ndarray, plain: np.ndarray, k: int, klass: Callable, A: int, pod_keys):
    """(picks, rows (R, k)) of one affinity segment: `plain` is a plain pick on the same tables, whose
    status and n_survivors the class entry gives; pod_idx and the row rank the class list by key."""
    out = plain.copy()
    rows = np.full((len(reqs), k), -1, dtype=np.int16)
    crit, a = FF.class_of(reqs, A)
    for i in range(len(reqs)):
        if out["status"][i] != LIG_OK:
            out["pod_idx"][i] = -1
            continue
        r = ranking(int(reqs["rand_key"][i]), klass(bool(crit[i]), int(a[i]))[1], pod_keys)
        out["pod_idx"][i] = r[0]
        rows[i, :min(k, len(r) - 1)] = r[1:1 + k]
    return out, rows


def run_chain_affinity(P: int, q0, calls: Sequence, specs: Sequence[Tuple[str, int]], window: int,
                       tables_for: FF.TablesFor, pod_keys):
    """(picks of every call, rows of every call (R, k), loads[P]) for the chain of `calls` with
    specs[i] = (kind, k) per call."""
    assert len(specs) == len(calls)
    bounds = np.cumsum([0] + [len(c) for c, _ in calls])
    rows: List[np.ndarray] = [np.full((len(c), max(int(k), 0)), -1, dtype=np.int16)
                              for (c, _), (_, k) in zip(calls, specs)]
    cursor = [0]

    def scheduler_for(q):
        schedule, klass, A = tables_for(q)

        def run(x, seed):
            pos = cursor[0]
            cursor[0] += len(x)
            ci = int(np.searchsorted(bounds, pos, side="right")) - 1     # run_chain never crosses a call
            off = pos - int(bounds[ci])
            kind, k = specs[ci]
            reqs = x["req"] if x.dtype == MC.MREQ_DTYPE else x
            ok = x["ok"] == 1 if x.dtype == MC.MREQ_DTYPE else np.ones(len(x), dtype=bool)
            out = np.zeros(len(x), dtype=B.PICK_DTYPE)
            out["pod_idx"] = -1
            out["status"] = MC.LIG_NO_MODEL
            if ok.any():
                out[ok] = schedule(np.ascontiguousarray(reqs[ok]), seed)
            if kind == "affinity":
                seg, seg_rows = affinity_segment(reqs, out, int(k), klass, A, pod_keys)
                seg["pod_idx"][~ok] = -1
                seg_rows[~ok] = -1
                out = seg
                rows[ci][off:off + len(x)] = seg_rows
            elif kind == "fallbacks" and k > 0:
                rows[ci][off:off + len(x)] = FF.segment_rows(reqs, out, seed, int(k), klass, A)
            return out
        return run

    outs, loads = run_chain(P, q0, calls, window, scheduler_for)
    return MC.finish(outs, calls), rows, loads


def schedule_chain_affinity(P, A, kv, q, n_active, max_active, bitmap, pod_keys, calls, specs, window: int,
                            thresholds=(0.8, 5, 50)):
    """The mixed chain on the class-table oracle: (picks, rows, loads)."""
    return run_chain_affinity(P, q, calls, specs, window,
                              FF.class_table_tables(P, A, kv, n_active, max_active, bitmap, thresholds), pod_keys)


def schedule_chain_affinity_tree(nodes, records: List[dict], names: List[str], pod_keys, calls, specs, window: int):
    """The mixed chain under a caller filter tree, on oracle_tree's port: (picks, rows, loads)."""
    import oracle_tree
    q0 = [r["waiting_queue_size"] for r in records]
    oracle_tree.set_filter_tree(nodes)
    try:
        return run_chain_affinity(len(records), q0, calls, specs, window, FF.tree_tables(records, names), pod_keys)
    finally:
        oracle_tree.set_filter_tree(None)
