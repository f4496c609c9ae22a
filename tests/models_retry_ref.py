"""Model-id retries (lig_schedule_models_batch[_feedback_chain]_excluding[_fallbacks], include/lig.h) by
their definition (test infrastructure).

A model-id retry resolves each request at a fixed target, without a draw, on the packed model table
(PackedModels: the arrays lig_upload_models takes), and then is the descriptor retry of the resolved
descriptor {adapter_id, Critical, rand_key = first_index + i}.  So every function here is
fixed_resolve followed by an existing definition: retry_ref.retry_batch, retry_fallbacks_ref's rows,
eject_ref for ejected epochs, and the chain references of feedback_chain_retry[_fallbacks]_ref, whose
window walk a model-retry call joins like any other call.  A request that does not resolve is
{-1, LIG_NO_MODEL, 255} with a row of -1; in a chain it holds its place in the window and adds no load.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

import numpy as np

import eject_ref as ER
import feedback_chain_fallbacks_ref as FR
import feedback_chain_retry_fallbacks_ref as CRF
import feedback_chain_retry_ref as CR
import oracle_tree as OT
import retry_fallbacks_ref as RF
import retry_ref as RR
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, PackedModels

LIG_NO_MODEL = 3
SELF = 255                       # target_idx of a model without TargetModels
M64 = (1 << 64) - 1
# one model-id retry request after the resolve: its descriptor, whether it resolved, its target
RESOLVED_DTYPE = np.dtype([("req", REQ_DTYPE), ("ok", "u1"), ("target_idx", "u1")])


def fixed_resolve(pm: PackedModels, ids, targets, first_index: int = 0) -> np.ndarray:
    """RESOLVED_DTYPE rows: request i is ids[i] at target targets[i], rand_key first_index + i."""
    ids = np.asarray(ids, dtype=np.uint32)
    targets = np.asarray(targets, dtype=np.uint8)
    out = np.zeros(len(ids), dtype=RESOLVED_DTYPE)
    out["target_idx"] = targets
    for i, (m, t) in enumerate(zip(ids.tolist(), targets.tolist())):
        out["req"]["rand_key"][i] = (first_index + i) & M64
        if m >= pm.n_models or not pm.present[m]:
            continue
        lo, hi = int(pm.target_offsets[m]), int(pm.target_offsets[m + 1])
        if (hi == lo and t != SELF) or (hi > lo and t >= hi - lo):
            continue
        out["req"]["adapter_id"][i] = pm.self_adapter_ids[m] if t == SELF else pm.target_adapter_ids[lo + t]
        out["req"]["flags"][i] = 1 if pm.critical[m] else 0
        out["ok"][i] = 1
    return out


def as_mpicks(picks: np.ndarray, res: np.ndarray) -> np.ndarray:
    """lig_mpick rows from the descriptor picks of the resolved requests (rows of `res` that did not
    resolve are LIG_NO_MODEL whatever `picks` holds there)."""
    ok = res["ok"] == 1
    out = np.zeros(len(res), dtype=MPICK_DTYPE)
    out["pod_idx"] = np.where(ok, picks["pod_idx"], -1)
    out["status"] = np.where(ok, picks["status"], LIG_NO_MODEL)
    out["target_idx"] = np.where(ok, res["target_idx"], 255)
    return out


def _resident(res, excluded, k, run):
    ok = res["ok"] == 1
    picks = np.zeros(len(res), dtype=PICK_DTYPE)
    rows = np.full((len(res), k), -1, dtype=np.int16)
    if ok.any():
        got = run(np.ascontiguousarray(res["req"][ok]), np.ascontiguousarray(excluded[ok]))
        if k:
            picks[ok], rows[ok] = got
        else:
            picks[ok] = got
    return as_mpicks(picks, res), rows


def retry_batch(snap, pm: PackedModels, ids, targets, excluded, seed: int, first_index: int = 0,
                thresholds=(0.8, 5, 50), nodes=None, ejected: Optional[Sequence[int]] = None) -> np.ndarray:
    """lig_schedule_models_batch_excluding: lig_mpick rows.  ejected: the pods lig_eject_pods removed
    from `snap` to make the epoch (None = an uploaded epoch)."""
    res = fixed_resolve(pm, ids, targets, first_index)
    excluded = np.asarray(excluded, dtype=np.int16).reshape(len(res), -1)
    if ejected is None:
        def run(r, x):
            return RR.retry_batch(snap, r, x, seed, thresholds, nodes)
    else:
        def run(r, x):
            return ER.retry_batch(snap, ejected, r, x, seed, thresholds, nodes)
    return _resident(res, excluded, 0, run)[0]


def retry_fallback_batch(snap, pm: PackedModels, ids, targets, excluded, seed: int, k: int, first_index: int = 0,
                         thresholds=(0.8, 5, 50), nodes=None, ejected: Optional[Sequence[int]] = None):
    """lig_schedule_models_batch_excluding_fallbacks: (lig_mpick rows, int16 rows (R, k))."""
    res = fixed_resolve(pm, ids, targets, first_index)
    excluded = np.asarray(excluded, dtype=np.int16).reshape(len(res), -1)
    if ejected is None:
        def run(r, x):
            return RF.retry_fallback_batch(snap, r, x, seed, k, thresholds, nodes)
    else:
        def run(r, x):
            return ER.retry_fallback_batch(snap, ejected, r, x, seed, k, thresholds, nodes)
    return _resident(res, excluded, k, run)


# ---- under the load-feedback chain ---------------------------------------------------------------
def model_retry_call(pm: PackedModels, ids, targets, excluded, seed: int, first_index: int = 0):
    """A model-id retry chain call for run_chain: (MRETRY rows, seed)."""
    res = fixed_resolve(pm, ids, targets, first_index)
    excluded = np.asarray(excluded, dtype=np.int16).reshape(len(res), -1)
    x = np.zeros(len(res), dtype=np.dtype([("req", REQ_DTYPE), ("excluded", np.int16, (excluded.shape[1],)),
                                           ("ok", "u1"), ("target_idx", "u1"), ("at", np.int64)]))
    for f in ("req", "ok", "target_idx"):
        x[f] = res[f]
    x["excluded"] = excluded
    return x, seed


def is_model_retry(x: np.ndarray) -> bool:
    return x.dtype.names is not None and "excluded" in x.dtype.names and "ok" in x.dtype.names


def with_model_retry_calls(tables_for: FR.TablesFor, snap, rows: np.ndarray, k_at: np.ndarray,
                           thresholds=(0.8, 5, 50), nodes=None) -> FR.TablesFor:
    """tables_for(q) whose schedule() also takes model-retry segments: the resolved requests are the
    descriptor retry (with rows when the call's k > 0) on `snap` with the chain's queue sizes q; the
    others are LIG_NO_MODEL, picked on nothing and counted on nothing."""
    def wrapped(q):
        schedule, klass, A = tables_for(q)
        snap_q = dataclasses.replace(snap, q=np.asarray(q, dtype=np.int64).astype(np.int32))

        def run(x, seed):
            if not is_model_retry(x):
                return schedule(x, seed)
            out = np.zeros(len(x), dtype=PICK_DTYPE)
            out["pod_idx"] = -1
            out["status"] = LIG_NO_MODEL
            ok = x["ok"] == 1
            if ok.any():
                at = x["at"][ok]
                k = int(k_at[at[0]])             # run_chain never crosses a call
                reqs, ex = np.ascontiguousarray(x["req"][ok]), np.ascontiguousarray(x["excluded"][ok])
                if k:
                    out[ok], rows[at, :k] = RF.retry_fallback_batch(snap_q, reqs, ex, seed, k, thresholds, nodes)
                else:
                    out[ok] = RR.retry_batch(snap_q, reqs, ex, seed, thresholds, nodes)
                if nodes is not None:            # retry_ref clears the tree the chain's other calls walk
                    OT.set_filter_tree(nodes)
            return out
        return run, klass, A
    return wrapped


def run_chain(snap, calls: Sequence, window: int, ks: Optional[Sequence[int]] = None, thresholds=(0.8, 5, 50),
              nodes=None, records: Optional[List[dict]] = None, names: Optional[List[str]] = None):
    """(picks of every call, rows of every call, loads[P]) for a chain over `snap` of every kind of call:
    plain, model-id and fallback calls (feedback_chain_fallbacks_ref), descriptor retry calls with or
    without rows (feedback_chain_retry_ref.retry_call, rows when ks[i] > 0) and model-retry calls
    (model_retry_call, rows when ks[i] > 0).  Model-retry calls give lig_mpick rows."""
    ks = [0] * len(calls) if ks is None else [int(k) for k in ks]
    bounds = np.cumsum([0] + [len(c) for c, _ in calls])
    rows = np.full((int(bounds[-1]), max([0] + ks)), -1, dtype=np.int16)
    k_at = np.repeat(np.array(ks, dtype=np.int64), np.diff(bounds))
    run_calls, run_ks, tagged = [], [], []
    for i, ((c, s), k) in enumerate(zip(calls, ks)):
        if is_model_retry(c):
            c = c.copy()
            c["at"] = bounds[i] + np.arange(len(c), dtype=np.int64)
        elif CR.is_retry(c) and k > 0:
            c = CRF._tagged(c, int(bounds[i]))
        else:
            run_calls.append((c, s))
            run_ks.append(k)
            tagged.append(False)
            continue
        run_calls.append((c, s))
        run_ks.append(0)
        tagged.append(True)

    def tables(tf):
        tf = CRF.with_retry_fallback_calls(CR.with_retry_calls(tf, snap, thresholds, nodes), snap, rows, k_at,
                                           thresholds, nodes)
        return with_model_retry_calls(tf, snap, rows, k_at, thresholds, nodes)
    if nodes is None:
        tf = FR.class_table_tables(snap.P, snap.A, snap.kv, snap.n_active, snap.max_active, snap.bitmap, thresholds)
        outs, call_rows, loads = FR.run_chain_fallbacks(snap.P, snap.q, run_calls, run_ks, window, tables(tf))
    else:
        OT.set_filter_tree(nodes)
        try:
            outs, call_rows, loads = FR.run_chain_fallbacks(snap.P, snap.q, run_calls, run_ks, window,
                                                            tables(FR.tree_tables(records, names)))
        finally:
            OT.set_filter_tree(None)
    for i, (c, _) in enumerate(calls):
        if tagged[i]:
            call_rows[i] = rows[bounds[i]:bounds[i + 1], :ks[i]].copy()
        if is_model_retry(c):
            outs[i] = as_mpicks(outs[i], c)
    return outs, call_rows, loads


def run_chain_snapshot(snap, calls: Sequence, window: int, ks: Optional[Sequence[int]] = None,
                       thresholds=(0.8, 5, 50), nodes=None, ejected: Optional[Sequence[int]] = None):
    """run_chain on the epoch made from `snap` (ejected: the pods lig_eject_pods removed; caller trees
    take the snapshot's oracle records).  Pod indices of calls and results are in `snap`'s order."""
    kept = np.arange(snap.P, dtype=np.int64)
    small = snap
    if ejected is not None:
        small, kept = ER.reduced(snap, ejected)
        red = []
        for c, s in calls:
            if is_model_retry(c) or CR.is_retry(c):
                c = c.copy()
                c["excluded"] = ER.to_reduced(kept, snap.P, c["excluded"])
            red.append((c, s))
        calls = red
    kw = {}
    if nodes is not None:
        kw = dict(nodes=nodes, records=RR.records(small), names=RR.adapter_names(small) + [WL.UNKNOWN_MODEL])
    outs, rows, loads = run_chain(small, calls, window, ks, thresholds=thresholds, **kw)
    if ejected is None:
        return outs, rows, loads
    full = np.zeros(snap.P, dtype=np.int64)
    full[kept] = loads
    back = []
    for o in outs:
        o = o.copy()
        o["pod_idx"] = ER.map_back(kept, o["pod_idx"])
        back.append(o)
    return back, [ER.map_back(kept, r).astype(np.int16) for r in rows], full
