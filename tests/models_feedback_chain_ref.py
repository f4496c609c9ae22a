"""Sequential definition of the feedback chain with model-id calls (include/lig.h,
lig_schedule_models_batch_feedback_chain), on top of feedback_chain_ref.run_chain.

A model-id call is one more chain call.  Request i of a call (ids, seed, first_index) has
rand_key = first_index + i; it is resolved on the host with the oracle's restatement of the
datastore (oracle.binding.Models.resolve, lig_oracle_models.c) and the descriptor it resolves to
is picked like any other request of the chain, on the tables of the current queue sizes.  A request
that does not resolve (absent model, id >= n_models) gives pod -1 / LIG_NO_MODEL / target 255 and
still counts toward its window.  The resolve does not depend on the queue sizes, so it runs once per
call, before the chain; run_chain sees the call as a structured array (MREQ_DTYPE) and the inner
scheduler picks its resolved rows.

Calls are (reqs, seed) descriptor calls, as in feedback_chain_ref, and model-id calls made by
model_call(); both kinds may alternate in one chain.  Descriptor calls give lig_pick rows, model-id
calls lig_mpick rows.
"""
from __future__ import annotations

from typing import Callable, List, Sequence

import numpy as np

from feedback_chain_ref import run_chain
from oracle import binding as B

LIG_NO_MODEL = 3
# one model-id request after the resolve: its descriptor, whether it resolved, the drawn target
MREQ_DTYPE = np.dtype([("req", B.REQ_DTYPE), ("ok", "u1"), ("target_idx", "u1")])


def resolve_call(models: "B.Models", adapter_id: Callable[[str], int], ids: np.ndarray, seed: int,
                 first_index: int = 0) -> np.ndarray:
    """The MREQ_DTYPE rows of one model-id call: the oracle's resolve of every id, the resolved name
    interned with adapter_id (the snapshot's dense id, A when no pod lists it)."""
    ids = np.asarray(ids, dtype=np.uint32)
    out = np.zeros(len(ids), dtype=MREQ_DTYPE)
    out["target_idx"] = 255
    for i, m in enumerate(ids.tolist()):
        key = (first_index + i) & ((1 << 64) - 1)
        out["req"]["rand_key"][i] = key
        if m >= models.n:
            continue
        rc, name, crit, k = models.resolve(m, seed, key)
        if rc != 0:                 # absent, or a draw that finds no target (packed as absent)
            continue
        out["req"]["adapter_id"][i] = adapter_id(name)
        out["req"]["flags"][i] = 1 if crit else 0
        out["ok"][i] = 1
        out["target_idx"][i] = k
    return out


def model_call(models, adapter_id, ids, seed: int, first_index: int = 0):
    """A model-id chain call for run_chain / schedule_chain: (MREQ_DTYPE rows, seed)."""
    return resolve_call(models, adapter_id, ids, seed, first_index), seed


def with_model_calls(scheduler_for):
    """Wraps a descriptor scheduler_for(q) of feedback_chain_ref so that its schedule() also takes
    MREQ_DTYPE slices: resolved rows are picked as descriptors, the others are LIG_NO_MODEL."""
    def wrapped(q):
        schedule = scheduler_for(q)

        def run(x, seed):
            if x.dtype != MREQ_DTYPE:
                return schedule(x, seed)
            out = np.zeros(len(x), dtype=B.PICK_DTYPE)
            out["pod_idx"] = -1
            out["status"] = LIG_NO_MODEL
            ok = x["ok"] == 1
            if ok.any():
                out[ok] = schedule(np.ascontiguousarray(x["req"][ok]), seed)
            return out
        return run
    return wrapped


def as_mpicks(picks: np.ndarray, call: np.ndarray) -> np.ndarray:
    """lig_mpick rows of a model-id call from run_chain's lig_pick rows."""
    out = np.zeros(len(call), dtype=B.MPICK_DTYPE)
    out["pod_idx"] = picks["pod_idx"]
    out["status"] = picks["status"]
    out["target_idx"] = np.where(call["ok"] == 1, call["target_idx"], 255)
    return out


def finish(outs: List[np.ndarray], calls: Sequence) -> List[np.ndarray]:
    return [as_mpicks(o, c) if c.dtype == MREQ_DTYPE else o for o, (c, _) in zip(outs, calls)]


def schedule_chain(P: int, A: int, kv, q, n_active, max_active, bitmap, calls, window: int,
                   thresholds=(0.8, 5, 50)):
    """The mixed chain on the class-table oracle: (picks of every call, loads[P])."""
    def scheduler_for(qs):
        return B.ClassTable(P, A, kv, qs.astype(np.int32), n_active, max_active, bitmap, thresholds).schedule_batch
    outs, loads = run_chain(P, q, calls, window, with_model_calls(scheduler_for))
    return finish(outs, calls), loads


def schedule_chain_tree(nodes, records: List[dict], names: List[str], calls, window: int):
    """The mixed chain with a caller filter tree, on oracle_tree's port (names = adapter names,
    then the model no pod lists)."""
    import oracle_tree
    q0 = [r["waiting_queue_size"] for r in records]

    def scheduler_for(qs):
        pool = oracle_tree.Pool([dict(r, waiting_queue_size=int(qs[i])) for i, r in enumerate(records)])
        return lambda reqs, seed: pool.schedule_batch(names[:-1], names[-1], reqs, seed)
    oracle_tree.set_filter_tree(nodes)
    try:
        outs, loads = run_chain(len(records), q0, calls, window, with_model_calls(scheduler_for))
    finally:
        oracle_tree.set_filter_tree(None)
    return finish(outs, calls), loads


def split_model_calls(models, adapter_id, ids: np.ndarray, bounds: Sequence[int], seeds, first_index: int = 0):
    """Model-id calls over ids[a:b] for consecutive bounds, first_index advancing by each call's
    size; seeds is one seed or one per call."""
    out = []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        seed = seeds if np.isscalar(seeds) else seeds[k]
        out.append(model_call(models, adapter_id, np.ascontiguousarray(ids[a:b]), int(seed), first_index + a))
    return out
