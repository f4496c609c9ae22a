"""Sequential definition of the load-feedback chain (include/lig.h, lig_schedule_batch_feedback_chain).

The requests of all chain calls against one epoch form one sequence, cut into windows of `window`
requests regardless of call boundaries.  Every request is scheduled against the current queue
sizes with its own call's seed; when a window fills, its picks per pod are added to
WaitingQueueSize (saturating at INT32_MAX) before the next request is scheduled:

    for each call (reqs, seed), for each request r in order:
        pick r against the tables of the CURRENT queue sizes, with `seed`
        filled += 1; if filled == window: q += picks of the window; filled = 0

With one seed for every call this is oracle/feedback.py's schedule_batch_feedback over the
concatenation with sub_batch = window, however the requests are split.  Three interchangeable
inner schedulers: the class-table oracle, the structure-preserving port (small pools) and the
caller-tree port (oracle_tree).
"""
from __future__ import annotations

from typing import Callable, List, Sequence, Tuple

import numpy as np

from oracle import binding as B

INT32_MAX = (1 << 31) - 1


def run_chain(P: int, q0, calls: Sequence[Tuple[np.ndarray, int]], window: int,
              scheduler_for: Callable[[np.ndarray], Callable[[np.ndarray, int], np.ndarray]]):
    """(picks of every call, loads[P]) for the chain of `calls` = [(reqs, seed), ...] starting from
    queue sizes q0.  scheduler_for(q) returns schedule(reqs, seed) -> picks on the tables of q."""
    assert window >= 1
    q = np.asarray(q0, dtype=np.int64).copy()
    closed = np.zeros(P, dtype=np.int64)
    hist = np.zeros(P, dtype=np.int64)
    filled = 0
    schedule = None
    outs: List[np.ndarray] = []
    for reqs, seed in calls:
        R = len(reqs)
        out = np.zeros(R, dtype=B.PICK_DTYPE)
        pos = 0
        while pos < R:
            n = min(R - pos, window - filled)
            if schedule is None:
                schedule = scheduler_for(q)
            picks = schedule(np.ascontiguousarray(reqs[pos:pos + n]), seed)
            out[pos:pos + n] = picks
            if P:
                hist += np.bincount(picks["pod_idx"][picks["pod_idx"] >= 0], minlength=P)
            pos += n
            filled += n
            if filled == window:
                q = np.minimum(q + hist, INT32_MAX)
                closed += hist
                hist[:] = 0
                filled = 0
                schedule = None
        outs.append(out)
    return outs, closed + hist


def schedule_batch_feedback_chain(P: int, A: int, kv, q, n_active, max_active, bitmap, calls, window: int,
                                  thresholds=(0.8, 5, 50)):
    """The chain on the class-table oracle: returns (picks of every call, loads[P])."""
    def scheduler_for(qs):
        tab = B.ClassTable(P, A, kv, qs.astype(np.int32), n_active, max_active, bitmap, thresholds)
        return tab.schedule_batch
    return run_chain(P, q, calls, window, scheduler_for)


def schedule_batch_feedback_chain_port(pods: List[dict], adapter_names: List[str], unknown: str, calls,
                                       window: int):
    """The same with the structure-preserving port of Scheduler.Schedule as the inner scheduler."""
    q0 = [p["waiting_queue_size"] for p in pods]

    def scheduler_for(qs):
        pool = B.Pool([dict(p, waiting_queue_size=int(qs[i])) for i, p in enumerate(pods)])
        return lambda reqs, seed: pool.schedule_batch(adapter_names, unknown, reqs, seed)[0]
    return run_chain(len(pods), q0, calls, window, scheduler_for)


def schedule_batch_feedback_chain_tree(nodes, records: List[dict], names: List[str], calls, window: int):
    """The chain with a caller filter tree: oracle_tree's port walks `nodes` over the pool with the
    current queue sizes (names = adapter names, then the model no pod lists)."""
    import oracle_tree
    q0 = [r["waiting_queue_size"] for r in records]

    def scheduler_for(qs):
        pool = oracle_tree.Pool([dict(r, waiting_queue_size=int(qs[i])) for i, r in enumerate(records)])
        return lambda reqs, seed: pool.schedule_batch(names[:-1], names[-1], reqs, seed)
    oracle_tree.set_filter_tree(nodes)
    try:
        return run_chain(len(records), q0, calls, window, scheduler_for)
    finally:
        oracle_tree.set_filter_tree(None)


def random_split(R: int, rng, window: int) -> List[int]:
    """Call boundaries 0 = b0 < ... < bk = R that include calls of size 0, 1, W-1, W, W+1 and calls
    spanning several windows, then random sizes."""
    sizes = [0, 1, max(window - 1, 0), window, window + 1, 3 * window + 2, 0]
    out, pos = [0], 0
    for s in sizes + list(rng.integers(0, 2 * window + 3, size=64)):
        if pos >= R:
            break
        pos = min(R, pos + int(s))
        out.append(pos)
    while pos < R:
        pos = min(R, pos + int(rng.integers(1, 4 * window + 2)))
        out.append(pos)
    return out


def split_calls(reqs: np.ndarray, bounds: Sequence[int], seed: int):
    return [(np.ascontiguousarray(reqs[a:b]), seed) for a, b in zip(bounds[:-1], bounds[1:])]
