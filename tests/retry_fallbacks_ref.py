"""Retry scheduling with fallback rows (lig_schedule_batch_excluding_fallbacks, include/lig.h) by its
definition (test infrastructure).

Composed from the two independent definitions and nothing else: out is retry_ref.retry_batch, each
request's reduced survivor list is retry_ref.survivors (which rebuilds the pool without the excluded
pods and never masks a full one), and fallback_ref.fallback_rows ranks those lists as a CSR.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

import fallback_ref as FR
import retry_ref as RR
from llm_instance_gateway_b200 import _native as N


def reduced_lists(snap, reqs: np.ndarray, excluded: np.ndarray, thresholds=(0.8, 5, 50),
                  nodes=None) -> List[Tuple[int, List[int]]]:
    """(status, survivors in the epoch's pod indices) per request, over its pool without its row.
    Requests with the same excluded pods and class share one retry_ref.survivors call."""
    excluded = np.asarray(excluded).reshape(len(reqs), -1)
    memo: Dict[tuple, Tuple[int, List[int]]] = {}
    out = []
    for i, r in enumerate(reqs):
        gone = tuple(sorted({int(e) for e in excluded[i] if 0 <= int(e) < snap.P}))
        a = int(r["adapter_id"])
        crit = bool(int(r["flags"]) & N.LIG_REQ_CRITICAL)
        key = (gone, crit, a if 0 <= a < snap.A else snap.A)
        if key not in memo:
            memo[key] = RR.survivors(snap, crit, a, excluded[i], thresholds, nodes)
        out.append(memo[key])
    return out


def retry_fallback_batch(snap, reqs: np.ndarray, excluded: np.ndarray, seed: int, k: int,
                         thresholds=(0.8, 5, 50), nodes=None):
    """(picks, rows (R, k) int16) of lig_schedule_batch_excluding_fallbacks by its definition."""
    excluded = np.asarray(excluded).reshape(len(reqs), -1)
    picks = RR.retry_batch(snap, reqs, excluded, seed, thresholds, nodes)
    lists = reduced_lists(snap, reqs, excluded, thresholds, nodes)
    counts = np.array([len(lst) for _, lst in lists], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64) if len(lists) else np.zeros(0, np.int64)
    pods = np.array([p for _, lst in lists for p in lst], dtype=np.int64)
    ok = picks["status"] == N.LIG_OK
    rows, _ = FR.fallback_rows(seed, reqs["rand_key"], ok, starts, counts, pods, k)
    return picks, rows
