"""CPU reference for caller filter trees: (*filter).Filter (filter.go:44-73) walked over a table of
LigFilterNode rows with the reference's node functions restated in numpy (Go semantics: int64 queue
arithmetic, three separately rounded binary64 operations in leastKVCacheFilterFunc, NaN never
updating min / max).  Pods are oracle records (dicts with waiting_queue_size,
kv_cache_usage_percent, max_active_models, active_models)."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

from llm_instance_gateway_b200 import _native as N

MAX_FLOAT64 = np.float64(1.7976931348623157e308)


class Pods:
    def __init__(self, records: Sequence[dict]):
        self.records = list(records)
        self.P = len(self.records)
        self.q = np.array([int(r["waiting_queue_size"]) for r in self.records], dtype=np.int64)
        self.kv = np.array([float(r["kv_cache_usage_percent"]) for r in self.records], dtype=np.float64)
        self.room = np.array([len(r["active_models"]) < int(r["max_active_models"]) for r in self.records], dtype=bool)
        self._aff = {}

    def affinity(self, model: str) -> np.ndarray:
        if model not in self._aff:
            self._aff[model] = np.array([model in r["active_models"] for r in self.records], dtype=bool)
        return self._aff[model]


def least_queuing(pods: Pods, member: np.ndarray) -> np.ndarray:            # filter.go:102-122
    n = int(member.sum())
    if n == 0:
        return member.copy()
    v = pods.q[member]
    mn, mx = int(v.min()), max(0, int(v.max()))
    thr = mn + (mx - mn) // n              # mx - mn >= 0: floor == Go's truncation
    return member & (pods.q >= mn) & (pods.q <= thr)


def least_kv(pods: Pods, member: np.ndarray) -> np.ndarray:                 # filter.go:134-154
    n = int(member.sum())
    if n == 0:
        return member.copy()
    v = pods.kv[member]
    v = v[~np.isnan(v)]
    mn = min(MAX_FLOAT64, np.float64(v.min())) if v.size else MAX_FLOAT64
    mx = max(np.float64(0.0), np.float64(v.max())) if v.size else np.float64(0.0)
    with np.errstate(all="ignore"):
        thr = mn + (mx - mn) / np.float64(n)
        return member & (pods.kv >= mn) & (pods.kv <= thr)


def predicate(pods: Pods, node, critical: bool, model: str) -> np.ndarray:
    k = node.kind
    if k == N.LIG_F_CRITICAL_REQUEST:
        return np.full(pods.P, bool(critical))
    if k == N.LIG_F_LOW_QUEUEING:
        return pods.q < node.queue_threshold
    if k == N.LIG_F_LORA_AFFINITY:
        return pods.affinity(model)
    if k == N.LIG_F_CAN_ACCEPT_NEW_LORA:
        return pods.room
    if k == N.LIG_F_LOW_LORA_COST:
        return pods.affinity(model) | pods.room
    assert k == N.LIG_F_NO_QUEUE_AND_LOW_KV
    return (pods.q <= node.queue_threshold) & (pods.kv <= node.kv_threshold)


def walk(nodes, pods: Pods, critical: bool, model: str) -> Tuple[int, List[int]]:
    """(status, survivors) of Schedule's filter call for one request class."""
    cur = np.ones(pods.P, dtype=bool)
    i = 0
    while True:
        nd = nodes[i]
        err = N.LIG_OK
        if nd.kind == N.LIG_F_LEAST_QUEUING:
            res = least_queuing(pods, cur)
        elif nd.kind == N.LIG_F_LEAST_KV_CACHE:
            res = least_kv(pods, cur)
        elif nd.kind == N.LIG_F_DROP:
            res, err = np.zeros(pods.P, dtype=bool), N.LIG_DROP
        else:
            res = cur & predicate(pods, nd, critical, model)
            if not res.any():
                err = N.LIG_NO_PODS_LEFT
        ok = err == N.LIG_OK and res.any()
        if ok:
            nxt = nd.next_on_success if nd.next_on_success >= 0 else nd.next_on_success_or_failure
        else:
            nxt = nd.next_on_failure if nd.next_on_failure >= 0 else nd.next_on_success_or_failure
        if nxt < 0:
            idx = np.nonzero(res)[0].tolist()
            return (err if err != N.LIG_OK else (N.LIG_OK if idx else N.LIG_EMPTY)), idx
        if ok:
            cur = res
        i = nxt


# ---- random trees and pools ------------------------------------------------------------------------
KV_SPECIAL = [0.0, -0.0, 0.8, 0.8000000000000002, 0.7999999999999999, 1.0, math.inf, -math.inf,
              math.nan, 1e-300, 5e-324, -0.25, 1.0 / 3.0]
Q_SPECIAL = [0, 5, 6, 49, 50, -1, 2**31 - 1, -(2**31)]
ADAPTERS = ["a0", "a1", "a2", "a3"]


def random_tree(rng: np.random.Generator, max_nodes: int = 16) -> List[N.LigFilterNode]:
    """A random forward-linked table: random kinds, thresholds from the special values, every
    combination of successor fields (next_on_success together with next_on_success_or_failure too)."""
    n = int(rng.integers(1, max_nodes + 1))
    nodes = []
    for i in range(n):
        def succ():
            if i + 1 >= n or rng.random() < 0.35:
                return -1
            return int(rng.integers(i + 1, n))
        kind = int(rng.integers(0, 9))
        nodes.append(N.LigFilterNode(kind, succ(), succ(), succ(), int(rng.choice(Q_SPECIAL + [1, 3, 10, 30])),
                                     float(rng.choice(KV_SPECIAL + [0.5, 0.3]))))
    return nodes


def random_pool(rng: np.random.Generator) -> List[dict]:
    """The value sets of the GPU parity suite's random adversarial pools."""
    P = int(rng.integers(1, 70))
    out = []
    for i in range(P):
        q = int(rng.choice(Q_SPECIAL)) if rng.random() < 0.2 else int(rng.integers(0, 70))
        kv = float(rng.choice(KV_SPECIAL)) if rng.random() < 0.25 else float(np.round(rng.random(), 2))
        out.append(dict(name=f"pod-{i}", address=f"address-{i}", waiting_queue_size=q, kv_cache_usage_percent=kv,
                        max_active_models=int(rng.integers(0, 4)),
                        active_models=[str(a) for a in rng.choice(ADAPTERS, size=int(rng.integers(0, 4)), replace=False)]))
    return out
