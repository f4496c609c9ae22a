"""Threshold values at the edges of their Go types, for the built-in tree's three thresholds and for
caller-tree nodes.  Go's thresholds are `int` (64 bit) and float64, so every value here is legal
configuration; a threshold narrowed to int32 anywhere turns 2^31 into -2^31 and flips `q < thr`."""
from __future__ import annotations

import itertools
import math
import sys
from typing import List, Sequence, Tuple

import numpy as np

from llm_instance_gateway_b200 import _native as N

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
DBL_MAX = sys.float_info.max

Q_FIXED = [INT64_MIN, INT64_MIN + 1, INT32_MIN - 1, INT32_MIN, -1, 0, 1, INT32_MAX, INT32_MAX + 1, 1 << 32, INT64_MAX]
KV_FIXED = [math.nan, -math.inf, math.inf, -0.0, 0.0, 5e-324, 1.0, DBL_MAX, -DBL_MAX]
# pods that sit on the thresholds' edges: appended to every pool the grid is tried on
Q_POD_EDGE = [INT32_MIN, INT32_MAX]
KV_POD_EDGE = [math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324]


def q_grid(pod_q: Sequence[int]) -> List[int]:
    vals = set(Q_FIXED)
    for q in pod_q:
        vals |= {int(q) - 1, int(q) + 1}
    return sorted(vals)


def kv_grid(pod_kv: Sequence[float]) -> List[float]:
    vals = list(KV_FIXED)
    for kv in pod_kv:
        if not math.isnan(kv):
            vals += [float(kv), float(np.nextafter(kv, -math.inf)), float(np.nextafter(kv, math.inf))]
    out, seen = [], set()
    for v in vals:                        # keeps -0.0 and 0.0 apart, one NaN
        key = struct_key(v)
        if key not in seen:
            seen.add(key)
            out.append(v)
    return out


def struct_key(v: float) -> bytes:
    return np.float64(math.nan if math.isnan(v) else v).tobytes()


def corner_triples() -> List[Tuple[float, int, int]]:
    """(kv_cache_threshold, queue_threshold_critical, queueing_threshold_lora) at the extremes."""
    return [(kv, qc, ql) for kv, qc, ql in itertools.product([math.nan, -math.inf, math.inf, -0.0, 5e-324],
                                                            [INT64_MIN, INT64_MAX], [INT64_MIN, INT64_MAX])]


def triples(pod_q, pod_kv, n_random: int, rng: np.random.Generator) -> List[Tuple[float, int, int]]:
    """The corner triples plus a seeded sample of the grid's product."""
    qs, kvs = q_grid(pod_q), kv_grid(pod_kv)
    out = corner_triples()
    for _ in range(n_random):
        out.append((float(kvs[int(rng.integers(len(kvs)))]), int(qs[int(rng.integers(len(qs)))]),
                    int(qs[int(rng.integers(len(qs)))])))
    return out


def edge_pods(rng: np.random.Generator, n: int, first: int, adapters: Sequence[str]) -> List[dict]:
    """Oracle records of n pods with queue and KV values on the edges of their types."""
    out = []
    for k in range(n):
        q = Q_POD_EDGE[k % 2] if k % 3 else int(rng.integers(0, 70))
        kv = KV_POD_EDGE[k % len(KV_POD_EDGE)]
        out.append(dict(name=f"pod-{first + k}", address=f"address-{first + k}", waiting_queue_size=q,
                        kv_cache_usage_percent=kv, max_active_models=int(rng.integers(0, 4)),
                        active_models=[str(a) for a in rng.choice(list(adapters), size=int(rng.integers(0, 3)),
                                                                  replace=False)]))
    return out


def default_tree(kv: float, q_crit: int, q_lora: int) -> List[N.LigFilterNode]:
    """defaultFilter (scheduler.go:26-91) as a caller tree with the given thresholds."""
    from llm_instance_gateway_b200 import scheduling as S
    out = []
    for n in S.DEFAULT_FILTER.flatten():
        q, k = n.queue_threshold, n.kv_threshold
        if n.kind == N.LIG_F_LOW_QUEUEING:
            q = q_lora
        elif n.kind == N.LIG_F_NO_QUEUE_AND_LOW_KV:
            q, k = q_crit, kv
        out.append(N.LigFilterNode(n.kind, n.next_on_success, n.next_on_failure, n.next_on_success_or_failure, q, k))
    return out


def with_grid_thresholds(nodes, rng: np.random.Generator, qs: Sequence[int], kvs: Sequence[float]):
    """The same table with every node's thresholds drawn from the grid."""
    return [N.LigFilterNode(n.kind, n.next_on_success, n.next_on_failure, n.next_on_success_or_failure,
                            int(qs[int(rng.integers(len(qs)))]), float(kvs[int(rng.integers(len(kvs)))]))
            for n in nodes]


def placed_trees(q: int, kv: float) -> List[List[N.LigFilterNode]]:
    """LOW_QUEUEING and NO_QUEUE_AND_LOW_KV nodes carrying (q, kv): at the root, after each range
    node, and on both the success and the failure branch of a predicate."""
    F = N.LigFilterNode
    out = []
    for kind in (N.LIG_F_LOW_QUEUEING, N.LIG_F_NO_QUEUE_AND_LOW_KV):
        out.append([F(kind, 1, -1, -1, q, kv), F(N.LIG_F_LEAST_QUEUING, -1, -1, -1, 0, 0.0)])
        for rng_kind in (N.LIG_F_LEAST_QUEUING, N.LIG_F_LEAST_KV_CACHE):
            out.append([F(rng_kind, -1, -1, 1, 0, 0.0), F(kind, -1, -1, -1, q, kv)])
        out.append([F(N.LIG_F_LORA_AFFINITY, 1, 2, -1, 0, 0.0), F(kind, -1, -1, -1, q, kv),
                    F(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0)])
        out.append([F(N.LIG_F_LORA_AFFINITY, 1, 2, -1, 0, 0.0), F(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0),
                    F(kind, -1, -1, -1, q, kv)])
    return out
