"""Shared test helpers: conversions between the golden-vector dicts, the oracle's records and
the product package's Go-named record types; a numpy restatement of the pick arithmetic."""
from __future__ import annotations

import numpy as np

from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics
from oracle import lig_oracle_py as PY

M64 = (1 << 64) - 1


def golden_to_podmetrics(p: dict) -> PodMetrics:
    return PodMetrics(Pod=Pod(Name=p["name"], Address=p["address"]),
                      Metrics=Metrics(WaitingQueueSize=p["waiting_queue_size"],
                                      KVCacheUsagePercent=p["kv_cache_usage_percent"],
                                      MaxActiveModels=p["max_active_models"],
                                      ActiveModels={m: 1 for m in p["active_models"]}))


def golden_to_py(p: dict) -> PY.PodMetrics:
    return PY.PodMetrics(pod=PY.Pod(p["name"], p["address"]),
                         metrics=PY.Metrics(active_models={m: 1 for m in p["active_models"]},
                                            max_active_models=p["max_active_models"],
                                            waiting_queue_size=p["waiting_queue_size"],
                                            kv_cache_usage_percent=p["kv_cache_usage_percent"]))


def pod_key(p: dict):
    """What cmp.Diff compares in the reference tests: the whole record."""
    return (p["name"], p["address"], p["waiting_queue_size"], p["kv_cache_usage_percent"],
            p["max_active_models"], tuple(sorted(p["active_models"])))


def fold(reqs: np.ndarray, seeds) -> np.ndarray:
    """The requests whose picks under seed 0 are those of `reqs` under `seeds`: the pick state is
    seed ^ rand_key, so the seed folds into the key.  `seeds` is a uint64 array that broadcasts
    against reqs (one seed per batch row)."""
    f = np.array(reqs, copy=True)
    f["rand_key"] ^= seeds
    return f


def np_splitmix_int31(state: np.ndarray):
    """Vectorised next()>>33 over uint64 states; returns (new_state, int31)."""
    with np.errstate(over="ignore"):
        state = state + np.uint64(0x9E3779B97F4A7C15)
        z = state.copy()
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return state, (z >> np.uint64(33)).astype(np.int64)


def np_int31n(seed: int, rand_key: np.ndarray, n: np.ndarray) -> np.ndarray:
    """Vectorised Go Int31n over per-request streams (n > 0 everywhere)."""
    state = (np.uint64(seed) ^ rand_key.astype(np.uint64))
    n = n.astype(np.int64)
    state, v = np_splitmix_int31(state)
    pow2 = (n & (n - 1)) == 0
    mx = (1 << 31) - 1 - ((1 << 31) % n)
    k = np.where(pow2, v & (n - 1), 0)
    pending = ~pow2 & (v > mx)
    while pending.any():
        state2, v2 = np_splitmix_int31(state)
        state = np.where(pending, state2, state)
        v = np.where(pending, v2, v)
        pending = ~pow2 & (v > mx)
    return np.where(pow2, k, v % n)
