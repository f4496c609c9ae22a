"""The per-batch seed folds into the request keys.

A pick's random stream starts from `seed ^ rand_key` (include/lig.h), so the picks of a batch under
seed s equal the picks of the same batch under seed 0 with every key replaced by `s ^ rand_key`.
tests/test_gpu_kernel_variants.py relies on this to check a queue of many batches (batch b runs
with seed + b, mod 2^64) with one call of the class-table CPU arm.  Shown here on that arm itself,
with the real per-batch seeds, on a pool whose picks depend on the key and on one whose classes
DROP and end EMPTY, for seeds that wrap past 2^64.
"""
import math

import numpy as np

from helpers import M64, fold
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics
from llm_instance_gateway_b200.packer import pack_pod_metrics
from oracle.binding import LIGO_DROP, LIGO_EMPTY, LIGO_OK


def test_seed_folds_into_the_keys(oracle):
    c3 = WL.make_snapshot(512, 256, seed=41).packed
    # queues 1-3 and NaN KV everywhere: sheddable classes DROP, critical ones end EMPTY
    all_nan_kv = [PodMetrics(Pod(f"pod-{i}", f"address-{i}"), Metrics(WaitingQueueSize=q, KVCacheUsagePercent=math.nan))
                  for i, q in enumerate((1, 2, 3))]
    pools = [c3, pack_pod_metrics(all_nan_kv)]
    seed, nb, R = M64 - 4, 12, 700                      # batch seeds 2^64-5 .. 2^64-1, 0 .. 6
    seeds = [(seed + b) & M64 for b in range(nb)]
    assert seeds[5] == 0 and seeds[-1] == 6
    statuses = set()
    for p in pools:
        table = oracle.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap)
        reqs = WL.make_requests(nb * R, p.A, seed=3).reshape(nb, R)
        reqs["adapter_id"][:, :4] = [-1, p.A, p.A + 1, 2**31 - 1]
        real = np.stack([table.schedule_batch(np.ascontiguousarray(reqs[b]), seeds[b]) for b in range(nb)])
        folded = table.schedule_batch(fold(reqs, np.array(seeds, dtype=np.uint64)[:, None]).reshape(-1), 0)
        assert np.array_equal(folded.reshape(nb, R), real)
        statuses |= set(np.unique(real["status"]).tolist())
        if p.A:
            # the picks do depend on the seed: the fold is not trivially true
            assert not np.array_equal(real[0], table.schedule_batch(np.ascontiguousarray(reqs[0]), 0))
            assert (real["n_survivors"] > 1).any()
    assert {LIGO_OK, LIGO_DROP, LIGO_EMPTY} <= statuses
