"""The references at extreme thresholds, without a GPU: the oracle's port of the reference, its Python
twin, the class-table oracle and the caller-tree oracle (with defaultFilter restated at the same
thresholds) give the same survivor sets for queue thresholds across the whole int64 range and KV
thresholds at NaN, the infinities, signed zeros, denormals and one ulp either side of a pod's value.
The GPU tests of the same values judge the device against these references.  Also: the C packer
refuses a pod record that claims more adapters than LIG_MAX_ADAPTERS."""
import numpy as np
import pytest

import oracle_tree
import threshold_grid as TG
from filter_tree_ref import ADAPTERS, Pods, random_pool, random_tree, walk
from helpers import golden_to_podmetrics, golden_to_py
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200.packer import REQ_DTYPE, pack_pod_metrics
from oracle import lig_oracle_py as PY


@pytest.fixture
def port(oracle):
    yield oracle
    oracle.set_thresholds()
    oracle_tree.set_filter_tree(None)


def extreme_pool(rng):
    recs = random_pool(rng)
    return recs + TG.edge_pods(rng, int(rng.integers(3, 10)), len(recs), ADAPTERS)


def packed_names(records):
    packed = pack_pod_metrics([golden_to_podmetrics(r) for r in records])
    names = [None] * packed.A
    for k, v in packed.adapter_ids.items():
        names[v] = k
    return packed, names + ["never-loaded"]


def class_requests(A):
    reqs = np.zeros(2 * (A + 1), dtype=REQ_DTYPE)
    reqs["adapter_id"] = list(range(A + 1)) * 2
    reqs["flags"] = [0] * (A + 1) + [1] * (A + 1)
    reqs["rand_key"] = np.arange(len(reqs), dtype=np.uint64)
    return reqs


def mask_list(row, P):
    return [p for p in range(P) if (int(row[p >> 5]) >> (p & 31)) & 1]


def test_references_agree_at_extreme_thresholds(port):
    rng = np.random.default_rng(2031)
    n_triples = 0
    for it in range(40):
        records = extreme_pool(rng)
        packed, names = packed_names(records)
        P, A = packed.P, packed.A
        pods = Pods(records)
        py_pods = [golden_to_py(r) for r in records]
        reqs = class_requests(A)
        tpool = oracle_tree.Pool(records)
        for kv, qc, ql in TG.triples(packed.q, packed.kv, 24, rng):
            n_triples += 1
            label = (it, kv, qc, ql)
            port.set_thresholds(kv, qc, ql)
            out, masks = port.Pool(records).schedule_batch(names[:-1], names[-1], reqs, 1, True)
            tab = port.ClassTable(P, A, packed.kv, packed.q, packed.n_active, packed.max_active, packed.bitmap,
                                  thresholds=(kv, qc, ql))
            twin = PY.Scheduler(PY.StaticProvider(py_pods), PY.Thresholds(kv, qc, ql))
            tree = TG.default_tree(kv, qc, ql)
            oracle_tree.set_filter_tree(tree)
            for i, (a, crit) in enumerate(zip(reqs["adapter_id"], reqs["flags"])):
                crit, model = bool(crit), names[int(a)]
                want = (int(out["status"][i]), mask_list(masks[i], P))
                st, surv = twin.filter_only(PY.LLMRequest(model=model, resolved_target_model=model, critical=crit))
                assert (st, [int(p.pod.name.split("-")[1]) for p in surv]) == want, label + ("twin", model, crit)
                t_st, _, t_list = tab.klass(crit, int(a))
                assert (t_st, t_list) == want, label + ("classtab", model, crit)
                assert tpool.filter(model, crit) == want, label + ("oracle_tree", model, crit)
                assert walk(tree, pods, crit, model) == want, label + ("filter_tree_ref", model, crit)
                assert int(out["n_survivors"][i]) == len(want[1])
    assert n_triples >= 40 * len(TG.corner_triples())


def test_the_grid_reaches_both_sides_of_every_comparison(port):
    """Some pod must pass and some fail each threshold comparison at some grid value, or the test
    above could not see a threshold read as another value."""
    records = TG.edge_pods(np.random.default_rng(1), 12, 0, ADAPTERS)
    q = np.array([r["waiting_queue_size"] for r in records])
    kv = np.array([r["kv_cache_usage_percent"] for r in records])
    for thr in (TG.INT32_MAX + 1, 1 << 32, TG.INT64_MAX):
        assert (q < thr).all()                 # read as int32 these would be negative or -1: all fail
    for thr in (TG.INT32_MIN - 1, TG.INT64_MIN):
        assert not (q <= thr).any()            # read as int32 they would keep the INT32_MIN pods
    with np.errstate(invalid="ignore"):
        assert (kv <= np.inf).sum() == (~np.isnan(kv)).sum() and not (kv <= np.nan).any()


def test_caller_trees_with_grid_thresholds_oracle_and_walker_agree(port):
    rng = np.random.default_rng(77)
    for it in range(120):
        records = extreme_pool(rng)
        pods, tpool = Pods(records), oracle_tree.Pool(records)
        qs, kvs = TG.q_grid(pods.q), TG.kv_grid(pods.kv)
        trees = [TG.with_grid_thresholds(random_tree(rng), rng, qs, kvs)]
        if it % 4 == 0:
            trees += TG.placed_trees(int(rng.choice(qs)), float(rng.choice(kvs)))
        for tree in trees:
            oracle_tree.set_filter_tree(tree)
            for model in sorted({m for r in records for m in r["active_models"]}) + ["never-loaded"]:
                for crit in (False, True):
                    assert tpool.filter(model, crit) == walk(tree, pods, crit, model), (it, model, crit)


def c_pack_snapshot(P, A, kv, q, na, ma, bm, blob_ok=True):
    lib = N.load()
    blob = np.full(max(lib.lig_snapshot_bytes(P, A), 16), 0x5A, dtype=np.uint8)
    p = lambda a: a.ctypes.data if a is not None and a.size else None
    rc = lib.lig_pack_snapshot(blob.ctypes.data if blob_ok else None, P, A, p(kv), p(q), p(na), p(ma), p(bm))
    return rc, blob


@pytest.mark.parametrize("pod", ["first", "last"])
def test_pack_snapshot_refuses_n_active_above_max_adapters(pod):
    P, A = 37, 3
    kv, q = np.zeros(P), np.zeros(P, dtype=np.int32)
    na, ma = np.full(P, N.LIG_MAX_ADAPTERS, dtype=np.uint16), np.full(P, 65535, dtype=np.uint16)
    bm = np.zeros((A, 2), dtype=np.uint32)
    assert c_pack_snapshot(P, A, kv, q, na, ma, bm)[0] == 0           # 65534 is the largest legal count
    na[0 if pod == "first" else P - 1] = 65535
    rc, blob = c_pack_snapshot(P, A, kv, q, na, ma, bm)
    assert rc == N.LIG_ERR_RANGE
    assert b"n_active 65535" in N.load().lig_last_error()
    assert (blob == 0x5A).all()                                      # refused before anything is written


def test_pack_snapshot_refuses_null_arrays():
    P, A = 5, 2
    cols = [np.zeros(P), np.zeros(P, dtype=np.int32), np.zeros(P, dtype=np.uint16), np.zeros(P, dtype=np.uint16),
            np.zeros((A, 1), dtype=np.uint32)]
    assert c_pack_snapshot(P, A, *cols)[0] == 0
    assert c_pack_snapshot(P, A, *cols, blob_ok=False)[0] == N.LIG_ERR_INVALID
    for k in range(5):
        bad = list(cols)
        bad[k] = None
        assert c_pack_snapshot(P, A, *bad)[0] == N.LIG_ERR_INVALID, k
    assert c_pack_snapshot(0, 0, None, None, None, None, None)[0] == 0
    assert c_pack_snapshot(P, 0, *cols[:4], None)[0] == 0            # no adapters: no bitmap needed
