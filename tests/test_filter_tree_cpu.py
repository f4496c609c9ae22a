"""Caller filter trees without a GPU: the Python chart builder, and the two CPU references of a caller
tree: the oracle's port of the reference walking a node table (oracle_tree, what the GPU tests check
against) and an independent numpy walker (filter_tree_ref).  DEFAULT_FILTER through either equals the
oracle's defaultFilter, one-node trees give the reference's TestFilterFunc survivor sets, and the two
agree on random trees."""
import numpy as np
import pytest

import oracle_tree
from filter_tree_ref import Pods, random_pool, random_tree, walk
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S


def names_of(records):
    return sorted({m for r in records for m in r["active_models"]}) + ["never-loaded"]


@pytest.fixture
def tree_oracle():
    yield oracle_tree
    oracle_tree.set_filter_tree(None)


def check_default_equals_oracle(oracle, records):
    pool = oracle.Pool(records)
    tpool = oracle_tree.Pool(records)
    pods = Pods(records)
    table = S.DEFAULT_FILTER.flatten()
    oracle_tree.set_filter_tree(table)
    for model in names_of(records):
        for crit in (False, True):
            want = pool.filter(model, crit)
            assert tpool.filter(model, crit) == want, (model, crit)
            assert walk(table, pods, crit, model) == want, (model, crit)


def test_default_filter_restates_scheduler_go():
    t = S.DEFAULT_FILTER.flatten()
    assert len(t) == 11
    kinds = [n.kind for n in t]
    assert kinds.count(N.LIG_F_LEAST_QUEUING) == 2 and kinds.count(N.LIG_F_LEAST_KV_CACHE) == 2
    # queueLoRAAndKVCacheFilter has two parents (sheddable success, low-queue failure) and
    # queueAndKVCacheFilter two (affinity success, can-accept either way): both stored once
    parents = {}
    for i, n in enumerate(t):
        for j in (n.next_on_success, n.next_on_failure, n.next_on_success_or_failure):
            if j >= 0:
                assert j > i
                parents.setdefault(j, set()).add(i)
    assert sorted(len(p) for p in parents.values()).count(2) == 2
    low_q = [n for n in t if n.kind == N.LIG_F_LOW_QUEUEING][0]
    shed = [n for n in t if n.kind == N.LIG_F_NO_QUEUE_AND_LOW_KV][0]
    assert low_q.queue_threshold == 50 and (shed.queue_threshold, shed.kv_threshold) == (5, 0.8)


def test_flatten_keeps_shared_subtrees_and_rejects_cycles():
    leaf = S.Filter("kv", S.LEAST_KV_CACHE)
    mid = S.Filter("q", S.LEAST_QUEUING, next_on_success_or_failure=leaf)
    root = S.Filter("r", S.LORA_AFFINITY, next_on_success=mid, next_on_failure=S.Filter("c", S.CAN_ACCEPT_NEW_LORA,
                                                                                            next_on_success=mid))
    t = root.flatten()
    assert len(t) == 4 and t[0].kind == N.LIG_F_LORA_AFFINITY
    assert t[0].next_on_success == t[t[0].next_on_failure].next_on_success
    a = S.Filter("a", S.LEAST_QUEUING)
    b = S.Filter("b", S.LEAST_KV_CACHE, next_on_failure=a)
    a.next_on_success = b
    with pytest.raises(ValueError, match="cycle"):
        a.flatten()
    self_loop = S.Filter("s", S.DROP)
    self_loop.next_on_failure = self_loop
    with pytest.raises(ValueError, match="cycle"):
        self_loop.flatten()
    chain = S.Filter("0", S.LEAST_QUEUING)
    node = chain
    for i in range(1, 33):
        node.next_on_success_or_failure = S.Filter(str(i), S.LEAST_QUEUING)
        node = node.next_on_success_or_failure
    with pytest.raises(ValueError, match="33 nodes"):
        chain.flatten()


def test_default_filter_tree_equals_oracle_on_golden_pools(golden, oracle, tree_oracle):
    for case in golden["TestFilter"]:
        check_default_equals_oracle(oracle, case["input"] or [])


def test_default_filter_tree_equals_oracle_on_random_pools(oracle, tree_oracle):
    rng = np.random.default_rng(2024)
    for _ in range(200):
        check_default_equals_oracle(oracle, random_pool(rng))


def one_node(kind, q_thr=0, kv_thr=0.0):
    return [N.LigFilterNode(kind, -1, -1, -1, q_thr, kv_thr)]


def test_golden_filter_funcs_as_one_node_trees(golden, tree_oracle):
    by_name = {c["name"]: c for c in golden["TestFilterFunc"]}
    cases = {
        "least queuing empty input": one_node(N.LIG_F_LEAST_QUEUING),
        "least queuing": one_node(N.LIG_F_LEAST_QUEUING),
        "least kv cache empty input": one_node(N.LIG_F_LEAST_KV_CACHE),
        "least kv cache": one_node(N.LIG_F_LEAST_KV_CACHE),
        "noQueueAndLessThanKVCacheThresholdPredicate": one_node(N.LIG_F_NO_QUEUE_AND_LOW_KV, 0, 0.8),
        "low LoRA cost": one_node(N.LIG_F_LOW_LORA_COST),
    }
    assert set(cases) == set(by_name)
    for name, tree in cases.items():
        c = by_name[name]
        req = c["req"] or {}
        model, crit = req.get("resolved_target_model", ""), bool(req.get("critical"))
        oracle_tree.set_filter_tree(tree)
        st, idx = oracle_tree.Pool(c["input"]).filter(model, crit)
        assert (st, idx) == walk(tree, Pods(c["input"]), crit, model), name
        want = [(p["waiting_queue_size"], p["kv_cache_usage_percent"], tuple(p["active_models"])) for p in c["output"]]
        got = [(c["input"][i]["waiting_queue_size"], c["input"][i]["kv_cache_usage_percent"],
                tuple(c["input"][i]["active_models"])) for i in idx]
        assert got == want, name
        assert st == (N.LIG_OK if want else N.LIG_EMPTY), name
    # a predicate leaf that keeps nothing: Go's "no pods left"
    c = by_name["low LoRA cost"]
    oracle_tree.set_filter_tree(one_node(N.LIG_F_LORA_AFFINITY))
    assert oracle_tree.Pool(c["input"]).filter("nobody-serves-this", False) == (N.LIG_NO_PODS_LEFT, [])
    assert walk(one_node(N.LIG_F_LORA_AFFINITY), Pods(c["input"]), False, "nobody-serves-this") == (N.LIG_NO_PODS_LEFT, [])


def test_random_trees_oracle_and_walker_agree(tree_oracle):
    """Every routing case (next_on_success with next_on_success_or_failure, predicate leaves, drop
    nodes with successors, ...) through both references."""
    rng = np.random.default_rng(5)
    kinds = set()
    for it in range(400):
        tree = random_tree(rng)
        kinds |= {n.kind for n in tree}
        records = random_pool(rng)
        oracle_tree.set_filter_tree(tree)
        tpool, pods = oracle_tree.Pool(records), Pods(records)
        for model in names_of(records):
            for crit in (False, True):
                assert tpool.filter(model, crit) == walk(tree, pods, crit, model), (it, model, crit)
    assert kinds == set(range(9))


def test_oracle_tree_rejects_invalid_tables(tree_oracle):
    row = lambda k, s=-1, f=-1, sf=-1: N.LigFilterNode(k, s, f, sf, 0, 0.0)
    for bad in ([row(N.LIG_F_LEAST_QUEUING, 0)], [row(N.LIG_F_LEAST_QUEUING, -1, -1, 1)], [row(9)], []):
        with pytest.raises(ValueError):
            oracle_tree.set_filter_tree(bad)


def test_no_pods_left_error_text():
    err = S._schedule_error(N.LIG_NO_PODS_LEFT)
    assert err.code == "Unknown"
    assert str(err) == "failed to apply filter, resulted 0 pods, this should never happen: no pods left"
