"""Caller filter trees on the GPU (lig_set_filter_tree): the tree build's class tables and picks
against the oracle's port of the reference walking the same table (oracle_tree), DEFAULT_FILTER as a
caller tree against the built-in build on every pick path, the LIG_NO_PODS_LEFT status, the tree's
lifecycle over epochs, and device groups."""
import math

import numpy as np
import pytest
import torch

import oracle_tree
from filter_tree_ref import random_pool, random_tree
from helpers import np_int31n
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics
from llm_instance_gateway_b200.engine import Engine, EngineGroup
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models, pack_pod_metrics

pytestmark = pytest.mark.gpu

DEFAULT = S.DEFAULT_FILTER.flatten()


def mkpods(qs, kvs, maxs=None, acts=None):
    n = len(qs)
    maxs = maxs or [0] * n
    acts = acts or [[] for _ in range(n)]
    return [PodMetrics(Pod(f"pod-{i}", f"address-{i}"),
                       Metrics(WaitingQueueSize=qs[i], KVCacheUsagePercent=kvs[i], MaxActiveModels=maxs[i],
                               ActiveModels={a: 1 for a in acts[i]})) for i in range(n)]


# the shapes of the parity suite's edge pools
EDGE_POOLS = {
    "single_pod": mkpods([0], [0.1]),
    "single_pod_busy": mkpods([60], [0.95]),
    "all_nan_kv": mkpods([1, 2, 3], [math.nan] * 3),
    "some_nan_kv": mkpods([0, 0, 0, 0], [math.nan, 0.2, math.nan, 0.1]),
    "inf_kv": mkpods([0, 0, 0], [math.inf, math.inf, math.inf]),
    "neg_inf_kv": mkpods([0, 0, 0], [-math.inf, 0.5, 0.2]),
    "signed_zero_kv": mkpods([0, 0, 0, 0], [0.0, -0.0, -0.0, 0.0]),
    "negative_q": mkpods([-10, -7, -1, 4], [0.1, 0.1, 0.1, 0.1]),
    "int32_extremes": mkpods([2**31 - 1, -(2**31), 0, 7], [0.1, 0.2, 0.3, 0.4]),
    "q_all_high": mkpods([50, 51, 99, 50, 200], [0.5, 0.4, 0.3, 0.2, 0.1],
                         [2, 2, 2, 2, 2], [["x"], [], ["x", "y"], ["y"], []]),
    "q_boundaries": mkpods([49, 50, 5, 6, 0], [0.8, 0.8, 0.8000000000000002, 0.1, 0.7999999999999999]),
    "ties": mkpods([3] * 40, [0.25] * 40),
    "max_active_zero": mkpods([0, 0, 0], [0.1, 0.2, 0.3], [0, 0, 0], [["a"], ["b"], []]),
    "overfull": mkpods([1, 1, 1, 1], [0.3, 0.2, 0.1, 0.4], [1, 1, 2, 70000], [["a", "b"], ["a"], ["b"], []]),
    "affinity_vs_room": mkpods([0, 1, 2, 3, 4, 5], [0.5, 0.1, 0.9, 0.3, 0.2, 0.6], [2, 1, 2, 2, 0, 3],
                               [["a"], ["b"], ["a", "b"], [], ["a"], ["c"]]),
    "drop_all": mkpods([10, 3, 10], [0.9, 0.85, 0.85]),
    "empty": [],
}


def class_requests(A, copies=4, seed=3):
    ids = list(range(A + 1)) + [-1, A + 7]
    reqs = np.zeros(2 * len(ids) * copies, dtype=REQ_DTYPE)
    reqs["adapter_id"] = (ids + ids) * copies
    reqs["flags"] = ([0] * len(ids) + [1] * len(ids)) * copies
    reqs["rand_key"] = np.random.default_rng(seed).integers(0, 1 << 64, size=len(reqs), dtype=np.uint64)
    return reqs


def read_tables(eng, ep, A, P):
    return [[eng.read_class(ep, bool(crit), a, P) for a in range(A + 1)] for crit in (0, 1)]


def ref_tables(nodes, records, names):
    """The oracle's (status, survivors) per class; names[a] for a in [0, A] is the adapter's name
    (names[A] = a model no pod lists)."""
    oracle_tree.set_filter_tree(nodes)
    try:
        pool = oracle_tree.Pool(records)
        return [[pool.filter(names[a], bool(crit)) for a in range(len(names))] for crit in (0, 1)]
    finally:
        oracle_tree.set_filter_tree(None)


def ref_picks(nodes, records, names, reqs, seed):
    """The oracle's Schedule with the caller's tree; names as for ref_tables (names[-1] = unknown)."""
    oracle_tree.set_filter_tree(nodes)
    try:
        return oracle_tree.Pool(records).schedule_batch(names[:-1], names[-1], reqs, seed)
    finally:
        oracle_tree.set_filter_tree(None)


def assert_tables_equal(got, want, label=""):
    for crit in (0, 1):
        for a, ((st, n, lst), (wst, widx)) in enumerate(zip(got[crit], want[crit])):
            assert (st, n, lst.tolist()) == (wst, len(widx), widx), (label, crit, a)


def expected_picks(tables, A, reqs, seed):
    """Picks from class tables [(status, list)]: list[Int31n(n)] on the request's stream."""
    crit = (reqs["flags"] & 1).astype(np.int64)
    a = np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)
    out = np.zeros(len(reqs), dtype=PICK_DTYPE)
    st = np.array([[t[0] for t in row] for row in tables])
    ns = np.array([[len(t[1]) for t in row] for row in tables])
    out["status"] = st[crit, a]
    out["n_survivors"] = ns[crit, a]
    out["pod_idx"] = -1
    ok = out["n_survivors"] > 0
    if ok.any():
        k = np_int31n(seed, reqs["rand_key"][ok], out["n_survivors"][ok].astype(np.int64))
        lists = [[t[1] for t in row] for row in tables]
        out["pod_idx"][ok] = [lists[c][x][j] for c, x, j in zip(crit[ok], a[ok], k)]
    return out


def device_paths(eng, ep, reqs, seed, ids=None):
    """The same batch through the host-buffer kernel, the persistent queue, the feedback mode, the
    doorbell stream and (with model ids) the model-request queue."""
    R = len(reqs)
    out = {"host": eng.schedule_batch(ep, seed, reqs)}
    d_reqs = torch.from_numpy(reqs.view(np.uint8).reshape(-1).copy()).cuda()
    d_q = [torch.zeros(R * 8, dtype=torch.uint8, device="cuda") for _ in range(2)]
    eng.schedule_batches_device(ep, seed, [d_reqs.data_ptr()] * 2, R, [t.data_ptr() for t in d_q])
    d_fb = torch.zeros(R * 8, dtype=torch.uint8, device="cuda")
    eng.schedule_batch_feedback_device(ep, seed, d_reqs.data_ptr(), R, d_fb.data_ptr(), max(1, R // 4))
    if ids is not None:
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        d_m = torch.zeros(len(ids) * 4, dtype=torch.uint8, device="cuda")
        eng.schedule_models_batches_device(ep, seed, 0, [d_ids.data_ptr()], len(ids), [d_m.data_ptr()])
    torch.cuda.synchronize()
    out["queue0"], out["queue1"] = [t.cpu().numpy().view(PICK_DTYPE) for t in d_q]
    out["feedback"] = d_fb.cpu().numpy().view(PICK_DTYPE)
    if ids is not None:
        out["models"] = d_m.cpu().numpy().view(MPICK_DTYPE)
    n = min(R, N.load().lig_stream_capacity())
    eng.stream_open()
    try:
        out["doorbell"] = eng.stream_submit(ep, seed, np.ascontiguousarray(reqs[:n]))
    finally:
        eng.stream_close()
    return out


@pytest.fixture(scope="module")
def pair():
    """Two ctxs: the built-in tree, and DEFAULT_FILTER as a caller tree."""
    builtin = Engine(0, max_pods=4096, max_adapters=1024, max_batch=1 << 20)
    caller = Engine(0, max_pods=4096, max_adapters=1024, max_batch=1 << 20)
    caller.set_filter_tree(S.DEFAULT_FILTER)
    yield builtin, caller
    builtin.close()
    caller.close()


_ep = [0]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


def check_equivalent(builtin, caller, packed, reqs, seed, ids=None, models=None, label=""):
    ep = next_epoch()
    for e in (builtin, caller):
        e.upload_snapshot(ep, packed)
        if models is not None:
            e.upload_models(ep, models)
    assert_tables_equal(read_tables(caller, ep, packed.A, packed.P),
                        [[(st, lst.tolist()) for st, _, lst in row] for row in read_tables(builtin, ep, packed.A, packed.P)],
                        label)
    got, want = device_paths(caller, ep, reqs, seed, ids), device_paths(builtin, ep, reqs, seed, ids)
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), (label, k)


# ---- 4. built-in equivalence ----------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C3", "C4"])
def test_default_filter_as_caller_tree_equals_builtin(cfg, pair):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"])
    reqs = WL.make_requests(c["R"], c["A"])
    models = pack_models(WL.make_models(c["A"]), snap.packed)
    ids = WL.make_model_requests(c["R"], c["A"])
    check_equivalent(*pair, snap.packed, reqs, 0xC0FFEE, ids, models, cfg)


@pytest.mark.parametrize("name", sorted(EDGE_POOLS))
def test_default_filter_as_caller_tree_equals_builtin_edge_pools(name, pair):
    packed = pack_pod_metrics(EDGE_POOLS[name])
    check_equivalent(*pair, packed, class_requests(packed.A), 77, label=name)


def test_default_filter_as_caller_tree_equals_builtin_unstaged():
    """P = 20000: the pod columns do not fit in shared memory, both builds read global memory."""
    P, A = 20000, 64
    builtin = Engine(0, max_pods=N.LIG_MAX_PODS, max_adapters=A, max_batch=1 << 16)
    caller = Engine(0, max_pods=N.LIG_MAX_PODS, max_adapters=A, max_batch=1 << 16)
    try:
        caller.set_filter_tree(S.DEFAULT_FILTER)
        snap = WL.make_snapshot(P, A, seed=5)
        check_equivalent(builtin, caller, snap.packed, WL.make_requests(1 << 14, A, seed=6), 9,
                         WL.make_model_requests(1 << 14, A, seed=7), pack_models(WL.make_models(A), snap.packed),
                         "P=20000")
    finally:
        builtin.close()
        caller.close()


# ---- 5. random trees against the oracle -----------------------------------------------------------
def test_random_trees_against_reference(pair):
    _, eng = pair
    rng = np.random.default_rng(77)
    try:
        for it in range(320):
            tree = random_tree(rng)
            records = random_pool(rng)
            pods = mkpods([r["waiting_queue_size"] for r in records], [r["kv_cache_usage_percent"] for r in records],
                          [r["max_active_models"] for r in records], [r["active_models"] for r in records])
            packed = pack_pod_metrics(pods)
            names = [None] * packed.A + ["never-loaded"]
            for k, v in packed.adapter_ids.items():
                names[v] = k
            eng.set_filter_tree(tree)
            ep = next_epoch()
            eng.upload_snapshot(ep, packed)
            want = ref_tables(tree, records, names)
            assert_tables_equal(read_tables(eng, ep, packed.A, packed.P), want, f"tree#{it}")
            reqs = class_requests(packed.A, seed=it)
            assert np.array_equal(eng.schedule_batch(ep, it, reqs), ref_picks(tree, records, names, reqs, it)), it
    finally:
        eng.set_filter_tree(S.DEFAULT_FILTER)


def c4_tree():
    """KV check before the queue check, no LoRA stage for critical traffic, drop leaves on both sides."""
    kv = S.Filter("least KV", S.LEAST_KV_CACHE)
    q_then_kv = S.Filter("least queuing", S.LEAST_QUEUING, next_on_success_or_failure=kv)
    crit = S.Filter("kv headroom", S.NO_QUEUE_AND_LOW_KV, queue_threshold=40, kv_threshold=0.9,
                    next_on_success=q_then_kv,
                    next_on_failure=S.Filter("low queue", S.LOW_QUEUEING, queue_threshold=60,
                                             next_on_success=kv, next_on_failure=S.Filter("drop", S.DROP)))
    shed = S.Filter("affinity", S.LORA_AFFINITY, next_on_success=q_then_kv,
                    next_on_failure=S.Filter("drop sheddable", S.DROP))
    return S.Filter("critical", S.CRITICAL_REQUEST, next_on_success=crit, next_on_failure=shed)


def test_nontrivial_tree_at_C4(pair):
    _, eng = pair
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    tree = c4_tree().flatten()
    try:
        eng.set_filter_tree(tree)
        ep = next_epoch()
        eng.upload_snapshot(ep, snap.packed)
        want = ref_tables(tree, snap.pod_records(), snap.adapter_names() + [WL.UNKNOWN_MODEL])
        assert_tables_equal(read_tables(eng, ep, c["A"], c["P"]), want, "C4")
        assert len({st for row in want for st, _ in row}) > 1
        reqs = WL.make_requests(c["R"], c["A"])
        sel = np.random.default_rng(4).choice(c["R"], 32768, replace=False)
        sub = np.ascontiguousarray(reqs[sel])
        got = eng.schedule_batch(ep, 0xC4, reqs)
        assert np.array_equal(got[sel], expected_picks(want, c["A"], sub, 0xC4))
        names = snap.adapter_names() + [WL.UNKNOWN_MODEL]
        assert np.array_equal(got[sel[:4096]], ref_picks(tree, snap.pod_records(), names,
                                                         np.ascontiguousarray(sub[:4096]), 0xC4))
    finally:
        eng.set_filter_tree(S.DEFAULT_FILTER)


# ---- 6. statuses ----------------------------------------------------------------------------------
def test_statuses_of_caller_trees():
    eng = Engine(0, max_pods=64, max_adapters=8, max_batch=4096)
    try:
        pods = mkpods([0, 1, 2], [0.1, 0.2, 0.3], [1, 1, 1], [["a"], [], ["b"]])
        packed = pack_pod_metrics(pods)
        A = packed.A
        # a lone LoRA-affinity node for an adapter no pod serves: "no pods left"
        eng.set_filter_tree([N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0)])
        eng.upload_snapshot(1, packed)
        reqs = np.zeros(64, dtype=REQ_DTYPE)
        reqs["adapter_id"] = A
        reqs["flags"] = np.arange(64) & 1
        reqs["rand_key"] = np.arange(64)
        ids = np.zeros(64, dtype=np.uint32)      # model-0 -> adapter-0, which no pod here lists
        eng.upload_models(1, pack_models(WL.make_models(1), packed))
        paths = device_paths(eng, 1, reqs, 5, ids)
        for k, v in paths.items():
            assert (v["status"] == N.LIG_NO_PODS_LEFT).all() and (v["pod_idx"] == -1).all(), k
            if k != "models":
                assert (v["n_survivors"] == 0).all(), k
        assert eng.read_class(1, False, A, packed.P)[:2] == (N.LIG_NO_PODS_LEFT, 0)
        assert eng.read_class(1, True, packed.adapter_id("a"), packed.P)[0] == N.LIG_OK
        # a drop leaf, and an all-NaN least-KV leaf
        eng.set_filter_tree([N.LigFilterNode(N.LIG_F_DROP, -1, -1, -1, 0, 0.0)])
        eng.upload_snapshot(2, packed)
        assert (eng.schedule_batch(2, 1, reqs)["status"] == N.LIG_DROP).all()
        eng.set_filter_tree([N.LigFilterNode(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0)])
        eng.upload_snapshot(3, pack_pod_metrics(mkpods([1, 2, 3], [math.nan] * 3)))
        got = eng.schedule_batch(3, 1, np.ascontiguousarray(reqs[:4]))
        assert (got["status"] == N.LIG_EMPTY).all() and (got["pod_idx"] == -1).all()
    finally:
        eng.close()


class StaticProvider:
    def __init__(self, pods):
        self.pods = list(pods)

    def AllPodMetrics(self):
        return list(self.pods)


def test_scheduler_mirror_errors_with_caller_tree():
    pods = mkpods([0, 1], [0.1, 0.2], [0, 0], [["a"], []])
    sched = S.NewScheduler(StaticProvider(pods), filter=S.Filter("affinity", S.LORA_AFFINITY), max_pods=64,
                           max_adapters=8, max_batch=64, seed=1)
    try:
        with pytest.raises(S.StatusError) as ei:
            sched.Schedule(S.LLMRequest(Model="b", ResolvedTargetModel="b"))
        assert ei.value.code == "Unknown"
        assert str(ei.value) == "failed to apply filter, resulted 0 pods, this should never happen: no pods left"
        assert sched.Schedule(S.LLMRequest(Model="a", ResolvedTargetModel="a")).Name == "pod-0"
        got, err = sched.Filter(S.LLMRequest(ResolvedTargetModel="b"))
        assert got == [] and str(err) == "no pods left"
        got, err = sched.Filter(S.LLMRequest(ResolvedTargetModel="a"))
        assert [p.Name for p in got] == ["pod-0"] and err is None
    finally:
        sched.close()
    sched = S.NewScheduler(StaticProvider(pods), filter=S.Filter("drop", S.DROP), max_pods=64, max_adapters=8,
                           max_batch=64, seed=1)
    try:
        with pytest.raises(S.StatusError) as ei:
            sched.Schedule(S.LLMRequest(Model="a", ResolvedTargetModel="a", Critical=True))
        assert ei.value.code == "ResourceExhausted"
    finally:
        sched.close()


def test_host_runtime_scheduler_maps_no_pods_left():
    from llm_instance_gateway_b200 import host as H
    prov = H.HostProvider(mkpods([0, 1], [0.1, 0.2], [0, 0], [["a"], []]))
    try:
        for doorbell in (False, True):        # the latency knobs pass through with a caller tree
            sched = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=64, use_doorbell=doorbell,
                                    busy_poll=doorbell, filter=S.Filter("affinity", S.LORA_AFFINITY))
            try:
                assert sched.Schedule("b", "b", False) == (
                    H.GRPC_UNKNOWN, None, "failed to apply filter, resulted 0 pods, this should never happen: no pods left")
                code, pod, _ = sched.Schedule("a", "a", True)
                assert code == H.GRPC_OK and pod.Name == "pod-0"
            finally:
                sched.close()
    finally:
        prov.close()


# ---- 7. lifecycle and validation ------------------------------------------------------------------
def test_tree_lifecycle_and_validation(oracle):
    eng = Engine(0, max_pods=512, max_adapters=64, max_batch=1 << 14)
    try:
        snap = WL.make_snapshot(300, 20, seed=8)
        names = snap.adapter_names() + [WL.UNKNOWN_MODEL]
        rec = snap.pod_records()
        tree_a = DEFAULT
        tree_b = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, 1, -1, -1, 20, 0.0),
                  N.LigFilterNode(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0)]
        tree_c = c4_tree().flatten()
        eng.set_filter_tree(tree_a)
        eng.upload_snapshot(1, snap.packed)
        eng.set_filter_tree(tree_b)
        eng.upload_snapshot(2, snap.packed)
        reqs = class_requests(20)
        for ep, tree in ((1, tree_a), (2, tree_b)):     # each epoch keeps the tree it was built with
            want = ref_tables(tree, rec, names)
            assert_tables_equal(read_tables(eng, ep, 20, 300), want, ep)
            assert np.array_equal(eng.schedule_batch(ep, 3, reqs), expected_picks(want, 20, reqs, 3))
        # a delta from epoch 2 follows the tree in force now
        eng.set_filter_tree(tree_c)
        eng.update_snapshot(3, 2, [0, 5], [0.95, 0.01], [70, 0], [0, 1], [4, 4], [0, 0, 1], [3])
        rec3 = [dict(r) for r in rec]
        rec3[0].update(kv_cache_usage_percent=0.95, waiting_queue_size=70, active_models=[], max_active_models=4)
        rec3[5].update(kv_cache_usage_percent=0.01, waiting_queue_size=0, active_models=[names[3]], max_active_models=4)
        assert_tables_equal(read_tables(eng, 3, 20, 300), ref_tables(tree_c, rec3, names), "delta")
        # thresholds do not affect a caller tree's build
        eng.set_thresholds(0.1, 0, 0)
        eng.upload_snapshot(4, snap.packed)
        assert_tables_equal(read_tables(eng, 4, 20, 300), ref_tables(tree_c, rec, names), "thresholds")
        eng.set_thresholds()
        # invalid tables: LIG_ERR_INVALID, the previous tree stays in force
        row = lambda k, s=-1, f=-1, sf=-1: N.LigFilterNode(k, s, f, sf, 0, 0.0)
        bad = [[row(N.LIG_F_LEAST_QUEUING), row(N.LIG_F_LEAST_KV_CACHE, 0)],     # backward edge
               [row(N.LIG_F_LEAST_QUEUING, -1, 0)],                               # self edge
               [row(N.LIG_F_LEAST_QUEUING, -1, -1, 1)],                           # past the end
               [],                                                                # 0 nodes
               [row(N.LIG_F_LEAST_QUEUING)] * 33,                                 # 33 nodes
               [row(9)], [row(-1)]]                                               # bad kinds
        for nodes in bad:
            with pytest.raises(N.LigError) as ei:
                eng.set_filter_tree(nodes)
            assert ei.value.code == N.LIG_ERR_INVALID
        eng.upload_snapshot(5, snap.packed)
        assert_tables_equal(read_tables(eng, 5, 20, 300), ref_tables(tree_c, rec, names), "after invalid")
        # the direct scan refuses an epoch whose tables a caller tree built
        with pytest.raises(N.LigError) as ei:
            eng.schedule_scan(5, 1, reqs, False)
        assert ei.value.code == N.LIG_ERR_INVALID
        # NULL restores the built-in tree
        eng.set_filter_tree(None)
        eng.upload_snapshot(6, snap.packed)
        pool = oracle.Pool(rec)
        for crit in (0, 1):
            for a in range(21):
                st, n, lst = eng.read_class(6, bool(crit), a, 300)
                assert (st, lst.tolist()) == pool.filter(names[a], bool(crit))
        got, _ = eng.schedule_scan(6, 1, reqs, False)
        assert np.array_equal(got, eng.schedule_batch(6, 1, reqs))
        with pytest.raises(N.LigError):                    # epoch 5 is still resident, still a caller tree's
            eng.schedule_scan(5, 1, reqs, False)
        eng.set_filter_tree(tree_c)                        # a built-in epoch stays scannable under a caller tree
        got, _ = eng.schedule_scan(6, 1, reqs, False)
        assert np.array_equal(got, eng.schedule_batch(6, 1, reqs))
    finally:
        eng.close()


# ---- 8. several GPUs ------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least 2 GPUs")
def test_group_filter_tree_matches_single_device():
    world = min(torch.cuda.device_count(), 8)
    P, A, R = 700, 48, 100_003
    snap = WL.make_snapshot(P, A, seed=61)
    reqs = WL.make_requests(R, A, seed=62)
    tree = c4_tree()
    with EngineGroup(list(range(world)), max_pods=1024, max_adapters=64, max_batch=R) as g, \
            Engine(0, max_pods=1024, max_adapters=64, max_batch=R) as one:
        with pytest.raises(N.LigError):
            g.set_filter_tree([N.LigFilterNode(N.LIG_F_DROP, 0, -1, -1, 0, 0.0)])
        g.set_filter_tree(tree)
        one.set_filter_tree(tree)
        g.upload_snapshot(1, snap.packed)
        one.upload_snapshot(1, snap.packed)
        want = one.schedule_batch(1, 17, reqs)
        assert np.array_equal(g.schedule_batch(1, 17, reqs), want)
        for m in range(world):
            assert_tables_equal(read_tables(g.member(m), 1, A, P),
                                [[(st, lst.tolist()) for st, _, lst in row] for row in read_tables(one, 1, A, P)], m)
