"""The C++ runtime's refresh tick (Scheduler::Refresh) against the oracle, tick by tick.

A seeded pool history (tests/pool_history.py) is fed through HostProvider, one Refresh per tick,
into a scheduler whose max_pods is the pool's size, so a tick with one pod more is refused.  After
every refresh, published or refused, the runtime must answer for the pool of the last published
tick (pool_history.expected_pools):

* Filter(name, critical) equals the oracle's survivor set, code and pod names in slice order, for
  every name of that pool, a never-loaded name and the names it has dropped since the tick before;
* a run of Schedule and ScheduleWithFallbacks calls from one caller equals the pick and fallback
  row of tests/fallback_ref.py over the oracle's survivors, with the runtime's rand_key sequence
  (splitmix_next from seed ^ 0xD1B54A32D192ED03, one key per request, batch seed = seed);
* ScheduleModel(model) (resolved on the device) equals oracle.Models over that pool, with the
  device request count continuing across ticks, while SetInferenceModels swaps lists whose targets
  come and go (built-in tree only; the model oracle walks the built-in tree);
* refreshes, failed_refreshes and excluded_pods follow the ticks' outcomes, and delta_refreshes
  moves where the tick kind makes the upload certain: a delta at the dirty * 4 == P boundary and
  for renamed pods, a full upload one pod past it and after a refused tick.

The regression tests replay a refused tick that swapped a pod's adapter names: the next refresh
must not leave that pod's old bitmap row on the device.
"""
import functools
import threading

import numpy as np
import pytest

import pool_history as PH
from fallback_ref import fallback_row
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import (CRITICAL, InferenceModel, InferenceModelSpec, Metrics, Pod,
                                               PodMetrics, TargetModel)
from oracle import binding as B
from test_gpu_snapshot_mutation import drop_and_no_pods_trees
from test_pool_history_cpu import CASES, case_history, case_sets

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1
PREFIX = "failed to find target pod: "
ERR0 = "failed to apply filter, resulted 0 pods, this should never happen: "
DROP_INNER = "rpc error: code = ResourceExhausted desc = dropping request due to limited backend resources"


def splitmix_next(state):
    """(next state, value): the runtime's rand_key generator."""
    state = (state + 0x9E3779B97F4A7C15) & MASK
    z = state
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    return state, z ^ (z >> 31)


def schedule_code(rc):
    return {N.LIG_OK: H.GRPC_OK, N.LIG_DROP: H.GRPC_RESOURCE_EXHAUSTED}.get(rc, H.GRPC_UNKNOWN)


def filter_result(rc, survivors):
    """Scheduler::Filter's (code, pods) for an oracle status and survivor list."""
    if rc == N.LIG_DROP:
        return H.GRPC_RESOURCE_EXHAUSTED, []
    if rc == N.LIG_NO_PODS_LEFT:
        return H.GRPC_UNKNOWN, []
    return H.GRPC_OK, survivors


def im(name, crit=None, targets=()):
    return InferenceModel(name, InferenceModelSpec(ModelName=name, Criticality=crit,
                                                   TargetModels=[TargetModel(n, w) for n, w in targets]))


def model_lists():
    """Two lists over names that come and go in the histories (lora-0..2 are listed at the start and
    replaced during the rebuild), a target no pod ever lists and a passthrough model."""
    a = [im("single", None, [("lora-0", 1)]), im("split", CRITICAL, [("lora-0", 3), ("lora-1", 5), ("ghost", 2)]),
         im("ghost-only", None, [("ghost", 1)]), im("plain")]
    b = [im("single", CRITICAL, [("lora-1", 1)]), im("split", None, [("lora-1", 2), ("lora-2", 7)]),
         im("ghost-only", CRITICAL, [("ghost", 4)]), im("other", None, [("lora-0", 1), ("lora-2", 1)])]
    return [sorted(a, key=lambda m: m.Spec.ModelName), sorted(b, key=lambda m: m.Spec.ModelName)]


@functools.lru_cache(maxsize=None)
def history(P, tree):
    return case_history(P, tree, seed=P + 7 * (tree or 0))


class Runtime:
    """A HostScheduler over a HostProvider, and what the oracle says it must answer."""

    def __init__(self, hist, P, tree, doorbell, seed):
        self.P, self.seed = P, seed
        self.sets = case_sets(tree)
        self.prov = H.HostProvider(hist[0].pods)
        kw = {} if tree is None else dict(filter=drop_and_no_pods_trees()[tree])
        self.s = H.HostScheduler(self.prov, max_pods=P, max_adapters=PH.MAX_ADAPTERS, max_batch=256,
                                 batch_window_us=20, seed=seed, use_doorbell=doorbell, **kw)
        self.keys = seed ^ 0xD1B54A32D192ED03
        self.rng = np.random.default_rng(seed)
        self.model_index = 0
        self.lists = self.stores = None
        if tree is None:
            self.lists = model_lists()
            self.stores = [H.HostDataStore(ms) for ms in self.lists]
            self.s.set_inference_models(self.stores[0])
            self.list = 0

    def close(self):
        for d in self.stores or ():
            d.close()
        self.s.close()
        self.prov.close()

    def next_key(self):
        self.keys, key = splitmix_next(self.keys)
        return key

    def check_survivors(self, pool, probes, where):
        want = self.sets(pool, probes)
        for (name, crit), (rc, survivors) in want.items():
            code, pods, _ = self.s.Filter(name, crit)
            assert (code, pods) == filter_result(rc, survivors), (where, name, crit, rc)
        return want

    def check_picks(self, want, where, n=6):
        classes = sorted(want.items())
        for j in range(n):
            (name, crit), (rc, survivors) = classes[int(self.rng.integers(0, len(classes)))]
            key = self.next_key()
            pick, row = fallback_row(self.seed, key, survivors, 8) if rc == N.LIG_OK else (-1, [])
            ok = rc == N.LIG_OK and survivors
            if j % 3 == 2:
                code, pods, _ = self.s.ScheduleWithFallbacks(name, crit, 8)
                assert (code, pods) == ((H.GRPC_OK, [pick] + [p for p in row if p != -1]) if ok
                                        else (schedule_code(rc), [])), (where, name, crit, j)
            else:
                code, pod, _ = self.s.Schedule(name, name, crit)
                assert (code, pod.Name if pod else None) == ((H.GRPC_OK, pick) if ok else (schedule_code(rc), None)), \
                    (where, name, crit, j)

    def check_models(self, pool, where):
        models = self.lists[self.list]
        ids = {m.Spec.ModelName: i for i, m in enumerate(models)}
        oracle_pool, mo = B.Pool(PH.records(pool)), B.Models(WL.model_records(models))
        for name in sorted(ids) + ["nope"]:
            code, resolved, pod, err = self.s.ScheduleModelOnDevice(name)
            if name not in ids:
                assert (code, err) == (H.GRPC_UNKNOWN, f"error finding a model object in InferenceModel for input {name}")
                continue
            mp = mo.schedule_batch(oracle_pool, np.array([ids[name]], dtype=np.uint32), self.seed, self.model_index)[0]
            self.model_index += 1
            t, st = int(mp["target_idx"]), int(mp["status"])
            assert resolved == (name if t == 255 else models[ids[name]].Spec.TargetModels[t].Name), (where, name)
            if st == N.LIG_OK:
                assert code == H.GRPC_OK and pod.Name == pool[int(mp["pod_idx"])].Pod.Name, (where, name)
            elif st == N.LIG_DROP:
                assert (code, err) == (H.GRPC_RESOURCE_EXHAUSTED, PREFIX + ERR0 + DROP_INNER), (where, name)
            else:
                assert (st, code, err) == (N.LIG_EMPTY, H.GRPC_UNKNOWN, PREFIX + ERR0 + "%!w(<nil>)"), (where, name)


def probes_for(pools, t, seen):
    """Every name of the expected pool, a never-loaded name, the names dropped since the previous
    tick's pool and one name dropped before that."""
    now = PH.names_of(pools[t])
    recent = sorted(PH.names_of(pools[t - 1]) - now) if t else []
    older = sorted(seen - now - set(recent))[:1]
    return sorted(now) + [PH.NEVER_LOADED] + recent + older


@pytest.mark.parametrize("doorbell", [False, True], ids=["launch", "doorbell"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_runtime_follows_pool_history(case, doorbell):
    follow_history(case, doorbell, eject=False)


EJECT_CASES = [c for c in CASES if c[0] in ("p1", "p33", "p1000", "p5000", "drop_tree", "no_pods_tree")]


@pytest.mark.parametrize("doorbell", [False, True], ids=["launch", "doorbell"])
@pytest.mark.parametrize("case", EJECT_CASES, ids=[c[0] for c in EJECT_CASES])
def test_runtime_follows_pool_history_with_ejections(case, doorbell):
    """The same history with EjectPods called at the ticks of pool_history.eject_schedule: every
    check runs on the expected pool without the ejected pods (by value), ejected_pods counts the
    ejected pods in that pool, and eject_publishes moves exactly where an epoch is derived: an
    EjectPods whose pods sit at other indices than the published epoch's set, a full upload with any
    ejected pod in the pool, and a delta whose ejected pods are not its base's (renamed pods)."""
    follow_history(case, doorbell, eject=True)


def follow_history(case, doorbell, eject):
    _, P, tree = case
    hist = history(P, tree)
    pools = PH.expected_pools(hist)
    ejections = PH.eject_schedule(hist, seed=P) if eject else {}
    rt = Runtime(hist, P, tree, doorbell, seed=1000 + P + (tree or 0))
    try:
        refreshes = 2 if rt.lists else 1      # NewScheduler's refresh, and SetInferenceModels'
        failed = delta = excluded = publishes = deltas_seen = 0
        seen, last_ok = set(), True
        gone, ejected = set(), []             # EjectPods' set, and its indices in the published pool

        def indices(pool):
            return [i for i, p in enumerate(pool) if p.Pod in gone]
        for t, tick in enumerate(hist):
            where = (t, tick.kind)
            if t:
                rt.prov.set_pods(tick.pods)
                try:
                    if rt.lists and t % 5 == 0:       # a new model list publishes through a refresh too
                        rt.s.set_inference_models(rt.stores[1 - rt.list])
                        rt.list = 1 - rt.list
                    else:
                        rt.s.Refresh()
                    ok = True
                except H.HostSchedulerError as e:
                    assert "lig_upload_snapshot" in str(e), (where, str(e))
                    ok = False
                assert ok == tick.published, where
            if tick.published:
                refreshes += t > 0
                excluded = len(tick.pods) - len(tick.kept())
            else:
                failed += 1
            st = rt.s.stats()
            if t and tick.published:          # a delta inherits its base's set, a full upload has none
                used_delta = st["delta_refreshes"] > deltas_seen
                publishes += (indices(pools[t]) != ejected) if used_delta else bool(indices(pools[t]))
                ejected = indices(pools[t])
            deltas_seen = st["delta_refreshes"]
            if t in ejections:
                rt.s.EjectPods(ejections[t])
                gone = set(ejections[t])
                publishes += indices(pools[t]) != ejected
                ejected = indices(pools[t])
                st = rt.s.stats()
            assert (st["eject_publishes"], st["ejected_pods"]) == (publishes, len(ejected)), (where, st)
            if t and tick.kind in ("qkv_boundary", "rename") and last_ok:
                delta += 1                            # at most P // 4 dirty pods, nothing else changed
            assert (st["refreshes"], st["failed_refreshes"], st["excluded_pods"]) == (refreshes, failed, excluded), \
                (where, st)
            seen |= PH.names_of(tick.kept())
            pool = [p for p in pools[t] if p.Pod not in gone]
            want = rt.check_survivors(pool, probes_for(pools, t, seen), where)
            rt.check_picks(want, where)
            if rt.lists:
                rt.check_models(pool, where)
            if t and (tick.kind in ("qkv_boundary", "rename", "qkv_past", "qkv_most", "after_refusal")):
                assert st["delta_refreshes"] == delta, (where, st)
            delta = st["delta_refreshes"]
            last_ok = tick.published
        st = rt.s.stats()
        assert st["stale_retries"] == 0 and st["delta_refreshes"] >= 3, st
        assert publishes >= (4 if eject else 0), publishes
    finally:
        rt.close()


def pod(i, active):
    return PodMetrics(Pod(f"pod-{i}", f"address-{i}"), Metrics(ActiveModels={a: 1 for a in active},
                                                                WaitingQueueSize=0, KVCacheUsagePercent=0.1))


def refuse_then_return(P, swapped):
    """P equal pods.  Pod `swapped` lists {a, b}, the next pod lists c, no other pod lists b.  A
    refused tick (P + 1 pods) swaps b for c on `swapped`; the next tick is the first pool with that
    swap kept.  Every class must then be the oracle's, b's above all: no pod lists b any more."""
    other = (swapped + 1) % P
    first = [pod(i, ["a", "b"] if i == swapped else ["c"] if i == other else []) for i in range(P)]
    after = [pod(i, ["a", "c"] if i == swapped else ["c"] if i == other else []) for i in range(P)]
    prov = H.HostProvider(first)
    s = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=64, seed=3)
    sets = PH.survivor_sets(None)
    try:
        assert s.Filter("b", True)[:2] == (H.GRPC_OK, [f"pod-{swapped}"])
        prov.set_pods(after + [pod(P, [])])
        with pytest.raises(H.HostSchedulerError):
            s.Refresh()
        prov.set_pods(after)
        s.Refresh()
        st = s.stats()
        assert (st["refreshes"], st["failed_refreshes"]) == (2, 1), st
        want = sets(after, ["a", "b", "c", PH.NEVER_LOADED])
        assert want[("b", True)] == (N.LIG_OK, [p.Pod.Name for p in after])
        assert s.Filter("b", True)[:2] == (H.GRPC_OK, [p.Pod.Name for p in after])
        got = {k: s.Filter(*k)[:2] for k in want}
        assert got == {k: filter_result(*v) for k, v in want.items()}
    finally:
        s.close()
        prov.close()


def test_refused_refresh_leaves_no_stale_adapter_row():
    """Eight pods with max_pods = 8: after the refused nine-pod tick and back, Filter("b", critical)
    is all eight pods (none lists b), not the swapped pod 0."""
    refuse_then_return(8, 0)


@pytest.mark.parametrize("swapped", [0, 39, 35], ids=["first_pod", "last_pod", "ragged_last_word"])
def test_refused_refresh_leaves_no_stale_adapter_row_at(swapped):
    """The same on 40 pods (the last bitmap word holds pods 32..39) with the swap on the first pod,
    the last pod and a pod inside the ragged last word."""
    refuse_then_return(40, swapped)


def test_refresh_that_derives_under_concurrent_callers():
    """A refresh that derives (a full upload with ejected pods) evicts the published epoch while it
    derives the next one: calls that captured it get LIG_ERR_STALE_EPOCH and must wait for the
    publication instead of spending their attempts at once.  Two slices hold the same 40 pods; the
    second rotates the 3 ejected pods among their own positions and reverses the kept pods among
    theirs, so every tick is a full upload that derives, and an ejected pod is at the same index in
    either slice."""
    names = ("a", "b", "c")
    gone_at = [0, 17, 33]
    pods = [pod(i, names) for i in range(40)]
    for i, pm in enumerate(pods):                            # distinct metrics: every moved pod is dirty
        pm.Metrics.WaitingQueueSize = i % 4
        pm.Metrics.KVCacheUsagePercent = 0.01 * i
    kept_at = [i for i in range(40) if i not in gone_at]
    other = list(pods)
    for a, b in zip(gone_at, gone_at[1:] + gone_at[:1]):
        other[b] = pods[a]
    for a, b in zip(kept_at, kept_at[::-1]):
        other[b] = pods[a]
    slices = [pods, other]
    gone = {pods[i].Pod for i in gone_at}
    assert {other[i].Pod for i in gone_at} == gone
    sets = PH.survivor_sets(None)
    for s_ in slices:                                        # every class keeps a survivor
        for (name, crit), (rc, surv) in sets([p for p in s_ if p.Pod not in gone], list(names)).items():
            assert rc == N.LIG_OK and surv, (name, crit)
    models = [im(f"model-{n}", CRITICAL, [(n, 1)]) for n in names]
    prov = H.HostProvider(pods)
    s = H.HostScheduler(prov, max_pods=40, max_adapters=8, max_batch=256, batch_window_us=20, seed=5)
    ds = H.HostDataStore(models)
    errors, stop = [], [False]
    try:
        s.set_inference_models(ds)
        s.EjectPods([pods[i].Pod for i in gone_at])
        before = s.stats()
        ticks = [0]

        def refresher():
            while not stop[0] or ticks[0] < 200:
                ticks[0] += 1
                prov.set_pods(slices[ticks[0] % 2])
                s.Refresh()

        def caller():                                        # keeps the errors and ejected picks
            while not stop[0]:
                code, got, err = s.Schedule("m", "a", True)
                if code != H.GRPC_OK or got in gone:
                    errors.append(err or f"ejected pod {got}")
        threads = [threading.Thread(target=refresher), threading.Thread(target=caller)]
        for t in threads:
            t.start()
        try:
            res = {}
            workers = [threading.Thread(target=lambda: res.update(d=s.schedule_concurrent(16, 200, list(names),
                                                                                         [False, True, False]))),
                       threading.Thread(target=lambda: res.update(m=s.schedule_models_concurrent(
                           16, 200, [f"model-{n}" for n in names])))]
            for w in workers:
                w.start()
            for w in workers:
                w.join()
        finally:
            stop[0] = True
            for t in threads:
                t.join()
        st = s.stats()
        (dcodes, dpods), (mcodes, mpods, _) = res["d"], res["m"]
        info = (st["stale_retries"], errors[:1], int((dcodes != H.GRPC_OK).sum()), int((mcodes != H.GRPC_OK).sum()), st)
        assert (dcodes == H.GRPC_OK).all() and (mcodes == H.GRPC_OK).all() and not errors, info
        assert not set(gone_at) & (set(dpods.tolist()) | set(mpods.tolist())), info
        assert st["failed_refreshes"] == 0 and ticks[0] >= 200, info
        assert st["eject_publishes"] - before["eject_publishes"] == st["refreshes"] - before["refreshes"], info
        assert st["refreshes"] - before["refreshes"] == ticks[0] and st["ejected_pods"] == 3, info
    finally:
        stop[0] = True
        s.close()
        ds.close()
        prov.close()
