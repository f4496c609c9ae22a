"""Model requests resolved on the device by the schedulers (Scheduler::SetInferenceModels and
Scheduler::ScheduleModel(model, ...) in the C++ runtime, scheduling.Scheduler.SetInferenceModels /
ScheduleModelBatch / ScheduleModel in Python).

* The k-th request of a scheduler that reaches the device is the oracle's model path
  (lig_oracle_schedule_models_batch) with the scheduler's seed and first_index = k: pod, resolved
  name and status, for the plain launch and the doorbell, which agree byte for byte.  Unknown and
  zero-weight models are answered on the host and take no key.  Caller trees are checked against
  Engine.schedule_models_batch on a ctx with the same tree.
* With load_feedback_window, interleaved descriptor and model calls equal the chain's sequential
  definition (models_feedback_chain_ref), and the window count is exact.
* The new calls do not move the key sequences of Schedule and ScheduleModel(datastore, ...).
* The model table travels with every epoch: SetInferenceModels publishes one, a target starts to
  match once a pod loads it (full and delta refreshes), and a refused list leaves the previous one.
* Concurrent callers with the refresher running, and the Python scheduler.
"""
import threading

import numpy as np
import pytest

import models_feedback_chain_ref as MC
from helpers import golden_to_podmetrics
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import (CRITICAL, InferenceModel, InferenceModelSpec, Metrics, Pod,
                                               PodMetrics, TargetModel)
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import REQ_DTYPE, pack_models, pack_pod_metrics
from oracle import binding as B
from test_gpu_feedback_chain import splitmix_keys
from test_gpu_snapshot_mutation import drop_and_no_pods_trees, random_state

pytestmark = pytest.mark.gpu

PREFIX = "failed to find target pod: "
ERR0 = "failed to apply filter, resulted 0 pods, this should never happen: "
DROP_MSG = (PREFIX + ERR0 + "rpc error: code = ResourceExhausted desc = dropping request due to limited backend "
            "resources")


def im(name, crit=None, targets=()):
    return InferenceModel(name, InferenceModelSpec(ModelName=name, Criticality=crit,
                                                   TargetModels=[TargetModel(n, w) for n, w in targets]))


def model_list(A):
    """make_models plus a three-way split, a zero-weight model and a model on an unloaded name."""
    return WL.make_models(A) + [
        im("three-way", CRITICAL, [(WL.adapter_name(0), 25), (WL.adapter_name(1), 55), (WL.adapter_name(2), 50)]),
        im("zero", None, [(WL.adapter_name(0), 0), (WL.adapter_name(1), 0)]),
        im("plain-unlisted", CRITICAL)]


def by_id(models):
    """The C++ runtime's model ids for a list pushed through ligh_datastore: sorted by ModelName."""
    return sorted(models, key=lambda m: m.Spec.ModelName)


def records_to_pms(records):
    return [golden_to_podmetrics(r) for r in records]


def pod_index(pod):
    return -1 if pod is None else int(pod.Name.split("-")[1])


class Rt:
    """A C++ runtime with a model list, and the oracle's view of the same pool and list."""

    def __init__(self, records, models, seed=1234, **kw):
        self.prov = H.HostProvider(records_to_pms(records))
        opts = dict(max_pods=max(64, len(records)), max_adapters=64, max_batch=4096, batch_window_us=20)
        opts.update(kw)
        self.s = H.HostScheduler(self.prov, seed=seed, **opts)
        self.ds = H.HostDataStore(models)
        self.s.set_inference_models(self.ds)
        self.models = by_id(models)
        self.ids = {m.Spec.ModelName: i for i, m in enumerate(self.models)}
        self.seed = seed
        self.set_records(records)

    def set_records(self, records):
        self.records = records
        self.pool = B.Pool(records)
        self.mo = B.Models(WL.model_records(self.models))

    def close(self):
        self.ds.close()
        self.s.close()
        self.prov.close()

    def expect(self, name, k):
        """(code, resolved, pod index, message) the oracle gives for `name` as device request k."""
        m = self.models[self.ids[name]]
        mp = self.mo.schedule_batch(self.pool, np.array([self.ids[name]], dtype=np.uint32), self.seed, k)[0]
        t, st = int(mp["target_idx"]), int(mp["status"])
        resolved = name if t == 255 else m.Spec.TargetModels[t].Name
        if st == N.LIG_OK:
            return 0, resolved, int(mp["pod_idx"]), ""
        if st == N.LIG_DROP:
            return H.GRPC_RESOURCE_EXHAUSTED, resolved, -1, DROP_MSG
        assert st == N.LIG_EMPTY, st
        return H.GRPC_UNKNOWN, resolved, -1, PREFIX + ERR0 + "%!w(<nil>)"


def run_sequence(rt, names):
    """Sends names one by one; returns [(code, resolved, pod index, err)] and checks every request
    against the oracle with its device key."""
    out, k = [], 0
    for name in names:
        code, resolved, pod, err = rt.s.ScheduleModelOnDevice(name)
        got = (code, resolved, pod_index(pod), err if code else "")
        if name not in rt.ids:
            assert got == (H.GRPC_UNKNOWN, "", -1, f"error finding a model object in InferenceModel for input {name}")
        elif name == "zero":
            assert got == (H.GRPC_UNKNOWN, "", -1, "error getting target model name for model zero")
        else:
            assert got == rt.expect(name, k), (name, k)
            k += 1
        out.append(got)
    return out, k


@pytest.mark.parametrize("doorbell", [False, True])
def test_hermetic_case(golden, doorbell):
    case = golden["TestHandleRequestBody"][0]
    tm = case["models"]["my-model"]["target_models"][0]
    rt = Rt(case["pods"], [im("my-model", None, [(tm["name"], tm["weight"])])], use_doorbell=doorbell)
    try:
        code, resolved, pod, _ = rt.s.ScheduleModelOnDevice("my-model")
        assert (code, resolved, pod.Address) == (H.GRPC_OK, "my-model-v1", "address-1")
        assert rt.expect("my-model", 0)[:3] == (0, "my-model-v1", 1)
    finally:
        rt.close()


def sequence_names(models, n, seed):
    rng = np.random.default_rng(seed)
    names = [m.Spec.ModelName for m in models] + ["nope"]
    seq = [names[i] for i in rng.integers(0, len(names), n)]
    seq[:6] = ["three-way", "nope", "three-way", "zero", "base-model", "plain-unlisted"]
    return seq


def test_one_caller_equals_oracle_plain_and_doorbell():
    state = random_state(64, 12, seed=101)
    models = model_list(12)
    seq = sequence_names(models, 300, seed=102) + ["three-way"] * 60
    results = []
    for doorbell in (False, True):
        rt = Rt(state.records(), models, seed=103, use_doorbell=doorbell)
        try:
            got, k = run_sequence(rt, seq)
            st = rt.s.stats()
            assert st["model_scheduled"] == len(seq) and st["model_batches"] == k
            assert st["scheduled"] == 0 and st["batches"] == 0                   # the descriptor lane is untouched
        finally:
            rt.close()
        results.append(got)
    assert results[0] == results[1]
    seen = {r[1] for n, r in zip(seq, results[0]) if n == "three-way"}
    assert seen == {WL.adapter_name(0), WL.adapter_name(1), WL.adapter_name(2)}
    assert any(r == (0, "base-model", r[2], "") for r in results[0])              # passthrough


@pytest.mark.parametrize("doorbell", [False, True])
def test_shed_pool(doorbell):
    records = [dict(name=f"pod-{i}", address=f"address-{i}", waiting_queue_size=10, kv_cache_usage_percent=0.9,
                    max_active_models=0, active_models=[WL.adapter_name(i % 3)]) for i in range(8)]
    models = [im("shed", None, [(WL.adapter_name(0), 1), (WL.adapter_name(1), 1)]), im("crit", CRITICAL)]
    rt = Rt(records, models, seed=7, use_doorbell=doorbell)
    try:
        got, k = run_sequence(rt, ["shed", "crit", "nope", "shed"])
        assert got[0][0] == H.GRPC_RESOURCE_EXHAUSTED and got[0][3] == DROP_MSG
        assert got[1][0] == H.GRPC_OK and k == 3
    finally:
        rt.close()


@pytest.mark.parametrize("tree", [0, 1])
@pytest.mark.parametrize("doorbell", [False, True])
def test_caller_trees_equal_engine(tree, doorbell):
    state = random_state(96, 12, seed=111 + tree)
    nodes = drop_and_no_pods_trees()[tree]
    models = model_list(12)
    seq = sequence_names(models, 250, seed=112)
    rt = Rt(state.records(), models, seed=113, use_doorbell=doorbell, filter=nodes)
    try:
        got = [rt.s.ScheduleModelOnDevice(n) for n in seq]
    finally:
        rt.close()
    snap = pack_pod_metrics(records_to_pms(state.records()))
    pm = pack_models(by_id(models), snap)
    sent = [n for n in seq if n in rt.ids and n != "zero"]
    with Engine(0, max_pods=96, max_adapters=64, max_batch=4096) as e:
        e.set_filter_tree(nodes)
        e.upload_snapshot(1, snap)
        e.upload_models(1, pm)
        want = e.schedule_models_batch(1, 113, np.array([rt.ids[n] for n in sent], dtype=np.uint32), first_index=0)
    statuses = set()
    k = 0
    for n, (code, resolved, pod, err) in zip(seq, got):
        if n not in rt.ids or n == "zero":
            assert code == H.GRPC_UNKNOWN and not err.startswith(PREFIX)
            continue
        w = want[k]
        k += 1
        st, t = int(w["status"]), int(w["target_idx"])
        statuses.add(st)
        assert resolved == (n if t == 255 else pm.target_names[rt.ids[n]][t])
        if st == N.LIG_OK:
            assert code == H.GRPC_OK and pod_index(pod) == int(w["pod_idx"]), (n, k)
        elif st == N.LIG_DROP:
            assert (code, err) == (H.GRPC_RESOURCE_EXHAUSTED, DROP_MSG)
        elif st == N.LIG_NO_PODS_LEFT:
            assert (code, err) == (H.GRPC_UNKNOWN, PREFIX + ERR0 + "no pods left")
        else:
            assert (code, err) == (H.GRPC_UNKNOWN, PREFIX + ERR0 + "%!w(<nil>)")
    assert N.LIG_OK in statuses and (N.LIG_DROP if tree == 0 else N.LIG_NO_PODS_LEFT) in statuses


@pytest.mark.parametrize("W", [1, 8, 64])
def test_feedback_chain_interleaved(W):
    state = random_state(64, 12, seed=121)
    state.q[:] = np.random.default_rng(122).integers(0, 4, state.P)
    records = state.records()
    names = state.names()
    models = model_list(12)
    rng = np.random.default_rng(123)
    seq = sequence_names(models, 240, seed=124)
    kinds = rng.integers(0, 2, len(seq))
    crit = rng.integers(0, 2, len(seq)).astype(bool)
    seed = 125
    rt = Rt(records, models, seed=seed, load_feedback_window=W)
    got = []
    try:
        for kind, n, c in zip(kinds, seq, crit):
            if kind == 0:                                     # a descriptor request for an adapter
                a = names[len(got) % len(names)]
                code, pod, _ = rt.s.Schedule(a, a, bool(c))
                got.append(("d", a, bool(c), pod_index(pod) if code == 0 else -1))
            else:
                code, resolved, pod, _ = rt.s.ScheduleModelOnDevice(n)
                got.append(("m", n, resolved, pod_index(pod) if code == 0 else -1, code))
        st = rt.s.stats()
    finally:
        rt.close()
    dkeys = iter(splitmix_keys(seed, len(got)))
    calls, k = [], 0
    packed = state.packed()
    for g in got:
        if g[0] == "d":
            r = np.zeros(1, dtype=REQ_DTYPE)
            r[0] = (names.index(g[1]), N.LIG_REQ_CRITICAL if g[2] else 0, next(dkeys))
            calls.append((r, seed))
        elif g[1] in rt.ids and g[1] != "zero":
            calls.append(MC.model_call(rt.mo, packed.adapter_id, np.array([rt.ids[g[1]]], dtype=np.uint32), seed, k))
            k += 1
    want, _ = MC.schedule_chain(packed.P, packed.A, packed.kv, state.q, packed.n_active, packed.max_active,
                                packed.bitmap, calls, W)
    it = iter(want)
    for g in got:
        if g[0] == "m" and (g[1] not in rt.ids or g[1] == "zero"):
            assert g[4] == H.GRPC_UNKNOWN
            continue
        w = next(it)[0]
        if g[0] == "d":
            assert g[3] == int(w["pod_idx"]), g
        else:
            t = int(w["target_idx"])
            m = rt.models[rt.ids[g[1]]]
            assert g[2] == (g[1] if t == 255 else m.Spec.TargetModels[t].Name), g
            assert g[3] == (int(w["pod_idx"]) if int(w["status"]) == N.LIG_OK else -1), g
    assert st["feedback_windows"] == len(calls) // W and st["feedback_restarts"] == 0
    assert st["model_batches"] == k and st["batches"] == sum(1 for g in got if g[0] == "d")


def test_new_calls_leave_the_other_key_sequences_alone():
    state = random_state(64, 12, seed=131)
    models = model_list(12)
    names = state.names()
    rng = np.random.default_rng(132)
    descs = [(names[i], bool(c)) for i, c in zip(rng.integers(0, len(names), 120), rng.integers(0, 2, 120))]
    mseq = sequence_names(models, 120, seed=133)

    def run(interleave):
        rt = Rt(state.records(), models, seed=134)
        out = []
        try:
            for i, (a, c) in enumerate(descs):
                if interleave:
                    rt.s.ScheduleModelOnDevice(mseq[i])
                code, pod, _ = rt.s.Schedule(a, a, c)
                out.append((code, pod_index(pod)))
                if interleave:
                    rt.s.ScheduleModelOnDevice(mseq[-1 - i])
                code, resolved, pod, _ = rt.s.ScheduleModel(rt.ds, mseq[i])
                out.append((code, resolved, pod_index(pod)))
        finally:
            rt.close()
        return out
    assert run(False) == run(True)


def pm_for(q, active, kv=0.1, ma=0):
    return [PodMetrics(Pod(f"pod-{i}", f"address-{i}"),
                       Metrics(WaitingQueueSize=q, KVCacheUsagePercent=kv, MaxActiveModels=ma,
                               ActiveModels={a: 1 for a in act}))
            for i, act in enumerate(active)]


def test_table_lifecycle():
    """MaxActiveModels = 0: the affinity filter decides, so a critical request for a target that one
    pod holds always lands there, and for a target nobody holds lands anywhere."""
    P = 40
    base = [["foo"] for _ in range(P)]
    prov = H.HostProvider(pm_for(0, base))
    s = H.HostScheduler(prov, max_pods=64, max_adapters=64, max_batch=1024, seed=9)
    ds = H.HostDataStore([im("late", CRITICAL, [("late-v1", 10)])])
    try:
        assert s.ScheduleModelOnDevice("late")[0] == H.GRPC_UNKNOWN        # no list yet: an empty datastore
        r0 = s.stats()["refreshes"]
        s.set_inference_models(ds)
        assert s.stats()["refreshes"] == r0 + 1
        picks = {pod_index(s.ScheduleModelOnDevice("late")[2]) for _ in range(40)}
        assert len(picks) > 1                                              # no pod lists late-v1
        # full refresh: a new adapter name enters the table
        active = [list(a) for a in base]
        active[17] = ["foo", "late-v1"]
        prov.set_pods(pm_for(0, active))
        d0 = s.stats()["delta_refreshes"]
        s.Refresh()
        assert s.stats()["delta_refreshes"] == d0
        for _ in range(20):
            code, resolved, pod, _ = s.ScheduleModelOnDevice("late")
            assert (code, resolved, pod_index(pod)) == (0, "late-v1", 17)
        # delta refreshes: the name stays interned while pod 17 drops it and pod 5 loads it
        active[17] = ["foo"]
        prov.set_pods(pm_for(0, active))
        s.Refresh()
        assert len({pod_index(s.ScheduleModelOnDevice("late")[2]) for _ in range(40)}) > 1
        active[5] = ["foo", "late-v1"]
        prov.set_pods(pm_for(0, active))
        s.Refresh()
        assert s.stats()["delta_refreshes"] == d0 + 2
        for _ in range(20):
            assert pod_index(s.ScheduleModelOnDevice("late")[2]) == 5
        # refused lists leave the previous one in force
        r1 = s.stats()["refreshes"]
        for bad, msg in ((im("wide", None, [(f"t{i}", 1) for i in range(256)]), "256 target models"),
                         (im("heavy", None, [("a", 2**30), ("b", 2**30)]), "sum to 2147483648")):
            ds2 = H.HostDataStore([im("late", CRITICAL, [("late-v1", 10)]), bad, im("new")])
            with pytest.raises(H.HostSchedulerError, match=msg) as ei:
                s.set_inference_models(ds2)
            assert bad.Spec.ModelName in str(ei.value)
            ds2.close()
        assert s.stats()["refreshes"] == r1
        assert s.ScheduleModelOnDevice("new")[0] == H.GRPC_UNKNOWN
        assert pod_index(s.ScheduleModelOnDevice("late")[2]) == 5
        # a new list applies from its epoch on
        ds.set_model(im("new"))
        s.set_inference_models(ds)
        code, resolved, _, _ = s.ScheduleModelOnDevice("new")
        assert (code, resolved) == (0, "new") and s.stats()["refreshes"] == r1 + 1
    finally:
        ds.close()
        s.close()
        prov.close()


def test_concurrent_callers_with_refresher():
    state = random_state(300, 24, seed=141)
    records = state.records()
    models = model_list(24)
    rt = Rt(records, models, seed=142, max_pods=512, flush_size=256, batch_window_us=200, refresh_interval_ms=2)
    names = [m.Spec.ModelName for m in models] + ["nope"]
    adapters = state.names()
    try:
        dres = {}
        th = threading.Thread(target=lambda: dres.update(
            r=rt.s.schedule_concurrent(8, 200, adapters, [True] * len(adapters))))
        th.start()
        codes, pods, targets = rt.s.schedule_models_concurrent(16, 200, names)
        th.join()
        st = rt.s.stats()
    finally:
        rt.close()
    assert st["refreshes"] > 2 and st["model_scheduled"] == len(codes)
    assert 0 < st["model_batches"] < st["model_scheduled"]
    pool = B.Pool(records)
    byname = {m.Spec.ModelName: m for m in models}
    cache = {}
    for i in range(len(codes)):
        n = names[i % len(names)]
        m = byname.get(n)
        if m is None or n == "zero":
            assert codes[i] == H.GRPC_UNKNOWN and pods[i] == -1
            continue
        t = int(targets[i])
        resolved = n if t == 255 else m.Spec.TargetModels[t].Name
        key = (resolved, m.Spec.Criticality == CRITICAL)
        if key not in cache:
            cache[key] = pool.filter(*key)
        rc, survivors = cache[key]
        if rc == B.LIGO_OK:
            assert codes[i] == H.GRPC_OK and pods[i] in survivors, (i, n, resolved)
        elif rc == B.LIGO_DROP:
            assert codes[i] == H.GRPC_RESOURCE_EXHAUSTED
        else:
            assert codes[i] == H.GRPC_UNKNOWN
    dcodes, dpods = dres["r"]
    for i in range(len(dcodes)):
        rc, survivors = pool.filter(adapters[i % len(adapters)], True)
        if rc == B.LIGO_OK:
            assert dcodes[i] == H.GRPC_OK and dpods[i] in survivors, i
        else:
            assert dcodes[i] == (H.GRPC_RESOURCE_EXHAUSTED if rc == B.LIGO_DROP else H.GRPC_UNKNOWN)


def test_python_scheduler():
    from llm_instance_gateway_b200 import scheduling as S
    state = random_state(80, 12, seed=151)
    pms = records_to_pms(state.records())

    class Provider:
        def AllPodMetrics(self):
            return pms

        def Version(self):
            return 1

    models = model_list(12)
    seq = sequence_names(models, 200, seed=152)
    sched = S.NewScheduler(Provider(), seed=153, max_pods=128, max_adapters=64)
    try:
        with pytest.raises(S.StatusError, match="for input three-way"):
            sched.ScheduleModel("three-way")                               # no list yet
        sched.SetInferenceModels(models)
        ep = sched._epoch
        got = sched.ScheduleModelBatch(seq[:120]) + sched.ScheduleModelBatch(seq[120:])
        with pytest.raises(ValueError, match="wide"):
            sched.SetInferenceModels([im("wide", None, [(f"t{i}", 1) for i in range(256)])])
        assert sched._epoch == ep
        with pytest.raises(S.StatusError) as ei:
            sched.ScheduleModel("zero")
        assert ei.value.code == "Unknown" and str(ei.value) == "error getting target model name for model zero"
    finally:
        sched.close()
    snap = pack_pod_metrics(pms)
    pm = pack_models(models, snap)
    sent = [n for n in seq if n in pm.model_ids and pm.present[pm.model_ids[n]]]
    with Engine(0, max_pods=128, max_adapters=64, max_batch=4096) as e:
        e.upload_snapshot(1, snap)
        e.upload_models(1, pm)
        want = e.schedule_models_batch(1, sched._seed, np.array([pm.model_ids[n] for n in sent], dtype=np.uint32))
    k = 0
    for n, (pod, resolved, err) in zip(seq, got):
        if n not in pm.model_ids or n == "zero":
            assert pod is None and err.code == "Unknown"
            continue
        w = want[k]
        k += 1
        t = int(w["target_idx"])
        assert resolved == (n if t == 255 else pm.target_names[pm.model_ids[n]][t])
        if int(w["status"]) == N.LIG_OK:
            assert err is None and pod == snap.pods[int(w["pod_idx"])]
        else:
            assert pod is None and str(err).startswith(PREFIX)
    assert k == len(sent)


@pytest.mark.parametrize("W", [1, 16])
def test_python_scheduler_chain(W):
    from llm_instance_gateway_b200 import scheduling as S
    state = random_state(64, 12, seed=161)
    state.q[:] = np.random.default_rng(162).integers(0, 4, state.P)
    records = state.records()
    pms = records_to_pms(records)

    class Provider:
        def AllPodMetrics(self):
            return pms

        def Version(self):
            return 1

    models = model_list(12)
    seq = sequence_names(models, 150, seed=163)
    sched = S.NewScheduler(Provider(), seed=164, max_pods=64, max_adapters=64, load_feedback_window=W)
    try:
        sched.SetInferenceModels(models)
        got = []
        for a, b in ((0, 1), (1, 40), (40, 41), (41, 150)):
            got += sched.ScheduleModelBatch(seq[a:b])
        seed = sched._seed
    finally:
        sched.close()
    packed = state.packed()
    pm = pack_models(models, packed)
    mo = B.Models(WL.model_records(models))
    calls, k = [], 0
    for a, b in ((0, 1), (1, 40), (40, 41), (41, 150)):
        ids = [pm.model_ids[n] for n in seq[a:b] if n in pm.model_ids and pm.present[pm.model_ids[n]]]
        if ids:
            calls.append(MC.model_call(mo, packed.adapter_id, np.array(ids, dtype=np.uint32), seed, k))
            k += len(ids)
    want, _ = MC.schedule_chain(packed.P, packed.A, packed.kv, state.q, packed.n_active, packed.max_active,
                                packed.bitmap, calls, W)
    flat = np.concatenate(want) if want else []
    sent = [(n, g) for n, g in zip(seq, got) if n in pm.model_ids and n != "zero"]
    assert len(sent) == len(flat)
    for (n, (pod, resolved, err)), w in zip(sent, flat):
        t = int(w["target_idx"])
        assert resolved == (n if t == 255 else pm.target_names[pm.model_ids[n]][t])
        assert pod_index(pod) == (int(w["pod_idx"]) if int(w["status"]) == N.LIG_OK else -1)


def test_python_scheduler_hermetic_case(golden):
    from llm_instance_gateway_b200 import scheduling as S
    case = golden["TestHandleRequestBody"][0]
    pms = [golden_to_podmetrics(p) for p in case["pods"]]

    class Provider:
        def AllPodMetrics(self):
            return pms

    tm = case["models"]["my-model"]["target_models"][0]
    sched = S.NewScheduler(Provider(), seed=5, max_pods=64, max_adapters=64)
    try:
        sched.SetInferenceModels([im("my-model", None, [(tm["name"], tm["weight"])])])
        resolved, pod = sched.ScheduleModel("my-model")
        assert (resolved, pod.Address) == ("my-model-v1", "address-1")
    finally:
        sched.close()


def test_multi_device_runtime_refuses_model_lists():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    prov = H.HostProvider(pm_for(0, [["foo"]] * 4))
    s = H.HostScheduler(prov, max_pods=8, max_adapters=8, max_batch=64, devices=[0, 1])
    ds = H.HostDataStore([im("m")])
    try:
        with pytest.raises(H.HostSchedulerError, match="single device"):
            s.set_inference_models(ds)
        assert s.ScheduleModelOnDevice("m")[0] == H.GRPC_UNKNOWN
    finally:
        ds.close()
        s.close()
        prov.close()


def test_handler_replay_takes_the_model_branch(golden):
    """The hermetic case through the handler surface when the scheduler holds the InferenceModels
    (the branch patch 0004 adds to HandleRequestBody): same headers and rewritten body, 429 for a
    shed request, the reference's error for an unknown model.  The datastore is empty, so a
    response can only come from the scheduler's own model table."""
    from llm_instance_gateway_b200 import scheduling as S
    from llm_instance_gateway_b200.backend import FakeDataStore
    from llm_instance_gateway_b200.handlers import NewServer, RequestContext, go_json_marshal
    case = golden["TestHandleRequestBody"][0]
    pms = [golden_to_podmetrics(p) for p in case["pods"]]

    class Provider:
        def AllPodMetrics(self):
            return pms

    def request(model):
        return {"request_body": {"body": go_json_marshal({"model": model, "prompt": "hello", "max_tokens": 100,
                                                          "temperature": 0})}}
    models = [im(name, None, [(t["name"], t["weight"]) for t in m["target_models"]])
              for name, m in case["models"].items()] + [im("sheddable")]
    sched = S.NewScheduler(Provider(), seed=5, max_pods=64, max_adapters=64)
    try:
        assert not sched.ResolvesModels()
        sched.SetInferenceModels(models)
        assert sched.ResolvesModels()
        server = NewServer(Provider(), sched, "target-pod", FakeDataStore({}))
        ctx = RequestContext()
        res = server.Process(ctx, request(case["request_model"]))
        want_headers = [{"header": {"key": h["key"], "raw_value": h["raw_value"].encode()}} for h in case["want_headers"]]
        assert res == {"request_body": {"response": {"header_mutation": {"set_headers": want_headers},
                                                     "body_mutation": {"body": case["want_body"].encode()}}}}
        assert ctx.TargetPod == Pod("pod-1", "address-1") and ctx.Model == "my-model"
        with pytest.raises(S.StatusError) as ei:
            server.Process(RequestContext(), request("nope"))
        assert str(ei.value) == ("failed to handle request: error finding a model object in InferenceModel for "
                                 "input nope")
        pms[:] = [PodMetrics(Pod(f"pod-{i}", f"address-{i}"), Metrics(WaitingQueueSize=10, KVCacheUsagePercent=0.9))
                  for i in range(3)]
        assert server.Process(RequestContext(), request("sheddable")) == {"immediate_response": {"status": {"code": 429}}}
    finally:
        sched.close()


def test_python_duplicate_names_last_wins():
    """Of two models with one ModelName the later is used, and only it is checked: an earlier entry
    the device could not take does not refuse the list."""
    from llm_instance_gateway_b200 import scheduling as S
    state = random_state(32, 6, seed=171)
    pms = records_to_pms(state.records())

    class Provider:
        def AllPodMetrics(self):
            return pms

        def Version(self):
            return 1

    sched = S.NewScheduler(Provider(), seed=172, max_pods=64, max_adapters=64)
    try:
        sched.SetInferenceModels([im("m", None, [(f"t{i}", 1) for i in range(256)]), im("other"),
                                  im("m", CRITICAL, [(WL.adapter_name(1), 7)])])
        assert [m.Spec.ModelName for m in sched._models] == ["m", "other"]
        for _ in range(10):
            resolved, _ = sched.ScheduleModel("m")
            assert resolved == WL.adapter_name(1)
        with pytest.raises(ValueError, match="model m has 256"):
            sched.SetInferenceModels([im("m", CRITICAL, [(WL.adapter_name(1), 7)]),
                                      im("m", None, [(f"t{i}", 1) for i in range(256)])])
    finally:
        sched.close()


def flip_records(P, phase):
    """Two pools whose adapter names intern to different ids: in phase 0 pod j holds fa-j and t-j
    (t-j gets id 2j + 1), in phase 1 pod j holds fb-j and pod 20 + j holds t-j (t-j gets id 12 + j).
    Together they hold 36 names, more than max_adapters = 32, so every switch re-interns from scratch.
    MaxActiveModels = 0 and empty queues: a critical request for t-j lands on the one pod holding it."""
    recs = []
    for i in range(P):
        if phase == 0:
            act = [f"fa-{i}", f"t-{i}"] if i < 12 else []
        else:
            act = [f"fb-{i}"] if i < 12 else ([f"t-{i - 20}"] if 20 <= i < 32 else [])
        recs.append(dict(name=f"pod-{i}", address=f"address-{i}", waiting_queue_size=0, kv_cache_usage_percent=0.1,
                         max_active_models=0, active_models=act))
    return recs


@pytest.mark.parametrize("doorbell", [False, True])
def test_epochs_change_under_concurrent_callers(doorbell):
    """Pods and adapter ids change while 16 callers send model requests: every pick must come from the
    epoch the request's table was packed for.  A table interned against another epoch's adapter ids
    would send t-j to a filler adapter's pod."""
    P = 40
    models = [im(f"m-{j}", CRITICAL, [(f"t-{j}", 1)]) for j in range(12)]
    prov = H.HostProvider(records_to_pms(flip_records(P, 0)))
    s = H.HostScheduler(prov, max_pods=64, max_adapters=32, max_batch=4096, seed=181, flush_size=64,
                        batch_window_us=100, refresh_interval_ms=1, use_doorbell=doorbell)
    ds = H.HostDataStore(models)
    stop = threading.Event()

    def flipper():
        phase = 0
        while not stop.is_set():
            phase ^= 1
            prov.set_pods(records_to_pms(flip_records(P, phase)))
            s.Refresh()

    try:
        s.set_inference_models(ds)
        th = threading.Thread(target=flipper)
        th.start()
        try:
            names = [f"m-{j}" for j in range(12)] + ["nope"]
            codes, pods, targets = s.schedule_models_concurrent(16, 300, names)
        finally:
            stop.set()
            th.join()
        st = s.stats()
    finally:
        ds.close()
        s.close()
        prov.close()
    assert st["refreshes"] > 20 and st["failed_refreshes"] == 0, st
    assert 0 < st["model_batches"] < st["model_scheduled"] == len(codes)
    seen = set()
    for i in range(len(codes)):
        n = names[i % len(names)]
        if n == "nope":
            assert codes[i] == H.GRPC_UNKNOWN
            continue
        j = int(n.split("-")[1])
        assert codes[i] == H.GRPC_OK and targets[i] == 0, (i, n)
        assert pods[i] in (j, 20 + j), (i, n, pods[i])
        seen.add(pods[i] == j)
    assert seen == {True, False}                   # both epochs served requests
