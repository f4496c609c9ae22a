"""Model-id retries through the schedulers: Scheduler::ScheduleModelRetry[WithFallbacks] in the C++ runtime
(through HostScheduler) and scheduling.Scheduler.ScheduleModel[Batch]Retry[WithFallbacks].  A model request,
then a refresh that adds adapters (every adapter id moves), then its retry at the target it drew: the pick
and the row are checked against the definition (models_retry_ref.py) on the new epoch with the request's
device key.  Also the host-answered errors (which take no key), the feedback opt-ins, the counters and
concurrent callers."""
import threading

import numpy as np
import pytest

import models_retry_ref as MR
from helpers import golden_to_podmetrics
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import CRITICAL, InferenceModel, InferenceModelSpec, Pod, TargetModel
from llm_instance_gateway_b200.packer import pack_models, pack_pod_metrics
from test_gpu_filter_batch import StaticProvider

pytestmark = pytest.mark.gpu

GRPC_INVALID_ARGUMENT = 3
SEED = 0x7E7_12


def im(name, crit=None, targets=()):
    return InferenceModel(name, InferenceModelSpec(ModelName=name, Criticality=crit,
                                                   TargetModels=[TargetModel(n, w) for n, w in targets]))


def models_for(A):
    return WL.make_models(A) + [
        im("three-way", CRITICAL, [(WL.adapter_name(0), 25), (WL.adapter_name(1), 55), (WL.adapter_name(2), 50)]),
        im("zero", None, [(WL.adapter_name(0), 0)]),
        im("late", CRITICAL, [(WL.adapter_name(A + 3), 1), (WL.adapter_name(1), 1)])]


def pms(P, A, seed):
    return [golden_to_podmetrics(r) for r in WL.make_snapshot(P, A, seed=seed).pod_records()]


def expect(pods, models, name, resolved, tried, seed, key, k=0):
    """(pod, row) the definition gives for one retry over the provider slice `pods`."""
    snap = pack_pod_metrics(pods)
    pm = pack_models(models, snap)
    m = pm.model_ids[name]
    tgt = pm.target_names[m]
    t = 255 if not tgt else tgt.index(resolved)
    row = [p for p, x in enumerate(pods) if x.Pod in set(tried)] or [-1]
    picks, rows = MR.retry_fallback_batch(snap, pm, np.array([m], np.uint32), np.array([t], np.uint8),
                                          np.array([row], np.int16), seed, max(k, 1), key)
    pk = picks[0]
    if pk["status"] != N.LIG_OK:
        return None, []
    return snap.pods[int(pk["pod_idx"])], [snap.pods[int(x)] for x in rows[0][:k] if x >= 0]


def test_cpp_runtime_after_a_refresh_that_adds_adapters():
    models = models_for(6)
    first_pods, later_pods = pms(48, 6, 1), pms(48, 10, 2)       # the refresh loads four more adapters
    prov = H.HostProvider(first_pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=64, max_batch=512, seed=SEED)
    ds = H.HostDataStore(models)
    try:
        hs.set_inference_models(ds)
        firsts = []
        for name in ("three-way", "model-2", "base-model", "split-1", "late"):
            code, resolved, pod, _ = hs.ScheduleModelOnDevice(name)
            firsts.append((name, resolved, pod))
        key = len(firsts)                                          # device keys 0 .. 4 taken
        prov.set_pods(later_pods)
        hs.Refresh()
        before = hs.stats()
        for name, resolved, pod in firsts:
            tried = [pod] if pod is not None else [Pod("ghost", "x")]
            code, got, _ = hs.ScheduleModelRetry(name, resolved, tried)
            want, _ = expect(later_pods, models, name, resolved, tried, SEED, key)
            key += 1
            assert (code == H.GRPC_OK) == (want is not None) and got == want, name
            code, names, _ = hs.ScheduleModelRetryWithFallbacks(name, resolved, tried, 3)
            want, row = expect(later_pods, models, name, resolved, tried, SEED, key, 3)
            key += 1
            if want is not None:
                assert code == H.GRPC_OK and names == [p.Name for p in [want] + row], name
        # answered on the host, with no key taken
        code, _, err = hs.ScheduleModelRetry("nope", "nope", [])
        assert code == H.GRPC_UNKNOWN and err == "error finding a model object in InferenceModel for input nope"
        code, _, err = hs.ScheduleModelRetry("zero", WL.adapter_name(0), [])
        assert code == H.GRPC_UNKNOWN and err == "error getting target model name for model zero"
        code, _, err = hs.ScheduleModelRetry("three-way", WL.adapter_name(5), [])
        assert code == GRPC_INVALID_ARGUMENT and "not a target model" in err
        code, _, _ = hs.ScheduleModelRetry("base-model", "something-else", [])
        assert code == GRPC_INVALID_ARGUMENT
        code, _, _ = hs.ScheduleModelRetry("model-0", WL.adapter_name(0), [Pod("p", "a")] * 33)
        assert code == GRPC_INVALID_ARGUMENT
        code, _, _ = hs.ScheduleModelRetryWithFallbacks("model-0", WL.adapter_name(0), [], 9)
        assert code == GRPC_INVALID_ARGUMENT
        # the model-id sequence continues where the retries left it
        code, resolved, pod, _ = hs.ScheduleModelOnDevice("model-3")
        want, _ = expect(later_pods, models, "model-3", resolved, [], SEED, key)
        assert pod == want
        after = hs.stats()
        assert after["retry_scheduled"] - before["retry_scheduled"] == 2 * len(firsts) + 4   # argument refusals: 0
        assert after["model_batches"] - before["model_batches"] == 2 * len(firsts) + 1
    finally:
        ds.close()
        hs.close()
        prov.close()


def test_cpp_runtime_feedback_opt_ins_and_concurrent_callers():
    models = models_for(6)
    pods = pms(40, 6, 3)
    prov = H.HostProvider(pods)
    ds = H.HostDataStore(models)
    try:
        for retries, fallbacks in ((False, False), (True, False), (True, True)):
            hs = H.HostScheduler(prov, max_pods=64, max_adapters=64, max_batch=512, seed=SEED,
                                 load_feedback_window=4, feedback_retries=retries, feedback_fallbacks=fallbacks)
            try:
                hs.set_inference_models(ds)
                code, _, _ = hs.ScheduleModelRetry("model-1", WL.adapter_name(1), [])
                assert (code == H.GRPC_OK) == retries
                code, names, _ = hs.ScheduleModelRetryWithFallbacks("model-1", WL.adapter_name(1), [], 2)
                assert (code == H.GRPC_OK) == (retries and fallbacks)
                if retries:
                    assert hs.stats()["feedback_windows"] == 0
                    for _ in range(3):
                        hs.ScheduleModelRetry("model-1", WL.adapter_name(1), [])
                    assert hs.stats()["feedback_windows"] >= 1
            finally:
                hs.close()
        hs = H.HostScheduler(prov, max_pods=64, max_adapters=64, max_batch=512, seed=SEED)
        try:
            hs.set_inference_models(ds)
            out, lock = [], threading.Lock()
            tried = [pods[0].Pod, pods[1].Pod]

            def caller(t):
                for i in range(40):
                    name = ("model-0", "three-way", "base-model")[(t + i) % 3]
                    res = {"model-0": WL.adapter_name(0), "three-way": WL.adapter_name(1), "base-model": name}[name]
                    code, pod, _ = hs.ScheduleModelRetry(name, res, tried)
                    with lock:
                        out.append((code, pod))

            th = [threading.Thread(target=caller, args=(t,)) for t in range(8)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert len(out) == 320 and hs.stats()["retry_scheduled"] == 320
            assert all(pod not in tried for code, pod in out if code == H.GRPC_OK)
            assert any(code == H.GRPC_OK for code, _ in out)
        finally:
            hs.close()
    finally:
        ds.close()
        prov.close()


def test_python_scheduler_after_a_refresh_and_opt_ins():
    models = models_for(6)
    first_pods, later_pods = pms(48, 6, 4), pms(48, 10, 5)
    prov = StaticProvider(first_pods)
    sched = S.NewScheduler(prov, max_pods=64, max_adapters=64, max_batch=512, seed=9)
    try:
        sched.SetInferenceModels(models)
        names = ["three-way", "model-2", "base-model", "split-0", "late"]
        firsts = [(res, pod) for pod, res, _ in sched.ScheduleModelBatch(names)]
        key = sched._model_index
        prov.pods = later_pods
        sched.Refresh()
        for name, (resolved, pod) in zip(names, firsts):
            want, _ = expect(later_pods, models, name, resolved, [pod], sched._seed, key)
            key += 1
            if want is None:
                with pytest.raises(S.StatusError):
                    sched.ScheduleModelRetry(name, resolved, [pod])
            else:
                assert sched.ScheduleModelRetry(name, resolved, [pod]) == want
        got = sched.ScheduleModelBatchRetryWithFallbacks(names, [r for r, _ in firsts], [[p] for _, p in firsts], 4)
        for name, (resolved, pod), (pods, res, err) in zip(names, firsts, got):
            want, row = expect(later_pods, models, name, resolved, [pod], sched._seed, key, 4)
            key += 1
            assert res == resolved and (pods == [want] + row if want is not None else err is not None)
        # host answers take no key
        out = sched.ScheduleModelBatchRetry(["nope", "zero", "three-way", "model-1"],
                                            ["nope", WL.adapter_name(0), "not-a-target", WL.adapter_name(1)],
                                            [[], [], [], []])
        assert out[0][2].code == "Unknown" and out[1][2].code == "Unknown" and out[2][2].code == "InvalidArgument"
        want, _ = expect(later_pods, models, "model-1", WL.adapter_name(1), [], sched._seed, key)
        assert out[3][0] == want and sched._model_index == key + 1
    finally:
        sched.close()
    for retries, fallbacks in ((False, False), (True, False), (True, True)):
        chain = S.NewScheduler(StaticProvider(later_pods), load_feedback_window=3, max_pods=64, max_adapters=64,
                               feedback_retries=retries, feedback_fallbacks=fallbacks, seed=9)
        try:
            chain.SetInferenceModels(models)
            if retries:
                assert len(chain.ScheduleModelBatchRetry(["model-1"], [WL.adapter_name(1)], [[]])) == 1
            else:
                with pytest.raises(ValueError, match="load_feedback_window"):
                    chain.ScheduleModelRetry("model-1", WL.adapter_name(1), [])
            if retries and fallbacks:
                assert len(chain.ScheduleModelBatchRetryWithFallbacks(["model-1"], [WL.adapter_name(1)], [[]], 2)) == 1
            else:
                with pytest.raises(ValueError, match="load_feedback_window"):
                    chain.ScheduleModelRetryWithFallbacks("model-1", WL.adapter_name(1), [], 2)
        finally:
            chain.close()
