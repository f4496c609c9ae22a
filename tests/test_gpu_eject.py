"""Outlier ejection (lig_eject_pods) on the GPU, against the definition (eject_ref.py: every call as on
an epoch uploaded from the literally reduced snapshot, pod indices mapped back).  Every class through
lig_read_class for each class-table build (fast at C4, general staged and unstaged, caller trees staged
and unstaged, ejected pods in the last partial word, an empty pool); the results of the host, queue
and model-id picks, the doorbell, lig_filter_batch, the fallback calls, the four retry calls, the
in-batch feedback call and the chain calls with their loads; and the lifecycle: n = 0, threshold
rebuilds, deltas, full uploads, refusals and the scan's refusal.  Then both schedulers: EjectPods and
lifting across delta and full refreshes, with a model list and with concurrent callers.  Each
built-in-build case has a fixed seed, and the queue kernels run in every variant
test_gpu_kernel_variants.py selects."""
import threading
import time

import numpy as np
import pytest
import torch

import eject_ref as ER
import feedback_chain_retry_ref as CR
from test_gpu_filter_batch import StaticProvider, dev
from test_gpu_filter_tree import c4_tree, mkpods
from test_gpu_kernel_variants import VARIANTS, make_engine
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import CRITICAL, InferenceModel, InferenceModelSpec, Pod, TargetModel
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import pack_models, pack_pod_metrics

pytestmark = pytest.mark.gpu

SEED = 0xE1EC_7000_0000_0001
UNSTAGED_P = 13000          # too many pods for staged columns in every walk and build
GENERIC_P = 5000            # past the fast build's 4096 pods, staged general build


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=16384, max_adapters=1024, max_batch=1 << 16)
    yield e
    e.close()


_ep = [9000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


def hot_pods(snap, reqs, k, rng, thresholds=(0.8, 5, 50), nodes=None):
    """k pods the base picks (so ejecting them changes results) plus a few at random."""
    base = ER.schedule_batch(snap, [], reqs[:256], SEED, thresholds, nodes)
    hot = np.unique(base["pod_idx"][base["pod_idx"] >= 0])
    pick = set(rng.choice(hot, size=min(k, len(hot)), replace=False).tolist())
    pick |= set(rng.choice(snap.P, size=min(3, snap.P), replace=False).tolist())
    return sorted(pick)


def upload_and_eject(eng, snap, ejected):
    base, ep = next_epoch(), next_epoch()
    eng.upload_snapshot(base, snap)
    eng.eject_pods(ep, base, ejected)
    return base, ep


def check_classes(eng, ep, snap, ejected, thresholds=(0.8, 5, 50), nodes=None, adapters=None):
    adapters = range(snap.A + 1) if adapters is None else adapters
    for crit in (False, True):
        for a in adapters:
            st, n, lst = eng.read_class(ep, crit, a, snap.P)
            want = ER.klass(snap, ejected, crit, a, thresholds, nodes)
            assert (st, lst.tolist()) == want, (crit, a)
            assert n == len(want[1])


@pytest.mark.parametrize("shape", ["fast_c4", "generic_staged", "generic_unstaged", "last_word"])
def test_every_class_of_the_built_in_builds(eng, shape):
    rng = np.random.default_rng({"fast_c4": 1, "generic_staged": 2, "generic_unstaged": 3, "last_word": 4}[shape])
    P, A = {"fast_c4": (WL.CONFIGS["C4"]["P"], WL.CONFIGS["C4"]["A"]), "generic_staged": (GENERIC_P, 40),
            "generic_unstaged": (UNSTAGED_P, 24), "last_word": (70, 6)}[shape]
    snap = WL.make_snapshot(P, A, seed=3).packed
    reqs = WL.make_requests(512, A, seed=4)
    ejected = hot_pods(snap, reqs, 10, rng)
    if shape == "last_word":
        ejected = sorted(set(ejected) | {64, 66, 69})
    _, ep = upload_and_eject(eng, snap, ejected)
    adapters = None if A <= 64 else list(range(0, A, max(1, A // 40))) + [A]
    check_classes(eng, ep, snap, ejected, adapters=adapters)
    got = eng.schedule_batch(ep, SEED, reqs)
    assert got.tobytes() == ER.schedule_batch(snap, ejected, reqs, SEED).tobytes()


@pytest.mark.parametrize("P", [300, UNSTAGED_P])
def test_every_class_of_a_caller_tree(eng, P):
    rng = np.random.default_rng(P)
    snap = WL.make_snapshot(P, 12, seed=5).packed
    reqs = WL.make_requests(256, 12, seed=6)
    nodes = c4_tree().flatten()
    ejected = hot_pods(snap, reqs, 8, rng, nodes=nodes)
    eng.set_filter_tree(nodes)
    try:
        base, ep = next_epoch(), next_epoch()
        eng.upload_snapshot(base, snap)
        eng.eject_pods(ep, base, ejected)
    finally:
        eng.set_filter_tree(None)
    check_classes(eng, ep, snap, ejected, nodes=nodes)
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == \
        ER.schedule_batch(snap, ejected, reqs, SEED, nodes=nodes).tobytes()
    ex = np.full((len(reqs), 3), -1, dtype=np.int16)      # four distinct rows: the reference rebuilds a pool per row
    ex[:, 0] = ejected[0]
    ex[:, 1] = rng.integers(0, P, size=4)[np.arange(len(reqs)) % 4]
    assert eng.schedule_batch_excluding(ep, SEED, reqs, ex).tobytes() == \
        ER.retry_batch(snap, ejected, reqs, ex, SEED, nodes=nodes).tobytes()
    with pytest.raises(N.LigError):                  # the scan refuses caller trees and ejected pools
        eng.schedule_scan(ep, SEED, reqs[:4], False)


@pytest.mark.parametrize("P", [40, GENERIC_P])
def test_ejecting_every_pod(eng, P):
    snap = WL.make_snapshot(P, 5, seed=7).packed
    reqs = WL.make_requests(64, 5, seed=8)
    _, ep = upload_and_eject(eng, snap, list(range(P)))
    got = eng.schedule_batch(ep, SEED, reqs)
    assert (got["status"] == N.LIG_DROP).all() and (got["pod_idx"] == -1).all()
    assert got.tobytes() == ER.schedule_batch(snap, list(range(P)), reqs, SEED).tobytes()
    rows = np.full((64, 2), -1, dtype=np.int16)
    assert eng.schedule_batch_excluding(ep, SEED, reqs, rows).tobytes() == got.tobytes()


@pytest.mark.parametrize("tree", ["no_pods_leaf", "c4"])
@pytest.mark.parametrize("P", [40, UNSTAGED_P])
def test_ejecting_every_pod_under_a_caller_tree(eng, tree, P):
    """The tree build and the retry walks start from an empty pool: the tree's answer for an empty
    slice (a predicate leaf keeps no pod: LIG_NO_PODS_LEFT)."""
    nodes = {"no_pods_leaf": [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 50, 0.0)],
             "c4": c4_tree().flatten()}[tree]
    snap = WL.make_snapshot(P, 5, seed=9).packed
    reqs = WL.make_requests(64, 5, seed=10)
    every = list(range(P))
    eng.set_filter_tree(nodes)
    try:
        base, ep = next_epoch(), next_epoch()
        eng.upload_snapshot(base, snap)
        eng.eject_pods(ep, base, every)
    finally:
        eng.set_filter_tree(None)
    check_classes(eng, ep, snap, every, nodes=nodes)
    want = ER.schedule_batch(snap, every, reqs, SEED, nodes=nodes)
    assert (want["pod_idx"] == -1).all()
    if tree == "no_pods_leaf":
        assert (want["status"] == N.LIG_NO_PODS_LEFT).all()
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == want.tobytes()
    rows = np.full((64, 2), -1, dtype=np.int16)
    rows[:, 0] = 3
    assert eng.schedule_batch_excluding(ep, SEED, reqs, rows).tobytes() == \
        ER.retry_batch(snap, every, reqs, rows, SEED, nodes=nodes).tobytes()
    p, fb = eng.schedule_batch_excluding_fallbacks(ep, SEED, reqs, rows, 3)
    wp, wf = ER.retry_fallback_batch(snap, every, reqs, rows, SEED, 3, nodes=nodes)
    assert p.tobytes() == wp.tobytes() and np.array_equal(fb, wf)


@pytest.fixture(scope="module")
def c4():
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=11).packed
    reqs = WL.make_requests(4096, c["A"], seed=12)
    ejected = hot_pods(snap, reqs, 16, np.random.default_rng(13))
    return snap, reqs, ejected


def test_every_table_reading_call(eng, c4):
    snap, reqs, ejected = c4
    _, ep = upload_and_eject(eng, snap, ejected)
    want = ER.schedule_batch(snap, ejected, reqs, SEED)
    assert (want["status"] == N.LIG_OK).sum() > 1000
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == want.tobytes()
    # the persistent queue kernel, three batches
    d_in = dev(reqs)
    outs = [torch.zeros(len(reqs) * 8, dtype=torch.uint8, device="cuda") for _ in range(3)]
    eng.schedule_batches_device(ep, SEED, [d_in.data_ptr()] * 3, len(reqs), [o.data_ptr() for o in outs])
    torch.cuda.synchronize()
    for b, o in enumerate(outs):
        assert o.cpu().numpy().tobytes() == ER.schedule_batch(snap, ejected, reqs, SEED + b).tobytes()
    # the doorbell
    eng.stream_open()
    try:
        assert eng.stream_submit(ep, SEED, reqs[:1000]).tobytes() == want[:1000].tobytes()
    finally:
        eng.stream_close()
    # lig_filter_batch: picks and every request's list
    picks, offsets, pods = eng.filter_batch(ep, SEED, reqs[:500])
    assert picks.tobytes() == want[:500].tobytes()
    for i in range(0, 500, 7):
        r = reqs[i]
        a = int(r["adapter_id"])
        st, lst = ER.klass(snap, ejected, bool(r["flags"] & 1), a if 0 <= a < snap.A else snap.A)
        got = pods[offsets[i]:offsets[i + 1]].tolist()
        assert got == (lst if st == N.LIG_OK else [])
    # fallbacks
    p, rows = eng.schedule_batch_fallbacks(ep, SEED, reqs, 5)
    wp, wr = ER.fallback_batch(snap, ejected, reqs, SEED, 5)
    assert p.tobytes() == wp.tobytes() and np.array_equal(rows, wr)
    # the four retry calls: rows name ejected pods, kept pods, the pick, padding and out-of-range entries.
    # The reference rebuilds a pool per distinct row and a class table per (row, class): 8 rows, 4 adapters.
    rng = np.random.default_rng(17)
    rreqs = np.ascontiguousarray(reqs[:1024].copy())
    rreqs["adapter_id"] = np.array([0, 1, 2, snap.A])[np.arange(1024) % 4]
    pattern = np.full((8, 4), -1, dtype=np.int16)
    pattern[:, 0] = rng.choice(ejected, size=8)
    pattern[:, 1] = rng.integers(0, snap.P, size=8)
    pattern[:, 2] = ER.schedule_batch(snap, ejected, rreqs[:8], SEED)["pod_idx"]
    pattern[::3, 3] = snap.P + 3
    ex_r = pattern[(np.arange(1024) // 4) % 8]
    wret = ER.retry_batch(snap, ejected, rreqs, ex_r, SEED)
    assert eng.schedule_batch_excluding(ep, SEED, rreqs, ex_r).tobytes() == wret.tobytes()
    p, rows = eng.schedule_batch_excluding_fallbacks(ep, SEED, rreqs, ex_r, 4)
    wp, wr = ER.retry_fallback_batch(snap, ejected, rreqs, ex_r, SEED, 4)
    assert p.tobytes() == wp.tobytes() and np.array_equal(rows, wr)
    # the chain: plain, fallback, retry and retry-with-rows calls, loads of every pod
    eng.feedback_chain_reset()
    calls, ks, got_outs, got_rows = [], [], [], []
    loads = np.zeros(snap.P, dtype=np.int32)
    a, b = reqs[:700], reqs[700:1500]
    c, d = np.ascontiguousarray(rreqs[:512]), np.ascontiguousarray(rreqs[512:1024])
    ea, eb = np.ascontiguousarray(ex_r[:512]), np.ascontiguousarray(ex_r[512:1024])
    got_outs.append(eng.schedule_batch_feedback_chain(ep, SEED, a, 256, loads))
    calls.append((a, SEED)); ks.append(0)
    o, r = eng.schedule_batch_feedback_chain_fallbacks(ep, SEED + 1, b, 3, 256, loads)
    got_outs.append(o); got_rows.append((1, r)); calls.append((b, SEED + 1)); ks.append(3)
    got_outs.append(eng.schedule_batch_feedback_chain_excluding(ep, SEED + 2, c, ea, 256, loads))
    calls.append(CR.retry_call(c, ea, SEED + 2)); ks.append(0)
    o, r = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED + 3, d, eb, 2, 256, loads)
    got_outs.append(o); got_rows.append((3, r)); calls.append(CR.retry_call(d, eb, SEED + 3)); ks.append(2)
    wouts, wrows, wloads = ER.chain(snap, ejected, calls, 256, ks)
    for g, w in zip(got_outs, wouts):
        assert g.tobytes() == w.tobytes()
    for i, r in got_rows:
        assert np.array_equal(r, wrows[i])
    assert np.array_equal(loads.astype(np.int64), wloads) and loads[ejected].sum() == 0
    # the in-batch feedback call: a one-call chain of windows of 512
    d_out = torch.zeros(len(reqs) * 8, dtype=torch.uint8, device="cuda")
    d_hist = torch.zeros(snap.P, dtype=torch.int32, device="cuda")
    eng.schedule_batch_feedback_device(ep, SEED, d_in.data_ptr(), len(reqs), d_out.data_ptr(), 512, 0,
                                       d_hist.data_ptr())
    torch.cuda.synchronize()
    wouts, _, wloads = ER.chain(snap, ejected, [(reqs, SEED)], 512)
    assert d_out.cpu().numpy().tobytes() == wouts[0].tobytes()
    assert np.array_equal(d_hist.cpu().numpy().astype(np.int64), wloads)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_queue_kernel_variants(variant, c4, monkeypatch):
    snap, reqs, ejected = c4
    e = make_engine(VARIANTS[variant], monkeypatch, max_pods=snap.P, max_adapters=snap.A, max_batch=1 << 12)
    try:
        _, ep = upload_and_eject(e, snap, ejected)
        d_in = dev(reqs)
        outs = [torch.zeros(len(reqs) * 8, dtype=torch.uint8, device="cuda") for _ in range(2)]
        e.schedule_batches_device(ep, SEED, [d_in.data_ptr()] * 2, len(reqs), [o.data_ptr() for o in outs])
        torch.cuda.synchronize()
        for b, o in enumerate(outs):
            assert o.cpu().numpy().tobytes() == ER.schedule_batch(snap, ejected, reqs, SEED + b).tobytes()
    finally:
        e.close()


def test_model_id_calls(eng, c4):
    """Model ids resolve without reading pods: each model-id call equals the descriptor call on the
    descriptors the device resolved."""
    snap, _, ejected = c4
    models = WL.make_models(snap.A)
    ids = WL.make_model_requests(3000, snap.A, seed=21)
    _, ep = upload_and_eject(eng, snap, ejected)
    with pytest.raises(N.LigError):                  # no model table until lig_upload_models
        eng.schedule_models_batch(ep, SEED, ids)
    eng.upload_models(ep, pack_models(models, snap))
    dreqs, res = eng.resolve_models(ep, SEED, ids)
    present = res["status"] != N.LIG_NO_MODEL
    want = ER.schedule_batch(snap, ejected, np.ascontiguousarray(dreqs[present]), SEED)
    got = eng.schedule_models_batch(ep, SEED, ids)
    assert np.array_equal(got["pod_idx"][present], want["pod_idx"])
    assert np.array_equal(got["status"][present], want["status"])
    assert not set(ejected) & set(got["pod_idx"][got["pod_idx"] >= 0].tolist())
    p, rows = eng.schedule_models_batch_fallbacks(ep, SEED, ids, 3)
    _, wr = ER.fallback_batch(snap, ejected, np.ascontiguousarray(dreqs[present]), SEED, 3)
    assert np.array_equal(rows[present], wr)
    # the model-id chain, on ids that all resolve
    ids = np.where(present, ids, ids[present][0]).astype(np.uint32)
    dreqs, _ = eng.resolve_models(ep, SEED, ids)
    eng.feedback_chain_reset()
    loads = np.zeros(snap.P, dtype=np.int32)
    got = eng.schedule_models_batch_feedback_chain(ep, SEED, ids, 128, loads=loads)
    wouts, _, wloads = ER.chain(snap, ejected, [(dreqs, SEED)], 128)
    assert np.array_equal(got["pod_idx"], wouts[0]["pod_idx"]) and np.array_equal(got["status"], wouts[0]["status"])
    assert np.array_equal(loads.astype(np.int64), wloads) and loads[ejected].sum() == 0


def test_lifecycle_and_refusals(eng):
    snap = WL.make_snapshot(600, 10, seed=31).packed
    reqs = WL.make_requests(1024, 10, seed=32)
    ejected = hot_pods(snap, reqs, 6, np.random.default_rng(33))
    base, ep = upload_and_eject(eng, snap, ejected)
    b_out = eng.schedule_batch(base, SEED, reqs)
    e_out = eng.schedule_batch(ep, SEED, reqs)
    assert e_out.tobytes() == ER.schedule_batch(snap, ejected, reqs, SEED).tobytes()
    assert b_out.tobytes() == ER.schedule_batch(snap, [], reqs, SEED).tobytes()
    # every refusal leaves both resident epochs answering as before
    bad = [(ep, ep, [1]), (next_epoch(), 123456789, [1]), (next_epoch(), base, [-1]), (next_epoch(), base, [600]),
           (next_epoch(), base, [3, 3]), (next_epoch(), base, list(range(601)))]
    for new, b, idx in bad:
        with pytest.raises(N.LigError):
            eng.eject_pods(new, b, idx)
    lib = N.load()
    assert lib.lig_eject_pods(eng._ctx, next_epoch(), base, None, 2) == N.LIG_ERR_INVALID
    assert lib.lig_eject_pods(eng._ctx, next_epoch(), base, None, -1) == N.LIG_ERR_INVALID
    assert lib.lig_eject_pods(eng._ctx, next_epoch(), 123456789, None, 0) == N.LIG_ERR_STALE_EPOCH
    # base is the older slot: the new epoch would overwrite it
    assert lib.lig_eject_pods(eng._ctx, next_epoch(), base, None, 0) == N.LIG_ERR_INVALID
    assert eng.schedule_batch(base, SEED, reqs).tobytes() == b_out.tobytes()
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == e_out.tobytes()
    # the scan refuses an ejected epoch
    with pytest.raises(N.LigError):
        eng.schedule_scan(ep, SEED, reqs[:4], False)
    # a threshold rebuild keeps the set
    try:
        eng.set_thresholds(0.5, 3, 20)
        assert eng.schedule_batch(ep, SEED, reqs).tobytes() == \
            ER.schedule_batch(snap, ejected, reqs, SEED, (0.5, 3, 20)).tobytes()
    finally:
        eng.set_thresholds()
    # a delta from the ejected epoch keeps the set
    d = next_epoch()
    dirty = np.array([ejected[0], 5], dtype=np.int32)
    kv = np.array([0.01, 0.02]); q = np.array([0, 0], dtype=np.int32)
    na = np.array([0, 0], dtype=np.uint16); ma = np.array([4, 4], dtype=np.uint16)
    eng.update_snapshot(d, ep, dirty, kv, q, na, ma, np.array([0, 0, 0], dtype=np.int32), np.zeros(0, np.int32))
    snap_d = ER.RR.reduce_snapshot(snap, np.arange(snap.P))       # a copy of the columns
    snap_d.kv[dirty] = kv
    snap_d.q[dirty] = q
    snap_d.n_active[dirty] = na
    snap_d.max_active[dirty] = ma
    for p in dirty:
        snap_d.bitmap[:, p >> 5] &= np.uint32(~(1 << (int(p) & 31)) & 0xFFFFFFFF)
    assert eng.schedule_batch(d, SEED, reqs).tobytes() == ER.schedule_batch(snap_d, ejected, reqs, SEED).tobytes()
    # n = 0 from the ejected epoch: every pod back, base's results byte for byte
    back = next_epoch()
    eng.eject_pods(back, d, [])
    assert eng.schedule_batch(back, SEED, reqs).tobytes() == ER.schedule_batch(snap_d, [], reqs, SEED).tobytes()
    # a full upload clears the set
    full = next_epoch()
    eng.upload_snapshot(full, snap)
    assert eng.schedule_batch(full, SEED, reqs).tobytes() == b_out.tobytes()
    assert eng.schedule_scan(full, SEED, reqs, False)[0].tobytes() == b_out.tobytes()


# ---- both schedulers: EjectPods and lifting across refreshes ------------------------------------------
def sched_pods(qs=None):
    qs = qs or [0, 3, 1, 7, 0, 2, 60, 4, 0, 1, 5, 0, 2, 9, 0, 3]
    n = len(qs)
    kvs = [0.1 + 0.05 * (i % 7) for i in range(n)]
    acts = [["a"] if i % 3 == 0 else ["b"] if i % 3 == 1 else ["a", "c"] for i in range(n)]
    return mkpods(qs, kvs, [2 + i % 3 for i in range(n)], acts)


def want_names(pods, gone, name, critical):
    """Survivor names of a class on the snapshot of `pods` without the pods `gone` (by value)."""
    snap = pack_pod_metrics(pods)
    idx = [p for p, pm in enumerate(pods) if pm.Pod in gone]
    st, lst = ER.klass(snap, idx, critical, snap.adapter_id(name))
    return st, [snap.pods[p].Name for p in lst]


def models_for_pods():
    return [InferenceModel(m, InferenceModelSpec(ModelName=m, Criticality=CRITICAL, TargetModels=[TargetModel(t, 1)]))
            for m, t in (("model-a", "a"), ("model-b", "b"), ("model-c", "c"))]


def test_python_scheduler_eject_and_lift():
    pods = sched_pods()
    prov = StaticProvider(pods)
    sched = S.NewScheduler(prov, max_pods=64, max_adapters=8, max_batch=256, seed=3)
    try:
        sched.SetInferenceModels(models_for_pods())
        reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "c", "zz") for c in (False, True)]
        picked = {pod for pod, err in sched.ScheduleBatch(reqs * 8) if pod is not None}
        gone = set(sorted(picked, key=lambda p: p.Name)[:3])
        sched.EjectPods(list(gone) + [Pod("not-a-pod", "nowhere")])

        def check(pods_now):
            for r in reqs:
                got, err = sched.Filter(r)
                st, names = want_names(pods_now, gone, r.ResolvedTargetModel, r.Critical)
                assert [p.Name for p in got] == (names if st == N.LIG_OK else []), r
            assert not gone & {p for p, _ in sched.ScheduleBatch(reqs * 16) if p is not None}
            for _ in range(32):
                for m in ("model-a", "model-b", "model-c"):
                    _, pod = sched.ScheduleModel(m)
                    assert pod not in gone
        check(pods)
        prov.pods = pods[::-1]                   # a refresh with every pod at a new index
        sched.Refresh()
        check(pods[::-1])
        sched.EjectPods([])                      # lifted: every pod back
        gone = set()
        check(pods[::-1])
    finally:
        sched.close()


def test_host_scheduler_eject_and_lift_across_refreshes():
    pods = sched_pods()
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=9)
    ds = H.HostDataStore(models_for_pods())
    try:
        hs.Refresh()
        hs.set_inference_models(ds)
        gone = {pods[0].Pod, pods[4].Pod, pods[11].Pod}

        def check(pods_now):
            for m in ("a", "b", "c", "zz"):
                for crit in (False, True):
                    code, names, _ = hs.Filter(m, crit)
                    st, want = want_names(pods_now, gone, m, crit)
                    assert names == (want if st == N.LIG_OK else []), (m, crit)
                    for _ in range(8):
                        code, pod, _ = hs.Schedule("m", m, crit)
                        assert pod not in gone
            for m in ("model-a", "model-b", "model-c"):
                for _ in range(16):
                    code, _, pod, _ = hs.ScheduleModelOnDevice(m)
                    assert code == H.GRPC_OK and pod not in gone

        before = hs.stats()
        hs.EjectPods(sorted(gone, key=lambda p: p.Name))
        st = hs.stats()
        assert st["ejected_pods"] == 3 and st["eject_publishes"] == before["eject_publishes"] + 1
        check(pods)
        # a delta tick (one pod's queue changes) inherits the set: no new derived epoch
        moved = sched_pods([0, 3, 1, 7, 0, 2, 60, 4, 0, 1, 5, 0, 2, 9, 0, 30])
        prov.set_pods(moved)
        hs.Refresh()
        st2 = hs.stats()
        assert st2["delta_refreshes"] == st["delta_refreshes"] + 1 and st2["eject_publishes"] == st["eject_publishes"]
        assert st2["ejected_pods"] == 3
        check(moved)
        # a full upload (every pod at a new index) derives once more
        prov.set_pods(moved[::-1])
        hs.Refresh()
        st3 = hs.stats()
        assert st3["eject_publishes"] == st2["eject_publishes"] + 1 and st3["ejected_pods"] == 3
        check(moved[::-1])
        # lifted
        hs.EjectPods([])
        gone = set()
        assert hs.stats()["ejected_pods"] == 0
        check(moved[::-1])
    finally:
        hs.close()
        ds.close()


def test_host_scheduler_eject_with_concurrent_callers():
    """Every Schedule call that starts after EjectPods returns avoids the ejected pods, while other
    threads keep scheduling through the ejection and the lifting."""
    pods = sched_pods()
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=11, batch_window_us=20)
    hs.Refresh()
    code, first, _ = hs.Schedule("m", "a", True)
    gone = {first}
    ejected = threading.Event()
    stop = threading.Event()
    bad, done = [], [0]

    def caller(k):
        m = ("a", "b", "c")[k % 3]
        while not stop.is_set():
            after = ejected.is_set()
            code, pod, _ = hs.Schedule("m", m, bool(k & 1))
            done[0] += 1
            if after and pod in gone:
                bad.append(pod)
    threads = [threading.Thread(target=caller, args=(k,)) for k in range(6)]
    try:
        for t in threads:
            t.start()
        time.sleep(0.05)
        hs.EjectPods(list(gone))
        ejected.set()
        time.sleep(0.2)
        n = done[0]
        stop.set()
        for t in threads:
            t.join()
        assert not bad and n > 100
    finally:
        stop.set()
        hs.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="a device group needs two GPUs")
def test_host_scheduler_over_several_devices_refuses():
    prov = H.HostProvider(sched_pods())
    hs = H.HostScheduler(prov, devices=[0, 1], max_pods=64, max_adapters=8)
    try:
        with pytest.raises(H.HostSchedulerError, match="several devices"):
            hs.EjectPods([Pod("pod-0", "address-0")])
    finally:
        hs.close()
