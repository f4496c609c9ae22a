"""Session affinity (lig_upload_pod_keys, lig_schedule_[models_]batch_affinity[_device]) on the GPU: `out`
and the rows byte for byte against the definition (affinity_ref.py) built from lig_filter_batch's lists, for
descriptors and model ids, pageable, page-locked and device buffers and n_fallbacks 0, 1 and 8, on the
bench pools, caller trees whose lists reach P = 32768, lists across the per-thread / per-warp boundary,
compact-pool overflow and ejected epochs; agreement with the plain calls; stability under pod reordering,
ejection, several ctxs and split batches; the refusals; and the Python and C++ schedulers."""
import numpy as np
import pytest
import torch

import affinity_ref as AR
from test_gpu_filter_batch import Pinned, StaticProvider, dev, im
from test_gpu_filter_tree import mkpods
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Pod
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_columns, pack_models, \
    pack_pod_metrics

pytestmark = pytest.mark.gpu

K = N.LIG_MAX_FALLBACKS
NS = (0, 1, 8)
KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]
LORA_ONLY = [N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0)]


def random_keys(R, seed):
    return np.random.default_rng(seed).integers(0, 1 << 64, size=R, dtype=np.uint64)


def expected(eng, ep, data, pod_keys, keys=None, pm=None):
    """(out, rows (R, K)) by the definition from lig_filter_batch's lists; the plain call's picks."""
    models = data.dtype == np.uint32
    if models:
        reqs, resolved, target = AR.affinity_resolve(pm, data, keys)
    else:
        reqs = data
    plain, offsets, pods = eng.filter_batch(ep, 0, reqs)
    assert plain.tobytes() == eng.schedule_batch(ep, 0, reqs).tobytes()
    ok = plain["status"] == N.LIG_OK
    if models:
        ok &= resolved
    pick, rows = AR.affinity_rows(reqs["rand_key"], ok, offsets, pods, pod_keys, K)
    if models:
        out = AR.as_mpicks(plain, resolved, target, pick)
    else:
        out = plain.copy()
        out["pod_idx"] = np.where(ok, pick, -1)
    # the pick and the row are distinct members of the request's survivor list
    for i in np.flatnonzero(ok)[:: max(1, int(ok.sum()) // 500)]:
        ranked = [int(pick[i])] + [int(x) for x in rows[i] if x >= 0]
        lst = set(pods[offsets[i]:offsets[i + 1]].tolist())
        assert len(set(ranked)) == len(ranked) and set(ranked) <= lst
    return out, rows


def run_device(eng, ep, data, n, keys=None):
    R = len(data)
    models = data.dtype == np.uint32
    d_in = dev(data)
    d_keys = dev(np.ascontiguousarray(keys, dtype=np.uint64)) if models else None
    d_out = torch.full((R * (4 if models else 8),), 0xAB, dtype=torch.uint8, device="cuda")
    d_rows = torch.full((max(R * n, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
    rp = d_rows.data_ptr() if n else 0
    if models:
        eng.schedule_models_batch_affinity_device(ep, d_in.data_ptr(), d_keys.data_ptr(), R, d_out.data_ptr(), n, rp)
    else:
        eng.schedule_batch_affinity_device(ep, d_in.data_ptr(), R, d_out.data_ptr(), n, rp)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().view(MPICK_DTYPE if models else PICK_DTYPE)
    return out, d_rows.cpu().numpy()[: R * n].reshape(R, n)


def run_pinned(eng, ep, data, n, keys=None):
    R = len(data)
    models = data.dtype == np.uint32
    odt = MPICK_DTYPE if models else PICK_DTYPE
    bufs = [Pinned(R, data.dtype), Pinned(R, odt), Pinned(max(R * n, 1), np.int16), Pinned(R, np.uint64)]
    try:
        b_in, b_out, b_rows, b_keys = bufs
        b_in.a[:] = data
        b_out.a.view(np.uint8)[:] = 0xAB
        if models:
            b_keys.a[:] = keys
            eng.schedule_models_batch_affinity_ptr(ep, b_in.ptr, b_keys.ptr, R, b_out.ptr, n, b_rows.ptr if n else 0)
        else:
            eng.schedule_batch_affinity_ptr(ep, b_in.ptr, R, b_out.ptr, n, b_rows.ptr if n else 0)
        return b_out.a.copy(), b_rows.a[: R * n].copy().reshape(R, n)
    finally:
        for b in bufs:
            b.free()


def check(eng, ep, data, pod_keys, keys=None, pm=None, ns=NS, forms=("pageable", "pinned", "device")):
    want, rows = expected(eng, ep, data, pod_keys, keys, pm)
    models = data.dtype == np.uint32
    for n in ns:
        for form in forms:
            if form == "pageable":
                out, got = (eng.schedule_models_batch_affinity(ep, data, keys, n) if models
                            else eng.schedule_batch_affinity(ep, data, n))
            elif form == "pinned":
                out, got = run_pinned(eng, ep, data, n, keys)
            else:
                out, got = run_device(eng, ep, data, n, keys)
            assert out.tobytes() == want.tobytes(), (form, n)
            assert np.array_equal(got, rows[:, :n]), (form, n)
    return want, rows


def upload(eng, ep, packed, tree=None, models=None, seed=0):
    eng.set_filter_tree(tree)
    try:
        eng.upload_snapshot(ep, packed)
    finally:
        eng.set_filter_tree(None)
    pod_keys = np.array([S.pod_key(p) for p in packed.pods], dtype=np.uint64)
    eng.upload_pod_keys(ep, pod_keys)
    pm = None
    if models is not None:
        pm = pack_models(models, packed)
        eng.upload_models(ep, pm)
    return pod_keys, pm


# ---- parity -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg,tree", [("C1", None), ("C1", "keep_all"), ("C4", None), ("C4", "keep_all")])
def test_parity_at_the_bench_pools(cfg, tree):
    c = WL.CONFIGS[cfg]
    e = Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=1 << 16)
    try:
        snap = WL.make_snapshot(c["P"], c["A"], seed=5)
        pod_keys, pm = upload(e, 1, snap.packed, KEEP_ALL if tree else None, WL.make_models(c["A"]))
        R = 2048 if (tree and cfg == "C4") else min(c["R"], 1 << 16)
        reqs = WL.make_requests(R, c["A"], seed=6)
        want, rows = check(e, 1, reqs, pod_keys)
        assert (want["status"] == N.LIG_OK).mean() > 0.3
        ids = WL.make_model_requests(R, c["A"], seed=7)
        check(e, 1, ids, pod_keys, random_keys(R, 8), pm)
    finally:
        e.close()


def test_predicate_tree_lists_reach_32768_pods():
    P = 32768
    e = Engine(0, max_pods=P, max_adapters=1, max_batch=4096)
    try:
        packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64), np.zeros(P, np.int64),
                              np.zeros((1, P // 32), np.uint32))
        pod_keys, _ = upload(e, 1, packed, KEEP_ALL)
        reqs = np.zeros(256, dtype=REQ_DTYPE)
        reqs["adapter_id"] = np.arange(256) % 2
        reqs["rand_key"] = random_keys(256, 9)
        want, _ = check(e, 1, reqs, pod_keys)
        assert (want["status"] == N.LIG_OK).all() and (want["n_survivors"] == P).all()
    finally:
        e.close()


@pytest.mark.parametrize("P", [31, 32, 33, 4096])
def test_lists_across_the_warp_boundary(P):
    e = Engine(0, max_pods=max(P, 64), max_adapters=1, max_batch=1 << 14)
    try:
        packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64), np.zeros(P, np.int64),
                              np.zeros((0, (P + 31) // 32), np.uint32))
        pod_keys, _ = upload(e, 1, packed, KEEP_ALL)
        R = 1024 if P == 4096 else 4096
        reqs = np.zeros(R, dtype=REQ_DTYPE)
        reqs["rand_key"] = random_keys(R, P)
        want, _ = check(e, 1, reqs, pod_keys)
        assert (want["n_survivors"] == P).all()
    finally:
        e.close()


def test_long_and_short_lists_in_one_warp():
    """A LoRA-affinity tree: adapter 0 on every pod (long), 1 on 5 pods (short), 2 on 40 pods (long), 3
    on none (no pods left), interleaved so every warp mixes per-thread and per-warp requests."""
    P, A = 100, 3
    W = (P + 31) // 32
    bm = np.zeros((A, W), np.uint32)
    for a, pods in ((0, range(P)), (1, [3, 17, 50, 51, 99]), (2, range(10, 90, 2))):
        for p in pods:
            bm[a, p // 32] |= np.uint32(1 << (p % 32))
    packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.ones(P, np.int64), np.full(P, 4, np.int64), bm)
    e = Engine(0, max_pods=128, max_adapters=4, max_batch=1 << 14)
    try:
        pod_keys, _ = upload(e, 1, packed, LORA_ONLY)
        R = 8192
        reqs = np.zeros(R, dtype=REQ_DTYPE)
        reqs["adapter_id"] = np.random.default_rng(3).integers(0, 4, R)
        reqs["rand_key"] = random_keys(R, 4)
        want, rows = check(e, 1, reqs, pod_keys)
        assert {N.LIG_OK, N.LIG_NO_PODS_LEFT} <= {int(s) for s in want["status"]}
        assert (rows[want["status"] != N.LIG_OK] == -1).all()
    finally:
        e.close()


def test_compact_overflow_and_ejected_epochs():
    P, A = 4096, 1024
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 15)
    try:
        W = (P + 31) // 32
        packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.full(P, 1, np.int64),
                              np.full(P, 2, np.int64), np.full((A, W), 0xFFFFFFFF, dtype=np.uint32))
        pod_keys, _ = upload(e, 1, packed)
        assert e.pick_kernel_info(1)["table_bytes"] == 0      # the strided rows serve
        reqs = WL.make_requests(1024, A, seed=8)
        check(e, 1, reqs, pod_keys)
        # an ejected epoch of a bench snapshot: the pool form of the build; keys uploaded again
        snap = WL.make_snapshot(P, A, seed=9)
        pod_keys, pm = upload(e, 2, snap.packed, None, WL.make_models(A))
        gone = np.sort(np.random.default_rng(1).choice(P, 600, replace=False)).astype(np.int32)
        e.eject_pods(3, 2, gone)
        e.upload_pod_keys(3, pod_keys)
        e.upload_models(3, pm)
        reqs = WL.make_requests(1 << 15, A, seed=10)
        want, _ = check(e, 3, reqs, pod_keys)
        assert not np.isin(want["pod_idx"], gone).any()
        check(e, 3, WL.make_model_requests(1 << 14, A, seed=11), pod_keys, random_keys(1 << 14, 12), pm)
    finally:
        e.close()


# ---- stability --------------------------------------------------------------------------------------
def test_reordered_pods_keep_their_pick():
    rng = np.random.default_rng(21)
    n = 300
    pods = mkpods(rng.integers(0, 8, n).tolist(), rng.random(n).round(2).tolist(), [4] * n,
                  [[f"ad-{x}" for x in rng.choice(12, 2, replace=False)] for _ in range(n)])
    perm = rng.permutation(n)
    names = [f"ad-{x}" for x in rng.integers(0, 13, 4096)]
    keys = random_keys(4096, 22)
    crit = rng.random(4096) < 0.5
    picked = []
    for order in (pods, [pods[i] for i in perm]):
        packed = pack_pod_metrics(order)
        e = Engine(0, max_pods=512, max_adapters=64, max_batch=8192)
        try:
            for tree in (None, KEEP_ALL):
                pod_keys, _ = upload(e, 1 if tree is None else 2, packed, tree)
                reqs = np.zeros(4096, dtype=REQ_DTYPE)
                reqs["adapter_id"] = [packed.adapter_id(x) for x in names]
                reqs["flags"] = crit.astype(np.uint32)
                reqs["rand_key"] = keys
                out, rows = e.schedule_batch_affinity(1 if tree is None else 2, reqs, K)
                picked.append(([packed.pods[p].Name if p >= 0 else None for p in out["pod_idx"]],
                               [[packed.pods[p].Name for p in r if p >= 0] for r in rows]))
        finally:
            e.close()
    assert picked[0] == picked[2] and picked[1] == picked[3]


def test_ejection_keeps_the_picks_that_survive():
    P, A = 512, 16
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 14)
    try:
        snap = WL.make_snapshot(P, A, seed=31)
        pod_keys, _ = upload(e, 1, snap.packed, KEEP_ALL)
        reqs = WL.make_requests(8192, A, seed=32)
        before, _ = e.schedule_batch_affinity(1, reqs)
        plain1, off1, pods1 = e.filter_batch(1, 0, reqs)
        gone = np.arange(0, P, 7, dtype=np.int32)
        e.set_filter_tree(KEEP_ALL)                # the derived epoch is built with the tree in force
        try:
            e.eject_pods(2, 1, gone)
        finally:
            e.set_filter_tree(None)
        e.upload_pod_keys(2, pod_keys)
        after, _ = e.schedule_batch_affinity(2, reqs)
        plain2, off2, pods2 = e.filter_batch(2, 0, reqs)
        kept = 0
        for i in range(len(reqs)):
            s1 = set(pods1[off1[i]:off1[i + 1]].tolist())
            s2 = set(pods2[off2[i]:off2[i + 1]].tolist())
            if before["pod_idx"][i] in s2 and s2 <= s1:
                assert after["pod_idx"][i] == before["pod_idx"][i]
                kept += 1
        assert kept > 4000
    finally:
        e.close()


def test_two_ctxs_and_split_batches_agree():
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=41)
    models = WL.make_models(c["A"])
    reqs = WL.make_requests(20000, c["A"], seed=42)
    ids = WL.make_model_requests(20000, c["A"], seed=43)
    keys = random_keys(20000, 44)
    outs = []
    for ep in (5, 9):
        e = Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=1 << 15)
        try:
            upload(e, ep, snap.packed, None, models)
            whole = (e.schedule_batch_affinity(ep, reqs, 3), e.schedule_models_batch_affinity(ep, ids, keys, 3))
            cuts = [0, 1, 777, 13000, 20000]
            parts = [(e.schedule_batch_affinity(ep, reqs[a:b], 3),
                      e.schedule_models_batch_affinity(ep, ids[a:b], keys[a:b], 3)) for a, b in zip(cuts, cuts[1:])]
            for j in range(2):
                assert np.concatenate([p[j][0] for p in parts]).tobytes() == whole[j][0].tobytes()
                assert np.array_equal(np.concatenate([p[j][1] for p in parts]), whole[j][1])
            outs.append(whole)
        finally:
            e.close()
    for j in range(2):
        assert outs[0][j][0].tobytes() == outs[1][j][0].tobytes() and np.array_equal(outs[0][j][1], outs[1][j][1])


# ---- refusals -----------------------------------------------------------------------------------------
def test_refusals_write_nothing():
    P, A = 64, 8
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=256)
    lib, ctx = e._lib, e._ctx
    try:
        snap = WL.make_snapshot(P, A, seed=51)
        e.upload_snapshot(1, snap.packed)
        reqs = WL.make_requests(128, A, seed=52)
        ids = WL.make_model_requests(128, A, seed=53)
        keys = random_keys(128, 54)
        pod_keys = np.array([S.pod_key(p) for p in snap.packed.pods], dtype=np.uint64)

        def refused(code, fn, args):
            out = np.full(128 * 8, 0xAB, np.uint8)
            rows = np.full(128 * K, 0x5A5A, np.int16)
            rc = fn(ctx, *args(out.ctypes.data, rows.ctypes.data))
            assert rc == code, (rc, lib.lig_last_error())
            assert (out == 0xAB).all() and (rows == 0x5A5A).all()

        p = lambda a: a.ctypes.data
        desc = lambda ep, n: (lambda o, r: (ep, p(reqs), 128, o, n, r))
        mod = lambda ep, n: (lambda o, r: (ep, p(ids), p(keys), 128, o, n, r))
        # an epoch without keys, descriptors and model ids
        refused(N.LIG_ERR_NO_SNAPSHOT, lib.lig_schedule_batch_affinity, desc(1, 2))
        assert b"lig_upload_pod_keys" in lib.lig_last_error()
        # key uploads: P mismatch, null keys, stale epoch
        assert lib.lig_upload_pod_keys(ctx, 1, P - 1, p(pod_keys)) == N.LIG_ERR_INVALID
        assert lib.lig_upload_pod_keys(ctx, 1, P, None) == N.LIG_ERR_INVALID
        assert lib.lig_upload_pod_keys(ctx, 77, P, p(pod_keys)) == N.LIG_ERR_STALE_EPOCH
        e.upload_pod_keys(1, pod_keys)
        # the model forms without a model table
        refused(N.LIG_ERR_NO_SNAPSHOT, lib.lig_schedule_models_batch_affinity, mod(1, 2))
        e.upload_models(1, pack_models(WL.make_models(A), snap.packed))
        # a refused upload keeps the keys; a threshold rebuild keeps them
        assert lib.lig_upload_pod_keys(ctx, 1, P + 1, p(pod_keys)) == N.LIG_ERR_INVALID
        e.set_thresholds(0.5, 3, 40)
        check(e, 1, reqs, pod_keys, ns=(0, 2), forms=("pageable",))
        check(e, 1, ids, pod_keys, keys, pack_models(WL.make_models(A), snap.packed), ns=(2,), forms=("pageable",))
        # bad arguments
        for n in (-1, K + 1):
            refused(N.LIG_ERR_INVALID, lib.lig_schedule_batch_affinity, desc(1, n))
            refused(N.LIG_ERR_INVALID, lib.lig_schedule_models_batch_affinity, mod(1, n))
        refused(N.LIG_ERR_INVALID, lib.lig_schedule_batch_affinity, lambda o, r: (1, p(reqs), 128, o, 2, None))
        refused(N.LIG_ERR_INVALID, lib.lig_schedule_models_batch_affinity,
                lambda o, r: (1, p(ids), None, 128, o, 0, r))
        big = WL.make_requests(257, A, seed=55)
        refused(N.LIG_ERR_INVALID, lib.lig_schedule_batch_affinity, lambda o, r: (1, p(big), 257, o, 0, None))
        refused(N.LIG_ERR_STALE_EPOCH, lib.lig_schedule_batch_affinity, desc(77, 2))
        d_reqs, d_out = dev(reqs), torch.zeros(128 * 8 + 8, dtype=torch.uint8, device="cuda")
        assert lib.lig_schedule_batch_affinity_device(ctx, 1, d_reqs.data_ptr() + 8, 128, d_out.data_ptr(), 0, None,
                                                      None) == N.LIG_ERR_INVALID
        d_ids, d_keys = dev(ids), dev(np.concatenate([keys, keys[:1]]))
        assert lib.lig_schedule_models_batch_affinity_device(ctx, 1, d_ids.data_ptr(), d_keys.data_ptr() + 4, 128,
                                                             d_out.data_ptr(), 0, None, None) == N.LIG_ERR_INVALID
        # a derived epoch and a delta epoch start without keys
        e.eject_pods(2, 1, [3, 4])
        refused(N.LIG_ERR_NO_SNAPSHOT, lib.lig_schedule_batch_affinity, desc(2, 0))
        e.update_snapshot(3, 2, [5], [0.3], [1], [0], [4], [0, 0], np.zeros(0, np.int32))
        refused(N.LIG_ERR_NO_SNAPSHOT, lib.lig_schedule_batch_affinity, desc(3, 1))
        e.upload_pod_keys(3, pod_keys)
        check(e, 3, reqs, pod_keys, ns=(1,), forms=("pageable", "device"))
    finally:
        e.close()


# ---- the schedulers ---------------------------------------------------------------------------------------
def pool(n, seed):
    rng = np.random.default_rng(seed)
    return mkpods(rng.integers(0, 8, n).tolist(), rng.random(n).round(2).tolist(), [4] * n,
                  [[f"ad-{x}" for x in rng.choice(6, 2, replace=False)] for _ in range(n)])


KEEP_ALL_CHART = S.Filter("keep all", S.LOW_QUEUEING, queue_threshold=1 << 62)


def test_python_scheduler():
    pods = pool(200, 61)
    prov = StaticProvider(pods)
    s = S.NewScheduler(prov, filter=KEEP_ALL_CHART, affinity=True, max_pods=256, max_adapters=16, max_batch=4096,
                       seed=1)
    try:
        keys = [int(k) for k in random_keys(500, 62)]
        req = S.LLMRequest(ResolvedTargetModel="ad-1", Critical=True)
        first = [s.ScheduleAffinity(req, k) for k in keys]
        prov.pods = list(reversed(pods))                  # a new order at the next refresh
        assert [s.ScheduleAffinity(req, k) for k in keys] == first
        rows = s.ScheduleBatchAffinity([req] * len(keys), keys, 4)
        assert [r[0][0] for r in rows] == first and all(len(r[0]) == 5 for r in rows)
        assert s.ScheduleAffinityWithFallbacks(req, keys[0], 4) == rows[0][0]
        gone = [pods[3].Pod, first[0], first[7]]
        s.EjectPods(gone)
        after = [s.ScheduleAffinity(req, k) for k in keys]
        for a, b in zip(first, after):
            assert (a == b) == (a not in gone) and b not in gone
        s.EjectPods([])
        assert [s.ScheduleAffinity(req, k) for k in keys] == first
        s.SetInferenceModels([im("m", [("ad-1", 3), ("ad-2", 5)]), im("plain")])
        resolved, pod = s.ScheduleModelAffinity("m", keys[1])
        assert (resolved, pod) == s.ScheduleModelAffinity("m", keys[1])
        r2, pods2 = s.ScheduleModelAffinityWithFallbacks("m", keys[1], 3)
        assert r2 == resolved and pods2[0] == pod and len(pods2) == 4
        out = s.ScheduleModelBatchAffinity(["m", "nope", "plain"], keys[:3])
        assert out[1][0] is None and out[1][2].code == "Unknown" and out[2][1] == "plain"
        with pytest.raises(ValueError):
            s.ScheduleBatchAffinity([req], keys[:2])
        with pytest.raises(ValueError):
            s.ScheduleAffinityWithFallbacks(req, 1, K + 1)
    finally:
        s.close()
    plain = S.NewScheduler(StaticProvider(pods), max_pods=256, max_adapters=16, max_batch=64)
    chain = S.NewScheduler(StaticProvider(pods), affinity=True, load_feedback_window=4, max_pods=256,
                           max_adapters=16, max_batch=64)
    try:
        for sch in (plain, chain):
            with pytest.raises(ValueError):
                sch.ScheduleAffinity(req, 1)
            with pytest.raises(ValueError):
                sch.ScheduleModelAffinity("m", 1)
    finally:
        plain.close()
        chain.close()


def test_cpp_runtime_matches_python():
    pods = pool(200, 71)
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=256, max_adapters=16, max_batch=512, seed=3, filter=KEEP_ALL_CHART,
                         affinity=True)
    sp = StaticProvider(pods)
    s = S.NewScheduler(sp, filter=KEEP_ALL_CHART, affinity=True, max_pods=256, max_adapters=16, max_batch=512)
    try:
        keys = [int(k) for k in random_keys(300, 72)]
        req = S.LLMRequest(ResolvedTargetModel="ad-2")

        def cpp(k, n=0):
            code, names, err = hs.ScheduleAffinity("ad-2", False, k, n)
            assert code == 0, err
            return names

        def py(k, n=0):
            return [p.Name for p in (s.ScheduleAffinityWithFallbacks(req, k, n) if n else [s.ScheduleAffinity(req, k)])]

        first = [cpp(k) for k in keys]
        assert first == [py(k) for k in keys]
        assert [cpp(k, 3) for k in keys[:50]] == [py(k, 3) for k in keys[:50]]
        prov.set_pods(list(reversed(pods)))
        sp.pods = list(reversed(pods))
        hs.Refresh()
        assert [cpp(k) for k in keys] == first
        gone = [pods[5].Pod, Pod(first[0][0], f"address-{first[0][0].split('-')[1]}")]
        hs.EjectPods(gone)
        s.EjectPods(gone)
        after = [cpp(k) for k in keys]
        assert after == [py(k) for k in keys]
        names_gone = {p.Name for p in gone}
        for a, b in zip(first, after):
            assert (a == b) == (a[0] not in names_gone) and b[0] not in names_gone
        assert hs.stats()["affinity_scheduled"] >= 2 * len(keys)
        models = [im("m", [("ad-1", 3), ("ad-2", 5)]), im("plain")]
        hs.set_inference_models(H.HostDataStore(models))
        s.SetInferenceModels(models)
        for k in keys[:40]:
            code, resolved, names, err = hs.ScheduleModelAffinity("m", k, 2)
            r2, pods2 = s.ScheduleModelAffinityWithFallbacks("m", k, 2)
            assert code == 0 and (resolved, names) == (r2, [p.Name for p in pods2])
        code, _, _, err = hs.ScheduleModelAffinity("nope", 1)
        assert code == H.GRPC_UNKNOWN
    finally:
        hs.close()
        s.close()
    plain = H.HostScheduler(H.HostProvider(pods), max_pods=256, max_adapters=16, max_batch=64)
    chain = H.HostScheduler(H.HostProvider(pods), max_pods=256, max_adapters=16, max_batch=64, affinity=True,
                            load_feedback_window=4)
    try:
        for hsx in (plain, chain):
            code, _, err = hsx.ScheduleAffinity("ad-1", False, 5)
            assert code == 3 and "ScheduleAffinity" in err
            code, _, _, err = hsx.ScheduleModelAffinity("m", 5, 2)
            assert code == 3
    finally:
        plain.close()
        chain.close()
