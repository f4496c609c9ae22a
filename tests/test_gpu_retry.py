"""Retry scheduling (lig_schedule_batch_excluding[_device]) on the GPU: every result against the definition
(retry_ref.py, which rebuilds each request's pool without its excluded pods), and rows that exclude
nothing also against lig_schedule_batch.  Pools at the bit-word edges, the bench configurations and one
too large for staged columns; the built-in tree at default and extreme thresholds and caller trees with
DROP and "no pods left" leaves; an epoch whose tree has since been replaced; rows of every kind; forced
Int31n rejections; delta epochs, threshold rebuilds, stale epochs and refusals; buffer kinds and two
streams; and the Python and C++ schedulers."""
import random

import numpy as np
import pytest
import torch

import retry_ref as RR
from draw_keys import accept_top, pick_keys, rejection_heavy_ns
from test_gpu_fallbacks import DROP_AND_NO_PODS, KEEP_ALL, splitmix_keys
from test_gpu_filter_batch import Pinned, StaticProvider, dev
from test_gpu_filter_tree import c4_tree, mkpods
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Pod
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, pack_columns, pack_pod_metrics

pytestmark = pytest.mark.gpu

X = N.LIG_MAX_EXCLUDED
SEED = 0x0DDB_A11_5EED
UNSTAGED_P = 13000          # 608 B of shared memory per 32 pods: past the 227 KB a CTA can have
# no pods left at the root for critical requests without affinity, DROP for sheddable ones
NO_PODS_TREE = [N.LigFilterNode(N.LIG_F_CRITICAL_REQUEST, 1, 2, -1, 0, 0.0),
                N.LigFilterNode(N.LIG_F_LORA_AFFINITY, 4, -1, -1, 0, 0.0),
                N.LigFilterNode(N.LIG_F_NO_QUEUE_AND_LOW_KV, 4, 3, -1, 5, 0.8),
                N.LigFilterNode(N.LIG_F_DROP, -1, -1, -1, 0, 0.0),
                N.LigFilterNode(N.LIG_F_LEAST_QUEUING, -1, -1, -1, 0, 0.0)]
# trees whose walk of an empty pool ends on a predicate leaf (no pods left) or a range leaf (empty)
NO_PODS_LEAF = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 50, 0.0)]
EMPTY_LEAF = [N.LigFilterNode(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0)]
EXTREME = [(0.8, 5, -(1 << 63)), (float("nan"), (1 << 63) - 1, (1 << 63) - 1), (0.0, 0, 0),
           (float("inf"), -(1 << 63), 1)]

_ep = [5000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=16384, max_adapters=1024, max_batch=1 << 16)
    yield e
    e.close()


def retry_device(eng, ep, seed, reqs, rows, stream=0):
    R, k = rows.shape
    d_in = dev(reqs) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda() if R else torch.zeros(1, dtype=torch.int16,
                                                                                     device="cuda")
    d_out = torch.full((max(R, 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    eng.schedule_batch_excluding_device(ep, seed, d_in.data_ptr(), R, d_rows.data_ptr(), k, d_out.data_ptr(), stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()[: R * 8].view(PICK_DTYPE)


def excludes_nothing(rows, P):
    return ((rows < 0) | (rows >= P)).all(axis=1)


def check(eng, ep, seed, snap, reqs, rows, thresholds=(0.8, 5, 50), nodes=None, device=True):
    """Host and device forms against the definition; rows that exclude nothing also against
    lig_schedule_batch."""
    want = RR.retry_batch(snap, reqs, rows, seed, thresholds, nodes)
    got = eng.schedule_batch_excluding(ep, seed, reqs, rows)
    assert got.tobytes() == want.tobytes()
    if device:
        assert retry_device(eng, ep, seed, reqs, rows).tobytes() == want.tobytes()
    keep = excludes_nothing(rows, snap.P)
    if keep.any():
        plain = eng.schedule_batch(ep, seed, np.ascontiguousarray(reqs[keep]))
        assert got[keep].tobytes() == plain.tobytes()
    return got


def row_templates(eng, ep, snap, rng, nodes=None):
    """Rows of every kind, as lists: nothing, random pods (duplicates and out-of-range entries mixed
    in), a class's whole survivor set, the largest queue, the bit-word edges, every pod of a small pool."""
    P = snap.P
    t = [[], [-1, P, 32767, -32768], [int(np.argmax(snap.q))], [31, 32, P - 1], [0]]
    for k in (1, 9, 32):
        r = rng.integers(0, P, size=k).tolist()
        if k > 2:
            r[1] = r[0]
            r[-1] = P + 3
        t.append(r)
    for crit, a in ((True, 0), (False, 0), (True, snap.A)):
        st, n, lst = eng.read_class(ep, crit, a, P)
        if 0 < n <= X:
            t.append([int(p) for p in lst])
    if P <= X:
        t.append(list(range(P))[::-1])
    return t


def rows_for(templates, R, width, rng):
    rows = np.full((R, width), -1, dtype=np.int16)
    for i in range(R):
        tpl = templates[int(rng.integers(0, len(templates)))][:width]
        rows[i, :len(tpl)] = tpl
    return rows


def class_reqs(A, R, rng):
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    ids = np.array([0, 1, 2, A, -1, A + 9] + list(range(min(A, 16))), dtype=np.int32)
    reqs["adapter_id"] = ids[rng.integers(0, len(ids), size=R)]
    reqs["flags"] = rng.integers(0, 2, size=R)
    reqs["rand_key"] = rng.integers(0, 1 << 64, size=R, dtype=np.uint64)
    return reqs


# ---- pools and trees --------------------------------------------------------------------------------------
POOLS = [(1, 4), (31, 4), (32, 4), (33, 4), (64, 32), (512, 256), (4096, 1024), (4097, 64), (UNSTAGED_P, 16)]


@pytest.mark.parametrize("P,A", POOLS)
def test_pools_built_in_tree(P, A, eng):
    rng = np.random.default_rng(P)
    snap = WL.make_snapshot(P, A, seed=P + 1).packed
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    tpl = row_templates(eng, ep, snap, rng)
    for width in (1, 9, 32):
        reqs = class_reqs(A, 96, rng)
        check(eng, ep, SEED + width, snap, reqs, rows_for(tpl, 96, width, rng))


@pytest.mark.parametrize("P,A", [(1, 4), (33, 4), (512, 256), (4096, 1024), (UNSTAGED_P, 16)])
@pytest.mark.parametrize("tree", ["drop_and_no_pods", "no_pods", "c4"])
def test_pools_caller_trees(P, A, tree, eng):
    nodes = {"drop_and_no_pods": DROP_AND_NO_PODS, "no_pods": NO_PODS_TREE, "c4": c4_tree().flatten()}[tree]
    rng = np.random.default_rng(P + 7)
    snap = WL.make_snapshot(P, A, seed=P + 2).packed
    ep = next_epoch()
    eng.set_filter_tree(nodes)
    try:
        eng.upload_snapshot(ep, snap)
    finally:
        eng.set_filter_tree(None)
    tpl = row_templates(eng, ep, snap, rng)
    for width in (1, 32):
        reqs = class_reqs(A, 64, rng)
        got = check(eng, ep, SEED, snap, reqs, rows_for(tpl, 64, width, rng), nodes=nodes)
        assert got["pod_idx"].max() < P


def test_statuses_of_caller_tree_leaves_and_empty_pools(eng):
    P, A = 5, 4
    snap = WL.make_snapshot(P, A, seed=3).packed
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    reqs["flags"] = [0, 1, 0, 1]
    reqs["adapter_id"] = [0, 0, A, A]
    everything = np.tile(np.arange(P, dtype=np.int16), (4, 1))
    seen = set()
    for nodes in (None, DROP_AND_NO_PODS, NO_PODS_TREE, NO_PODS_LEAF, EMPTY_LEAF):
        ep = next_epoch()
        eng.set_filter_tree(nodes)
        try:
            eng.upload_snapshot(ep, snap)
        finally:
            eng.set_filter_tree(None)
        got = check(eng, ep, SEED, snap, reqs, everything, nodes=nodes)
        assert (got["pod_idx"] == -1).all() and (got["n_survivors"] == 0).all()
        if nodes is None:                        # an empty pool drops critical and sheddable requests alike
            assert (got["status"] == N.LIG_DROP).all()
        seen |= set(got["status"].tolist())
    assert seen == {N.LIG_DROP, N.LIG_NO_PODS_LEFT, N.LIG_EMPTY}


@pytest.mark.parametrize("thresholds", EXTREME)
def test_extreme_thresholds(thresholds, eng):
    P, A = 200, 16
    rng = np.random.default_rng(11)
    snap = WL.make_snapshot(P, A, seed=12).packed
    eng.set_thresholds(*thresholds)
    try:
        ep = next_epoch()
        eng.upload_snapshot(ep, snap)
        tpl = row_templates(eng, ep, snap, rng)
        reqs = class_reqs(A, 128, rng)
        reqs["flags"][::2] = 1
        check(eng, ep, SEED, snap, reqs, rows_for(tpl, 128, 32, rng), thresholds)
    finally:
        eng.set_thresholds()


def test_low_queueing_failure_forwards_the_pool_not_every_pod(eng):
    """Every queue at or above queueingThresholdLoRA: the critical walk ranges over the pool itself."""
    pods = mkpods([50, 60, 100, 1000, 55], [0.5] * 5, [4] * 5)
    snap = pack_pod_metrics(pods)
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    reqs = np.zeros(3, dtype=REQ_DTYPE)
    reqs["flags"] = 1
    reqs["rand_key"] = [1, 2, 3]
    rows = np.array([[3, -1], [0, 1], [-1, -1]], dtype=np.int16)
    got = check(eng, ep, SEED, snap, reqs, rows)
    assert got["n_survivors"].tolist() == [3, 2, 4]     # 50 + 50 / 4 = 62; 55 + 945 / 3 = 370; 50 + 950 / 5 = 240


def test_epoch_keeps_the_tree_it_was_built_with(eng):
    P, A = 300, 16
    rng = np.random.default_rng(13)
    snap = WL.make_snapshot(P, A, seed=14).packed
    built_with = c4_tree().flatten()
    ep = next_epoch()
    eng.set_filter_tree(built_with)
    eng.upload_snapshot(ep, snap)
    reqs = class_reqs(A, 128, rng)
    tpl = row_templates(eng, ep, snap, rng)
    for replacement in (DROP_AND_NO_PODS, None):   # another caller tree, then the built-in tree
        eng.set_filter_tree(replacement)
        nothing = np.full((128, 3), -1, dtype=np.int16)
        assert eng.schedule_batch_excluding(ep, SEED, reqs, nothing).tobytes() == \
            eng.schedule_batch(ep, SEED, reqs).tobytes()
        check(eng, ep, SEED, snap, reqs, rows_for(tpl, 128, 9, rng), nodes=built_with)
    eng.set_filter_tree(None)


def test_forced_int31n_rejections(eng):
    for n in rejection_heavy_ns(40, 4000, 2):
        P = n + 3
        snap = WL.make_snapshot(P, 4, seed=n).packed
        ep = next_epoch()
        eng.set_filter_tree(KEEP_ALL)
        try:
            eng.upload_snapshot(ep, snap)
        finally:
            eng.set_filter_tree(None)
        rng = np.random.default_rng(n)
        keys = pick_keys(SEED, rng.integers(accept_top(n), 1 << 31, size=64), rng)
        reqs = np.zeros(64, dtype=REQ_DTYPE)
        reqs["rand_key"] = keys
        rows = np.tile(np.array([0, P // 2, P - 1], dtype=np.int16), (64, 1))
        got = check(eng, ep, SEED, snap, reqs, rows, nodes=KEEP_ALL)
        assert (got["n_survivors"] == n).all() and (got["status"] == N.LIG_OK).all()


# ---- epochs, thresholds, refusals -------------------------------------------------------------------------
def test_delta_epoch_and_threshold_rebuild(eng):
    P, A = 1000, 64
    rng = np.random.default_rng(15)
    snap = WL.make_snapshot(P, A, seed=16).packed
    base = next_epoch()
    eng.upload_snapshot(base, snap)
    dirty = np.sort(rng.choice(P, 40, replace=False)).astype(np.int32)
    acts = [rng.choice(A, int(rng.integers(0, 4)), replace=False) for _ in dirty]
    kv, q = rng.random(40), rng.integers(0, 60, 40)
    offs = np.concatenate([[0], np.cumsum([len(x) for x in acts])]).astype(np.int32)
    new = next_epoch()
    eng.update_snapshot(new, base, dirty, kv, q, [len(x) for x in acts], np.full(40, 4), offs,
                        np.concatenate(acts + [np.zeros(0, np.int64)]))
    bitmap = snap.bitmap.copy()
    kv2, q2, na2, ma2 = snap.kv.copy(), snap.q.astype(np.int64), snap.n_active.astype(np.int64), \
        snap.max_active.astype(np.int64)
    for j, p in enumerate(dirty):
        kv2[p], q2[p], na2[p], ma2[p] = kv[j], q[j], len(acts[j]), 4
        bitmap[:, p >> 5] &= ~np.uint32(1 << (p & 31))
        for a in acts[j]:
            bitmap[a, p >> 5] |= np.uint32(1 << (p & 31))
    updated = pack_columns(kv2, q2, na2, ma2, bitmap, snap.adapter_ids, snap.pods)
    reqs = class_reqs(A, 128, rng)
    rows = rows_for([[int(d) for d in dirty[:9]], [int(dirty[0])], [], [31, 32, P - 1]], 128, 9, rng)
    check(eng, new, SEED, updated, reqs, rows)
    # lig_set_thresholds rebuilds the resident epoch; the retry walks the new thresholds
    eng.set_thresholds(0.5, 3, 20)
    try:
        check(eng, new, SEED, updated, reqs, rows, (0.5, 3, 20))
    finally:
        eng.set_thresholds()
    check(eng, new, SEED, updated, reqs, rows)


def test_refusals_leave_out_untouched():
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=16)
    try:
        reqs = class_reqs(8, 16, np.random.default_rng(1))
        rows = np.full((16, X + 1), -1, dtype=np.int16)
        out = np.full(16 * 8, 0x7B, dtype=np.uint8)
        p = lambda a: a.ctypes.data

        def refused(code, fn):
            with pytest.raises(N.LigError) as err:
                fn()
            assert err.value.code == code
            assert (out == 0x7B).all()

        # no snapshot yet, then a stale epoch
        refused(N.LIG_ERR_NO_SNAPSHOT, lambda: e.schedule_batch_excluding_ptr(1, 2, p(reqs), 16, p(rows), 1, p(out)))
        e.upload_snapshot(1, WL.make_snapshot(40, 8, seed=2).packed)
        refused(N.LIG_ERR_STALE_EPOCH, lambda: e.schedule_batch_excluding_ptr(9, 2, p(reqs), 16, p(rows), 1, p(out)))
        for k in (0, X + 1, -3):
            refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_ptr(1, 2, p(reqs), 16, p(rows), k, p(out)))
        refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_ptr(1, 2, 0, 16, p(rows), 1, p(out)))
        refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_ptr(1, 2, p(reqs), 16, 0, 1, p(out)))
        big = class_reqs(8, 17, np.random.default_rng(2))
        big_rows = np.full((17, 1), -1, dtype=np.int16)
        refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_ptr(1, 2, p(big), 17, p(big_rows), 1, p(out)))
        # device forms: misaligned buffers
        d_in, d_rows = dev(reqs), torch.full((16 * 2 + 1,), -1, dtype=torch.int16, device="cuda")
        d_out = torch.full((16 * 8 + 8,), 0x7B, dtype=torch.uint8, device="cuda")
        for a, b, c in ((d_in.data_ptr() + 8, d_rows.data_ptr(), d_out.data_ptr()),
                        (d_in.data_ptr(), d_rows.data_ptr() + 1, d_out.data_ptr()),
                        (d_in.data_ptr(), d_rows.data_ptr(), d_out.data_ptr() + 4)):
            refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_device(1, 2, a, 16, b, 2, c))
        refused(N.LIG_ERR_STALE_EPOCH, lambda: e.schedule_batch_excluding_device(
            7, 2, d_in.data_ptr(), 16, d_rows.data_ptr(), 2, d_out.data_ptr()))
        torch.cuda.synchronize()
        assert (d_out.cpu().numpy() == 0x7B).all()
        # R = 0 is a no-op, R > max_batch is fine on the device form
        e.schedule_batch_excluding_ptr(1, 2, 0, 0, 0, 1, 0)
    finally:
        e.close()


# ---- buffers and streams ----------------------------------------------------------------------------------
def test_buffer_kinds_and_two_streams(eng):
    P, A, R, k = 512, 256, 3000, 9
    rng = np.random.default_rng(17)
    snap = WL.make_snapshot(P, A, seed=18).packed
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    reqs = WL.make_requests(R, A, seed=19)
    rows = rows_for(row_templates(eng, ep, snap, rng), R, k, rng)
    want = check(eng, ep, SEED, snap, reqs, rows, device=False)
    for mask in range(27):
        kinds = [mask // 3 ** i % 3 for i in range(3)]   # 0 pageable, 1 page-locked, 2 page-locked misaligned
        bufs = []

        def mk(kind, arr, shift):
            if kind == 0:
                a = np.ascontiguousarray(arr).copy()
                return a, a.ctypes.data
            nbytes = arr.nbytes
            b = Pinned(nbytes + 16, np.uint8)
            bufs.append(b)
            s = shift if kind == 2 else 0
            raw = b.a[s: s + nbytes]
            raw[:] = np.frombuffer(np.ascontiguousarray(arr).tobytes(), np.uint8)
            return raw, b.ptr + s

        try:
            h_in, pin = mk(kinds[0], reqs, 8)                     # +8: a request array at an odd 8 bytes
            h_rows, prows = mk(kinds[1], rows, 1)
            out, pout = mk(kinds[2], np.zeros(R, PICK_DTYPE), 4)
            eng.schedule_batch_excluding_ptr(ep, SEED, pin, R, prows, k, pout)
            assert out.tobytes() == want.tobytes(), kinds
            assert h_in.tobytes() == reqs.tobytes() and h_rows.tobytes() == rows.tobytes()
        finally:
            for b in bufs:
                b.free()
    d_in, d_rows = dev(reqs), torch.from_numpy(rows.reshape(-1).copy()).cuda()
    torch.cuda.synchronize()
    outs = []
    for s in (torch.cuda.Stream(), torch.cuda.Stream()):
        o = torch.zeros(R * 8, dtype=torch.uint8, device="cuda")
        eng.schedule_batch_excluding_device(ep, SEED, d_in.data_ptr(), R, d_rows.data_ptr(), k, o.data_ptr(),
                                            s.cuda_stream)
        outs.append(o)
    torch.cuda.synchronize()
    for o in outs:
        assert o.cpu().numpy().tobytes() == want.tobytes()


# ---- schedulers -------------------------------------------------------------------------------------------
def pool_pods(P=40):
    rng = np.random.default_rng(21)
    return mkpods(rng.integers(0, 12, P).tolist(), np.round(rng.random(P), 2).tolist(),
                  rng.integers(0, 4, P).tolist(), [list(rng.choice(["a", "b", "c"], int(rng.integers(0, 3)),
                                                               replace=False)) for _ in range(P)])


def expect_one(pods, seed, key, model, critical, tried, nodes=None):
    """The pod the definition picks for one retry over the provider slice `pods`."""
    snap = pack_pod_metrics(pods)
    row = [p for p, pm in enumerate(pods) if pm.Pod in set(tried)] or [-1]
    reqs = np.zeros(1, dtype=REQ_DTYPE)
    reqs[0] = (snap.adapter_id(model), int(critical), key)
    pk = RR.retry_batch(snap, reqs, np.array([row], dtype=np.int16), seed, nodes=nodes)[0]
    return (snap.pods[int(pk["pod_idx"])] if pk["status"] == N.LIG_OK else None), int(pk["status"])


@pytest.mark.parametrize("tree", [None, "c4"])
def test_python_scheduler(tree):
    nodes = None if tree is None else c4_tree()
    pods = pool_pods()
    prov = StaticProvider(pods)
    sched = S.NewScheduler(prov, filter=nodes, max_pods=64, max_adapters=8, max_batch=256, seed=5)
    flat = None if nodes is None else nodes.flatten()
    keys = random.Random(5)
    keys.getrandbits(64)                                  # the scheduler's seed
    try:
        req = S.LLMRequest(ResolvedTargetModel="a", Critical=True)
        first = sched.Schedule(req)
        keys.getrandbits(64)
        prov.pods = pods[::-1]                            # the provider reorders its slice
        tried = [first, Pod("ghost", "nowhere")]          # a pod that left the pool is ignored
        got = sched.ScheduleRetry(req, tried)
        want, _ = expect_one(prov.pods, sched._seed, keys.getrandbits(64), "a", True, tried, flat)
        assert got == want and got != first
        # a batch, tried lists of every width, and the plain calls after it keep the key sequence
        reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "zz") for c in (False, True)]
        tried_lists = [[pm.Pod for pm in prov.pods[:w]] for w in (0, 1, 5, 9, 31, 32)]
        got = sched.ScheduleBatchRetry(reqs, tried_lists)
        for r, t, (pod, err) in zip(reqs, tried_lists, got):
            want, st = expect_one(prov.pods, sched._seed, keys.getrandbits(64), r.ResolvedTargetModel, r.Critical, t,
                                  flat)
            assert pod == want and (err is None) == (st == N.LIG_OK)
            if err is not None:
                assert str(err) == str(S._schedule_error(st))
            assert pod is None or pod not in t
        after = sched.ScheduleBatch(reqs[:2])
        snap = pack_pod_metrics(prov.pods)
        arr = np.zeros(2, dtype=REQ_DTYPE)
        for i, r in enumerate(reqs[:2]):
            arr[i] = (snap.adapter_id(r.ResolvedTargetModel), int(r.Critical), keys.getrandbits(64))
        plain = RR.retry_batch(snap, arr, np.full((2, 1), -1, np.int16), sched._seed, nodes=flat)
        assert [p for p, _ in after] == [snap.pods[int(x)] if x >= 0 else None for x in plain["pod_idx"]]
        # every pod tried: an empty pool
        small = S.NewScheduler(StaticProvider(pods[:3]), filter=nodes, max_pods=64, max_adapters=8, seed=6)
        try:
            with pytest.raises(S.StatusError, match="dropping request"):
                small.ScheduleRetry(S.LLMRequest(ResolvedTargetModel="a", Critical=True),
                                    [pm.Pod for pm in pods[:3]])
        finally:
            small.close()
        with pytest.raises(ValueError):
            sched.ScheduleRetry(req, [pm.Pod for pm in prov.pods[:X + 1]])
    finally:
        sched.close()
    chain = S.NewScheduler(StaticProvider(pods), load_feedback_window=4, max_pods=64, max_adapters=8, seed=5)
    try:
        with pytest.raises(ValueError, match="load_feedback_window"):
            chain.ScheduleRetry(S.LLMRequest(ResolvedTargetModel="a"), [])
    finally:
        chain.close()


@pytest.mark.parametrize("use_doorbell", [False, True])
def test_cpp_runtime(use_doorbell):
    from llm_instance_gateway_b200 import host as H
    pods = pool_pods()
    seed = 0x4321
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, use_doorbell=use_doorbell)
    keys = splitmix_keys(seed, 64)
    try:
        code, first, _ = hs.Schedule("m", "a", True)
        assert code == H.GRPC_OK
        prov.set_pods(pods[::-1])
        hs.Refresh()
        k = 1
        for model, crit, width in (("a", True, 1), ("b", False, 9), ("zz", True, 32), ("a", False, 0)):
            tried = [first] + [pm.Pod for pm in prov.pods[:max(width - 1, 0)]] if width else [Pod("ghost", "x")]
            code, pod, err = hs.ScheduleRetry(model, crit, tried)
            want, st = expect_one(prov.pods, seed, int(keys[k]), model, crit, tried)
            k += 1
            assert pod == want, (model, crit, width)
            assert (code == H.GRPC_OK) == (st == N.LIG_OK)
            if st == N.LIG_DROP:
                assert code == H.GRPC_RESOURCE_EXHAUSTED
        # a plain Schedule after the retries takes the next key
        code, pod, _ = hs.Schedule("m", "b", False)
        want, _ = expect_one(prov.pods, seed, int(keys[k]), "b", False, [])
        assert pod == want
        code, pod, err = hs.ScheduleRetry("a", True, [pm.Pod for pm in prov.pods[:X + 1]])
        assert code == 3 and pod is None and str(X) in err
        assert hs.stats()["retry_scheduled"] == 4
    finally:
        hs.close()
    chain = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=8)
    try:
        code, pod, err = chain.ScheduleRetry("a", False, [])
        assert code == 3 and "load_feedback_window" in err
    finally:
        chain.close()
        prov.close()
