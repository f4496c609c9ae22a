"""Retry scheduling with fallback rows (lig_schedule_batch_excluding_fallbacks[_device]) on the GPU: every
result against the definition (retry_fallbacks_ref.py), every pick against lig_schedule_batch_excluding
byte for byte, and rows that exclude nothing against lig_schedule_batch_fallbacks.  Pools at the bit-word
edges, one too large for staged columns and the widest mask (P = 32768); the built-in tree and caller
trees (defaultFilter restated, one that keeps every pod, drop and "no pods left" leaves); rows of every
kind and width; forced Int31n rejections on the pick and on a ranking step; delta epochs, threshold
rebuilds and refusals; buffer kinds and two streams; the feedback chain left alone; and the Python and
C++ schedulers."""
import threading

import numpy as np
import pytest
import torch

import retry_fallbacks_ref as RF
import retry_ref as RR
from draw_keys import GAMMA, M64, accept_top, pick_keys, rejection_heavy_ns, states_for
from fallback_ref import fallback_rows
from test_gpu_fallbacks import DROP_AND_NO_PODS, KEEP_ALL, splitmix_keys
from test_gpu_filter_batch import Pinned, StaticProvider, dev
from test_gpu_filter_tree import mkpods
from test_gpu_retry import (EMPTY_LEAF, NO_PODS_LEAF, NO_PODS_TREE, UNSTAGED_P, class_reqs, excludes_nothing,
                            pool_pods, row_templates, rows_for)
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Pod
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, pack_columns, pack_pod_metrics

pytestmark = pytest.mark.gpu

X = N.LIG_MAX_EXCLUDED
K = N.LIG_MAX_FALLBACKS
SEED = 0x0DDB_A11_F00D
WIDEST_P = 32768            # W = 1024 mask words: the widest a select crosses

_ep = [9000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=WIDEST_P, max_adapters=1024, max_batch=1 << 16)
    yield e
    e.close()


def device_call(eng, ep, seed, reqs, rows, k, stream=0):
    R, w = rows.shape
    d_in = dev(reqs) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda() if R else torch.zeros(1, dtype=torch.int16,
                                                                                     device="cuda")
    d_out = torch.full((max(R, 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    d_fb = torch.full((max(R, 1) * k,), 0x5A5A, dtype=torch.int16, device="cuda")
    eng.schedule_batch_excluding_fallbacks_device(ep, seed, d_in.data_ptr(), R, d_rows.data_ptr(), w,
                                                  d_out.data_ptr(), k, d_fb.data_ptr(), stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()[: R * 8].view(PICK_DTYPE), d_fb.cpu().numpy()[: R * k].reshape(R, k)


def check(eng, ep, seed, snap, reqs, rows, thresholds=(0.8, 5, 50), nodes=None, ks=(1, 4, K), device=True):
    """Host and device forms at every k against the definition; picks against lig_schedule_batch_excluding;
    rows that exclude nothing against lig_schedule_batch_fallbacks.  Returns (picks, rows at k = 8)."""
    want, want_rows = RF.retry_fallback_batch(snap, reqs, rows, seed, max(ks), thresholds, nodes)
    retry = eng.schedule_batch_excluding(ep, seed, reqs, rows)
    assert retry.tobytes() == want.tobytes()
    keep = excludes_nothing(rows, snap.P)
    for k in ks:
        got, got_rows = eng.schedule_batch_excluding_fallbacks(ep, seed, reqs, rows, k)
        assert got.tobytes() == retry.tobytes(), k
        assert np.array_equal(got_rows, want_rows[:, :k]), k
        if device:
            d_got, d_rows = device_call(eng, ep, seed, reqs, rows, k)
            assert d_got.tobytes() == retry.tobytes() and np.array_equal(d_rows, want_rows[:, :k]), k
        if keep.any():
            plain, plain_rows = eng.schedule_batch_fallbacks(ep, seed, np.ascontiguousarray(reqs[keep]), k)
            assert got[keep].tobytes() == plain.tobytes() and np.array_equal(got_rows[keep], plain_rows), k
    for i in np.flatnonzero(want["status"] == N.LIG_OK):      # no entry excluded, entries distinct
        ranked = [int(want["pod_idx"][i])] + [int(x) for x in want_rows[i] if x >= 0]
        assert len(set(ranked)) == len(ranked) and not set(ranked) & set(rows[i].tolist())
    return want, want_rows


def int16_templates(tpl):
    """Row templates without the entries an int16 cannot hold (at P = 32768 every int16 >= 0 is a pod)."""
    return [[v for v in t if -32768 <= v <= 32767] for t in tpl]


# ---- pools and trees --------------------------------------------------------------------------------------
POOLS = [(1, 4), (31, 4), (32, 4), (33, 4), (64, 32), (512, 256), (4096, 1024), (4097, 64), (UNSTAGED_P, 16),
         (WIDEST_P, 16)]


@pytest.mark.parametrize("P,A", POOLS)
def test_pools_built_in_tree(P, A, eng):
    rng = np.random.default_rng(P + 100)
    snap = WL.make_snapshot(P, A, seed=P + 3).packed
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    tpl = int16_templates(row_templates(eng, ep, snap, rng))
    R = 64 if P < UNSTAGED_P else 24
    for width in (1, 9, 32):
        reqs = class_reqs(A, R, rng)
        check(eng, ep, SEED + width, snap, reqs, rows_for(tpl, R, width, rng))


def default_filter():
    return S.DEFAULT_FILTER.flatten()


@pytest.mark.parametrize("P,A", [(1, 4), (33, 4), (512, 256), (4096, 1024), (UNSTAGED_P, 16), (WIDEST_P, 16)])
@pytest.mark.parametrize("tree", ["default_filter", "keep_all", "drop_and_no_pods", "no_pods"])
def test_pools_caller_trees(P, A, tree, eng):
    if P == WIDEST_P and tree not in ("keep_all",):
        pytest.skip("the widest pool runs with the tree whose rows always fill")
    nodes = {"default_filter": default_filter(), "keep_all": KEEP_ALL, "drop_and_no_pods": DROP_AND_NO_PODS,
             "no_pods": NO_PODS_TREE}[tree]
    rng = np.random.default_rng(P + 17)
    snap = WL.make_snapshot(P, A, seed=P + 4).packed
    ep = next_epoch()
    eng.set_filter_tree(nodes)
    try:
        eng.upload_snapshot(ep, snap)
    finally:
        eng.set_filter_tree(None)
    tpl = int16_templates(row_templates(eng, ep, snap, rng))
    R = 48 if P < UNSTAGED_P else 12
    for width in (1, 32):
        reqs = class_reqs(A, R, rng)
        got, rows = check(eng, ep, SEED, snap, reqs, rows_for(tpl, R, width, rng), nodes=nodes)
        if tree == "keep_all" and P > X + K:   # every survivor set is P minus the excluded pods: rows fill
            full = got["n_survivors"] > K
            assert full.any() and (rows[full] >= 0).all()


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
        got, rows = check(eng, ep, SEED, snap, reqs, everything, nodes=nodes)
        assert (got["pod_idx"] == -1).all() and (got["n_survivors"] == 0).all() and (rows == -1).all()
        seen |= set(got["status"].tolist())
    assert seen == {N.LIG_DROP, N.LIG_NO_PODS_LEFT, N.LIG_EMPTY}


def test_rows_that_exclude_nothing_are_the_class_table_rows(eng):
    """A C4 pool: the walk over the full pool against the class tables, request by request."""
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=23).packed
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    reqs = WL.make_requests(20000, c["A"], seed=24)
    nothing = np.tile(np.array([-1, snap.P, 32767, -32768], dtype=np.int16), (len(reqs), 1))
    for k in (1, 4, K):
        want, want_rows = eng.schedule_batch_fallbacks(ep, SEED, reqs, k)
        got, rows = eng.schedule_batch_excluding_fallbacks(ep, SEED, reqs, nothing, k)
        assert got.tobytes() == want.tobytes() and np.array_equal(rows, want_rows), k
        d_got, d_rows = device_call(eng, ep, SEED, reqs, nothing, k)
        assert d_got.tobytes() == want.tobytes() and np.array_equal(d_rows, want_rows), k
    assert (rows >= 0).sum() > len(reqs)


def forced_epoch(eng, n):
    P = n + 3
    snap = WL.make_snapshot(P, 4, seed=n).packed
    ep = next_epoch()
    eng.set_filter_tree(KEEP_ALL)
    try:
        eng.upload_snapshot(ep, snap)
    finally:
        eng.set_filter_tree(None)
    row = np.array([0, P // 2, P - 1], dtype=np.int16)
    return snap, ep, row


def test_forced_int31n_rejection_on_the_pick(eng):
    for n in rejection_heavy_ns(40, 4000, 2):
        snap, ep, row = forced_epoch(eng, n)
        rng = np.random.default_rng(n)
        reqs = np.zeros(64, dtype=REQ_DTYPE)
        reqs["rand_key"] = pick_keys(SEED, rng.integers(accept_top(n), 1 << 31, size=64), rng)
        got, _ = check(eng, ep, SEED, snap, reqs, np.tile(row, (64, 1)), nodes=KEEP_ALL)
        assert (got["n_survivors"] == n).all() and (got["status"] == N.LIG_OK).all()


def test_forced_int31n_rejection_on_a_ranking_step(eng):
    for n1 in rejection_heavy_ns(40, 4000, 2):
        n = n1 + 1
        snap, ep, row = forced_epoch(eng, n)
        v = np.random.default_rng(n).integers(accept_top(n1), 1 << 31, size=256)
        with np.errstate(over="ignore"):
            keys = (states_for(v) - np.uint64(GAMMA)) ^ np.uint64(SEED & M64)
        kept = RR.kept_pods(snap.P, row)
        _, _, _, rejects = fallback_rows(SEED, keys, np.ones(len(keys), bool), np.zeros(len(keys), np.int64),
                                         np.full(len(keys), n), kept, K, with_draws=True)
        hit = (rejects[:, 0] == 0) & (rejects[:, 1] >= 1)
        assert hit.sum() >= 32, n
        reqs = np.zeros(int(hit.sum()), dtype=REQ_DTYPE)
        reqs["rand_key"] = keys[hit]
        got, _ = check(eng, ep, SEED, snap, reqs, np.tile(row, (len(reqs), 1)), nodes=KEEP_ALL)
        assert (got["n_survivors"] == n).all()


# ---- epochs, thresholds, refusals -------------------------------------------------------------------------
def test_delta_epoch_and_threshold_rebuild(eng):
    P, A = 1000, 64
    rng = np.random.default_rng(25)
    snap = WL.make_snapshot(P, A, seed=26).packed
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
    reqs = class_reqs(A, 96, rng)
    rows = rows_for([[int(d) for d in dirty[:9]], [int(dirty[0])], [], [31, 32, P - 1]], 96, 9, rng)
    check(eng, new, SEED, updated, reqs, rows)
    eng.set_thresholds(0.5, 3, 20)      # rebuilds the resident epoch in place
    try:
        check(eng, new, SEED, updated, reqs, rows, (0.5, 3, 20))
    finally:
        eng.set_thresholds()
    check(eng, new, SEED, updated, reqs, rows)


def test_refusals_leave_buffers_untouched():
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=16)
    try:
        reqs = class_reqs(8, 16, np.random.default_rng(1))
        rows = np.full((16, X + 1), -1, dtype=np.int16)
        out = np.full(16 * 8, 0x7B, dtype=np.uint8)
        fb = np.full(16 * (K + 1), 0x7B7B, dtype=np.int16)
        p = lambda a: a.ctypes.data

        def refused(code, fn, text="lig_schedule_batch_excluding_fallbacks"):
            with pytest.raises(N.LigError) as err:
                fn()
            assert err.value.code == code
            assert (out == 0x7B).all() and (fb == 0x7B7B).all()
            if code == N.LIG_ERR_INVALID:
                assert text in str(err.value)

        call = lambda ep, r, R, x, nx, o, nf, f: e.schedule_batch_excluding_fallbacks_ptr(ep, 2, r, R, x, nx, o, nf, f)
        refused(N.LIG_ERR_NO_SNAPSHOT, lambda: call(1, p(reqs), 16, p(rows), 1, p(out), 1, p(fb)))
        e.upload_snapshot(1, WL.make_snapshot(40, 8, seed=2).packed)
        refused(N.LIG_ERR_STALE_EPOCH, lambda: call(9, p(reqs), 16, p(rows), 1, p(out), 1, p(fb)))
        for nx, nf in ((0, 1), (X + 1, 1), (-3, 1), (1, 0), (1, K + 1), (1, -1)):
            refused(N.LIG_ERR_INVALID, lambda: call(1, p(reqs), 16, p(rows), nx, p(out), nf, p(fb)))
        for args in ((0, p(rows), p(out), p(fb)), (p(reqs), 0, p(out), p(fb)), (p(reqs), p(rows), 0, p(fb)),
                     (p(reqs), p(rows), p(out), 0)):
            refused(N.LIG_ERR_INVALID, lambda: call(1, args[0], 16, args[1], 1, args[2], 2, args[3]))
        big = class_reqs(8, 17, np.random.default_rng(2))
        big_rows = np.full((17, 1), -1, dtype=np.int16)
        refused(N.LIG_ERR_INVALID, lambda: call(1, p(big), 17, p(big_rows), 1, p(out), 1, p(fb)), "max_batch")
        # device form: each misaligned buffer, a stale epoch
        d_in, d_rows = dev(reqs), torch.full((16 * 2 + 1,), -1, dtype=torch.int16, device="cuda")
        d_out = torch.full((16 * 8 + 8,), 0x7B, dtype=torch.uint8, device="cuda")
        d_fb = torch.full((16 * 2 + 2,), 0x7B, dtype=torch.uint8, device="cuda")
        a0, b0, c0, f0 = d_in.data_ptr(), d_rows.data_ptr(), d_out.data_ptr(), d_fb.data_ptr()
        for a, b, c, f in ((a0 + 8, b0, c0, f0), (a0, b0 + 1, c0, f0), (a0, b0, c0 + 4, f0), (a0, b0, c0, f0 + 1)):
            refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_fallbacks_device(1, 2, a, 16, b, 2, c, 1, f),
                    "lig_schedule_batch_excluding_fallbacks_device")
        for nx, nf in ((0, 1), (1, 0), (1, K + 1)):
            refused(N.LIG_ERR_INVALID, lambda: e.schedule_batch_excluding_fallbacks_device(1, 2, a0, 16, b0, nx, c0,
                                                                                           nf, f0))
        refused(N.LIG_ERR_STALE_EPOCH, lambda: e.schedule_batch_excluding_fallbacks_device(7, 2, a0, 16, b0, 2, c0,
                                                                                           1, f0))
        torch.cuda.synchronize()
        assert (d_out.cpu().numpy() == 0x7B).all() and (d_fb.cpu().numpy() == 0x7B).all()
        call(1, 0, 0, 0, 1, 0, 1, 0)      # R = 0 is a no-op
    finally:
        e.close()


def test_feedback_chain_is_neither_ended_nor_advanced():
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=27).packed
    reqs = WL.make_requests(600, c["A"], seed=28)
    a, b = np.ascontiguousarray(reqs[:300]), np.ascontiguousarray(reqs[300:])
    rows = np.tile(np.array([0, 3, -1], dtype=np.int16), (len(reqs), 1))
    e = Engine(0, max_pods=64, max_adapters=32, max_batch=4096)
    try:
        e.upload_snapshot(1, snap)
        want = [e.schedule_batch_feedback_chain(1, 5, a, 100), e.schedule_batch_feedback_chain(1, 5, b, 100)]
        e.feedback_chain_reset()
        got = [e.schedule_batch_feedback_chain(1, 5, a, 100)]
        picks, _ = e.schedule_batch_excluding_fallbacks(1, 5, reqs, rows, K)
        got.append(e.schedule_batch_feedback_chain(1, 5, b, 100))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got, want))
        assert picks.tobytes() == e.schedule_batch_excluding(1, 5, reqs, rows).tobytes()   # the resident epoch
    finally:
        e.close()


# ---- buffers and streams ----------------------------------------------------------------------------------
def test_buffer_kinds_and_two_streams(eng):
    P, A, R, w, k = 512, 256, 1500, 9, 5
    rng = np.random.default_rng(29)
    snap = WL.make_snapshot(P, A, seed=30).packed
    ep = next_epoch()
    eng.upload_snapshot(ep, snap)
    reqs = WL.make_requests(R, A, seed=31)
    rows = rows_for(row_templates(eng, ep, snap, rng), R, w, rng)
    want, want_rows = check(eng, ep, SEED, snap, reqs, rows, ks=(k,), device=False)
    for mask in range(81):
        kinds = [mask // 3 ** i % 3 for i in range(4)]   # 0 pageable, 1 page-locked, 2 page-locked misaligned
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
            fb, pfb = mk(kinds[3], np.zeros((R, k), np.int16), 1)
            eng.schedule_batch_excluding_fallbacks_ptr(ep, SEED, pin, R, prows, w, pout, k, pfb)
            assert out.tobytes() == want.tobytes(), kinds
            assert fb.tobytes() == want_rows.tobytes(), kinds
            assert h_in.tobytes() == reqs.tobytes() and h_rows.tobytes() == rows.tobytes()
        finally:
            for b in bufs:
                b.free()
    d_in, d_rows = dev(reqs), torch.from_numpy(rows.reshape(-1).copy()).cuda()
    torch.cuda.synchronize()
    outs = []
    for s in (torch.cuda.Stream(), torch.cuda.Stream()):
        o = torch.zeros(R * 8, dtype=torch.uint8, device="cuda")
        f = torch.zeros(R * k, dtype=torch.int16, device="cuda")
        eng.schedule_batch_excluding_fallbacks_device(ep, SEED, d_in.data_ptr(), R, d_rows.data_ptr(), w,
                                                      o.data_ptr(), k, f.data_ptr(), s.cuda_stream)
        outs.append((o, f))
    torch.cuda.synchronize()
    for o, f in outs:
        assert o.cpu().numpy().tobytes() == want.tobytes() and f.cpu().numpy().tobytes() == want_rows.tobytes()


# ---- schedulers -------------------------------------------------------------------------------------------
def expect_ranked(pods, seed, key, model, critical, tried, k, nodes=None):
    """(pods [pick, row...], status) by the definition for one retry over the provider slice `pods`."""
    snap = pack_pod_metrics(pods)
    row = [p for p, pm in enumerate(pods) if pm.Pod in set(tried)] or [-1]
    reqs = np.zeros(1, dtype=REQ_DTYPE)
    reqs[0] = (snap.adapter_id(model), int(critical), key)
    pk, rows = RF.retry_fallback_batch(snap, reqs, np.array([row], dtype=np.int16), seed, k, nodes=nodes)
    if pk[0]["status"] != N.LIG_OK:
        return [], int(pk[0]["status"])
    return [snap.pods[int(pk[0]["pod_idx"])]] + [snap.pods[int(p)] for p in rows[0] if p >= 0], N.LIG_OK


@pytest.mark.parametrize("tree", [None, "keep_all"])
def test_python_scheduler(tree):
    import random
    nodes = None if tree is None else S.Filter("keep all", S.LOW_QUEUEING, queue_threshold=1 << 62)
    flat = None if nodes is None else nodes.flatten()
    pods = pool_pods()
    prov = StaticProvider(pods)
    sched = S.NewScheduler(prov, filter=nodes, max_pods=64, max_adapters=8, max_batch=256, seed=5)
    keys = random.Random(5)
    keys.getrandbits(64)                                  # the scheduler's seed
    try:
        req = S.LLMRequest(ResolvedTargetModel="a", Critical=True)
        first = sched.Schedule(req)
        keys.getrandbits(64)
        prov.pods = pods[::-1]                            # the provider reorders its slice
        tried = [first, Pod("ghost", "nowhere")]          # a pod that left the pool is ignored
        got = sched.ScheduleRetryWithFallbacks(req, tried, 4)
        want, _ = expect_ranked(prov.pods, sched._seed, keys.getrandbits(64), "a", True, tried, 4, flat)
        assert got == want and first not in got and len(got) >= 1
        # a plain retry takes the next key of the same sequence
        plain = sched.ScheduleRetry(req, tried)
        want, _ = expect_ranked(prov.pods, sched._seed, keys.getrandbits(64), "a", True, tried, 1, flat)
        assert plain == want[0]
        reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "zz") for c in (False, True)]
        tried_lists = [[pm.Pod for pm in prov.pods[:w]] for w in (0, 1, 5, 9, 31, 32)]
        for n in (1, 8):
            got = sched.ScheduleBatchRetryWithFallbacks(reqs, tried_lists, n)
            for r, t, (ranked, err) in zip(reqs, tried_lists, got):
                want, st = expect_ranked(prov.pods, sched._seed, keys.getrandbits(64), r.ResolvedTargetModel,
                                         r.Critical, t, n, flat)
                assert ranked == want and (err is None) == (st == N.LIG_OK)
                if err is not None:
                    assert str(err) == str(S._schedule_error(st))
                assert not set(ranked) & set(t) and len(ranked) <= n + 1
        # the batch retry after these calls takes the next keys
        after = sched.ScheduleBatchRetry(reqs[:2], tried_lists[:2])
        for r, t, (pod, _) in zip(reqs[:2], tried_lists[:2], after):
            want, _ = expect_ranked(prov.pods, sched._seed, keys.getrandbits(64), r.ResolvedTargetModel, r.Critical,
                                    t, 1, flat)
            assert pod == (want[0] if want else None)
        for bad in (0, K + 1):
            with pytest.raises(ValueError):
                sched.ScheduleRetryWithFallbacks(req, [], bad)
        with pytest.raises(ValueError):
            sched.ScheduleRetryWithFallbacks(req, [pm.Pod for pm in prov.pods[:X + 1]], 2)
    finally:
        sched.close()
    for retries in (False, True):
        chain = S.NewScheduler(StaticProvider(pods), load_feedback_window=4, feedback_retries=retries, max_pods=64,
                               max_adapters=8, seed=5)
        try:
            with pytest.raises(ValueError, match="load_feedback_window"):
                chain.ScheduleRetryWithFallbacks(S.LLMRequest(ResolvedTargetModel="a"), [], 2)
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
        for model, crit, width, n in (("a", True, 1, 8), ("b", False, 9, 3), ("zz", True, 32, 1), ("a", False, 0, 8)):
            tried = [first] + [pm.Pod for pm in prov.pods[:max(width - 1, 0)]] if width else [Pod("ghost", "x")]
            code, names, err = hs.ScheduleRetryWithFallbacks(model, crit, tried, n)
            want, st = expect_ranked(prov.pods, seed, int(keys[k]), model, crit, tried, n)
            k += 1
            assert names == [p.Name for p in want], (model, crit, width)
            assert (code == H.GRPC_OK) == (st == N.LIG_OK)
            if st == N.LIG_DROP:
                assert code == H.GRPC_RESOURCE_EXHAUSTED
        code, pod, _ = hs.ScheduleRetry("a", True, [first])       # the next key, the same lane
        want, _ = expect_ranked(prov.pods, seed, int(keys[k]), "a", True, [first], 1)
        assert pod == (want[0] if want else None)
        st = hs.stats()
        assert st["retry_scheduled"] == 5 and st["fallback_scheduled"] == 0
        for tried, n in (([], 0), ([], K + 1), ([pm.Pod for pm in prov.pods[:X + 1]], 2)):
            code, names, err = hs.ScheduleRetryWithFallbacks("a", True, tried, n)
            assert code == 3 and names == [] and "ScheduleRetryWithFallbacks" in err
        assert hs.stats()["retry_scheduled"] == 5
    finally:
        hs.close()
    for retries in (False, True):
        chain = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=8,
                                feedback_retries=retries)
        try:
            code, names, err = chain.ScheduleRetryWithFallbacks("a", False, [], 2)
            assert code == 3 and "load_feedback_window" in err
        finally:
            chain.close()
    prov.close()


def test_cpp_runtime_mixes_retry_and_retry_with_fallbacks_callers():
    """Concurrent callers folded into shared flushes: plain ScheduleRetry callers get the picks the
    fallback call makes, and every caller's pods are the pick and a row prefix of one key."""
    from llm_instance_gateway_b200 import host as H
    P = 64
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)])
    tried = [pm.Pod for pm in pods[:3]]
    seed = 0x2468
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200,
                         seed=seed, filter=KEEP_ALL)
    results = []
    lock = threading.Lock()

    def caller(t):
        mine = []
        for j in range(40):
            n = (t + j) % 9           # 0: ScheduleRetry
            if n == 0:
                code, pod, _ = hs.ScheduleRetry("a", False, tried)
                mine.append((0, code, [pod.Name] if pod else []))
            else:
                code, names, _ = hs.ScheduleRetryWithFallbacks("a", False, tried, n)
                mine.append((n, code, names))
        with lock:
            results.extend(mine)

    try:
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(12)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        total = len(results)
        assert total == 480 and all(code == H.GRPC_OK for _, code, _ in results)
        st = hs.stats()
        assert st["retry_scheduled"] == total and st["fallback_scheduled"] == 0
        assert st["batches"] < total                   # callers were folded into shared flushes
        e = Engine(0, max_pods=P, max_adapters=8, max_batch=4096)
        try:
            e.set_filter_tree(KEEP_ALL)
            e.upload_snapshot(1, pack_pod_metrics(pods))
            reqs = np.zeros(total, dtype=REQ_DTYPE)
            reqs["rand_key"] = splitmix_keys(seed, total)
            reqs["adapter_id"] = 1                      # any adapter: the tree keeps every pod
            rows = np.tile(np.arange(3, dtype=np.int16), (total, 1))
            picks = e.schedule_batch_excluding(1, seed, reqs, rows)
            out, fb = e.schedule_batch_excluding_fallbacks(1, seed, reqs, rows, K)
            assert out.tobytes() == picks.tobytes()
        finally:
            e.close()
        name = lambda i: f"pod-{i}"
        expect = [[name(picks["pod_idx"][j])] + [name(p) for p in fb[j] if p >= 0] for j in range(total)]
        assert sorted(r[2][0] for r in results) == sorted(x[0] for x in expect)
        prefixes = {tuple(x[:m]) for x in expect for m in range(1, K + 2)}
        for n, _, names in results:
            assert len(names) == n + 1 if n else len(names) == 1
            assert tuple(names) in prefixes and not {"pod-0", "pod-1", "pod-2"} & set(names)
    finally:
        hs.close()
        prov.close()
