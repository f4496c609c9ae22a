"""Fallback endpoints (lig_schedule_batch_fallbacks[_device], lig_schedule_models_batch_fallbacks[_device]):
`out` byte for byte the schedule calls' picks for every n, the rows against the definition
(fallback_ref.py) built from the survivor lists lig_read_class or lig_filter_batch return, on the built-in tree, caller
trees, edge pools and shapes, compact-pool overflow and delta epochs, forced Int31n rejections and
power-of-two steps; buffer kinds and streams, a model upload behind a queued call, refusals, and the
Python and C++ schedulers."""
import threading

import numpy as np
import pytest
import torch

from draw_keys import GAMMA, M64, accept_top, pick_keys, rejection_heavy_ns, states_for
from fallback_ref import fallback_rows
from test_gpu_filter_batch import Pinned, StaticProvider, class_tables, dev, im, scheduler_pods
from test_gpu_filter_tree import EDGE_POOLS, c4_tree, class_requests, mkpods
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_columns, pack_models, \
    pack_pod_metrics

pytestmark = pytest.mark.gpu

K = N.LIG_MAX_FALLBACKS
ALL_N = tuple(range(1, K + 1))
# a caller tree of one predicate node that keeps every pod whose queue is below 2^62: full rows
KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]
DROP_AND_NO_PODS = [N.LigFilterNode(N.LIG_F_CRITICAL_REQUEST, 1, 2, -1, 0, 0.0),
                    N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0),
                    N.LigFilterNode(N.LIG_F_DROP, -1, -1, -1, 0, 0.0)]


def model_keys(first_index, R):
    with np.errstate(over="ignore"):
        return np.uint64(first_index & M64) + np.arange(R, dtype=np.uint64)


def fb_device(eng, ep, seed, data, n, first_index=0, stream=0):
    """The device form with torch buffers: (picks, rows (R, n))."""
    R = len(data)
    models = data.dtype == np.uint32
    d_in = dev(data) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_out = torch.full((max(R, 1) * (4 if models else 8),), 0xAB, dtype=torch.uint8, device="cuda")
    d_rows = torch.full((max(R * n, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
    if models:
        eng.schedule_models_batch_fallbacks_device(ep, seed, first_index, d_in.data_ptr(), R, d_out.data_ptr(), n,
                                                   d_rows.data_ptr(), stream)
    else:
        eng.schedule_batch_fallbacks_device(ep, seed, d_in.data_ptr(), R, d_out.data_ptr(), n, d_rows.data_ptr(),
                                            stream)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()[: R * (4 if models else 8)].view(MPICK_DTYPE if models else PICK_DTYPE)
    return out, d_rows.cpu().numpy()[: R * n].reshape(R, n)


def expected(eng, ep, seed, data, first_index=0, A=None, P=None):
    """(picks of the schedule call, rows for n = K by the definition).  The lists are the class
    tables lig_read_class returns (one list per class, shared by its requests; model ids resolved by
    lig_resolve_models), or with A = None the CSR of lig_filter_batch."""
    R = len(data)
    models = data.dtype == np.uint32
    if models:
        picks = eng.schedule_models_batch(ep, seed, data, first_index)
        keys = model_keys(first_index, R)
    else:
        picks = eng.schedule_batch(ep, seed, data)
        keys = data["rand_key"]
    ok = picks["status"] == N.LIG_OK
    if A is None:
        fp, offsets, pods = (eng.filter_models_batch(ep, seed, data, first_index) if models
                             else eng.filter_batch(ep, seed, data))
        assert fp.tobytes() == picks.tobytes()
        starts, counts = offsets[:-1], np.diff(offsets)
    else:
        reqs = eng.resolve_models(ep, seed, data, first_index)[0] if models else data
        tables = class_tables(eng, ep, A, P)
        ncls = np.array([len(l) for _, l in tables], dtype=np.int64)
        pods = np.concatenate([l for _, l in tables] + [np.zeros(0, np.uint16)]).astype(np.int64)
        first = np.concatenate([[0], np.cumsum(ncls)])[:-1]
        c = (reqs["flags"] & 1).astype(np.int64) * (A + 1) + np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)
        starts, counts = first[c], ncls[c]
        if not models:
            assert np.array_equal(np.where(ok, counts, 0), np.where(ok, picks["n_survivors"], 0))
    rows, r0 = fallback_rows(seed, keys, ok, starts, counts, pods, K)
    # the definition's step 0 is the pick
    idx = np.where(ok, starts + np.maximum(r0, 0), 0)
    assert np.array_equal(np.where(ok, pods.astype(np.int64)[idx] if len(pods) else -1, -1),
                          picks["pod_idx"].astype(np.int64))
    return picks, rows


def check(eng, ep, seed, data, first_index=0, ns=ALL_N, device=True, A=None, P=None):
    """Host (pageable) and device forms for every n against the schedule call and the definition."""
    picks, rows = expected(eng, ep, seed, data, first_index, A, P)
    models = data.dtype == np.uint32
    for n in ns:
        if models:
            out, got = eng.schedule_models_batch_fallbacks(ep, seed, data, n, first_index)
        else:
            out, got = eng.schedule_batch_fallbacks(ep, seed, data, n)
        assert out.tobytes() == picks.tobytes(), n
        assert np.array_equal(got, rows[:, :n]), n
        if device:
            dout, dgot = fb_device(eng, ep, seed, data, n, first_index)
            assert dout.tobytes() == picks.tobytes() and np.array_equal(dgot, rows[:, :n]), n
    return picks, rows


_ep = [1000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=4096, max_adapters=1024, max_batch=1 << 20)
    yield e
    e.close()


# ---- built-in tree and caller trees at the bench configurations ---------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C3", "C4"])
def test_configs(cfg, eng):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"])
    reqs = WL.make_requests(c["R"], c["A"])
    ids = WL.make_model_requests(c["R"], c["A"])
    for tree in (None, KEEP_ALL):
        eng.set_filter_tree(tree)
        try:
            ep = next_epoch()
            eng.upload_snapshot(ep, snap.packed)
            eng.upload_models(ep, pack_models(WL.make_models(c["A"]), snap.packed))
        finally:
            eng.set_filter_tree(None)
        picks, rows = check(eng, ep, 0xC0FFEE, reqs, A=c["A"], P=c["P"])
        n = picks["n_survivors"].astype(np.int64)
        ok = picks["status"] == N.LIG_OK
        assert np.array_equal((rows >= 0).sum(axis=1), np.where(ok, np.minimum(n, K + 1) - 1, 0))
        if tree is not None:
            assert (rows[:, -1] >= 0).mean() > 0.9      # the rows are mostly full
        check(eng, ep, 0xC0FFEE, ids, first_index=(1 << 64) - 77, A=c["A"], P=c["P"])
        if cfg != "C4" or tree is None:     # the same rows from lig_filter_batch's lists
            assert np.array_equal(expected(eng, ep, 0xC0FFEE, reqs)[1], rows)


def test_caller_tree_at_C4_and_drop_leaves(eng):
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    reqs = WL.make_requests(1 << 18, c["A"], seed=4)
    eng.set_filter_tree(c4_tree())
    try:
        ep = next_epoch()
        eng.upload_snapshot(ep, snap.packed)
    finally:
        eng.set_filter_tree(None)
    check(eng, ep, 0xC4, reqs, ns=(1, 5, 8), A=c["A"], P=c["P"])
    # drop and "no pods left" leaves, descriptors and model ids
    pods = mkpods([0, 1, 2, 60, 3, 4], [0.1, 0.2, 0.3, 0.95, 0.4, 0.5], [2, 2, 1, 1, 2, 2],
                  [["a"], ["b"], ["a", "b"], [], ["a"], ["a"]])
    packed = pack_pod_metrics(pods)
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=8192)
    try:
        e.set_filter_tree(DROP_AND_NO_PODS)
        e.upload_snapshot(1, packed)
        pm = pack_models([im("m-a", [("a", 1)], critical=True), im("m-b", [("b", 2), ("zz", 1)]), im("m-self"),
                          im("m-none", [("zz", 1)], critical=True)], packed)
        e.upload_models(1, pm)
        reqs = class_requests(packed.A, copies=64)
        picks, rows = check(e, 1, 9, reqs)
        assert {N.LIG_OK, N.LIG_DROP, N.LIG_NO_PODS_LEFT} <= {int(s) for s in picks["status"]}
        assert (rows[picks["status"] != N.LIG_OK] == -1).all()
        ids = np.random.default_rng(2).integers(0, pm.n_models + 2, 3000).astype(np.uint32)
        mp, _ = check(e, 1, 9, ids, first_index=5)
        assert {N.LIG_OK, N.LIG_DROP, N.LIG_NO_PODS_LEFT, N.LIG_NO_MODEL} <= {int(s) for s in mp["status"]}
    finally:
        e.close()


# ---- pools and shapes -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(EDGE_POOLS))
def test_edge_pools(name, eng):
    packed = pack_pod_metrics(EDGE_POOLS[name])
    for tree in (None, KEEP_ALL):
        eng.set_filter_tree(tree)
        try:
            ep = next_epoch()
            eng.upload_snapshot(ep, packed)
        finally:
            eng.set_filter_tree(None)
        check(eng, ep, 77, class_requests(packed.A, copies=16))


@pytest.mark.parametrize("P,A", [(1, 1), (33, 5), (4097, 64), (20000, 64), (300, 0)])
def test_shapes(P, A):
    e = Engine(0, max_pods=max(P, 4096), max_adapters=max(A, 1), max_batch=1 << 16)
    try:
        packed = WL.make_snapshot(P, A, seed=P + 3).packed
        reqs = WL.make_requests(20000, A, seed=P + 4)
        for ep, tree in ((1, None), (2, KEEP_ALL)):
            e.set_filter_tree(tree)
            e.upload_snapshot(ep, packed)
            e.set_filter_tree(None)
            check(e, ep, 11, reqs, ns=(1, 2, 7, 8), A=A, P=P)
    finally:
        e.close()


def test_compact_overflow_and_delta_epochs():
    """Every affinity class owns a list of all P pods, so the compact pool overflows and the lists
    come from the strided rows; then a full epoch and a delta epoch on it."""
    P, A = 4096, 1024
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 16)
    try:
        W = (P + 31) // 32
        packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.full(P, 1, np.int64),
                              np.full(P, 2, np.int64), np.full((A, W), 0xFFFFFFFF, dtype=np.uint32))
        e.upload_snapshot(1, packed)
        assert e.pick_kernel_info(1)["table_bytes"] == 0      # the pool overflowed
        reqs = WL.make_requests(20000, A, seed=8)
        _, rows = check(e, 1, 3, reqs, A=A, P=P)
        assert (rows[:, -1] >= 0).mean() > 0.5
        e.upload_snapshot(2, WL.make_snapshot(P, A, seed=9).packed)
        check(e, 2, 3, reqs, A=A, P=P)
        rng = np.random.default_rng(10)
        dirty = np.sort(rng.choice(P, 300, replace=False)).astype(np.int32)
        acts = [rng.choice(A, int(rng.integers(0, 4)), replace=False) for _ in dirty]
        offs = np.concatenate([[0], np.cumsum([len(x) for x in acts])]).astype(np.int32)
        e.update_snapshot(3, 2, dirty, rng.random(300), rng.integers(0, 60, 300), [len(x) for x in acts],
                          np.full(300, 4), offs, np.concatenate(acts + [np.zeros(0, np.int64)]))
        check(e, 3, 3, reqs, A=A, P=P)
    finally:
        e.close()


# ---- the draws: power-of-two steps and forced rejections ----------------------------------------------
def keep_all_engine(P):
    e = Engine(0, max_pods=max(P, 64), max_adapters=1, max_batch=1 << 16)
    e.set_filter_tree(KEEP_ALL)
    e.upload_snapshot(1, pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64),
                                      np.zeros(P, np.int64), np.zeros((0, (P + 31) // 32), np.uint32)))
    return e


def reqs_with_keys(keys):
    reqs = np.zeros(len(keys), dtype=REQ_DTYPE)
    reqs["adapter_id"] = 0
    reqs["rand_key"] = keys
    return reqs


@pytest.mark.parametrize("P", [2, 5, 9, 12, 17, 36])
def test_power_of_two_steps(P):
    """Lists of n pods with n - j a power of two at some step j <= 8."""
    e = keep_all_engine(P)
    try:
        reqs = reqs_with_keys(np.random.default_rng(P).integers(0, 1 << 64, size=8192, dtype=np.uint64))
        picks, rows = check(e, 1, P, reqs)
        assert (picks["n_survivors"] == P).all()
        assert any((P - j) & (P - j - 1) == 0 for j in range(1, min(P, K + 1)))
    finally:
        e.close()


def test_forced_rejections_on_the_pick_and_on_a_fallback_step():
    seed = 0x5EED
    for n in rejection_heavy_ns(3, 4096, 3):
        e = keep_all_engine(n)
        try:
            rng = np.random.default_rng(n)
            # the pick's first draw rejected
            k_pick = pick_keys(seed, rng.integers(accept_top(n), 1 << 31, size=64), rng)
            # the second value of the stream (step 1's first draw) in Int31n(n - 1)'s rejection band
            v = rng.integers(accept_top(n - 1), 1 << 31, size=256)
            with np.errstate(over="ignore"):
                k_step = (states_for(v, rng) - np.uint64(GAMMA)) ^ np.uint64(seed)
            keys = np.concatenate([k_pick, k_step])
            _, _, _, rejects = fallback_rows(seed, keys, np.ones(len(keys), bool), np.zeros(len(keys), np.int64),
                                             np.full(len(keys), n), np.arange(n), K, with_draws=True)
            assert (rejects[:64, 0] >= 1).all()
            assert ((rejects[64:, 0] == 0) & (rejects[64:, 1] >= 1)).sum() >= 128
            check(e, 1, seed, reqs_with_keys(keys))
        finally:
            e.close()


# ---- buffers, streams, uploads, refusals ------------------------------------------------------------------
def test_buffer_kinds_and_two_streams(eng):
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"])
    ep = next_epoch()
    eng.set_filter_tree(KEEP_ALL)
    try:
        eng.upload_snapshot(ep, snap.packed)
    finally:
        eng.set_filter_tree(None)
    eng.upload_models(ep, pack_models(WL.make_models(c["A"]), snap.packed))
    reqs = WL.make_requests(5000, c["A"], seed=2)
    ids = WL.make_model_requests(5000, c["A"], seed=3)
    n = 6
    for models, data in ((False, reqs), (True, ids)):
        picks, rows = expected(eng, ep, 9, data, 17 if models else 0)
        rows = rows[:, :n]
        R = len(data)
        odt = MPICK_DTYPE if models else PICK_DTYPE
        # page-locked or pageable, and page-locked but misaligned (staged)
        for mask in range(27):
            kinds = [mask // 3 ** i % 3 for i in range(3)]   # 0 pageable, 1 page-locked, 2 misaligned
            bufs = []

            def mk(kind, count, dt, init=None):
                if kind == 0:
                    a = np.array(init) if init is not None else np.zeros(count, dt)
                    return a, a.ctypes.data
                shift = np.dtype(dt).itemsize // 2 if kind == 2 else 0   # half an element off
                b = Pinned(count * np.dtype(dt).itemsize + 16, np.uint8)
                bufs.append(b)
                raw = b.a[shift: shift + count * np.dtype(dt).itemsize]
                if init is not None:
                    raw[:] = np.frombuffer(np.ascontiguousarray(init).tobytes(), np.uint8)
                return raw, b.ptr + shift

            try:
                _, pin = mk(kinds[0], R, data.dtype, data)
                out, pout = mk(kinds[1], R, odt)
                rws, prows = mk(kinds[2], R * n, np.int16)
                if models:
                    eng.schedule_models_batch_fallbacks_ptr(ep, 9, 17, pin, R, pout, n, prows)
                else:
                    eng.schedule_batch_fallbacks_ptr(ep, 9, pin, R, pout, n, prows)
                assert out.tobytes() == picks.tobytes(), (models, kinds)
                assert np.frombuffer(rws.tobytes(), np.int16).reshape(R, n).tolist() == rows.tolist(), (models, kinds)
            finally:
                for b in bufs:
                    b.free()
        # two streams at once
        d_in = dev(data)
        torch.cuda.synchronize()
        outs = []
        for s in (torch.cuda.Stream(), torch.cuda.Stream()):
            o = torch.zeros(R * (4 if models else 8), dtype=torch.uint8, device="cuda")
            r = torch.zeros(R * n, dtype=torch.int16, device="cuda")
            if models:
                eng.schedule_models_batch_fallbacks_device(ep, 9, 17, d_in.data_ptr(), R, o.data_ptr(), n, r.data_ptr(),
                                                           s.cuda_stream)
            else:
                eng.schedule_batch_fallbacks_device(ep, 9, d_in.data_ptr(), R, o.data_ptr(), n, r.data_ptr(),
                                                    s.cuda_stream)
            outs.append((o, r))
        torch.cuda.synchronize()
        for o, r in outs:
            assert o.cpu().numpy().tobytes() == picks.tobytes()
            assert np.array_equal(r.cpu().numpy().reshape(R, n), rows)


def test_model_upload_while_a_device_call_is_queued():
    packed = pack_pod_metrics(mkpods([0] * 8, [0.1] * 8, [1] * 8, [["x"]] * 4 + [["y"]] * 4))
    old = pack_models([im("m", [("x", 1)], critical=True)], packed)
    new = pack_models([im("m", [("y", 1)])], packed)
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=4096)
    try:
        e.set_filter_tree([N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0)])
        e.upload_snapshot(1, packed)
        ids = np.zeros(3000, dtype=np.uint32)
        e.upload_models(1, old)
        want_old = e.schedule_models_batch_fallbacks(1, 4, ids, 8)
        e.upload_models(1, new)
        want_new = e.schedule_models_batch_fallbacks(1, 4, ids, 8)
        assert not np.array_equal(want_old[1], want_new[1])
        e.upload_models(1, old)
        st = torch.cuda.Stream()
        d_in = dev(ids)
        d_out = torch.zeros(3000 * 4, dtype=torch.uint8, device="cuda")
        d_rows = torch.zeros(3000 * 8, dtype=torch.int16, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(100_000_000)                 # keep the call queued behind ~50 ms of work
            e.schedule_models_batch_fallbacks_device(1, 4, 0, d_in.data_ptr(), 3000, d_out.data_ptr(), 8,
                                                     d_rows.data_ptr(), st.cuda_stream)
        e.upload_models(1, new)
        st.synchronize()
        assert d_out.cpu().numpy().view(MPICK_DTYPE).tobytes() == want_old[0].tobytes()
        assert np.array_equal(d_rows.cpu().numpy().reshape(3000, 8), want_old[1])
        got = e.schedule_models_batch_fallbacks(1, 4, ids, 8)
        assert got[0].tobytes() == want_new[0].tobytes() and np.array_equal(got[1], want_new[1])
    finally:
        e.close()


def test_refusals():
    lib = N.load()
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=100)
    try:
        snap = WL.make_snapshot(64, 8, seed=1)
        reqs = WL.make_requests(50, 8)
        ids = np.zeros(50, dtype=np.uint32)
        out, mout = np.zeros(50, PICK_DTYPE), np.zeros(50, MPICK_DTYPE)
        rows = np.full(50 * 8, 7, np.int16)
        p = lambda a: a.ctypes.data
        ctx = e._ctx
        # no snapshot yet
        assert lib.lig_schedule_batch_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), 2, p(rows)) == N.LIG_ERR_NO_SNAPSHOT
        e.upload_snapshot(1, snap.packed)
        # stale epoch
        assert lib.lig_schedule_batch_fallbacks(ctx, 2, 0, p(reqs), 50, p(out), 2, p(rows)) == N.LIG_ERR_STALE_EPOCH
        d_reqs, d_ids = dev(reqs), dev(ids)
        d_out = torch.zeros(50 * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.zeros(50 * 8, dtype=torch.int16, device="cuda")
        assert lib.lig_schedule_batch_fallbacks_device(ctx, 2, 0, d_reqs.data_ptr(), 50, d_out.data_ptr(), 2,
                                                       d_rows.data_ptr(), None) == N.LIG_ERR_STALE_EPOCH
        # no model table
        assert lib.lig_schedule_models_batch_fallbacks(ctx, 1, 0, 0, p(ids), 50, p(mout), 2,
                                                       p(rows)) == N.LIG_ERR_NO_SNAPSHOT
        assert lib.lig_schedule_models_batch_fallbacks_device(ctx, 1, 0, 0, d_ids.data_ptr(), 50, d_out.data_ptr(), 2,
                                                              d_rows.data_ptr(), None) == N.LIG_ERR_NO_SNAPSHOT
        e.upload_models(1, pack_models(WL.make_models(8), snap.packed))
        # n outside [1, 8], null buffers, negative R
        for nf in (0, 9, -1, 1 << 20):
            assert lib.lig_schedule_batch_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), nf, p(rows)) == N.LIG_ERR_INVALID
            assert lib.lig_schedule_models_batch_fallbacks_device(ctx, 1, 0, 0, d_ids.data_ptr(), 50, d_out.data_ptr(),
                                                                  nf, d_rows.data_ptr(), None) == N.LIG_ERR_INVALID
        for a, b, r, R in ((None, p(out), p(rows), 50), (p(reqs), None, p(rows), 50), (p(reqs), p(out), None, 50),
                           (p(reqs), p(out), p(rows), -1)):
            assert lib.lig_schedule_batch_fallbacks(ctx, 1, 0, a, R, b, 2, r) == N.LIG_ERR_INVALID
            assert lib.lig_schedule_batch_fallbacks_device(ctx, 1, 0, a, R, b, 2, r, None) == N.LIG_ERR_INVALID
            assert lib.lig_schedule_models_batch_fallbacks(ctx, 1, 0, 0, a, R, b, 2, r) == N.LIG_ERR_INVALID
        # device buffers not aligned to their element
        assert lib.lig_schedule_batch_fallbacks_device(ctx, 1, 0, d_reqs.data_ptr() + 8, 40, d_out.data_ptr(), 2,
                                                       d_rows.data_ptr(), None) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_fallbacks_device(ctx, 1, 0, d_reqs.data_ptr(), 40, d_out.data_ptr(), 2,
                                                       d_rows.data_ptr() + 1, None) == N.LIG_ERR_INVALID
        # R > max_batch on the host forms only
        big = WL.make_requests(101, 8)
        assert lib.lig_schedule_batch_fallbacks(ctx, 1, 0, p(big), 101, p(np.zeros(101, PICK_DTYPE)), 1,
                                                p(np.zeros(101, np.int16))) == N.LIG_ERR_INVALID
        assert b"max_batch" in lib.lig_last_error()
        assert lib.lig_schedule_models_batch_fallbacks(ctx, 1, 0, 0, p(np.zeros(101, np.uint32)), 101,
                                                       p(np.zeros(101, MPICK_DTYPE)), 1,
                                                       p(np.zeros(101, np.int16))) == N.LIG_ERR_INVALID
        # nothing was written by a refused call; R = 0 succeeds and writes nothing
        assert (rows == 7).all() and (out["pod_idx"] == 0).all()
        assert lib.lig_schedule_batch_fallbacks(ctx, 1, 0, None, 0, None, 3, None) == 0
        assert lib.lig_schedule_models_batch_fallbacks_device(ctx, 1, 0, 0, None, 0, None, 3, None, None) == 0
        torch.cuda.synchronize()
        with pytest.raises(N.LigError):
            e.schedule_batch_fallbacks(1, 0, reqs, 9)
    finally:
        e.close()


def test_feedback_chain_is_neither_ended_nor_advanced():
    """A fallback call between two chain calls leaves the chain's windows and loads as they were."""
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=21)
    reqs = WL.make_requests(600, c["A"], seed=22)
    a, b = np.ascontiguousarray(reqs[:300]), np.ascontiguousarray(reqs[300:])
    e = Engine(0, max_pods=64, max_adapters=32, max_batch=4096)
    try:
        e.upload_snapshot(1, snap.packed)
        want = [e.schedule_batch_feedback_chain(1, 5, a, 100), e.schedule_batch_feedback_chain(1, 5, b, 100)]
        e.feedback_chain_reset()
        got = [e.schedule_batch_feedback_chain(1, 5, a, 100)]
        picks, _ = check(e, 1, 5, reqs, ns=(8,))
        got.append(e.schedule_batch_feedback_chain(1, 5, b, 100))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got, want))
        assert picks.tobytes() == e.schedule_batch(1, 5, reqs).tobytes()   # the resident tables
    finally:
        e.close()


# ---- schedulers -------------------------------------------------------------------------------------
def test_python_scheduler():
    pods = scheduler_pods()
    reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "c", "zz", "") for c in (False, True)]
    reqs = reqs * 20
    models = [im("m-a", [("a", 1)]), im("m-split", [("a", 3), ("b", 5), ("c", 2)], critical=True), im("m-self"),
              im("m-zero", [("a", 0)]), im("b")]
    names = ["m-a", "m-split", "unknown", "m-zero", "m-self", "b", "m-split", "m-split"] * 10
    for tree in (None, S.Filter("all", S.LOW_QUEUEING, queue_threshold=1 << 40)):
        plain = S.NewScheduler(StaticProvider(pods), filter=tree, max_pods=64, max_adapters=8, max_batch=256, seed=5)
        fb = S.NewScheduler(StaticProvider(pods), filter=tree, max_pods=64, max_adapters=8, max_batch=256, seed=5)
        try:
            for n in (1, 3, 8):
                want = plain.ScheduleBatch(reqs)
                got = fb.ScheduleBatchWithFallbacks(reqs, n)
                for r, (pod, err), (ranked, ferr) in zip(reqs, want, got):
                    assert (err is None) == (ferr is None)
                    if err is not None:
                        assert (err.code, str(err)) == (ferr.code, str(ferr)) and ranked == []
                        continue
                    survivors, _ = fb.Filter(r)
                    names_ = [p.Name for p in ranked]
                    assert ranked[0] == pod and len(set(names_)) == len(names_)
                    assert len(ranked) == min(len(survivors), n + 1)
                    assert set(names_) <= {p.Name for p in survivors}
            # single requests raise like Schedule
            for r in reqs[:10]:
                try:
                    pod = plain.Schedule(r)
                except S.StatusError as err:
                    with pytest.raises(S.StatusError) as got_err:
                        fb.ScheduleWithFallbacks(r, 4)
                    assert str(got_err.value) == str(err)
                else:
                    assert fb.ScheduleWithFallbacks(r, 4)[0] == pod
            # model names: host-answered errors, resolved names and the rand_key sequence
            plain.SetInferenceModels(models)
            fb.SetInferenceModels(models)
            want = plain.ScheduleModelBatch(names)
            got = fb.ScheduleModelBatchWithFallbacks(names, 8)
            assert plain._model_index == fb._model_index
            for (pod, resolved, err), (ranked, fres, ferr) in zip(want, got):
                assert resolved == fres and (err is None) == (ferr is None)
                if err is None:
                    assert ranked[0] == pod and len({p.Name for p in ranked}) == len(ranked)
                else:
                    assert (err.code, str(err)) == (ferr.code, str(ferr)) and ranked == []
            with pytest.raises(ValueError):
                fb.ScheduleBatchWithFallbacks(reqs, 0)
            with pytest.raises(ValueError):
                fb.ScheduleModelBatchWithFallbacks(names, 9)
        finally:
            plain.close()
            fb.close()
    chain = S.NewScheduler(StaticProvider(pods), load_feedback_window=4, max_pods=64, max_adapters=8, seed=5)
    try:
        for call in (lambda: chain.ScheduleBatchWithFallbacks(reqs, 2), lambda: chain.ScheduleWithFallbacks(reqs[0], 2),
                     lambda: chain.ScheduleModelBatchWithFallbacks(names, 2)):
            with pytest.raises(ValueError, match="load_feedback_window"):
                call()
    finally:
        chain.close()


def splitmix_keys(seed, count):
    """The C++ runtime's rand_key sequence: splitmix_next(rng_state_), rng_state_ = seed ^ 0xD1B54A32D192ED03."""
    s = (seed ^ 0xD1B54A32D192ED03) & M64
    out = []
    for _ in range(count):
        s = (s + GAMMA) & M64
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        out.append(z ^ (z >> 31))
    return np.array(out, dtype=np.uint64)


def test_cpp_runtime_mixes_schedule_and_fallback_callers():
    from llm_instance_gateway_b200 import host as H
    P = 64
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)])
    seed = 0x1234
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200,
                         seed=seed, filter=KEEP_ALL)
    results = []
    lock = threading.Lock()

    def caller(t):
        mine = []
        for k in range(60):
            n = (t + k) % 9           # 0: Schedule
            if n == 0:
                code, pod, err = hs.Schedule("m", "a", False)
                mine.append((0, code, [pod.Name] if pod else []))
            else:
                code, names, err = hs.ScheduleWithFallbacks("a", False, n)
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
        assert total == 720 and all(code == H.GRPC_OK for _, code, _ in results)
        st = hs.stats()
        assert st["fallback_scheduled"] == sum(1 for n, _, _ in results if n > 0)
        assert st["batches"] < total                   # callers were folded into shared flushes
        # the same keys through the library: every caller holds the pick and the row prefix of one key
        e = Engine(0, max_pods=P, max_adapters=8, max_batch=4096)
        try:
            e.set_filter_tree(KEEP_ALL)
            e.upload_snapshot(1, pack_pod_metrics(pods))
            reqs = reqs_with_keys(splitmix_keys(seed, total))
            reqs["adapter_id"] = 1                      # any adapter: the tree keeps every pod
            picks = e.schedule_batch(1, seed, reqs)
            out, rows = e.schedule_batch_fallbacks(1, seed, reqs, K)
            assert out.tobytes() == picks.tobytes()
        finally:
            e.close()
        name = lambda i: f"pod-{i}"
        expect = [[name(picks["pod_idx"][k])] + [name(p) for p in rows[k] if p >= 0] for k in range(total)]
        assert sorted(r[2][0] for r in results) == sorted(x[0] for x in expect)
        free = {}
        for k, x in enumerate(expect):
            free.setdefault(tuple(x[:4]), []).append(k)
        used = set()
        for n, _, names in sorted(results, key=lambda r: -r[0]):
            if n < 3:
                continue
            assert len(names) == n + 1
            ks = [k for k in free.get(tuple(names[:4]), []) if k not in used and expect[k][:n + 1] == names]
            assert ks, names
            used.add(ks[0])
        # refusals
        assert hs.ScheduleWithFallbacks("a", False, 0)[0] == 3
        assert hs.ScheduleWithFallbacks("a", False, K + 1)[0] == 3
    finally:
        hs.close()
    chain = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=8)
    try:
        code, names, err = chain.ScheduleWithFallbacks("a", False, 2)
        assert code == 3 and "load_feedback_window" in err and names == []
    finally:
        chain.close()
        prov.close()
