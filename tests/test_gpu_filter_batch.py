"""Survivor lists of whole batches (lig_filter_batch[_device], lig_filter_models_batch[_device]): the
picks byte for byte those of the schedule calls they mirror, the CSR lists against the class tables
(lig_read_class), the direct scan's masks and the oracles, the capacity and offset contract, buffer
kinds and streams, refusals, and the Python and C++ schedulers' Filter calls."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import oracle_tree
from filter_tree_ref import random_pool, random_tree
from test_gpu_filter_tree import EDGE_POOLS, c4_tree, class_requests, mkpods, ref_tables
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import CRITICAL, InferenceModel, InferenceModelSpec, TargetModel
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models, pack_pod_metrics

pytestmark = pytest.mark.gpu

TILE = 1024          # requests per tile of the survivor-list kernel


def class_tables(eng, ep, A, P):
    """[(status, list)] per class c = critical * (A + 1) + a, read with lig_read_class."""
    rows = []
    for crit in (0, 1):
        for a in range(A + 1):
            st, _, lst = eng.read_class(ep, bool(crit), a, P)
            rows.append((st, lst.astype(np.uint16)))
    return rows


def expected_lists(tables, A, reqs, keep=None):
    """(offsets, pods) the contract gives for descriptors `reqs` with class tables `tables`; keep
    (bool per request, optional) empties the lists of the others (NO_MODEL)."""
    crit = (reqs["flags"] & 1).astype(np.int64)
    a = np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)
    c = crit * (A + 1) + a
    n_cls = np.array([len(l) if st == N.LIG_OK else 0 for st, l in tables], dtype=np.int64)
    pool = np.concatenate([l for _, l in tables] + [np.zeros(0, np.uint16)]).astype(np.uint16)
    start = np.concatenate([[0], np.cumsum([len(l) for _, l in tables])])[:-1].astype(np.int64)
    n = n_cls[c] if len(c) else np.zeros(0, np.int64)
    if keep is not None:
        n = np.where(keep, n, 0)
    offsets = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    total = int(offsets[-1])
    idx = np.repeat(start[c] - offsets[:-1], n) + np.arange(total, dtype=np.int64)
    return offsets, pool[idx]


def dev(a: np.ndarray):
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).cuda()


def filter_device(eng, ep, seed, data, capacity=None, first_index=None, stream=0, out_bytes=None):
    """The device form with torch buffers: (picks, offsets, pods[:offsets[R]] clipped to capacity)."""
    R = len(data)
    models = data.dtype == np.uint32
    d_in = dev(data) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_out = torch.full((max(R, 1) * (4 if models else 8),), 0xAB, dtype=torch.uint8, device="cuda")
    d_off = torch.full((R + 1,), -7, dtype=torch.int64, device="cuda")
    cap = 8 * R + 64 if capacity is None else capacity
    d_pods = torch.full((max(cap, 1),), 0xABCD - 65536, dtype=torch.int16, device="cuda")
    if models:
        eng.filter_models_batch_device(ep, seed, first_index or 0, d_in.data_ptr(), R, d_out.data_ptr(),
                                       d_off.data_ptr(), d_pods.data_ptr() if cap else 0, cap, stream)
    else:
        eng.filter_batch_device(ep, seed, d_in.data_ptr(), R, d_out.data_ptr(), d_off.data_ptr(),
                                d_pods.data_ptr() if cap else 0, cap, stream)
    torch.cuda.synchronize()
    offsets = d_off.cpu().numpy()
    out = d_out.cpu().numpy()[: R * (4 if models else 8)].view(MPICK_DTYPE if models else PICK_DTYPE)
    pods = d_pods.cpu().numpy().view(np.uint16)
    return out, offsets, pods[: min(int(offsets[R]), cap)], pods


def check_batch(eng, ep, seed, reqs, A, P, tables=None, device=True):
    """filter_batch (host, pageable) and the device form against schedule_batch and the class tables."""
    tables = tables if tables is not None else class_tables(eng, ep, A, P)
    want_off, want_pods = expected_lists(tables, A, reqs)
    picks, offsets, pods = eng.filter_batch(ep, seed, reqs)
    assert picks.tobytes() == eng.schedule_batch(ep, seed, reqs).tobytes()
    assert np.array_equal(offsets, want_off)
    assert np.array_equal(pods, want_pods)
    if device:
        dp, doff, dpods, _ = filter_device(eng, ep, seed, reqs, capacity=int(want_off[-1]))
        assert dp.tobytes() == picks.tobytes()
        assert np.array_equal(doff, want_off) and np.array_equal(dpods, want_pods)
    return picks, offsets, pods, tables


def check_scan(eng, ep, seed, reqs, P, W, offsets, pods):
    """The built-in tree: the lists equal the direct scan's masks (statuses other than OK: empty)."""
    picks, masks = eng.schedule_scan(ep, seed, reqs, True, W)
    for i in range(len(reqs)):
        lst = pods[offsets[i]:offsets[i + 1]].tolist()
        if picks[i]["status"] != N.LIG_OK:
            assert lst == [], i
            continue
        bits = [p for p in range(P) if (int(masks[i, p >> 5]) >> (p & 31)) & 1]
        assert lst == bits, i


def records_of(pods):
    """Oracle records of PodMetrics."""
    return [dict(name=p.Pod.Name, address=p.Pod.Address, waiting_queue_size=p.Metrics.WaitingQueueSize,
                 kv_cache_usage_percent=p.Metrics.KVCacheUsagePercent, max_active_models=p.Metrics.MaxActiveModels,
                 active_models=list(p.Metrics.ActiveModels)) for p in pods]


_ep = [0]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=4096, max_adapters=1024, max_batch=1 << 20)
    yield e
    e.close()


# ---- built-in tree --------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C3", "C4"])
def test_builtin_configs(cfg, eng):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"])
    ep = next_epoch()
    eng.upload_snapshot(ep, snap.packed)
    reqs = WL.make_requests(c["R"], c["A"])
    before = class_tables(eng, ep, c["A"], c["P"])
    _, offsets, pods, _ = check_batch(eng, ep, 0xC0FFEE, reqs, c["A"], c["P"], before)
    sub = np.ascontiguousarray(reqs[:2048])
    check_scan(eng, ep, 0xC0FFEE, sub, c["P"], snap.packed.W, offsets[:2049], pods)
    after = class_tables(eng, ep, c["A"], c["P"])             # resident tables untouched
    assert all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(before, after))


@pytest.mark.parametrize("name", sorted(EDGE_POOLS))
def test_builtin_edge_pools(name, eng):
    packed = pack_pod_metrics(EDGE_POOLS[name])
    ep = next_epoch()
    eng.upload_snapshot(ep, packed)
    reqs = class_requests(packed.A)
    _, offsets, pods, tables = check_batch(eng, ep, 77, reqs, packed.A, packed.P)
    check_scan(eng, ep, 77, reqs, packed.P, max(packed.W, 1), offsets, pods)
    # the port oracle's survivors (defaultFilter)
    names = [None] * packed.A + ["never-loaded"]
    for k, v in packed.adapter_ids.items():
        names[v] = k
    want = ref_tables(S.DEFAULT_FILTER.flatten(), records_of(EDGE_POOLS[name]), names)
    for crit in (0, 1):
        for a in range(packed.A + 1):
            st, lst = tables[crit * (packed.A + 1) + a]
            wst, widx = want[crit][a]
            assert (st, lst.tolist() if st == N.LIG_OK else []) == (wst, widx if wst == N.LIG_OK else []), (crit, a)


@pytest.mark.parametrize("P,A", [(0, 0), (1, 1), (33, 5), (4097, 64), (20000, 64), (300, 0)])
def test_builtin_shapes(P, A):
    e = Engine(0, max_pods=max(P, 1) if P > 4096 else 4096, max_adapters=max(A, 1), max_batch=1 << 16)
    try:
        snap = WL.make_snapshot(P, A, seed=P + 3) if P else None
        packed = snap.packed if snap else pack_pod_metrics([])
        e.upload_snapshot(1, packed)
        reqs = WL.make_requests(5000, A, seed=P + 4)
        _, offsets, pods, _ = check_batch(e, 1, 11, reqs, A, P)
        sub = np.ascontiguousarray(reqs[:256])
        check_scan(e, 1, 11, sub, P, max(packed.W, 1), offsets[:257], pods)
    finally:
        e.close()


def test_compact_overflow_and_delta_epochs():
    """Identical pods that serve every adapter: every affinity class owns a list of all P pods, so
    the compact pool overflows and the lists come from the strided rows; then a delta epoch."""
    P, A = 4096, 1024
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 16)
    try:
        W = (P + 31) // 32
        from llm_instance_gateway_b200.packer import pack_columns
        packed = pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.full(P, 1, np.int64),
                              np.full(P, 2, np.int64), np.full((A, W), 0xFFFFFFFF, dtype=np.uint32))
        e.upload_snapshot(1, packed)
        assert e.pick_kernel_info(1)["table_bytes"] == 0      # the pool overflowed
        reqs = WL.make_requests(2000, A, seed=8)
        _, offsets, _, _ = check_batch(e, 1, 3, reqs, A, P)
        assert offsets[-1] > 1000 * 2000
        base = WL.make_snapshot(P, A, seed=9).packed
        e.upload_snapshot(2, base)
        check_batch(e, 2, 3, reqs, A, P)
        rng = np.random.default_rng(10)
        dirty = np.sort(rng.choice(P, 300, replace=False)).astype(np.int32)
        acts = [rng.choice(A, int(rng.integers(0, 4)), replace=False) for _ in dirty]
        offs = np.concatenate([[0], np.cumsum([len(x) for x in acts])]).astype(np.int32)
        e.update_snapshot(3, 2, dirty, rng.random(300), rng.integers(0, 60, 300), [len(x) for x in acts],
                          np.full(300, 4), offs, np.concatenate(acts + [np.zeros(0, np.int64)]))
        check_batch(e, 3, 3, reqs, A, P)
    finally:
        e.close()


# ---- caller trees ---------------------------------------------------------------------------------
def test_random_caller_trees_against_oracle():
    e = Engine(0, max_pods=128, max_adapters=16, max_batch=4096)
    rng = np.random.default_rng(91)
    try:
        for it in range(80):
            tree = random_tree(rng)
            if it % 10 == 0:          # a drop leaf, and a predicate that keeps nothing
                tree = [N.LigFilterNode(N.LIG_F_LORA_AFFINITY, 1, -1, -1, 0, 0.0),
                        N.LigFilterNode(N.LIG_F_CRITICAL_REQUEST, 2, 3, -1, 0, 0.0),
                        N.LigFilterNode(N.LIG_F_LEAST_QUEUING, -1, -1, -1, 0, 0.0),
                        N.LigFilterNode(N.LIG_F_DROP, -1, -1, -1, 0, 0.0)]
            records = random_pool(rng)
            pods = mkpods([r["waiting_queue_size"] for r in records], [r["kv_cache_usage_percent"] for r in records],
                          [r["max_active_models"] for r in records], [r["active_models"] for r in records])
            packed = pack_pod_metrics(pods)
            names = [None] * packed.A + ["never-loaded"]
            for k, v in packed.adapter_ids.items():
                names[v] = k
            e.set_filter_tree(tree)
            ep = next_epoch()
            e.upload_snapshot(ep, packed)
            want = ref_tables(tree, records, names)
            tables = [(st, np.array(lst if st == N.LIG_OK else [], dtype=np.uint16))
                      for row in want for st, lst in row]
            reqs = class_requests(packed.A, seed=it)
            picks, _, _, got_tables = check_batch(e, ep, it, reqs, packed.A, packed.P, tables)
            assert {int(s) for s in picks["status"]} <= {N.LIG_OK, N.LIG_DROP, N.LIG_EMPTY, N.LIG_NO_PODS_LEFT}
            # lig_read_class agrees with the oracle too
            for (st, lst), (rst, rlst) in zip(tables, class_tables(e, ep, packed.A, packed.P)):
                assert st == rst and (st != N.LIG_OK or lst.tolist() == rlst.tolist())
    finally:
        e.close()


def test_caller_trees_at_C4(eng):
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    reqs = WL.make_requests(c["R"], c["A"])
    rng = np.random.default_rng(5)
    trees = [c4_tree().flatten()]
    while len(trees) < 3:          # random trees whose survivor sets differ between classes
        t = random_tree(rng)
        if any(n.kind in (N.LIG_F_LORA_AFFINITY, N.LIG_F_LOW_LORA_COST) for n in t):
            trees.append(t)
    try:
        for k, tree in enumerate(trees):
            eng.set_filter_tree(tree)
            ep = next_epoch()
            eng.upload_snapshot(ep, snap.packed)
            want = ref_tables(tree, snap.pod_records(), snap.adapter_names() + [WL.UNKNOWN_MODEL])
            tables = [(st, np.array(lst if st == N.LIG_OK else [], dtype=np.uint16)) for row in want for st, lst in row]
            # as many requests as keep the lists to ~2e7 entries (a random tree may keep most pods)
            mean_n = np.mean([len(l) for st, l in tables])
            R = int(min(c["R"], max(4096, 2e7 / max(mean_n, 1.0))))
            check_batch(eng, ep, 0xC4 + k, np.ascontiguousarray(reqs[:R]), c["A"], c["P"], tables)
    finally:
        eng.set_filter_tree(None)


# ---- model ids ------------------------------------------------------------------------------------
def im(name, targets=(), critical=False):
    return InferenceModel(Name=name, Spec=InferenceModelSpec(
        ModelName=name, Criticality=CRITICAL if critical else None,
        TargetModels=[TargetModel(Name=n, Weight=w) for n, w in targets]))


def check_models(e, ep, seed, ids, first_index, A, P):
    reqs, res = e.resolve_models(ep, seed, ids, first_index)
    keep = res["status"] == N.LIG_OK
    tables = class_tables(e, ep, A, P)
    want_off, want_pods = expected_lists(tables, A, reqs, keep)
    picks, offsets, pods = e.filter_models_batch(ep, seed, ids, first_index)
    assert picks.tobytes() == e.schedule_models_batch(ep, seed, ids, first_index).tobytes()
    assert np.array_equal(offsets, want_off) and np.array_equal(pods, want_pods)
    # the same lists as lig_filter_batch on the resolved descriptors
    _, doff, dpods = e.filter_batch(ep, seed, reqs)
    for i in np.flatnonzero(keep)[:4096]:
        assert pods[offsets[i]:offsets[i + 1]].tolist() == dpods[doff[i]:doff[i + 1]].tolist()
    mp, moff, mpods, _ = filter_device(e, ep, seed, ids, first_index=first_index, capacity=int(offsets[-1]))
    assert mp.tobytes() == picks.tobytes() and np.array_equal(moff, offsets) and np.array_equal(mpods, pods)
    return picks


def test_model_ids_configs():
    for cfg in ("C2", "C3"):
        c = WL.CONFIGS[cfg]
        e = Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=1 << 17)
        try:
            snap = WL.make_snapshot(c["P"], c["A"])
            e.upload_snapshot(1, snap.packed)
            e.upload_models(1, pack_models(WL.make_models(c["A"]), snap.packed))
            check_models(e, 1, 0xBEEF, WL.make_model_requests(c["R"], c["A"]), 12345, c["A"], c["P"])
        finally:
            e.close()


def test_model_table_edges():
    pods = mkpods([0, 1, 2, 60], [0.1, 0.2, 0.3, 0.95], [2, 2, 1, 1], [["a"], ["b"], ["a", "b"], []])
    packed = pack_pod_metrics(pods)
    many = [(f"t{k}", 1 + k % 3) for k in range(254)] + [("a", 5)]
    models = [im("none"), im("one", [("b", 3)]), im("many", many, critical=True), im("crit", [("a", 1), ("b", 2)], True),
              im("shed", [("a", 1), ("nope", 1)]), im("zero", [("a", 0)]), im("self-a"), im("a")]
    e = Engine(0, max_pods=64, max_adapters=8, max_batch=8192)
    try:
        e.upload_snapshot(1, packed)
        pm = pack_models(models, packed)
        e.upload_models(1, pm)
        ids = np.random.default_rng(3).integers(0, pm.n_models + 3, 5000).astype(np.uint32)
        ids[:4] = [pm.n_models, 2**32 - 1, 0, pm.model_ids["zero"]]
        picks = check_models(e, 1, 7, ids, 99, packed.A, packed.P)
        assert (picks["status"][:2] == N.LIG_NO_MODEL).all()
        assert (picks["status"] == N.LIG_OK).any()
        # n_models = 0
        e.upload_models(1, pack_models([], packed))
        picks = check_models(e, 1, 7, ids[:100], 0, packed.A, packed.P)
        assert (picks["status"] == N.LIG_NO_MODEL).all()
        # caller tree with drop and "no pods left" leaves
        e.set_filter_tree([N.LigFilterNode(N.LIG_F_CRITICAL_REQUEST, 1, 2, -1, 0, 0.0),
                           N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0),
                           N.LigFilterNode(N.LIG_F_DROP, -1, -1, -1, 0, 0.0)])
        e.upload_snapshot(2, packed)
        e.upload_models(2, pm)
        picks = check_models(e, 2, 8, ids, 5, packed.A, packed.P)
        assert {N.LIG_DROP, N.LIG_NO_PODS_LEFT, N.LIG_OK} <= {int(s) for s in picks["status"]}
    finally:
        e.close()


# ---- capacity and offsets -------------------------------------------------------------------------
def test_capacity_and_tile_boundaries(eng):
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"])
    ep = next_epoch()
    eng.upload_snapshot(ep, snap.packed)
    tables = class_tables(eng, ep, c["A"], c["P"])
    lib = N.load()
    for R in [0, 1, 31, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 37 * TILE + 5, 300 * TILE + 1]:
        reqs = WL.make_requests(R, c["A"], seed=R + 1)
        want_off, want_pods = expected_lists(tables, c["A"], reqs)
        total = int(want_off[-1])
        picks, offsets, pods = eng.filter_batch(ep, 21, reqs)
        assert np.array_equal(offsets, want_off) and np.array_equal(pods, want_pods), R
        for cap in sorted({0, total, max(total - 1, 0)}):
            out = np.zeros(R, dtype=PICK_DTYPE)
            off = np.full(R + 1, -7, dtype=np.int64)
            buf = np.full(cap + 16, 0xABCD, dtype=np.uint16)
            rc = lib.lig_filter_batch(eng._ctx, ep, 21, reqs.ctypes.data if R else None, R,
                                      out.ctypes.data if R else None, off.ctypes.data, buf.ctypes.data if cap else None,
                                      cap)
            assert rc == (0 if cap >= total else N.LIG_ERR_INVALID), (R, cap)
            assert np.array_equal(off, want_off) and out.tobytes() == picks.tobytes(), (R, cap)
            assert np.array_equal(buf[:cap], want_pods[:cap]) and (buf[cap:] == 0xABCD).all(), (R, cap)
            _, doff, dclip, draw = filter_device(eng, ep, 21, reqs, capacity=cap)
            assert np.array_equal(doff, want_off) and np.array_equal(dclip, want_pods[:cap]), (R, cap)
            assert (draw[cap:] == 0xABCD).all()


def test_offsets_beyond_2_to_31():
    """32768 identical pods all survive every class: R = 70000 requests need 2.29e9 entries; only
    the picks and the offsets are allocated (capacity 0)."""
    P, R = N.LIG_MAX_PODS, 70000
    e = Engine(0, max_pods=P, max_adapters=1, max_batch=R)
    try:
        from llm_instance_gateway_b200.packer import pack_columns
        e.upload_snapshot(1, pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64),
                                          np.zeros(P, np.int64), np.zeros((0, P // 32), np.uint32)))
        reqs = WL.make_requests(R, 0, seed=4)
        reqs["flags"] = np.arange(R) & 1
        out, offsets, _, _ = filter_device(e, 1, 5, reqs, capacity=0)
        assert (out["status"] == N.LIG_OK).all() and (out["n_survivors"] == P).all()
        assert np.array_equal(offsets, np.arange(R + 1, dtype=np.int64) * P)
        assert offsets[-1] > 2**31
        off = np.full(R + 1, -1, dtype=np.int64)
        o = np.zeros(R, dtype=PICK_DTYPE)
        assert N.load().lig_filter_batch(e._ctx, 1, 5, reqs.ctypes.data, R, o.ctypes.data, off.ctypes.data,
                                         None, 0) == N.LIG_ERR_INVALID
        assert np.array_equal(off, offsets) and o.tobytes() == out.tobytes()
    finally:
        e.close()


# ---- buffers, streams, refusals -------------------------------------------------------------------
class Pinned:
    def __init__(self, n, dtype):
        lib = N.load()
        self.lib = lib
        nbytes = max(n, 1) * np.dtype(dtype).itemsize
        self.ptr = lib.lig_host_alloc(nbytes)
        assert self.ptr
        self.a = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr)).view(dtype)[:n]

    def free(self):
        self.lib.lig_host_free(self.ptr)


def test_pinned_pageable_device_and_two_streams(eng):
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"])
    ep = next_epoch()
    eng.upload_snapshot(ep, snap.packed)
    eng.upload_models(ep, pack_models(WL.make_models(c["A"]), snap.packed))
    reqs = WL.make_requests(5000, c["A"], seed=2)
    ids = WL.make_model_requests(5000, c["A"], seed=3)
    want = eng.filter_batch(ep, 9, reqs)
    mwant = eng.filter_models_batch(ep, 9, ids, 17)
    for models, data, ref in ((False, reqs, want), (True, ids, mwant)):
        R, cap = len(data), int(ref[1][-1])
        # every mix of page-locked and pageable buffers
        for mask in range(16):
            bufs = []
            def mk(i, n, dt, init=None):
                if mask >> i & 1:
                    b = Pinned(n, dt)
                    bufs.append(b)
                    if init is not None:
                        b.a[:] = init
                    return b.a, b.ptr
                a = np.array(init) if init is not None else np.zeros(n, dt)
                return a, a.ctypes.data
            try:
                _, pin = mk(0, R, data.dtype, data)
                out, pout = mk(1, R, MPICK_DTYPE if models else PICK_DTYPE)
                off, poff = mk(2, R + 1, np.int64)
                pods, ppods = mk(3, cap, np.uint16)
                if models:
                    eng.filter_models_batch_ptr(ep, 9, 17, pin, R, pout, poff, ppods, cap)
                else:
                    eng.filter_batch_ptr(ep, 9, pin, R, pout, poff, ppods, cap)
                assert out.tobytes() == ref[0].tobytes() and np.array_equal(off, ref[1]), (models, mask)
                assert np.array_equal(pods, ref[2]), (models, mask)
            finally:
                for b in bufs:
                    b.free()
        # two streams at once
        d_in = dev(data)
        bufs = []
        torch.cuda.synchronize()
        for s in (torch.cuda.Stream(), torch.cuda.Stream()):
            b = (torch.zeros(R * (4 if models else 8), dtype=torch.uint8, device="cuda"),
                 torch.zeros(R + 1, dtype=torch.int64, device="cuda"), torch.zeros(cap, dtype=torch.int16, device="cuda"))
            args = (d_in.data_ptr(), R, b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), cap, s.cuda_stream)
            if models:
                eng.filter_models_batch_device(ep, 9, 17, *args)
            else:
                eng.filter_batch_device(ep, 9, *args)
            bufs.append(b)
        torch.cuda.synchronize()
        for out, off, pods in bufs:
            assert out.cpu().numpy().tobytes() == ref[0].tobytes() and np.array_equal(off.cpu().numpy(), ref[1])
            assert np.array_equal(pods.cpu().numpy().view(np.uint16), ref[2])


def test_model_upload_while_a_device_call_is_queued():
    P, A = 64, 8
    packed = pack_pod_metrics(mkpods([0] * 8, [0.1] * 8, [1] * 8, [["x"]] * 4 + [["y"]] * 4))
    old = pack_models([im("m", [("x", 1)], critical=True)], packed)
    new = pack_models([im("m", [("y", 1)])], packed)
    e = Engine(0, max_pods=P, max_adapters=A, max_batch=4096)
    try:
        e.upload_snapshot(1, packed)
        e.upload_models(1, old)
        ids = np.zeros(3000, dtype=np.uint32)
        want_old = e.filter_models_batch(1, 4, ids)
        e.upload_models(1, new)
        want_new = e.filter_models_batch(1, 4, ids)
        assert not np.array_equal(want_old[2], want_new[2])
        e.upload_models(1, old)
        st = torch.cuda.Stream()
        d_in = dev(ids)
        d_out = torch.zeros(3000 * 4, dtype=torch.uint8, device="cuda")
        d_off = torch.zeros(3001, dtype=torch.int64, device="cuda")
        d_pods = torch.zeros(64 * 3000, dtype=torch.int16, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(100_000_000)                 # keep the call queued behind ~50 ms of work
            e.filter_models_batch_device(1, 4, 0, d_in.data_ptr(), 3000, d_out.data_ptr(), d_off.data_ptr(),
                                         d_pods.data_ptr(), 64 * 3000, st.cuda_stream)
        e.upload_models(1, new)
        st.synchronize()
        off = d_off.cpu().numpy()
        assert d_out.cpu().numpy().view(MPICK_DTYPE).tobytes() == want_old[0].tobytes()
        assert np.array_equal(off, want_old[1])
        assert np.array_equal(d_pods.cpu().numpy().view(np.uint16)[: off[-1]], want_old[2])
        got = e.filter_models_batch(1, 4, ids)
        assert got[0].tobytes() == want_new[0].tobytes() and np.array_equal(got[2], want_new[2])
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
        off, pods = np.zeros(51, np.int64), np.zeros(4096, np.uint16)
        p = lambda a: a.ctypes.data
        # no snapshot yet
        assert lib.lig_filter_batch(e._ctx, 1, 0, p(reqs), 50, p(out), p(off), p(pods), 4096) == N.LIG_ERR_NO_SNAPSHOT
        e.upload_snapshot(1, snap.packed)
        assert lib.lig_filter_batch(e._ctx, 2, 0, p(reqs), 50, p(out), p(off), p(pods), 4096) == N.LIG_ERR_STALE_EPOCH
        assert lib.lig_filter_batch_device(e._ctx, 2, 0, p(reqs), 50, p(out), p(off), p(pods), 4096,
                                           None) == N.LIG_ERR_STALE_EPOCH
        # no model table
        assert lib.lig_filter_models_batch(e._ctx, 1, 0, 0, p(ids), 50, p(mout), p(off), p(pods),
                                           4096) == N.LIG_ERR_NO_SNAPSHOT
        assert lib.lig_filter_models_batch_device(e._ctx, 1, 0, 0, p(ids), 50, p(mout), p(off), p(pods), 4096,
                                                  None) == N.LIG_ERR_NO_SNAPSHOT
        # null buffers, negative sizes, R > max_batch on the host forms
        bad = [(None, p(out), p(off), p(pods), 4096, 50), (p(reqs), None, p(off), p(pods), 4096, 50),
               (p(reqs), p(out), None, p(pods), 4096, 50), (p(reqs), p(out), p(off), None, 4096, 50),
               (p(reqs), p(out), p(off), p(pods), -1, 50), (p(reqs), p(out), p(off), p(pods), 4096, -1)]
        for a, b, o, q, cap, R in bad:
            assert lib.lig_filter_batch(e._ctx, 1, 0, a, R, b, o, q, cap) == N.LIG_ERR_INVALID
            assert lib.lig_filter_batch_device(e._ctx, 1, 0, a, R, b, o, q, cap, None) == N.LIG_ERR_INVALID
            assert lib.lig_filter_models_batch(e._ctx, 1, 0, 0, a, R, b, o, q, cap) == N.LIG_ERR_INVALID
        assert lib.lig_filter_batch(None, 1, 0, p(reqs), 50, p(out), p(off), p(pods), 4096) == N.LIG_ERR_INVALID
        big = WL.make_requests(101, 8)
        assert lib.lig_filter_batch(e._ctx, 1, 0, p(big), 101, p(np.zeros(101, PICK_DTYPE)), p(np.zeros(102, np.int64)),
                                    p(pods), 4096) == N.LIG_ERR_INVALID
        assert b"max_batch" in lib.lig_last_error()
        # R = 0: offsets[0] = 0 and nothing else
        off[:] = -5
        assert lib.lig_filter_batch(e._ctx, 1, 0, None, 0, None, p(off), None, 0) == 0
        assert off[0] == 0 and (off[1:] == -5).all()
        # the device form leaves the capacity check to the caller
        _, doff, clip, _ = filter_device(e, 1, 0, reqs, capacity=3)
        assert doff[-1] > 3 and len(clip) == 3
    finally:
        e.close()


# ---- schedulers -----------------------------------------------------------------------------------
class StaticProvider:
    def __init__(self, pods):
        self.pods = list(pods)

    def AllPodMetrics(self):
        return list(self.pods)


def scheduler_pods():
    return mkpods([0, 3, 7, 60, 2, 0], [0.1, 0.5, 0.85, 0.95, 0.2, 0.1], [2, 1, 2, 1, 0, 3],
                  [["a"], ["b"], ["a", "b"], [], ["a"], ["c"]])


def as_tuple(res):
    pods, err = res
    return [p.Name for p in pods], (None if err is None else (err.code, str(err)))


@pytest.mark.parametrize("tree", [None, "affinity", "drop", "c4"])
def test_scheduler_filter_batch_agrees_with_filter(tree):
    from llm_instance_gateway_b200 import host as H
    filt = {None: None, "affinity": S.Filter("affinity", S.LORA_AFFINITY), "drop": S.Filter("drop", S.DROP),
            "c4": c4_tree()}[tree]
    pods = scheduler_pods()
    reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "c", "zz", "") for c in (False, True)]
    sched = S.NewScheduler(StaticProvider(pods), filter=filt, max_pods=64, max_adapters=8, max_batch=64, seed=1)
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=64, filter=filt)
    try:
        batch = [as_tuple(r) for r in sched.FilterBatch(reqs)]
        single = [as_tuple(sched.Filter(r)) for r in reqs]
        assert batch == single
        # the oracle: the port walking the same chart
        nodes = (filt or S.DEFAULT_FILTER).flatten()
        records = records_of(pods)
        oracle_tree.set_filter_tree(nodes)
        try:
            pool = oracle_tree.Pool(records)
            for r, (names, err) in zip(reqs, batch):
                st, idx = pool.filter(r.ResolvedTargetModel, r.Critical)
                want_err = {N.LIG_DROP: ("ResourceExhausted", S._DROP_DESC),
                            N.LIG_NO_PODS_LEFT: ("Unknown", "no pods left")}.get(st)
                assert err == want_err, r
                assert names == ([f"pod-{i}" for i in idx] if st == N.LIG_OK else []), r
        finally:
            oracle_tree.set_filter_tree(None)
        # the C++ runtime's Scheduler::Filter
        for r, (names, err) in zip(reqs, batch):
            code, got, msg = hs.Filter(r.ResolvedTargetModel, r.Critical)
            want_code = {None: H.GRPC_OK, "ResourceExhausted": 8, "Unknown": H.GRPC_UNKNOWN}[err and err[0]]
            assert (code, got, msg) == (want_code, names, err[1] if err else ""), r
        assert sched.FilterBatch([]) == []
    finally:
        hs.close()
        prov.close()
        sched.close()


def test_scheduler_filter_model_batch():
    pods = scheduler_pods()
    models = [im("m-a", [("a", 1)]), im("m-split", [("a", 3), ("b", 5), ("c", 2)], critical=True), im("m-self"),
              im("m-zero", [("a", 0)]), im("b")]
    sched = S.NewScheduler(StaticProvider(pods), max_pods=64, max_adapters=8, max_batch=64, seed=3)
    try:
        sched.SetInferenceModels(models)
        names = ["m-a", "m-split", "unknown", "m-zero", "m-self", "b", "m-split", "m-split"]
        got = [as_tuple(r) for r in sched.FilterModelBatch(names)]
        # the same draws as the next ScheduleModelBatch (FilterModelBatch leaves the key sequence alone)
        sch = sched.ScheduleModelBatch(names)
        for name, (pnames, err), (pod, resolved, serr) in zip(names, got, sch):
            if name == "unknown":
                assert err == ("Unknown", f"error finding a model object in InferenceModel for input {name}")
                continue
            if name == "m-zero":
                assert err == ("Unknown", f"error getting target model name for model {name}")
                continue
            crit = name == "m-split"
            want = as_tuple(sched.Filter(S.LLMRequest(ResolvedTargetModel=resolved, Critical=crit)))
            assert (pnames, err) == want, name
            if serr is None:
                assert pod.Name in pnames
    finally:
        sched.close()
