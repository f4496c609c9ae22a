"""The feedback chain for model-id requests on the device (include/lig.h,
lig_schedule_models_batch_feedback_chain[_device]): resolve, pick and count in one kernel.

Every check compares picks byte for byte and the per-pod loads exactly:
* with no closed window the chain is lig_schedule_models_batch;
* the chain equals its sequential definition (models_feedback_chain_ref) over pool shapes, window
  sizes, random call splits and per-call seeds, and the descriptor chain fed with the descriptors
  lig_resolve_models returns;
* descriptor calls and model-id calls alternate in one chain;
* model-table edges, caller trees, buffer forms and streams, model uploads between and during
  calls, refusals, resident epochs left untouched, and exact counting at 2^20 requests.
"""
import numpy as np
import pytest

import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import CRITICAL, SHEDDABLE, InferenceModel, InferenceModelSpec, TargetModel
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, pack_models
from oracle import binding as B
from test_gpu_feedback_chain import Pinned, pool_cases
from test_gpu_snapshot_mutation import PodState, drop_and_no_pods_trees, feedback_engine, mixed_requests, random_state

pytestmark = pytest.mark.gpu


# ---- calls: ("m", ids, seed, first_index) model-id calls, ("d", reqs, seed) descriptor calls -------
class Tables:
    """A model list interned against one pool: the device table and the oracle's datastore."""

    def __init__(self, state, models, absent=()):
        self.packed = state.packed()
        self.pm = pack_models(models, self.packed)
        recs = WL.model_records(models)
        for i in absent:
            recs[i] = None
        self.mo = B.Models(recs)
        self.n = len(models)

    def ref_call(self, call):
        if call[0] == "d":
            return call[1], call[2]
        return MC.model_call(self.mo, self.packed.adapter_id, call[1], call[2], call[3])


def ref_chain(state, calls, W, tables, thr=(0.8, 5, 50)):
    """tables: one Tables for every call, or one per call (the table each call resolves against)."""
    tabs = tables if isinstance(tables, list) else [tables] * len(calls)
    p = state.packed()
    return MC.schedule_chain(p.P, p.A, p.kv, state.q, p.n_active, p.max_active, p.bitmap,
                             [t.ref_call(c) for t, c in zip(tabs, calls)], W, thr)


def model_calls(ids, bounds, seeds, first_index=0):
    return [("m", np.ascontiguousarray(ids[a:b]), int(seeds if np.isscalar(seeds) else seeds[k]), first_index + a)
            for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]


def host_call(e, ep, call, W, P):
    """One call with pageable buffers; returns (picks, loads)."""
    loads = np.full(max(P, 1), -7, dtype=np.int32)
    if call[0] == "m":
        out = e.schedule_models_batch_feedback_chain(ep, call[2], call[1], W, first_index=call[3], loads=loads)
    else:
        out = e.schedule_batch_feedback_chain(ep, call[2], call[1], W, loads)
    return out, loads[:P].astype(np.int64)


def pinned_call(e, ep, call, W, P):
    lib = N.load()
    data = call[1]
    n = len(data)
    bi = Pinned(lib, n, data.dtype)
    bo = Pinned(lib, n, MPICK_DTYPE if call[0] == "m" else PICK_DTYPE)
    loads = Pinned(lib, max(P, 1), np.int32)
    try:
        bi.a[:] = data
        if call[0] == "m":
            e.schedule_models_batch_feedback_chain_ptr(ep, call[2], call[3], bi.ptr if n else 0, n, bo.ptr if n else 0,
                                                       W, loads.ptr)
        else:
            e.schedule_batch_feedback_chain_ptr(ep, call[2], bi.ptr if n else 0, n, bo.ptr if n else 0, W, loads.ptr)
        return bo.a.copy(), loads.a[:P].astype(np.int64)
    finally:
        for b in (bi, bo, loads):
            b.free()


def device_calls(e, ep, calls, W, P, streams=None, sync_between=True):
    """Device buffers; calls round-robin over `streams` (no host synchronisation between them when
    sync_between is False).  Returns (picks of every call, loads after the last)."""
    import torch
    streams = streams or [torch.cuda.Stream()]
    ins = [torch.from_numpy(c[1].view(np.uint8).reshape(-1).copy()).cuda() if len(c[1]) else None for c in calls]
    sizes = [4 if c[0] == "m" else 8 for c in calls]
    outs = [torch.full((max(len(c[1]), 1) * s,), 0xAB, dtype=torch.uint8, device="cuda") for c, s in zip(calls, sizes)]
    d_loads = torch.full((max(P, 1),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for k, c in enumerate(calls):
        st = streams[k % len(streams)]
        d_in = ins[k].data_ptr() if len(c[1]) else 0
        with torch.cuda.stream(st):
            if c[0] == "m":
                e.schedule_models_batch_feedback_chain_device(ep, c[2], c[3], d_in, len(c[1]), outs[k].data_ptr(), W,
                                                              d_loads.data_ptr(), st.cuda_stream)
            else:
                e.schedule_batch_feedback_chain_device(ep, c[2], d_in, len(c[1]), outs[k].data_ptr(), W,
                                                       d_loads.data_ptr(), st.cuda_stream)
        if sync_between:
            st.synchronize()
    torch.cuda.synchronize()
    picks = [o[: len(c[1]) * s].cpu().numpy().view(MPICK_DTYPE if c[0] == "m" else PICK_DTYPE)
             for o, c, s in zip(outs, calls, sizes)]
    return picks, d_loads[:P].cpu().numpy().astype(np.int64)


def run_calls(e, ep, calls, W, P, form=host_call):
    outs, loads = [], None
    for c in calls:
        o, loads = form(e, ep, c, W, P)
        outs.append(o)
    return outs, loads


def assert_same(got, want, label):
    outs, loads = got
    assert len(outs) == len(want[0]), label
    for k, (g, w) in enumerate(zip(outs, want[0])):
        assert g.dtype == w.dtype, (label, k)
        bad = np.nonzero(g != w)[0]
        assert bad.size == 0, (label, k, bad[:5], g[bad[:5]], w[bad[:5]])
    assert np.array_equal(loads, want[1]), (label, np.nonzero(loads != want[1])[0][:5])


def edge_ids(R, A, n_models, seed):
    ids = WL.make_model_requests(R, A, seed=seed)
    if R >= 8:
        ids[:6] = [n_models, n_models + 5, 2**32 - 1, 2**31, A, A + 1]   # absent x4, pass-through, a split model
    return ids


# ---- 1. no window closes -------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["C3", "C5"])
def test_no_closed_window_equals_models_batch(cfg):
    c = WL.CONFIGS[cfg]
    state = random_state(c["P"], c["A"], seed=c["P"] + 1)
    tab = Tables(state, WL.make_models(c["A"]))
    R = 30000
    ids = edge_ids(R, c["A"], tab.n, seed=2)
    bounds = FC.random_split(R, np.random.default_rng(3), 500)
    calls = model_calls(ids, bounds, 9, first_index=1 << 35)
    with feedback_engine(state.P, c["A"], R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        want = e.schedule_models_batch(1, 9, ids, first_index=1 << 35)
        for form in (host_call, pinned_call):
            e.feedback_chain_reset()
            outs, loads = run_calls(e, 1, calls, 1 << 30, state.P, form)
            got = np.concatenate(outs)
            assert np.array_equal(got, want), form.__name__
            assert np.array_equal(loads, np.bincount(got["pod_idx"][got["pod_idx"] >= 0], minlength=state.P))
        e.feedback_chain_reset()
        outs, _ = device_calls(e, 1, calls, 1 << 30, state.P)
        assert np.array_equal(np.concatenate(outs), want)
        assert (want["status"] == N.LIG_NO_MODEL).sum() >= 4 and ((want["target_idx"] > 0) & (want["target_idx"] < 255)).any()


# ---- 2. against the definition -------------------------------------------------------------------
@pytest.mark.parametrize("pool", ["C2", "C3", "C5", "P=0", "P=1", "P=33", "P=4097", "P=20000", "A=0"])
def test_chain_equals_the_definition(pool):
    for label, state in pool_cases(pool):
        P, A = state.P, state.A
        tab = Tables(state, WL.make_models(A))
        for W in (1, 7, 64, 4096):
            R = {1: 150, 7: 900, 64: 3000, 4096: 13000}[W]
            if P >= 4096:
                R = min(R, 600) if W < 64 else R
            ids = edge_ids(R, A, tab.n, seed=P + W)
            rng = np.random.default_rng(P * 7 + W)
            bounds = FC.random_split(R, rng, W)
            seeds = rng.integers(0, 1 << 63, len(bounds), dtype=np.uint64)
            calls = model_calls(ids, bounds, seeds, first_index=W * 1000)
            want = ref_chain(state, calls, W, tab)
            with feedback_engine(P, A, R) as e:
                e.upload_snapshot(1, state.packed())
                e.upload_models(1, tab.pm)
                assert_same(run_calls(e, 1, calls, W, P), want, (label, W, "host"))
                e.feedback_chain_reset()
                assert_same(device_calls(e, 1, calls, W, P), want, (label, W, "device"))
            got = np.concatenate(want[0])
            assert want[1].sum() == (got["pod_idx"] >= 0).sum()


# ---- 3. against the descriptor chain -------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 64, 4096])
def test_chain_equals_the_descriptor_chain_on_resolved_descriptors(W):
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=31)
    tab = Tables(state, WL.make_models(c["A"]))
    R = 12000 if W > 1 else 1500
    ids = WL.make_model_requests(R + R // 100 + 50, c["A"], seed=32)
    ids = np.ascontiguousarray(ids[ids < tab.n][:R])                 # every id resolves
    R = len(ids)
    rng = np.random.default_rng(33)
    bounds = FC.random_split(R, rng, W)
    seeds = [int(s) for s in rng.integers(0, 1 << 63, len(bounds), dtype=np.uint64)]
    calls = model_calls(ids, bounds, seeds, first_index=77)
    with feedback_engine(state.P, c["A"], R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        got = run_calls(e, 1, calls, W, state.P)
        dcalls, res = [], []
        for m in calls:
            reqs, r = e.resolve_models(1, m[2], m[1], first_index=m[3])
            assert (r["status"] == N.LIG_OK).all()
            dcalls.append(("d", reqs, m[2]))
            res.append(r)
        e.feedback_chain_reset()
        want = run_calls(e, 1, dcalls, W, state.P)
    assert np.array_equal(got[1], want[1])
    for g, w, r in zip(got[0], want[0], res):
        assert np.array_equal(g["pod_idx"].astype(np.int32), w["pod_idx"])
        assert np.array_equal(g["status"], w["status"].astype(np.uint8))
        assert np.array_equal(g["target_idx"], r["target_idx"])


# ---- 4. mixed chain ------------------------------------------------------------------------------
def test_descriptor_and_model_calls_alternate_in_one_chain():
    c = WL.CONFIGS["C5"]
    state = random_state(c["P"], c["A"], seed=41)
    tab = Tables(state, WL.make_models(c["A"]))
    W, R = 97, 8000
    ids = edge_ids(R, c["A"], tab.n, seed=42)
    reqs = mixed_requests(c["A"], R, seed=43)[:R]
    rng = np.random.default_rng(44)
    bounds = FC.random_split(R, rng, W)
    calls = []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        if k % 2:
            calls.append(("m", np.ascontiguousarray(ids[a:b]), 500 + k, a))
        else:
            calls.append(("d", np.ascontiguousarray(reqs[a:b]), 500 + k))
    want = ref_chain(state, calls, W, tab)
    with feedback_engine(state.P, c["A"], R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        assert_same(run_calls(e, 1, calls, W, state.P), want, "host")
        e.feedback_chain_reset()
        assert_same(device_calls(e, 1, calls, W, state.P), want, "device")
        e.feedback_chain_reset()
        outs, loads = [], None
        for k, call in enumerate(calls):                             # forms alternate as well
            if k % 3 == 2:
                o, loads = device_calls(e, 1, [call], W, state.P)
                o = o[0]
            else:
                o, loads = (host_call, pinned_call)[k % 3](e, 1, call, W, state.P)
            outs.append(o)
        assert_same((outs, loads), want, "forms alternate")


# ---- 5. model-table edges ------------------------------------------------------------------------
def mk(name, crit, targets):
    return InferenceModel(name, InferenceModelSpec(ModelName=name, Criticality=crit,
                                                   TargetModels=[TargetModel(n, w) for n, w in targets]))


def edge_models(A, rng):
    an = WL.adapter_name
    models = [
        mk(an(3), None, []),                                              # no target: its own name
        mk("no-target-unlisted", CRITICAL, []),                           # no target, no pod lists it
        mk("one", CRITICAL, [(an(1), 5)]),
        mk("one-sheddable", SHEDDABLE, [(an(2), 1)]),
        mk("many", None, [(an(k % A), int(w)) for k, w in enumerate(rng.integers(0, 1000, 255))]),
        mk("many-critical", CRITICAL, [(an((7 * k) % A), 1 + k) for k in range(255)]),
        mk("max-sum", CRITICAL, [(an(0), 2**30), (an(4), 2**30 - 1)]),
        mk("max-sum-3", None, [(an(5), 1), (an(6), 2**31 - 3), (an(7), 1)]),
        mk("on-A", CRITICAL, [(WL.UNKNOWN_MODEL, 3), ("unloaded", 4)]),    # targets on adapter id A
        mk("on-A-one", None, [("unloaded", 9)]),
        mk("zero-sum", None, [(an(0), 0)]),                               # packed as absent
        mk("half", SHEDDABLE, [(an(8), 50), (an(9), 50)]),
    ]
    return models, [10]


@pytest.mark.parametrize("tree", [None, 0, 1])
def test_model_table_edges(tree):
    P, A, W = 96, 12, 40
    rng = np.random.default_rng(51)
    state = random_state(P, A, seed=52)
    models, absent = edge_models(A, rng)
    tab = Tables(state, models, absent)
    assert tab.pm.present.tolist().count(0) == 1
    R = 6000
    ids = rng.integers(0, len(models) + 3, R).astype(np.uint32)
    ids[:3] = [2**32 - 1, len(models), 2**31]
    bounds = FC.random_split(R, rng, W)
    calls = model_calls(ids, bounds, [int(s) for s in rng.integers(0, 1 << 62, len(bounds))], first_index=5)
    def ref(calls, tabs):
        if tree is None:
            return ref_chain(state, calls, W, tabs)
        return MC.schedule_chain_tree(drop_and_no_pods_trees()[tree], state.records(), state.names(),
                                      [t.ref_call(c) for t, c in zip(tabs, calls)], W)
    want = ref(calls, [tab] * len(calls))
    got_all = np.concatenate(want[0])
    st = got_all["status"]
    assert (st == N.LIG_NO_MODEL).any() and (st == N.LIG_OK).any()
    if tree is not None:
        assert (st == (N.LIG_DROP if tree == 0 else N.LIG_NO_PODS_LEFT)).any()
    tg = got_all["target_idx"]
    assert (tg[ids == 4] > 200).any() and (tg[ids == 5] > 200).any()       # late targets of 255 drawn
    with feedback_engine(P, A, R) as e:
        if tree is not None:
            e.set_filter_tree(drop_and_no_pods_trees()[tree])
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        assert_same(run_calls(e, 1, calls, W, P), want, ("edges", tree))
        # n_models = 0: every id is LIG_NO_MODEL and every request still counts toward its window
        e.upload_models(1, pack_models([], tab.packed))
        empty = Tables(state, [])
        cont = model_calls(ids[:500], [0, 7, 40, 41, 500], 3)
        want2 = ref(calls + cont, [tab] * len(calls) + [empty] * len(cont))
        got2 = run_calls(e, 1, cont, W, P)
        assert_same(got2, (want2[0][len(calls):], want2[1]), ("n_models = 0", tree))
        assert (np.concatenate(got2[0])["status"] == N.LIG_NO_MODEL).all()


# ---- 6. buffers and streams ----------------------------------------------------------------------
def test_buffer_forms_and_two_streams():
    import torch
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=61)
    tab = Tables(state, WL.make_models(c["A"]))
    W, R = 333, 20000
    ids = edge_ids(R, c["A"], tab.n, seed=62)
    calls = model_calls(ids, FC.random_split(R, np.random.default_rng(63), W), 77, first_index=1 << 20)
    want = ref_chain(state, calls, W, tab)
    with feedback_engine(state.P, c["A"], R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        assert_same(run_calls(e, 1, calls, W, state.P, pinned_call), want, "pinned")
        e.feedback_chain_reset()
        assert_same(run_calls(e, 1, calls, W, state.P, host_call), want, "pageable")
        e.feedback_chain_reset()
        assert_same(device_calls(e, 1, calls, W, state.P), want, "device")
        e.feedback_chain_reset()
        assert_same(device_calls(e, 1, calls, W, state.P, [torch.cuda.Stream(), torch.cuda.Stream()],
                                 sync_between=False), want, "two streams")
        L = np.zeros(state.P, dtype=np.int32)                        # R = 0 reads the loads
        e.schedule_models_batch_feedback_chain(1, 5, np.zeros(0, dtype=np.uint32), W, loads=L)
        assert np.array_equal(L, want[1])


# ---- 7. model-table uploads ----------------------------------------------------------------------
def shuffled_models(A, seed):
    """make_models with the targets of the single-target models moved: another resolve for most ids."""
    models = WL.make_models(A)
    r = np.random.default_rng(seed)
    for m in models[:A]:
        m.Spec.TargetModels = [TargetModel(WL.adapter_name(int(r.integers(0, A))), 100)]
    return models


def test_model_uploads_between_and_during_calls():
    import torch
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=71)
    tabs = [Tables(state, shuffled_models(c["A"], 72 + k) if k else WL.make_models(c["A"])) for k in range(4)]
    W, R = 200, 3000
    ids = [WL.make_model_requests(R, c["A"], seed=80 + k) for k in range(6)]
    calls = [("m", ids[k], 90 + k, k * R) for k in range(6)]
    P = state.P
    with feedback_engine(P, c["A"], R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tabs[0].pm)
        # a blocking upload between calls: the next call resolves against it, the loads go on
        got = run_calls(e, 1, calls[:2], W, P)
        e.upload_models(1, tabs[1].pm)
        got2 = run_calls(e, 1, calls[2:3], W, P)
        want = ref_chain(state, calls[:3], W, [tabs[0], tabs[0], tabs[1]])
        assert_same((got[0] + got2[0], got2[1]), want, "upload between calls")
        assert not np.array_equal(got2[0][0], ref_chain(state, calls[:3], W, tabs[0])[0][2])
        # an async upload right before a device-form call is seen by that call
        e.upload_models(1, tabs[2].pm, block=False)
        got3 = device_calls(e, 1, calls[3:4], W, P)
        want = ref_chain(state, calls[:4], W, [tabs[0], tabs[0], tabs[1], tabs[2]])
        assert_same((got3[0], got3[1]), (want[0][3:], want[1]), "async upload before a device call")
        # a blocking upload while a device-form call is still in flight on another stream: that
        # call keeps the old table, the next one sees the new one
        st = torch.cuda.Stream()
        d_in = torch.from_numpy(ids[4].view(np.uint8).copy()).cuda()
        d_out = torch.full((R * 4,), 0xAB, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(100_000_000)                           # keep the call queued behind ~50 ms of work
            e.schedule_models_batch_feedback_chain_device(1, calls[4][2], calls[4][3], d_in.data_ptr(), R,
                                                          d_out.data_ptr(), W, 0, st.cuda_stream)
        e.upload_models(1, tabs[3].pm)
        st.synchronize()
        in_flight = d_out.cpu().numpy().view(MPICK_DTYPE).copy()
        got5 = run_calls(e, 1, calls[5:6], W, P)
        seq = [tabs[0], tabs[0], tabs[1], tabs[2], tabs[2], tabs[3]]
        want = ref_chain(state, calls, W, seq)
        assert np.array_equal(in_flight, want[0][4]), "the in-flight call saw the new table"
        assert_same(got5, (want[0][5:], want[1]), "the call after the upload")


# ---- 8. refusals ---------------------------------------------------------------------------------
def test_refused_calls_leave_the_chain_untouched():
    P, A, W = 128, 16, 30
    state = random_state(P, A, seed=81)
    tab = Tables(state, WL.make_models(A))
    ids = edge_ids(2000, A, tab.n, seed=82)
    calls = model_calls(ids, FC.random_split(2000, np.random.default_rng(83), W), 84)
    want = ref_chain(state, calls, W, tab)
    lib = N.load()
    with feedback_engine(P, A, 700) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        e.upload_snapshot(2, state.packed())                        # resident, no model table
        ctx = e._ctx
        junk = edge_ids(800, A, tab.n, seed=85)
        out = np.zeros(800, dtype=MPICK_DTYPE)
        f, fd = lib.lig_schedule_models_batch_feedback_chain, lib.lig_schedule_models_batch_feedback_chain_device
        refusals = [
            (lambda: f(ctx, 1, 84, 0, junk.ctypes.data, 10, out.ctypes.data, 0, None), N.LIG_ERR_INVALID),
            (lambda: f(ctx, 1, 84, 0, junk.ctypes.data, -1, out.ctypes.data, W, None), N.LIG_ERR_INVALID),
            (lambda: f(ctx, 1, 84, 0, None, 10, out.ctypes.data, W, None), N.LIG_ERR_INVALID),
            (lambda: f(ctx, 1, 84, 0, junk.ctypes.data, 10, None, W, None), N.LIG_ERR_INVALID),
            (lambda: f(ctx, 1, 84, 0, junk.ctypes.data, 800, out.ctypes.data, W, None), N.LIG_ERR_INVALID),
            (lambda: f(ctx, 9, 84, 0, junk.ctypes.data, 10, out.ctypes.data, W, None), N.LIG_ERR_STALE_EPOCH),
            (lambda: f(ctx, 2, 84, 0, junk.ctypes.data, 10, out.ctypes.data, W, None), N.LIG_ERR_NO_SNAPSHOT),
            (lambda: fd(ctx, 2, 84, 0, None, 0, None, W, None, None), N.LIG_ERR_NO_SNAPSHOT),
            (lambda: fd(ctx, 1, 84, 0, None, 10, None, W, None, None), N.LIG_ERR_INVALID),
            (lambda: fd(ctx, 1, 84, 0, None, 0, None, -3, None, None), N.LIG_ERR_INVALID),
        ]
        outs, loads = [], None
        for k, call in enumerate(calls):
            o, loads = host_call(e, 1, call, W, P)
            outs.append(o)
            fn, code = refusals[k % len(refusals)]
            assert fn() == code, k
        assert len(calls) >= len(refusals)
        assert_same((outs, loads), want, "refusals interleaved")
    # a doorbell stream open before the scratch exists
    with feedback_engine(P, A, 2000) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        e.stream_open()
        try:
            with pytest.raises(N.LigError) as ei:
                e.schedule_models_batch_feedback_chain(1, 84, calls[0][1], W)
            assert ei.value.code == N.LIG_ERR_INVALID and "doorbell" in str(ei.value)
        finally:
            e.stream_close()
        assert_same(run_calls(e, 1, calls, W, P), want, "after the doorbell refusal")
    # a ctx with a (single-rank) communicator
    with feedback_engine(P, A, 2000) as e:
        try:
            e.comm_init_rank(1, 0, e.comm_unique_id())
        except N.LigError as err:
            pytest.skip(f"no NCCL: {err}")
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        with pytest.raises(N.LigError) as ei:
            e.schedule_models_batch_feedback_chain(1, 84, calls[0][1], W)
        assert ei.value.code == N.LIG_ERR_INVALID and "communicator" in str(ei.value)


# ---- 9. resident state untouched -----------------------------------------------------------------
def test_resident_epochs_and_model_tables_untouched():
    P, A = 64, 8
    state = random_state(P, A, seed=91)
    state.q[:] = 0
    tab = Tables(state, WL.make_models(A))
    ids = np.zeros(20000, dtype=np.uint32)                            # model-0: one class, a herd without feedback
    with feedback_engine(P, A, 20000) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        e.upload_snapshot(2, random_state(P, A, seed=92).packed())
        e.upload_models(2, tab.pm)
        mix = WL.make_model_requests(20000, A, seed=93)
        classes = lambda ep: [e.read_class(ep, cr, a, P) for cr in (0, 1) for a in range(A + 1)]   # noqa: E731
        before = [(classes(ep), e.schedule_models_batch(ep, 3, mix, first_index=11)) for ep in (1, 2)]
        herd = e.schedule_models_batch(1, 3, ids)
        loads = np.zeros(P, dtype=np.int32)
        for lo in range(0, 20000, 2500):
            e.schedule_models_batch_feedback_chain(1, 3, np.ascontiguousarray(ids[lo:lo + 2500]), 8, first_index=lo,
                                                   loads=loads)
        assert loads.max() < np.bincount(herd["pod_idx"][herd["pod_idx"] >= 0], minlength=P).max()
        for ep, (cls, picks) in zip((1, 2), before):
            after = classes(ep)
            assert all(b[0] == a[0] and b[1] == a[1] and np.array_equal(b[2], a[2]) for b, a in zip(cls, after))
            assert np.array_equal(e.schedule_models_batch(ep, 3, mix, first_index=11), picks)


# ---- 10. exact counting --------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 64])
def test_single_survivor_counts_are_exact(P):
    """2^20 requests of single-target critical models whose class has exactly one survivor, in one
    open window: every warp counts runs of equal pods with one atomic per pod."""
    R = 1 << 20
    A = max(P, 1)
    state = PodState(A, np.full(P, 0.1), np.zeros(P), np.full(P, 4), [[p] for p in range(P)])
    models = [mk(f"m{a}", CRITICAL, [(WL.adapter_name(a), 7)]) for a in range(A)]
    tab = Tables(state, models)
    rng = np.random.default_rng(P)
    ids = (np.sort(rng.integers(0, A, R)) if P > 1 else np.zeros(R)).astype(np.uint32)
    with feedback_engine(P, A, R) as e:
        e.upload_snapshot(1, state.packed())
        e.upload_models(1, tab.pm)
        loads = np.zeros(P, dtype=np.int32)
        out = e.schedule_models_batch_feedback_chain(1, 3, ids, 1 << 30, first_index=0, loads=loads)
        assert (out["status"] == N.LIG_OK).all() and (out["target_idx"] == 0).all()
        assert np.array_equal(out["pod_idx"].astype(np.int64), ids.astype(np.int64))
        assert np.array_equal(loads, np.bincount(ids, minlength=P))
        assert np.array_equal(out, e.schedule_models_batch(1, 3, ids))
