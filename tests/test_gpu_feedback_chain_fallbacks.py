"""Fallback rows under the load-feedback chain on the device (include/lig.h,
lig_schedule_[models_]batch_feedback_chain_fallbacks[_device]), bit for bit:

* picks and loads are the plain chain's for every n, with calls with and without rows, descriptor and
  model-id calls alternating in one chain; with no closed window everything equals the resident
  lig_schedule_[models_]batch_fallbacks;
* rows against the sequential definition (feedback_chain_fallbacks_ref) on the bench configurations,
  edge pools and shapes, W in {1, 7, 64, 4096} with random splits and per-call seeds, the built-in
  tree and caller trees (full rows, DROP and "no pods left" leaves), model-id edges;
* a herd that moves pods across the queue thresholds: the rows follow the chain's tables;
* page-locked, pageable, +8-byte and device buffers mixed in one chain, two streams, a model upload
  behind a queued call; refusals leave the chain untouched; resident epochs stay as they were;
* one C4 call at R = 2^20;
* the Python scheduler's and the C++ runtime's feedback_fallbacks option.
"""
import random
import threading

import numpy as np
import pytest
import torch

import feedback_chain_fallbacks_ref as FF
import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
from test_gpu_fallbacks import KEEP_ALL, splitmix_keys
from test_gpu_feedback_chain import Pinned, pool_cases
from test_gpu_filter_batch import StaticProvider, im
from test_gpu_filter_tree import mkpods
from test_gpu_snapshot_mutation import INT32_MAX, drop_and_no_pods_trees, feedback_engine, mixed_requests, random_state
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models, pack_pod_metrics
from oracle import binding as B

pytestmark = pytest.mark.gpu

K = N.LIG_MAX_FALLBACKS
FORMS = ("pageable", "pinned", "pinned+8", "device")


# ---- calls: ("d", reqs, seed, k) or ("m", ids, seed, first_index, k); k = 0 is a plain chain call -------
def ref_calls(calls, mo=None, adapter_id=None):
    out = []
    for c in calls:
        if c[0] == "d":
            out.append((c[1], c[2]))
        else:
            out.append(MC.model_call(mo, adapter_id, c[1], c[2], c[3]))
    return out


def ks_of(calls):
    return [c[-1] for c in calls]


def oracle(state, calls, W, models=None, thr=(0.8, 5, 50)):
    p = state.packed()
    mo = B.Models(WL.model_records(models)) if models is not None else None
    return FF.schedule_chain_fallbacks(p.P, p.A, p.kv, state.q, p.n_active, p.max_active, p.bitmap,
                                       ref_calls(calls, mo, p.adapter_id), ks_of(calls), W, thr)


def _host_buf(lib, arr, shift, keep):
    """A page-locked copy of `arr` (or zeros of its size) `shift` bytes into a fresh buffer."""
    nbytes = arr.nbytes
    b = Pinned(lib, nbytes + 16, np.uint8)
    keep.append(b)
    raw = b.a[shift:shift + nbytes]
    raw[:] = np.frombuffer(np.ascontiguousarray(arr).tobytes(), np.uint8)
    return raw, b.ptr + shift


def run_call(e, ep, call, W, P, form="pageable", stream=None, sync=True):
    """One chain call in `form`: (picks, rows (R, k), loads[P]); with sync=False (device form) the
    device tensors, to be read after a synchronise."""
    kind, data, seed = call[0], call[1], call[2]
    first = call[3] if kind == "m" else 0
    k = call[-1]
    R = len(data)
    models = kind == "m"
    odt = MPICK_DTYPE if models else PICK_DTYPE
    if form == "device":
        d_in = (torch.from_numpy(data.view(np.uint8).reshape(-1).copy()).cuda() if R
                else torch.zeros(16, dtype=torch.uint8, device="cuda"))
        d_out = torch.full((max(R, 1) * odt.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
        d_rows = torch.full((max(R * k, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
        d_loads = torch.full((max(P, 1),), -7, dtype=torch.int32, device="cuda")
        st = stream or torch.cuda.current_stream()
        if sync:
            torch.cuda.synchronize()
        inp = d_in.data_ptr() if R else 0
        if models and k:
            e.schedule_models_batch_feedback_chain_fallbacks_device(ep, seed, first, inp, R, d_out.data_ptr(), k,
                                                                    d_rows.data_ptr(), W, d_loads.data_ptr(),
                                                                    st.cuda_stream)
        elif models:
            e.schedule_models_batch_feedback_chain_device(ep, seed, first, inp, R, d_out.data_ptr(), W,
                                                          d_loads.data_ptr(), st.cuda_stream)
        elif k:
            e.schedule_batch_feedback_chain_fallbacks_device(ep, seed, inp, R, d_out.data_ptr(), k, d_rows.data_ptr(),
                                                             W, d_loads.data_ptr(), st.cuda_stream)
        else:
            e.schedule_batch_feedback_chain_device(ep, seed, inp, R, d_out.data_ptr(), W, d_loads.data_ptr(),
                                                   st.cuda_stream)

        def read():
            return (d_out[: R * odt.itemsize].cpu().numpy().view(odt), d_rows[: R * k].cpu().numpy().reshape(R, k),
                    d_loads[:P].cpu().numpy().astype(np.int64))
        if not sync:
            return read, (d_in, d_out, d_rows, d_loads)
        st.synchronize()
        return read()
    lib, keep = N.load(), []
    try:
        loads = np.full(max(P, 1), -7, dtype=np.int32)
        if form == "pageable":
            inp, out, rows = np.ascontiguousarray(data), np.zeros(R, odt), np.zeros((R, k), np.int16)
            pin, pout, prows = inp.ctypes.data, out.ctypes.data, rows.ctypes.data
        else:
            s_in, s_rows = (8, 1) if form == "pinned+8" else (0, 0)     # +1 byte: rows staged
            _, pin = _host_buf(lib, data, s_in, keep)
            out, pout = _host_buf(lib, np.zeros(R, odt), s_in, keep)
            rows, prows = _host_buf(lib, np.zeros(R * k, np.int16), s_rows, keep)
        if not R:
            pin = pout = prows = 0
        if models and k:
            e.schedule_models_batch_feedback_chain_fallbacks_ptr(ep, seed, first, pin, R, pout, k, prows, W,
                                                                 loads.ctypes.data)
        elif models:
            e.schedule_models_batch_feedback_chain_ptr(ep, seed, first, pin, R, pout, W, loads.ctypes.data)
        elif k:
            e.schedule_batch_feedback_chain_fallbacks_ptr(ep, seed, pin, R, pout, k, prows, W, loads.ctypes.data)
        else:
            e.schedule_batch_feedback_chain_ptr(ep, seed, pin, R, pout, W, loads.ctypes.data)
        return (np.frombuffer(out.tobytes(), odt).copy(), np.frombuffer(rows.tobytes(), np.int16).reshape(R, k).copy(),
                loads[:P].astype(np.int64))
    finally:
        for b in keep:
            b.free()


def run_chain(e, ep, calls, W, P, forms=("pageable",)):
    outs, rows, loads = [], [], None
    for i, c in enumerate(calls):
        o, r, loads = run_call(e, ep, c, W, P, forms[i % len(forms)])
        outs.append(o)
        rows.append(r)
    return outs, rows, loads


def assert_same(got, want, label):
    outs, rows, loads = got
    assert len(outs) == len(want[0]), label
    for i, (o, w) in enumerate(zip(outs, want[0])):
        assert o.tobytes() == w.tobytes(), (label, i, np.nonzero(o != w)[0][:5])
    for i, (r, w) in enumerate(zip(rows, want[1])):
        assert np.array_equal(r, w), (label, i, np.nonzero((r != w).any(axis=1))[0][:5])
    assert np.array_equal(loads, want[2]), label


def split(data, bounds, seeds, ks, kind="d", first_index=0):
    calls = []
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        chunk = np.ascontiguousarray(data[a:b])
        if kind == "d":
            calls.append(("d", chunk, seeds[i], ks[i]))
        else:
            calls.append(("m", chunk, seeds[i], (first_index + a) & ((1 << 64) - 1), ks[i]))
    return calls


def mixed_chain(A, n_models, R, seed, ks=None, window=64):
    """Descriptor and model-id calls alternating, per-call seeds; ks cycles through 0..K."""
    reqs = mixed_requests(A, R, seed)
    ids = np.random.default_rng(seed).integers(0, n_models + 3, len(reqs)).astype(np.uint32)
    bounds = FC.random_split(len(reqs), np.random.default_rng(seed + 1), window)
    calls, first = [], (1 << 64) - 1000
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        k = (i % (K + 1)) if ks is None else ks[i % len(ks)]
        if i % 2:
            calls.append(("m", np.ascontiguousarray(ids[a:b]), 300 + i, first & ((1 << 64) - 1), k))
            first += b - a
        else:
            calls.append(("d", np.ascontiguousarray(reqs[a:b]), 300 + i, k))
    return calls


def engine_for(state, R, models=None):
    e = feedback_engine(state.P, state.A, R)
    p = state.packed()
    e.upload_snapshot(1, p)
    if models is not None:
        e.upload_models(1, pack_models(models, p))
    return e


# ---- picks and loads are the plain chain's; no closed window = the resident call -------------------------
def test_picks_and_loads_equal_the_plain_chain():
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=7)
    models = WL.make_models(c["A"])
    for W in (7, 64, 333):
        calls = mixed_chain(c["A"], len(models), 6000, seed=W)
        plain = [x[:-1] + (0,) for x in calls]
        with engine_for(state, 8000, models) as e:
            want_plain = run_chain(e, 1, plain, W, state.P)
            e.feedback_chain_reset()
            got = run_chain(e, 1, calls, W, state.P, FORMS)
            for n in range(1, K + 1):             # every n, all calls with rows
                e.feedback_chain_reset()
                same_n = run_chain(e, 1, [x[:-1] + (n,) for x in calls], W, state.P)
                assert all(o.tobytes() == w.tobytes() for o, w in zip(same_n[0], want_plain[0])), (W, n)
                assert np.array_equal(same_n[2], want_plain[2]), (W, n)
                assert all(np.array_equal(r, g[:, :n]) for r, g, x in zip(same_n[1], got[1], calls)
                           if x[-1] >= n), (W, n)                   # prefix rows
        assert all(o.tobytes() == w.tobytes() for o, w in zip(got[0], want_plain[0])), W
        assert np.array_equal(got[2], want_plain[2]) and got[2].sum() > 0, W
        assert_same(got, oracle(state, calls, W, models), ("definition", W))


def test_no_closed_window_equals_the_resident_fallbacks():
    c = WL.CONFIGS["C2"]
    state = random_state(c["P"], c["A"], seed=9)
    models = WL.make_models(c["A"])
    reqs = mixed_requests(c["A"], 3000, seed=10)
    ids = np.random.default_rng(11).integers(0, len(models) + 2, 3000).astype(np.uint32)
    with engine_for(state, 8000, models) as e:
        for n in (1, 4, 8):
            e.feedback_chain_reset()
            out, rows = e.schedule_batch_fallbacks(1, 5, reqs, n)
            got = run_call(e, 1, ("d", reqs, 5, n), 1 << 20, state.P, "device")
            assert got[0].tobytes() == out.tobytes() and np.array_equal(got[1], rows), n
            mout, mrows = e.schedule_models_batch_fallbacks(1, 6, ids, n, first_index=(1 << 64) - 9)
            got = run_call(e, 1, ("m", ids, 6, (1 << 64) - 9, n), 1 << 20, state.P, "pinned")
            assert got[0].tobytes() == mout.tobytes() and np.array_equal(got[1], mrows), n


# ---- rows against the definition ----------------------------------------------------------------------
@pytest.mark.parametrize("pool", ["C2", "C3", "C5", "edge_pools", "P=0", "P=1", "P=33", "P=4097", "P=20000", "A=0"])
def test_rows_against_the_definition(pool):
    for label, state in pool_cases(pool):
        P = state.P
        for W in (1, 7, 64, 4096):
            R = {1: 120, 7: 700, 64: 2500, 4096: 10000}[W]
            if P >= 4096 and W < 64:
                R = min(R, 400)
            reqs = mixed_requests(state.A, R, seed=P + W)
            rng = np.random.default_rng(P * 3 + W)
            bounds = FC.random_split(len(reqs), rng, W)
            n = len(bounds) - 1
            calls = split(reqs, bounds, (1000 + 7 * np.arange(n)).tolist(), rng.integers(0, K + 1, n).tolist())
            want = oracle(state, calls, W)
            with engine_for(state, len(reqs)) as e:
                assert_same(run_chain(e, 1, calls, W, P, FORMS), want, (label, W))
            ok = np.concatenate(want[0])["status"] == N.LIG_OK
            assert P == 0 or not ok.any() or want[2].sum() == ok.sum()


@pytest.mark.parametrize("tree", ["keep_all", "drop", "no_pods"])
def test_caller_trees(tree):
    P, A, W = 96, 12, 40
    state = random_state(P, A, seed=41)
    nodes = {"keep_all": KEEP_ALL, "drop": drop_and_no_pods_trees()[0], "no_pods": drop_and_no_pods_trees()[1]}[tree]
    reqs = mixed_requests(A, 3000, seed=42)
    rng = np.random.default_rng(43)
    bounds = FC.random_split(len(reqs), rng, W)
    n = len(bounds) - 1
    calls = split(reqs, bounds, [5 + i for i in range(n)], rng.integers(1, K + 1, n).tolist())
    want = FF.schedule_chain_fallbacks_tree(nodes, state.records(), state.names(), ref_calls(calls), ks_of(calls), W)
    st = {int(s) for s in np.concatenate(want[0])["status"]}
    if tree == "keep_all":
        rows = np.concatenate([r[:, :1] for r in want[1]])
        assert (rows >= 0).all()                              # full rows: every pod survives
    else:
        assert (N.LIG_DROP if tree == "drop" else N.LIG_NO_PODS_LEFT) in st
    e = feedback_engine(P, A, len(reqs))
    with e:
        e.set_filter_tree(nodes)
        e.upload_snapshot(1, state.packed())
        assert_same(run_chain(e, 1, calls, W, P, FORMS), want, tree)


def test_model_id_edges():
    """0, 1 and 255 targets, absent models (weights summing to 0), ids >= n_models, first_index
    wrapping 2^64, in one chain with descriptor calls."""
    pods = mkpods(list(range(40)), [0.05 * (i % 9) for i in range(40)], [4] * 40,
                  [["a"], ["b"], ["a", "b"], []] * 10)
    models = [im("m0"), im("m1", [("a", 1)], critical=True), im("m255", [("a" if j % 2 else "b", 1 + j % 3)
                                                                          for j in range(255)]),
              im("m-absent", [("a", 0)]), im("m-unloaded", [("zz", 1)])]
    from test_gpu_snapshot_mutation import PodState
    ids_of = {m: i for i, m in enumerate(("a", "b"))}
    state = PodState(2, [p.Metrics.KVCacheUsagePercent for p in pods], [p.Metrics.WaitingQueueSize for p in pods],
                     [p.Metrics.MaxActiveModels for p in pods],
                     [[ids_of[m] for m in p.Metrics.ActiveModels] for p in pods])
    # state.packed() names adapters by WL.adapter_name: use the workload names in the models
    nm = {"a": WL.adapter_name(0), "b": WL.adapter_name(1), "zz": "zz"}
    models = [im(m.Spec.ModelName, [(nm[t.Name], t.Weight) for t in m.Spec.TargetModels],
                 critical=m.Spec.Criticality == WL.CRITICAL) for m in models]
    ids = np.random.default_rng(5).integers(0, len(models) + 3, 4000).astype(np.uint32)
    bounds = FC.random_split(len(ids), np.random.default_rng(6), 50)
    n = len(bounds) - 1
    calls = split(ids, bounds, [9] * n, [(i % K) + 1 for i in range(n)], kind="m", first_index=(1 << 64) - 1500)
    calls.insert(3, ("d", mixed_requests(2, 200, 7), 9, 8))
    want = oracle(state, calls, 50, models)
    mo = [o for o, c in zip(want[0], calls) if c[0] == "m"]
    st = {int(s) for o in mo for s in o["status"]}
    assert N.LIG_NO_MODEL in st and N.LIG_OK in st
    assert {0, 255} <= {int(t) for o in mo for t in o["target_idx"]} and want[2].sum() > 0
    with engine_for(state, 4000, models) as e:
        assert_same(run_chain(e, 1, calls, 50, state.P, FORMS), want, "model edges")


# ---- a herd moves pods: the rows follow the chain's tables ----------------------------------------------
def test_herding_rows_follow_the_chain_tables():
    thr = (0.8, 5, 50)
    P, A, W = 48, 8, 50
    rng = np.random.default_rng(90)
    state = random_state(P, A, seed=91)
    state.q[:] = rng.integers(0, thr[1] + 1, P)
    state.kv[:] = np.round(rng.random(P) * 0.6, 2)
    reqs = WL.make_requests(4000, A, seed=92)
    reqs["adapter_id"] = rng.choice([0, 1, A], len(reqs))
    calls = split(reqs, list(range(0, 4001, 8)), [93] * 500, [K] * 500)          # micro-batches of 8
    want = oracle(state, calls, W)
    q_end = np.minimum(state.q + want[2], INT32_MAX)
    assert ((state.q <= thr[1]) & (q_end > thr[1])).any() and ((state.q < thr[2]) & (q_end >= thr[2])).any()
    with engine_for(state, 4000) as e:
        got = run_chain(e, 1, calls, W, P)
        assert_same(got, want, "herd")
        _, resident = e.schedule_batch_fallbacks(1, 93, reqs, K)
    rows = np.concatenate(got[1])
    assert np.array_equal(rows[:W], resident[:W])                    # no window closed yet: the resident rows
    differ = (rows[W:] != resident[W:]).any(axis=1)
    assert differ.mean() > 0.3, differ.mean()
    # every row is inside the survivor set of the chain's tables at its window (the definition asserts
    # the pick; here the entries): replay the windows
    p = state.packed()
    picks = np.concatenate(got[0])
    q = state.q.copy()
    for w0 in range(0, len(reqs), W):
        tab = B.ClassTable(P, A, p.kv, q.astype(np.int32), p.n_active, p.max_active, p.bitmap)
        crit, a = FF.class_of(reqs[w0:w0 + W], A)
        for i, (cr, ai) in enumerate(zip(crit.tolist(), a.tolist())):
            r = rows[w0 + i]
            assert set(r[r >= 0].tolist()) <= set(tab.klass(bool(cr), int(ai))[2])
        seg = picks["pod_idx"][w0:w0 + W]
        q = np.minimum(q + np.bincount(seg[seg >= 0], minlength=P), INT32_MAX)


# ---- buffers and streams --------------------------------------------------------------------------------
def test_two_streams_without_host_synchronisation():
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=11)
    models = WL.make_models(c["A"])
    W = 333
    calls = mixed_chain(c["A"], len(models), 20000, seed=12, ks=[8, 3, 0, 5], window=W)
    want = oracle(state, calls, W, models)
    with engine_for(state, 20000, models) as e:
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        pending = []
        torch.cuda.synchronize()
        for i, call in enumerate(calls):
            with torch.cuda.stream(streams[i % 2]):
                pending.append(run_call(e, 1, call, W, state.P, "device", streams[i % 2], sync=False))
        torch.cuda.synchronize()
        got = [read() for read, _ in pending]
        assert_same(([g[0] for g in got], [g[1] for g in got], got[-1][2]), want, "two streams")


def test_model_upload_while_a_device_call_is_queued():
    packed = pack_pod_metrics(mkpods([0] * 8, [0.1] * 8, [1] * 8, [["x"]] * 4 + [["y"]] * 4))
    old = pack_models([im("m", [("x", 1)], critical=True)], packed)
    new = pack_models([im("m", [("y", 1)])], packed)
    with feedback_engine(8, 2, 4096) as e:
        e.set_filter_tree([N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0)])
        e.upload_snapshot(1, packed)
        ids = np.zeros(3000, dtype=np.uint32)
        e.upload_models(1, old)
        want_old = e.schedule_models_batch_fallbacks(1, 4, ids, 8)
        e.upload_models(1, new)
        want_new = e.schedule_models_batch_fallbacks(1, 4, ids, 8, first_index=3000)
        assert not np.array_equal(want_old[1], want_new[1])
        e.upload_models(1, old)
        st = torch.cuda.Stream()
        W = 1 << 20                                   # no window closes: the resident rows
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(100_000_000)            # keep the call queued behind ~50 ms of work
            read, _bufs = run_call(e, 1, ("m", ids, 4, 0, 8), W, 8, "device", st, sync=False)
        e.upload_models(1, new)
        st.synchronize()
        out, rows, _ = read()
        assert out.tobytes() == want_old[0].tobytes() and np.array_equal(rows, want_old[1])
        out, rows, _ = run_call(e, 1, ("m", ids, 4, 3000, 8), W, 8, "pinned")
        assert out.tobytes() == want_new[0].tobytes() and np.array_equal(rows, want_new[1])


# ---- refusals and resident epochs -----------------------------------------------------------------------
def test_refusals_leave_the_chain_untouched():
    lib = N.load()
    P, A, W = 64, 8, 30
    state = random_state(P, A, seed=51)
    models = WL.make_models(A)
    calls = mixed_chain(A, len(models), 600, seed=52, ks=[8, 2], window=W)
    want = oracle(state, calls, W, models)
    reqs, ids = WL.make_requests(50, A), np.zeros(50, np.uint32)
    out, mout = np.zeros(50, PICK_DTYPE), np.zeros(50, MPICK_DTYPE)
    rows = np.full(50 * 8, 7, np.int16)
    loads = np.full(P, 9, np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    with engine_for(state, 100, models) as e:
        ctx = e._ctx
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_out = torch.zeros(50 * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.zeros(50 * 8 + 1, dtype=torch.int16, device="cuda")

        def refuse():
            codes = [
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), 0, p(rows), W, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), 9, p(rows), W, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), 2, None, W, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, p(reqs), 50, p(out), 2, p(rows), 0, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 2, 0, p(reqs), 50, p(out), 2, p(rows), W, p(loads)),
                lib.lig_schedule_models_batch_feedback_chain_fallbacks(ctx, 1, 0, 0, p(ids), 50, p(mout), -1, p(rows),
                                                                       W, p(loads)),
                lib.lig_schedule_models_batch_feedback_chain_fallbacks(ctx, 2, 0, 0, p(ids), 50, p(mout), 2, p(rows),
                                                                       W, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, p(WL.make_requests(101, A)), 101,
                                                                p(np.zeros(101, PICK_DTYPE)), 1,
                                                                p(np.zeros(101, np.int16)), W, p(loads)),
                lib.lig_schedule_batch_feedback_chain_fallbacks_device(ctx, 1, 0, d_reqs.data_ptr(), 50,
                                                                       d_out.data_ptr(), 2, d_rows.data_ptr() + 1, W,
                                                                       None, None),
                lib.lig_schedule_batch_feedback_chain_fallbacks_device(ctx, 1, 0, d_reqs.data_ptr(), 50,
                                                                       d_out.data_ptr(), 9, d_rows.data_ptr(), W,
                                                                       None, None),
                lib.lig_schedule_models_batch_feedback_chain_fallbacks_device(ctx, 1, 0, 0, d_reqs.data_ptr(), 50,
                                                                              d_out.data_ptr(), 2, None, W, None,
                                                                              None),
            ]
            return codes

        half = len(calls) // 2
        got = run_chain(e, 1, calls[:half], W, P, FORMS)
        codes = refuse()
        assert codes[:4] == [N.LIG_ERR_INVALID] * 4 and codes[4] == N.LIG_ERR_STALE_EPOCH, codes
        assert codes[5] == N.LIG_ERR_INVALID and codes[6] == N.LIG_ERR_STALE_EPOCH, codes
        assert codes[7:] == [N.LIG_ERR_INVALID] * 4, codes
        assert (rows == 7).all() and (out["pod_idx"] == 0).all() and (loads == 9).all()
        rest = run_chain(e, 1, calls[half:], W, P, FORMS)
        assert_same((got[0] + rest[0], got[1] + rest[1], rest[2]), want, "refusals in the middle")
        # R = 0 with loads reads them without scheduling
        L = np.zeros(P, np.int32)
        assert lib.lig_schedule_batch_feedback_chain_fallbacks(ctx, 1, 0, None, 0, None, 3, None, W, p(L)) == 0
        assert np.array_equal(L, want[2])


def test_resident_epochs_are_untouched_by_a_herd():
    P, A = 64, 8
    state = random_state(P, A, seed=31)
    state.q[:] = 0
    reqs = WL.make_requests(20000, A, seed=32)
    reqs["adapter_id"] = 0
    with engine_for(state, 20000) as e:
        classes = lambda: [e.read_class(1, cr, a, P) for cr in (0, 1) for a in range(A + 1)]   # noqa: E731
        before_cls, before = classes(), e.schedule_batch_fallbacks(1, 3, reqs, K)
        calls = split(reqs, list(range(0, 20001, 2500)), [3] * 8, [K] * 8)
        _, _, loads = run_chain(e, 1, calls, 8, P, FORMS)
        assert loads.max() < np.bincount(before[0]["pod_idx"][before[0]["pod_idx"] >= 0], minlength=P).max()
        after = classes()
        assert all(b[0] == a[0] and b[1] == a[1] and np.array_equal(b[2], a[2]) for b, a in zip(before_cls, after))
        again = e.schedule_batch_fallbacks(1, 3, reqs, K)
        assert again[0].tobytes() == before[0].tobytes() and np.array_equal(again[1], before[1])


def test_c4_one_call_at_2_to_20():
    c = WL.CONFIGS["C4"]
    state = random_state(c["P"], c["A"], seed=61)
    reqs = WL.make_requests(1 << 20, c["A"], seed=62)
    want = oracle(state, [("d", reqs, 63, K)], 4096)
    with engine_for(state, 1 << 20) as e:
        assert_same(run_chain(e, 1, [("d", reqs, 63, K)], 4096, state.P, ("device",)), want, "C4")
    # the built-in tree keeps at most 4 survivors per class at C4: short rows, but rows
    assert (want[1][0][:, 0] >= 0).mean() > 0.1 and want[2].sum() > 0


# ---- schedulers -----------------------------------------------------------------------------------------
def test_python_scheduler_feedback_fallbacks():
    from test_gpu_filter_batch import scheduler_pods
    pods = scheduler_pods()
    reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=c) for m in ("a", "b", "c", "zz", "") for c in (False, True)]
    reqs = reqs * 20
    models = [im("m-a", [("a", 1)]), im("m-split", [("a", 3), ("b", 5), ("c", 2)], critical=True), im("m-self"),
              im("m-zero", [("a", 0)]), im("b")]
    names = ["m-a", "m-split", "unknown", "m-zero", "m-self", "b", "m-split", "m-split"] * 10
    W = 6
    kw = dict(max_pods=64, max_adapters=8, max_batch=256, seed=5, load_feedback_window=W)
    twin = S.NewScheduler(StaticProvider(pods), **kw)
    fb = S.NewScheduler(StaticProvider(pods), feedback_fallbacks=True, **kw)
    check = feedback_engine(64, 8, 256)
    try:
        twin.SetInferenceModels(models)
        fb.SetInferenceModels(models)
        check.upload_snapshot(1, fb._snap)
        check.upload_models(1, fb._packed_models)
        for n in (1, 3, 8):
            keys = random.Random()
            keys.setstate(fb._rng.getstate())
            want = twin.ScheduleBatch(reqs)
            got = fb.ScheduleBatchWithFallbacks(reqs, n)
            arr = np.zeros(len(reqs), dtype=REQ_DTYPE)
            for i, r in enumerate(reqs):
                arr[i] = (fb._snap.adapter_id(r.ResolvedTargetModel), 1 if r.Critical else 0, keys.getrandbits(64))
            check.feedback_chain_reset()          # the provider has no Version(): every call is a new epoch
            picks, rows = check.schedule_batch_feedback_chain_fallbacks(1, fb._seed, arr, n, W)
            for (pod, err), (ranked, ferr), pk, row in zip(want, got, picks, rows):
                assert (err is None) == (ferr is None)
                if err is not None:
                    assert (err.code, str(err)) == (ferr.code, str(ferr)) and ranked == []
                    continue
                assert ranked[0] == pod and ranked[0] == fb._snap.pods[int(pk["pod_idx"])]
                assert [p.Name for p in ranked[1:]] == [fb._snap.pods[int(x)].Name for x in row if x >= 0]
            first = fb._model_index
            want = twin.ScheduleModelBatch(names)
            got = fb.ScheduleModelBatchWithFallbacks(names, n)
            assert twin._model_index == fb._model_index
            sent = [fb._packed_models.model_ids[m] for m in names
                    if m in fb._packed_models.model_ids and fb._packed_models.present[fb._packed_models.model_ids[m]]]
            check.feedback_chain_reset()
            mp, mrows = check.schedule_models_batch_feedback_chain_fallbacks(1, fb._seed, np.array(sent, np.uint32), n,
                                                                             W, first_index=first)
            j = 0
            for name, (pod, resolved, err), (ranked, fres, ferr) in zip(names, want, got):
                assert resolved == fres and (err is None) == (ferr is None)
                if err is None:
                    assert ranked[0] == pod and [p.Name for p in ranked[1:]] == \
                        [fb._snap.pods[int(x)].Name for x in mrows[j] if x >= 0]
                else:
                    assert (err.code, str(err)) == (ferr.code, str(ferr)) and ranked == []
                j += name in fb._packed_models.model_ids and fb._packed_models.present[fb._packed_models.model_ids[name]]
            assert j == len(sent) == len(mp)
        # single requests: the same pod as the twin's Schedule
        for r in reqs[:10]:
            try:
                pod = twin.Schedule(r)
            except S.StatusError as err:
                with pytest.raises(S.StatusError) as got_err:
                    fb.ScheduleWithFallbacks(r, 4)
                assert str(got_err.value) == str(err)
            else:
                assert fb.ScheduleWithFallbacks(r, 4)[0] == pod
        with pytest.raises(ValueError):
            fb.ScheduleBatchWithFallbacks(reqs, 0)
    finally:
        twin.close()
        fb.close()
        check.close()


def test_cpp_runtime_feedback_fallbacks_under_concurrent_callers():
    """W = 8 with the opt-in; every pod survives (KEEP_ALL), so each result is the ranking of its own
    key over the whole pool, whatever window it fell in, and the windows equal a run without rows."""
    from llm_instance_gateway_b200 import host as H
    P, seed, W = 64, 0x5151, 8
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)], [4] * P, [["a"]] * P)
    prov = H.HostProvider(pods)
    results = []
    lock = threading.Lock()

    def run(hs, with_rows):
        def caller(t):
            mine = []
            for k in range(40):
                kind = (t + k) % 4
                n = 1 + (t + k) % K if with_rows else 0
                if kind == 0 or (kind == 1 and not with_rows):
                    code, pod, _ = hs.Schedule("m", "a", False)
                    mine.append(("d", 0, code, [pod.Name] if pod else [], None))
                elif kind == 1:
                    code, names, _ = hs.ScheduleWithFallbacks("a", False, n)
                    mine.append(("d", n, code, names, None))
                elif kind == 2 or not with_rows:
                    code, resolved, pod, _ = hs.ScheduleModelOnDevice("m")
                    mine.append(("m", 0, code, [pod.Name] if pod else [], resolved))
                else:
                    code, resolved, names, _ = hs.ScheduleModelWithFallbacks("m", n)
                    mine.append(("m", n, code, names, resolved))
            with lock:
                results.extend(mine)
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(12)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()

    def scheduler():
        hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200,
                             seed=seed, filter=KEEP_ALL, load_feedback_window=W, feedback_fallbacks=True)
        store = H.HostDataStore([im("m", [("a", 1)])])
        hs.set_inference_models(store)
        return hs, store

    hs, store = scheduler()
    try:
        run(hs, True)
        st = hs.stats()
        total = len(results)
        assert total == 480 and all(r[2] == H.GRPC_OK for r in results)
        assert st["fallback_scheduled"] == sum(1 for r in results if r[1] > 0)
        assert all(r[4] == "a" for r in results if r[0] == "m")
        n_desc = sum(1 for r in results if r[0] == "d")
        n_model = total - n_desc
        assert st["feedback_windows"] == total // W or st["feedback_restarts"] > 0
        windows_with_rows = st["feedback_windows"]
        # refusals
        assert hs.ScheduleModelWithFallbacks("m", 0)[0] == 3 and hs.ScheduleModelWithFallbacks("m", K + 1)[0] == 3
    finally:
        hs.close()
    results_rows = list(results)
    results.clear()
    plain, store2 = scheduler()
    try:
        run(plain, False)
        assert plain.stats()["feedback_windows"] == windows_with_rows
    finally:
        plain.close()
    # the library over the runtime's key sequences: descriptors take splitmix keys, model ids k = 0, 1, ...
    e = feedback_engine(P, 8, 4096)
    try:
        e.set_filter_tree(KEEP_ALL)
        packed = pack_pod_metrics(pods)
        e.upload_snapshot(1, packed)
        e.upload_models(1, pack_models([im("m", [("a", 1)])], packed))
        dreqs = np.zeros(n_desc, dtype=REQ_DTYPE)
        dreqs["adapter_id"] = packed.adapter_id("a")
        dreqs["rand_key"] = splitmix_keys(seed, n_desc)
        dp, drows = e.schedule_batch_fallbacks(1, seed, dreqs, K)
        mp, mrows = e.schedule_models_batch_fallbacks(1, seed, np.zeros(n_model, np.uint32), K)
    finally:
        e.close()
    name = lambda i: f"pod-{i}"                                                  # noqa: E731
    for kind, picks, rows in (("d", dp, drows), ("m", mp, mrows)):
        expect = [[name(picks["pod_idx"][k])] + [name(x) for x in rows[k] if x >= 0] for k in range(len(picks))]
        mine = [r for r in results_rows if r[0] == kind]
        assert sorted(r[3][0] for r in mine) == sorted(x[0] for x in expect), kind
        used = set()
        by_pick = {}
        for k, x in enumerate(expect):
            by_pick.setdefault(x[0], []).append(k)
        for _, n, _, names, _ in sorted(mine, key=lambda r: -r[1]):
            if n == 0:
                continue
            assert len(names) == n + 1
            ks = [k for k in by_pick[names[0]] if k not in used and expect[k][:n + 1] == names]
            assert ks, (kind, names)
            used.add(ks[0])
    prov.close()
    store.close()
    store2.close()


def test_cpp_runtime_model_fallbacks_without_feedback_and_refusals():
    from llm_instance_gateway_b200 import host as H
    P, seed = 32, 0x77
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)], [4] * P, [["a"], ["b"]] * (P // 2))
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, seed=seed, filter=KEEP_ALL)
    try:
        store = H.HostDataStore([im("m", [("a", 1), ("b", 3)], critical=True)])
        hs.set_inference_models(store)
        got = [hs.ScheduleModelWithFallbacks(name, 1 + k % K) for k, name in enumerate(["m", "nope"] * 20)]
        assert all(g[0] == H.GRPC_OK for g in got[::2]) and all(g[0] == 2 and g[2] == [] for g in got[1::2])
        assert "error finding a model object" in got[1][3]
        e = feedback_engine(P, 8, 64)
        try:
            e.set_filter_tree(KEEP_ALL)
            packed = pack_pod_metrics(pods)
            e.upload_snapshot(1, packed)
            e.upload_models(1, pack_models([im("m", [("a", 1), ("b", 3)], critical=True)], packed))
            mp, mrows = e.schedule_models_batch_fallbacks(1, seed, np.zeros(20, np.uint32), K)
        finally:
            e.close()
        tnames = ["a", "b"]
        for k, g in enumerate(got[::2]):
            n = 1 + (2 * k) % K
            assert g[1] == tnames[mp["target_idx"][k]]
            assert g[2] == [f"pod-{mp['pod_idx'][k]}"] + [f"pod-{x}" for x in mrows[k][:n] if x >= 0]
        st = hs.stats()
        assert st["fallback_scheduled"] == 40 and st["model_scheduled"] == 40
        assert hs.ScheduleModelWithFallbacks("m", 0)[0] == 3
        store.close()
    finally:
        hs.close()
    chain = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=8)
    try:
        code, resolved, names, err = chain.ScheduleModelWithFallbacks("m", 2)
        assert code == 3 and "load_feedback_window" in err and names == []
    finally:
        chain.close()
        prov.close()
