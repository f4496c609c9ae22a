"""Session affinity under the load-feedback chain on the device (include/lig.h,
lig_schedule_[models_]batch_feedback_chain_affinity[_device]), bit for bit:

* `out`, rows and loads against the sequential definition (feedback_chain_affinity_ref) at C1 and C4, with
  the built-in tree and a keep-all caller tree, W in {1, 7, 64}, n in {0, 1, 8}, random call splits, and
  pageable, page-locked, +8-byte and device buffers;
* with no window closed, the resident lig_schedule_[models_]batch_affinity byte for byte;
* one chain mixing plain, fallback and affinity calls of both kinds;
* long lists under the count form (the warp path and the full-warp match), an ejected epoch's pool and
  model ids that do not resolve;
* a pod-key upload and a model upload behind a queued device call; refusals leave the chain untouched;
  resident epochs stay as they were;
* the Python scheduler's and the C++ runtime's feedback_affinity option, and concurrent callers.
"""
import threading
from collections import namedtuple

import numpy as np
import pytest
import torch

import affinity_ref as AR
import feedback_chain_affinity_ref as FA
import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
import test_gpu_feedback_chain_fallbacks as FCF
from test_gpu_affinity import KEEP_ALL, KEEP_ALL_CHART, LORA_ONLY
from test_gpu_affinity import pool as scheduler_pool
from test_gpu_filter_batch import im
from test_gpu_filter_tree import mkpods
from test_gpu_snapshot_mutation import feedback_engine, mixed_requests, random_state
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_columns, pack_models, \
    pack_pod_metrics
from oracle import binding as B

pytestmark = pytest.mark.gpu

K = N.LIG_MAX_FALLBACKS
FORMS = FCF.FORMS
# kind "d" (descriptors: rand_key is the affinity key) or "m" (model ids with keys); what "plain",
# "fallbacks" or "affinity"; k the rows (0 = none); seed and first are ignored by affinity calls
Call = namedtuple("Call", "kind data keys seed first what k")


def d_call(reqs, what="affinity", k=0, seed=0):
    return Call("d", np.ascontiguousarray(reqs), None, seed, 0, what, k)


def m_call(ids, keys=None, what="affinity", k=0, seed=0, first=0):
    return Call("m", np.ascontiguousarray(ids, dtype=np.uint32),
                None if keys is None else np.ascontiguousarray(keys, dtype=np.uint64), seed, first, what, k)


def ref_calls(calls, mo=None, adapter_id=None):
    out = []
    for c in calls:
        if c.kind == "d":
            out.append((c.data, c.seed))
        elif c.what == "affinity":
            out.append(FA.affinity_model_call(mo, adapter_id, c.data, c.keys))
        else:
            out.append(MC.model_call(mo, adapter_id, c.data, c.seed, c.first))
    return out, [(c.what, c.k) for c in calls]


def oracle(state, pod_keys, calls, W, models=None, tree=None):
    p = state.packed()
    mo = B.Models(WL.model_records(models)) if models is not None else None
    rc, specs = ref_calls(calls, mo, p.adapter_id)
    if tree is not None:
        return FA.schedule_chain_affinity_tree(tree, state.records(), state.names(), pod_keys, rc, specs, W)
    return FA.schedule_chain_affinity(p.P, p.A, p.kv, state.q, p.n_active, p.max_active, p.bitmap, pod_keys, rc,
                                      specs, W)


def dev(arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1).copy()).cuda()


def run_affinity(e, ep, c, W, P, form, stream=None, sync=True):
    """One chain affinity call in `form`: (picks, rows (R, k), loads[P]); with sync=False (device form)
    a reader to call after a synchronise, and the buffers to keep alive."""
    R, k, models = len(c.data), c.k, c.kind == "m"
    odt = MPICK_DTYPE if models else PICK_DTYPE
    if form == "device":
        d_in = dev(c.data) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
        d_keys = dev(c.keys) if models and R else None
        d_out = torch.full((max(R, 1) * odt.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
        d_rows = torch.full((max(R * k, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
        d_loads = torch.full((max(P, 1),), -7, dtype=torch.int32, device="cuda")
        st = stream or torch.cuda.current_stream()
        if sync:
            torch.cuda.synchronize()
        inp = d_in.data_ptr() if R else 0
        rp = d_rows.data_ptr() if k else 0
        if models:
            e.schedule_models_batch_feedback_chain_affinity_device(ep, inp, d_keys.data_ptr() if R else 0, R,
                                                                   d_out.data_ptr(), k, rp, W, d_loads.data_ptr(),
                                                                   st.cuda_stream)
        else:
            e.schedule_batch_feedback_chain_affinity_device(ep, inp, R, d_out.data_ptr(), k, rp, W, d_loads.data_ptr(),
                                                            st.cuda_stream)

        def read():
            return (d_out[: R * odt.itemsize].cpu().numpy().view(odt), d_rows[: R * k].cpu().numpy().reshape(R, k),
                    d_loads[:P].cpu().numpy().astype(np.int64))
        if not sync:
            return read, (d_in, d_keys, d_out, d_rows, d_loads)
        st.synchronize()
        return read()
    lib, keep = N.load(), []
    try:
        loads = np.full(max(P, 1), -7, dtype=np.int32)
        keys = c.keys if models else np.zeros(0, np.uint64)
        if form == "pageable":
            inp, out, rows = c.data, np.zeros(R, odt), np.zeros((R, k), np.int16)
            pin, pout, prows, pkeys = inp.ctypes.data, out.ctypes.data, rows.ctypes.data, keys.ctypes.data
        else:
            shift = 8 if form == "pinned+8" else 0          # +8: requests and picks bounce, rows and keys staged
            _, pin = FCF._host_buf(lib, c.data, shift, keep)
            out, pout = FCF._host_buf(lib, np.zeros(R, odt), shift, keep)
            rows, prows = FCF._host_buf(lib, np.zeros(R * k, np.int16), 1 if shift else 0, keep)
            _, pkeys = FCF._host_buf(lib, keys, 4 if shift else 0, keep)
        if not R:
            pin = pout = prows = pkeys = 0
        if not k:
            prows = 0
        if models:
            e.schedule_models_batch_feedback_chain_affinity_ptr(ep, pin, pkeys, R, pout, k, prows, W, loads.ctypes.data)
        else:
            e.schedule_batch_feedback_chain_affinity_ptr(ep, pin, R, pout, k, prows, W, loads.ctypes.data)
        return (np.frombuffer(out.tobytes(), odt).copy(), np.frombuffer(rows.tobytes(), np.int16).reshape(R, k).copy(),
                loads[:P].astype(np.int64))
    finally:
        for b in keep:
            b.free()


def run_call(e, ep, c, W, P, form="pageable", stream=None, sync=True):
    if c.what == "affinity":
        return run_affinity(e, ep, c, W, P, form, stream, sync)
    k = c.k if c.what == "fallbacks" else 0
    legacy = ("d", c.data, c.seed, k) if c.kind == "d" else ("m", c.data, c.seed, c.first, k)
    return FCF.run_call(e, ep, legacy, W, P, form, stream, sync)


def run_chain(e, ep, calls, W, P, forms=("pageable",)):
    outs, rows, loads = [], [], None
    for i, c in enumerate(calls):
        o, r, loads = run_call(e, ep, c, W, P, forms[i % len(forms)])
        outs.append(o)
        rows.append(r)
    return outs, rows, loads


def engine_for(state, R, models=None, tree=None, seed=0):
    e = feedback_engine(state.P, state.A, R)
    p = state.packed()
    if tree is not None:
        e.set_filter_tree(tree)
    e.upload_snapshot(1, p)
    pod_keys = np.random.default_rng(seed).integers(0, 1 << 64, size=state.P, dtype=np.uint64)
    e.upload_pod_keys(1, pod_keys)
    if models is not None:
        e.upload_models(1, pack_models(models, p))
    return e, pod_keys


def keyed(A, R, seed, n_keys=200, classes=True):
    """mixed_requests (or, without classes, workload requests only) with session keys: a few hundred
    keys, each repeated."""
    reqs = mixed_requests(A, R, seed) if classes else WL.make_requests(R, A, seed=seed + 1)
    reqs["rand_key"] = AR.mix(np.random.default_rng(seed).integers(1, n_keys + 1, len(reqs)).astype(np.uint64))
    return reqs


def affinity_split(data, bounds, ks, kind="d", keys=None):
    if kind == "d":
        return [d_call(data[a:b], k=ks[i]) for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]
    return [m_call(data[a:b], keys[a:b], k=ks[i]) for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]


# ---- against the definition ---------------------------------------------------------------------------
@pytest.mark.parametrize("cfg,tree", [("C1", None), ("C1", "keep_all"), ("C4", None), ("C4", "keep_all")])
def test_parity_against_the_definition(cfg, tree):
    c = WL.CONFIGS[cfg]
    state = random_state(c["P"], c["A"], seed=c["P"] + 3)
    nodes = KEEP_ALL if tree else None
    models = WL.make_models(c["A"])
    for W in (1, 7, 64):
        # C1 takes one request of every class as well; at C4 (2 x 1025 classes) the CPU reference would
        # spend minutes on them, so C4 takes workload requests only, enough for every split size
        if cfg == "C4":
            reqs = keyed(c["A"], {1: 60, 7: 200, 64: 700}[W], seed=W, classes=False)
        else:
            reqs = keyed(c["A"], {1: 300, 7: 1200, 64: 4000}[W], seed=W)
        ids = np.random.default_rng(W).integers(0, len(models), len(reqs)).astype(np.uint32)
        ids[::7] = len(models) + 1                 # ids that do not resolve: LIG_NO_MODEL, counted, no pick
        rng = np.random.default_rng(W + 1)
        bounds = FC.random_split(len(reqs), rng, W)
        ks = [(0, 1, K)[i % 3] for i in range(len(bounds) - 1)]
        calls = [d_call(reqs[a:b], k=ks[i]) if i % 2 == 0 else m_call(ids[a:b], reqs["rand_key"][a:b], k=ks[i])
                 for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]
        e, pod_keys = engine_for(state, len(reqs), models, nodes)
        with e:
            got = run_chain(e, 1, calls, W, state.P, FORMS)
        want = oracle(state, pod_keys, calls, W, models, nodes)
        FCF.assert_same(got, want, (cfg, tree, W))
        picks = np.concatenate([o["pod_idx"] for o in want[0]]).astype(np.int64)
        assert np.array_equal(want[2], np.bincount(picks[picks >= 0], minlength=state.P)) and want[2].sum() > 0
        assert N.LIG_NO_MODEL in {int(s) for o, x in zip(want[0], calls) if x.kind == "m" for s in o["status"]}


def test_no_closed_window_equals_resident_affinity():
    c = WL.CONFIGS["C2"]
    state = random_state(c["P"], c["A"], seed=9)
    models = WL.make_models(c["A"])
    reqs = keyed(c["A"], 3000, seed=10)
    ids = np.random.default_rng(11).integers(0, len(models) + 2, len(reqs)).astype(np.uint32)
    keys = np.random.default_rng(12).integers(0, 1 << 64, size=len(reqs), dtype=np.uint64)
    e, _ = engine_for(state, 8000, models)
    with e:
        for n in (0, 1, 8):
            for form in ("pageable", "pinned", "device"):
                e.feedback_chain_reset()
                out, rows = e.schedule_batch_affinity(1, reqs, n)
                got = run_call(e, 1, d_call(reqs, k=n), 1 << 20, state.P, form)
                assert got[0].tobytes() == out.tobytes() and np.array_equal(got[1], rows), (n, form)
                mout, mrows = e.schedule_models_batch_affinity(1, ids, keys, n)
                got = run_call(e, 1, m_call(ids, keys, k=n), 1 << 20, state.P, form)
                assert got[0].tobytes() == mout.tobytes() and np.array_equal(got[1], mrows), (n, form)


def test_one_chain_mixes_every_kind():
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=13)
    models = WL.make_models(c["A"])
    W = 97
    reqs = keyed(c["A"], 6000, seed=14)
    ids = np.random.default_rng(15).integers(0, len(models) + 3, len(reqs)).astype(np.uint32)
    bounds = FC.random_split(len(reqs), np.random.default_rng(16), W)
    calls, first = [], (1 << 64) - 700
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        what = ("plain", "fallbacks", "affinity")[i % 3]
        k = 0 if what == "plain" else (1, 4, K, 0)[i % 4] if what == "affinity" else 1 + i % K
        if (i // 3) % 2:
            calls.append(m_call(ids[a:b], reqs["rand_key"][a:b], what, k, seed=50 + i, first=first % (1 << 64)))
            first += b - a
        else:
            calls.append(d_call(reqs[a:b], what, k, seed=50 + i))
    e, pod_keys = engine_for(state, len(reqs), models)
    with e:
        got = run_chain(e, 1, calls, W, state.P, FORMS)
    FCF.assert_same(got, oracle(state, pod_keys, calls, W, models), "mixed")
    assert {(x.kind, x.what) for x in calls} == {(a, b) for a in "dm" for b in ("plain", "fallbacks", "affinity")}


# ---- long lists under the count form ------------------------------------------------------------------
def test_long_and_short_lists_in_one_warp_under_load():
    """The built-in tree over an idle pool: adapter 0 on every pod (lists of 100 that shrink as the chain
    loads pods), 1 on 5 pods, 2 on 40 pods, 3 on none, interleaved; R not a multiple of 32."""
    P, A = 100, 3
    mask = {0: range(P), 1: [3, 17, 50, 51, 99], 2: range(10, 90, 2)}
    from test_gpu_snapshot_mutation import PodState
    state = PodState(A, [0.1] * P, [0] * P, [4] * P, [[a for a in range(A) if p in mask[a]] for p in range(P)])
    reqs = np.zeros(4097, dtype=REQ_DTYPE)
    rng = np.random.default_rng(3)
    reqs["adapter_id"] = rng.integers(0, 4, len(reqs))
    reqs["flags"] = rng.integers(0, 2, len(reqs))
    reqs["rand_key"] = AR.mix(rng.integers(1, 300, len(reqs)).astype(np.uint64))
    for W in (7, 64):
        bounds = FC.random_split(len(reqs), np.random.default_rng(W), W)
        calls = affinity_split(reqs, bounds, [(0, 1, K)[i % 3] for i in range(len(bounds) - 1)])
        e, pod_keys = engine_for(state, len(reqs))
        with e:
            got = run_chain(e, 1, calls, W, P, FORMS)
        want = oracle(state, pod_keys, calls, W)
        FCF.assert_same(got, want, W)
        out = np.concatenate(want[0])
        assert (out["n_survivors"][out["status"] == N.LIG_OK] > 32).any()
        assert (out["n_survivors"][out["status"] == N.LIG_OK] <= 32).any()


@pytest.mark.parametrize("P", [33, 4096, 32768])
def test_keep_all_lists_up_to_32768_pods(P):
    """A keep-all tree keeps every pod whatever the loads: every call equals resident affinity, and the
    loads are the bincount of the picks (lists past 32 pods take the warp path)."""
    e = feedback_engine(P, 1, 4096)
    with e:
        e.set_filter_tree(KEEP_ALL)
        e.upload_snapshot(1, pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64),
                                          np.zeros(P, np.int64), np.zeros((1, (P + 31) // 32), np.uint32)))
        e.upload_pod_keys(1, np.random.default_rng(P).integers(0, 1 << 64, size=P, dtype=np.uint64))
        reqs = np.zeros(1000, dtype=REQ_DTYPE)
        reqs["adapter_id"] = np.arange(1000) % 2
        reqs["rand_key"] = np.random.default_rng(P + 1).integers(0, 1 << 64, size=1000, dtype=np.uint64)
        want, want_rows = e.schedule_batch_affinity(1, reqs, K)
        assert (want["n_survivors"] == P).all()
        for W, form in ((1, "device"), (7, "pinned"), (64, "pageable")):
            e.feedback_chain_reset()
            outs, rows, loads = run_chain(e, 1, affinity_split(reqs, [0, 31, 33, 500, 1000], [K, 0, 1, K]), W, P,
                                          (form,))
            got = np.concatenate(outs)
            assert got.tobytes() == want.tobytes(), (P, W)
            assert np.array_equal(rows[0], want_rows[:31]) and np.array_equal(rows[3], want_rows[500:])
            assert np.array_equal(loads, np.bincount(want["pod_idx"], minlength=P))


def test_ejected_epoch_and_models_that_do_not_resolve():
    P, A = 256, 16
    snap = WL.make_snapshot(P, A, seed=21)
    models = WL.make_models(A)
    pm = pack_models(models, snap.packed)
    gone = np.sort(np.random.default_rng(22).choice(P, 60, replace=False)).astype(np.int32)
    pod_keys = np.random.default_rng(23).integers(0, 1 << 64, size=P, dtype=np.uint64)
    e = feedback_engine(P, A, 8192)
    with e:
        e.upload_snapshot(2, snap.packed)
        e.eject_pods(3, 2, gone)
        e.upload_models(3, pm)
        reqs = WL.make_requests(4000, A, seed=24)
        ids = np.random.default_rng(25).integers(0, len(models) + 5, 4000).astype(np.uint32)
        keys = np.random.default_rng(26).integers(0, 1 << 64, size=4000, dtype=np.uint64)
        out = np.zeros(4000, PICK_DTYPE)
        assert e._lib.lig_schedule_batch_feedback_chain_affinity(e._ctx, 3, reqs.ctypes.data, 4000, out.ctypes.data, 0,
                                                                 None, 8, None) == N.LIG_ERR_NO_SNAPSHOT   # no keys
        e.upload_pod_keys(3, pod_keys)
        want, want_rows = e.schedule_batch_affinity(3, reqs, K)
        mwant, mrows = e.schedule_models_batch_affinity(3, ids, keys, K)
        got = run_chain(e, 3, [d_call(reqs, k=K), m_call(ids, keys, k=K)], 1 << 20, P, ("device", "pinned+8"))
        assert got[0][0].tobytes() == want.tobytes() and np.array_equal(got[1][0], want_rows)
        assert got[0][1].tobytes() == mwant.tobytes() and np.array_equal(got[1][1], mrows)
        assert N.LIG_NO_MODEL in set(mwant["status"].tolist())
        for W in (1, 16):
            results = []
            for forms, split in ((("device",), [0, 4000]), (FORMS, [0, 1, 17, 900, 2500, 4000])):
                e.feedback_chain_reset()
                calls = affinity_split(reqs, split, [K] * (len(split) - 1)) + \
                    affinity_split(ids, split, [K] * (len(split) - 1), "m", keys)
                outs, rows, loads = run_chain(e, 3, calls, W, P, forms)
                results.append((np.concatenate([o["pod_idx"] for o in outs]), loads))
                for o, r in zip(outs, rows):
                    ok = o["pod_idx"] >= 0
                    assert not np.isin(o["pod_idx"], gone).any() and not np.isin(r, gone).any()
                    assert (r[~ok] == -1).all()
                picks = results[-1][0].astype(np.int64)
                assert np.array_equal(loads, np.bincount(picks[picks >= 0], minlength=P))
            assert np.array_equal(results[0][0], results[1][0]) and np.array_equal(results[0][1], results[1][1])


# ---- uploads, refusals, resident epochs -------------------------------------------------------------------
def test_key_and_model_uploads_behind_a_queued_call():
    packed = pack_pod_metrics(mkpods([0] * 8, [0.1] * 8, [1] * 8, [["x"]] * 4 + [["y"]] * 4))
    old_m = pack_models([im("m", [("x", 1)], critical=True)], packed)
    new_m = pack_models([im("m", [("y", 1)])], packed)
    old_k = np.arange(1, 9, dtype=np.uint64)
    new_k = np.arange(101, 109, dtype=np.uint64)
    ids = np.zeros(3000, dtype=np.uint32)
    keys = np.random.default_rng(1).integers(0, 1 << 64, size=3000, dtype=np.uint64)
    W = 1 << 20                                         # no window closes: the resident picks, loads add up
    with feedback_engine(8, 2, 4096) as e:
        e.set_filter_tree(LORA_ONLY)
        e.upload_snapshot(1, packed)
        e.upload_models(1, new_m)
        e.upload_pod_keys(1, new_k)
        want_new = e.schedule_models_batch_affinity(1, ids, keys, 8)
        e.upload_models(1, old_m)
        e.upload_pod_keys(1, old_k)
        want_old = e.schedule_models_batch_affinity(1, ids, keys, 8)
        assert not np.array_equal(want_old[1], want_new[1])
        e.feedback_chain_reset()
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(100_000_000)              # keep the call queued behind ~50 ms of work
            read, _bufs = run_call(e, 1, m_call(ids, keys, k=8), W, 8, "device", st, sync=False)
        e.upload_models(1, new_m)
        e.upload_pod_keys(1, new_k)
        st.synchronize()
        out, rows, loads1 = read()
        assert out.tobytes() == want_old[0].tobytes() and np.array_equal(rows, want_old[1])
        out, rows, loads2 = run_call(e, 1, m_call(ids, keys, k=8), W, 8, "pinned")
        assert out.tobytes() == want_new[0].tobytes() and np.array_equal(rows, want_new[1])
        assert loads1.sum() == 3000 and loads2.sum() == 6000           # the chain did not restart


def test_refusals_leave_the_chain_untouched():
    lib = N.load()
    P, A, W = 64, 8, 30
    state = random_state(P, A, seed=51)
    models = WL.make_models(A)
    reqs = keyed(A, 600, seed=52)
    ids = np.random.default_rng(53).integers(0, len(models), len(reqs)).astype(np.uint32)
    bounds = FC.random_split(len(reqs), np.random.default_rng(54), W)
    calls = [m_call(ids[a:b], reqs["rand_key"][a:b], k=2) if i % 2 else d_call(reqs[a:b], k=(i // 2) % 3)
             for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]
    rq, mids, mkeys = WL.make_requests(50, A), np.zeros(50, np.uint32), np.zeros(50, np.uint64)
    big, big_out = WL.make_requests(201, A), np.zeros(201, PICK_DTYPE)
    out, mout = np.zeros(50, PICK_DTYPE), np.zeros(50, MPICK_DTYPE)
    rows = np.full(50 * 8, 7, np.int16)
    loads = np.full(P, 9, np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    e, pod_keys = engine_for(state, 200, models)
    with e:
        ctx = e._ctx
        e.upload_snapshot(4, state.packed())
        e.upload_models(4, pack_models(models, state.packed()))
        d_reqs = dev(rq)
        d_keys = torch.zeros(51, dtype=torch.int64, device="cuda")
        d_out = torch.zeros(50 * 8 + 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.zeros(50 * 8 + 1, dtype=torch.int16, device="cuda")
        bp, mp = lib.lig_schedule_batch_feedback_chain_affinity, lib.lig_schedule_models_batch_feedback_chain_affinity
        bd = lib.lig_schedule_batch_feedback_chain_affinity_device
        md = lib.lig_schedule_models_batch_feedback_chain_affinity_device
        dr, dk, do, dw = d_reqs.data_ptr(), d_keys.data_ptr(), d_out.data_ptr(), d_rows.data_ptr()

        def refuse():
            return [
                bp(ctx, 1, p(rq), 50, p(out), 9, p(rows), W, p(loads)),
                bp(ctx, 1, p(rq), 50, p(out), -1, p(rows), W, p(loads)),
                bp(ctx, 1, p(rq), 50, p(out), 2, None, W, p(loads)),
                bp(ctx, 1, p(rq), 50, None, 0, None, W, p(loads)),
                bp(ctx, 1, p(rq), 50, p(out), 2, p(rows), 0, p(loads)),
                mp(ctx, 1, p(mids), None, 50, p(mout), 0, None, W, p(loads)),
                bp(ctx, 1, p(big), 201, p(big_out), 0, None, W, p(loads)),
                bd(ctx, 1, dr, 50, do, 2, dw + 1, W, None, None),
                bd(ctx, 1, dr + 8, 50, do, 0, None, W, None, None),
                bd(ctx, 1, dr, 50, do + 4, 0, None, W, None, None),
                md(ctx, 1, dr, dk + 4, 50, do, 0, None, W, None, None),
                md(ctx, 1, dr, dk, 50, do, 9, dw, W, None, None),
                bp(ctx, 2, p(rq), 50, p(out), 2, p(rows), W, p(loads)),               # stale epoch
                mp(ctx, 2, p(mids), p(mkeys), 50, p(mout), 2, p(rows), W, p(loads)),
                bp(ctx, 4, p(rq), 50, p(out), 2, p(rows), W, p(loads)),               # no pod keys
                md(ctx, 4, dr, dk, 50, do, 0, None, W, None, None),
            ]

        half = len(calls) // 2
        got = run_chain(e, 1, calls[:half], W, P, FORMS)
        codes = refuse()
        assert codes[:12] == [N.LIG_ERR_INVALID] * 12, codes
        assert codes[12:14] == [N.LIG_ERR_STALE_EPOCH] * 2 and codes[14:] == [N.LIG_ERR_NO_SNAPSHOT] * 2, codes
        assert (rows == 7).all() and (out["pod_idx"] == 0).all() and (mout["pod_idx"] == 0).all()
        assert (loads == 9).all()
        rest = run_chain(e, 1, calls[half:], W, P, FORMS)
        FCF.assert_same((got[0] + rest[0], got[1] + rest[1], rest[2]), oracle(state, pod_keys, calls, W, models),
                        "refusals in the middle")
        L = np.zeros(P, np.int32)
        assert bp(ctx, 1, None, 0, None, 0, None, W, p(L)) == 0                   # R = 0 reads the loads
        assert np.array_equal(L, rest[2])


def test_resident_epochs_are_untouched_by_a_herd():
    P, A = 64, 8
    state = random_state(P, A, seed=31)
    state.q[:] = 0
    reqs = WL.make_requests(20000, A, seed=32)
    reqs["adapter_id"] = 0
    reqs["flags"] = N.LIG_REQ_CRITICAL
    reqs["rand_key"] = AR.mix(np.minimum(np.random.default_rng(33).zipf(1.3, len(reqs)), 10 ** 6).astype(np.uint64))
    e, _ = engine_for(state, 20000)
    with e:
        classes = lambda: [e.read_class(1, cr, a, P) for cr in (0, 1) for a in range(A + 1)]   # noqa: E731
        before_cls, before = classes(), e.schedule_batch_affinity(1, reqs, K)
        _, _, loads = run_chain(e, 1, affinity_split(reqs, list(range(0, 20001, 2500)), [K] * 8), 8, P, FORMS)
        resident_max = np.bincount(before[0]["pod_idx"][before[0]["pod_idx"] >= 0], minlength=P).max()
        assert loads.max() < resident_max, (loads.max(), resident_max)
        after = classes()
        assert all(b[0] == a[0] and b[1] == a[1] and np.array_equal(b[2], a[2]) for b, a in zip(before_cls, after))
        again = e.schedule_batch_affinity(1, reqs, K)
        assert again[0].tobytes() == before[0].tobytes() and np.array_equal(again[1], before[1])


def test_concurrent_library_callers_loads_sum_to_the_picks():
    """Eight threads of chain affinity calls on one ctx: the chain serialises them, so the loads are the
    bincount of every OK pick, whatever the order."""
    c = WL.CONFIGS["C2"]
    state = random_state(c["P"], c["A"], seed=41)
    e, _ = engine_for(state, 4096, WL.make_models(c["A"]))
    picks, lock = [], threading.Lock()
    with e:
        def caller(t):
            rng = np.random.default_rng(t)
            for j in range(20):
                reqs = keyed(c["A"], int(rng.integers(1, 200)), seed=t * 100 + j)
                if j % 2:
                    ids = rng.integers(0, 40, len(reqs)).astype(np.uint32)
                    out, _ = e.schedule_models_batch_feedback_chain_affinity(1, ids, reqs["rand_key"], j % 3, 16)
                else:
                    out, _ = e.schedule_batch_feedback_chain_affinity(1, reqs, j % 3, 16)
                with lock:
                    picks.append(out["pod_idx"].astype(np.int64))
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(8)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        L = np.zeros(state.P, np.int32)
        e.schedule_batch_feedback_chain_affinity(1, np.zeros(0, REQ_DTYPE), 0, 16, loads=L)
    allp = np.concatenate(picks)
    assert np.array_equal(L, np.bincount(allp[allp >= 0], minlength=state.P)) and L.sum() > 1000


# ---- the schedulers -----------------------------------------------------------------------------------
class VersionedProvider:
    """One scrape for the whole test: the schedulers keep one epoch, so the chain runs across calls."""
    def __init__(self, pods):
        self.pods = list(pods)

    def AllPodMetrics(self):
        return list(self.pods)

    def Version(self):
        return 1


def test_python_scheduler_feedback_affinity():
    pods = scheduler_pool(120, 61)
    W = 8
    kw = dict(max_pods=128, max_adapters=16, max_batch=1024, seed=3, load_feedback_window=W)
    s = S.NewScheduler(VersionedProvider(pods), affinity=True, feedback_affinity=True, **kw)
    check = feedback_engine(128, 16, 1024)
    try:
        models = [im("m", [("ad-1", 3), ("ad-2", 5)]), im("plain")]
        s.SetInferenceModels(models)
        check.upload_snapshot(1, s._snap)
        check.upload_pod_keys(1, s._pod_keys)
        check.upload_models(1, s._packed_models)
        reqs = [S.LLMRequest(ResolvedTargetModel=f"ad-{i % 7}", Critical=i % 3 == 0) for i in range(300)]
        keys = [int(k) for k in AR.mix(np.random.default_rng(62).integers(1, 40, 300).astype(np.uint64))]
        arr = np.zeros(len(reqs), dtype=REQ_DTYPE)
        for i, r in enumerate(reqs):
            arr[i] = (s._snap.adapter_id(r.ResolvedTargetModel), 1 if r.Critical else 0, keys[i])
        names = ["m", "plain", "nope", "m"] * 25
        mkeys = keys[:100]
        sent = [i for i, nm in enumerate(names) if nm != "nope"]
        mids = np.array([s._packed_models.model_ids[names[i]] for i in sent], np.uint32)
        for n in (None, 3):
            got = s.ScheduleBatchAffinity(reqs, keys, n)
            want, wrows = check.schedule_batch_feedback_chain_affinity(1, arr, n or 0, W)
            for g, pk, row in zip(got, want, wrows):
                pods_got = (g[0] if n else [g[0]]) if g[1] is None else []
                if pk["status"] != N.LIG_OK:
                    assert g[1] is not None
                    continue
                assert [p.Name for p in pods_got] == [s._snap.pods[int(x)].Name for x in [pk["pod_idx"]] + list(row)
                                                      if x >= 0]
            mgot = s.ScheduleModelBatchAffinity(names, mkeys, n)
            mwant, mrows = check.schedule_models_batch_feedback_chain_affinity(
                1, mids, np.array([mkeys[i] for i in sent], np.uint64), n or 0, W)
            assert mgot[2][2] is not None and mgot[2][2].code == "Unknown"
            for j, i in enumerate(sent):
                if mwant[j]["status"] != N.LIG_OK:
                    assert mgot[i][2] is not None
                    continue
                pods_got = mgot[i][0] if n else [mgot[i][0]]
                assert [p.Name for p in pods_got] == [s._snap.pods[int(x)].Name
                                                      for x in [mwant[j]["pod_idx"]] + list(mrows[j]) if x >= 0]
        assert s.ScheduleAffinity(reqs[0], keys[0]) == s._snap.pods[
            int(check.schedule_batch_feedback_chain_affinity(1, arr[:1], 0, W)[0][0]["pod_idx"])]
        with pytest.raises(ValueError):
            s.ScheduleAffinityWithFallbacks(reqs[0], 1, K + 1)
    finally:
        s.close()
        check.close()
    # without the opt-in the refusal stays; without load_feedback_window the opt-in changes nothing
    refuse = S.NewScheduler(VersionedProvider(pods), affinity=True, **kw)
    plain = S.NewScheduler(VersionedProvider(pods), affinity=True, feedback_affinity=True, max_pods=128,
                           max_adapters=16, max_batch=1024)
    twin = S.NewScheduler(VersionedProvider(pods), affinity=True, max_pods=128, max_adapters=16, max_batch=1024)
    try:
        with pytest.raises(ValueError, match="load_feedback_window"):
            refuse.ScheduleAffinity(reqs[0], 1)
        assert [plain.ScheduleAffinity(r, k) for r, k in zip(reqs[:50], keys)] == \
            [twin.ScheduleAffinity(r, k) for r, k in zip(reqs[:50], keys)]
    finally:
        refuse.close()
        plain.close()
        twin.close()


def test_cpp_runtime_matches_python_with_one_caller():
    pods = scheduler_pool(120, 71)
    W = 5
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=128, max_adapters=16, max_batch=512, seed=3, affinity=True,
                         load_feedback_window=W, feedback_affinity=True)
    s = S.NewScheduler(VersionedProvider(pods), affinity=True, feedback_affinity=True, load_feedback_window=W,
                       max_pods=128, max_adapters=16, max_batch=512)
    try:
        models = [im("m", [("ad-1", 3), ("ad-2", 5)]), im("plain")]
        store = H.HostDataStore(models)
        hs.set_inference_models(store)
        s.SetInferenceModels(models)
        keys = [int(k) for k in AR.mix(np.random.default_rng(72).integers(1, 20, 200).astype(np.uint64))]
        for i, k in enumerate(keys):
            ad, n = f"ad-{i % 5}", i % 3
            if i % 4 == 3:
                code, resolved, names, err = hs.ScheduleModelAffinity("m", k, n)
                if n:
                    r2, pods2 = s.ScheduleModelAffinityWithFallbacks("m", k, n)
                else:
                    r2, pod = s.ScheduleModelAffinity("m", k)
                    pods2 = [pod]
                assert code == 0 and (resolved, names) == (r2, [p.Name for p in pods2]), i
                continue
            code, names, err = hs.ScheduleAffinity(ad, False, k, n)
            req = S.LLMRequest(ResolvedTargetModel=ad)
            try:
                py = [p.Name for p in (s.ScheduleAffinityWithFallbacks(req, k, n) if n else
                                       [s.ScheduleAffinity(req, k)])]
            except S.StatusError:
                assert code != 0, (i, err)
                continue
            assert code == 0 and names == py, i
        st = hs.stats()
        assert st["affinity_scheduled"] == len(keys) and st["feedback_windows"] == len(keys) // W
        assert st["feedback_restarts"] == 0
        store.close()
    finally:
        hs.close()
        s.close()
    chain = H.HostScheduler(prov, max_pods=128, max_adapters=16, max_batch=64, affinity=True, load_feedback_window=4)
    try:
        code, _, err = chain.ScheduleAffinity("ad-1", False, 5)
        assert code == 3 and "load_feedback_window" in err
    finally:
        chain.close()
        prov.close()


def test_cpp_runtime_under_concurrent_callers():
    """W = 8; a keep-all tree keeps every pod, so each answer is its key's ranking over the whole pool
    whatever window it fell in; the windows count every call."""
    P, W = 64, 8
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)], [4] * P, [["a"]] * P)
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200, seed=9,
                         filter=KEEP_ALL_CHART, affinity=True, load_feedback_window=W, feedback_affinity=True)
    store = H.HostDataStore([im("m", [("a", 1)])])
    results, lock = [], threading.Lock()
    try:
        hs.set_inference_models(store)

        def caller(t):
            mine = []
            for j in range(40):
                key = int(AR.mix(np.uint64(t * 1000 + j % 7)))
                n = (t + j) % 4
                if j % 2:
                    code, _, names, _ = hs.ScheduleModelAffinity("m", key, n)
                else:
                    code, names, _ = hs.ScheduleAffinity("a", False, key, n)
                mine.append((key, n, code, names))
            with lock:
                results.extend(mine)
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(12)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        st = hs.stats()
    finally:
        hs.close()
        store.close()
        prov.close()
    assert len(results) == 480 and all(r[2] == H.GRPC_OK for r in results)
    assert st["affinity_scheduled"] == 480 and st["feedback_windows"] == 480 // W and st["feedback_restarts"] == 0
    pod_keys = np.array([S.pod_key(p.Pod) for p in pods], dtype=np.uint64)
    for key, n, _, names in results:
        want = AR.ranking(key, range(P), pod_keys)[:1 + n]
        assert names == [f"pod-{x}" for x in want]
