"""The model-id feedback chain's sequential definition (models_feedback_chain_ref) without a GPU: one
call over ids that all resolve is oracle/feedback.py over the resolved descriptors, a chain whose
window never closes is the oracle's model-request path, the result does not depend on how the ids
are split into calls, and model-id calls mix with descriptor calls in one sequence."""
import numpy as np
import pytest

import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from oracle import binding as B
from oracle import feedback as FB


def setup(cfg, snap_seed=1):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"], seed=snap_seed)
    models = WL.make_models(c["A"])
    return c, snap, B.Models(WL.model_records(models)), len(models)


def chain_of(snap, calls, window):
    p = snap.packed
    return MC.schedule_chain(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap, calls, window)


@pytest.mark.parametrize("cfg,window", [("C2", 256), ("C2", 1), ("C5", 700)])
def test_one_call_is_the_in_batch_definition_over_resolved_descriptors(cfg, window):
    c, snap, mo, n_models = setup(cfg)
    p = snap.packed
    ids = WL.make_model_requests(3000 if window > 1 else 600, c["A"], seed=2)
    ids = np.ascontiguousarray(ids[ids < n_models])              # no absent models
    rows = MC.resolve_call(mo, p.adapter_id, ids, 5, first_index=40)
    assert (rows["ok"] == 1).all()
    reqs = np.ascontiguousarray(rows["req"])
    want, want_total, _ = FB.schedule_batch_feedback(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap,
                                                     reqs, 5, window)
    (got,), loads = chain_of(snap, [MC.model_call(mo, p.adapter_id, ids, 5, 40)], window)
    assert np.array_equal(got["pod_idx"], want["pod_idx"]) and np.array_equal(got["status"], want["status"])
    assert np.array_equal(got["target_idx"], rows["target_idx"])
    assert np.array_equal(loads, want_total) and loads.sum() == (got["pod_idx"] >= 0).sum() > 0
    if c["A"] >= 32:
        assert ((got["target_idx"] > 0) & (got["target_idx"] < 255)).any()     # weighted draws ran


@pytest.mark.parametrize("cfg", ["C2", "C5"])
def test_no_closed_window_is_the_model_request_path(cfg):
    c, snap, mo, n_models = setup(cfg, snap_seed=3)
    p = snap.packed
    ids = WL.make_model_requests(4000, c["A"], seed=4)
    ids[:5] = [n_models, n_models + 9, 2**32 - 1, 2**31, c["A"]]     # absent ids and the pass-through model
    want = mo.schedule_batch(B.Pool(snap.pod_records()), ids, 17, first_index=1 << 40)
    bounds = FC.random_split(len(ids), np.random.default_rng(5), 300)
    calls = MC.split_model_calls(mo, p.adapter_id, ids, bounds, 17, first_index=1 << 40)
    outs, loads = chain_of(snap, calls, 1 << 30)
    got = np.concatenate(outs)
    assert np.array_equal(got, want)
    assert (got["status"] == N.LIG_NO_MODEL).sum() >= 4
    assert np.array_equal(loads, np.bincount(got["pod_idx"][got["pod_idx"] >= 0], minlength=p.P))


@pytest.mark.parametrize("window", [1, 7, 64, 4096])
def test_random_splits_give_one_result(window):
    c, snap, mo, _ = setup("C2", snap_seed=6)
    p = snap.packed
    R = max(5000, 5 * window + 300) if window > 1 else 700
    ids = WL.make_model_requests(R, c["A"], seed=7)
    (whole,), whole_loads = chain_of(snap, [MC.model_call(mo, p.adapter_id, ids, 9, 123)], window)
    rng = np.random.default_rng(window)
    for trial in range(3):
        bounds = FC.random_split(R, rng, window)
        sizes = np.diff(bounds)
        if trial == 0:
            assert {0, 1, window}.issubset(set(sizes.tolist())) and sizes.max() > 2 * window
        outs, loads = chain_of(snap, MC.split_model_calls(mo, p.adapter_id, ids, bounds, 9, first_index=123), window)
        assert np.array_equal(np.concatenate(outs), whole), (window, trial)
        assert np.array_equal(loads, whole_loads)


def test_mixed_calls_follow_the_descriptor_chain():
    """Model-id calls whose ids all resolve, alternating with descriptor calls, give the descriptor
    chain over the resolved descriptors; an id that does not resolve is LIG_NO_MODEL and picks nothing."""
    c, snap, mo, n_models = setup("C2", snap_seed=8)
    p = snap.packed
    W = 50
    ids = WL.make_model_requests(1200, c["A"], seed=9)
    ids = np.ascontiguousarray(ids[ids < n_models][:1000])
    reqs = WL.make_requests(1000, c["A"], seed=10)
    bounds = FC.random_split(1000, np.random.default_rng(11), W)
    calls, desc_calls = [], []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        if k % 2:
            call = MC.model_call(mo, p.adapter_id, np.ascontiguousarray(ids[a:b]), 100 + k, a)
            desc_calls.append((np.ascontiguousarray(call[0]["req"]), call[1]))
        else:
            call = (np.ascontiguousarray(reqs[a:b]), 100 + k)
            desc_calls.append(call)
        calls.append(call)
    outs, loads = chain_of(snap, calls, W)
    want, want_loads = FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active,
                                                        p.bitmap, desc_calls, W)
    assert np.array_equal(loads, want_loads)
    for (call, _), o, w in zip(calls, outs, want):
        if call.dtype == MC.MREQ_DTYPE:
            assert o.dtype == B.MPICK_DTYPE and np.array_equal(o["target_idx"], call["target_idx"])
            assert np.array_equal(o["pod_idx"], w["pod_idx"]) and np.array_equal(o["status"], w["status"])
        else:
            assert np.array_equal(o, w)
    # an absent id is LIG_NO_MODEL / target 255 and picks nothing
    bad = ids[:200].copy()
    bad[::3] = n_models + 1
    (o,), bad_loads = chain_of(snap, [MC.model_call(mo, p.adapter_id, bad, 3)], W)
    assert (o["status"][::3] == N.LIG_NO_MODEL).all() and (o["pod_idx"][::3] == -1).all()
    assert (o["target_idx"][::3] == 255).all() and (o["status"][1::3] != N.LIG_NO_MODEL).all()
    assert bad_loads.sum() == (o["pod_idx"] >= 0).sum()
