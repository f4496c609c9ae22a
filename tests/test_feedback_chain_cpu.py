"""The load-feedback chain's sequential definition (feedback_chain_ref) without a GPU: one call is the
in-batch definition of oracle/feedback.py, the result does not depend on how the requests are split
into calls when every call has the same seed, and the class-table chain equals its port twin on the
golden pools and on adversarial pools."""
import numpy as np
import pytest

import feedback_chain_ref as FC
from filter_tree_ref import random_pool
from helpers import golden_to_podmetrics
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import REQ_DTYPE, pack_pod_metrics
from oracle import binding as B
from oracle import feedback as FB


def chain_of(snap, calls, window, thresholds=(0.8, 5, 50)):
    p = snap.packed
    return FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap, calls,
                                            window, thresholds)


@pytest.mark.parametrize("cfg,window", [("C2", 256), ("C2", 1), ("C5", 700)])
def test_one_call_is_the_in_batch_definition(cfg, window):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"], seed=1)
    p = snap.packed
    reqs = WL.make_requests(3000 if window > 1 else 600, c["A"], seed=2)
    want, want_total, _ = FB.schedule_batch_feedback(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap,
                                                     reqs, 5, window)
    (got,), loads = chain_of(snap, [(reqs, 5)], window)
    assert np.array_equal(got, want) and np.array_equal(loads, want_total)
    assert loads.sum() == (got["pod_idx"] >= 0).sum() > 0


@pytest.mark.parametrize("window", [1, 7, 64, 4096])
def test_random_splits_with_one_seed_give_one_result(window):
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=3)
    R = max(5000, 5 * window + 300) if window > 1 else 700
    reqs = WL.make_requests(R, c["A"], seed=4)
    (whole,), whole_loads = chain_of(snap, [(reqs, 9)], window)
    rng = np.random.default_rng(window)
    for trial in range(3):
        bounds = FC.random_split(R, rng, window)
        sizes = np.diff(bounds)
        if trial == 0:              # the edge call sizes are there, and a call spans several windows
            assert {0, 1, window}.issubset(set(sizes.tolist())) and sizes.max() > 2 * window
        outs, loads = chain_of(snap, FC.split_calls(reqs, bounds, 9), window)
        assert np.array_equal(np.concatenate(outs), whole), (window, trial)
        assert np.array_equal(loads, whole_loads)


def test_per_call_seeds_follow_the_definition():
    """Every request uses its own call's seed against the tables of the window it falls in."""
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=5)
    p = snap.packed
    reqs = WL.make_requests(900, c["A"], seed=6)
    W = 100
    bounds = [0, 30, 30, 250, 251, 600, 900]
    calls = [(np.ascontiguousarray(reqs[a:b]), 1000 + k) for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]
    outs, loads = chain_of(snap, calls, W)
    got = np.concatenate(outs)
    seeds = np.concatenate([np.full(b - a, 1000 + k) for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))])
    q = snap.q64.copy()
    for w in range(0, 900, W):
        tab = B.ClassTable(p.P, p.A, p.kv, q.astype(np.int32), p.n_active, p.max_active, p.bitmap, (0.8, 5, 50))
        for i in range(w, w + W):
            assert got[i] == tab.schedule_batch(np.ascontiguousarray(reqs[i:i + 1]), int(seeds[i]))[0], i
        sel = got["pod_idx"][w:w + W]
        q = np.minimum(q + np.bincount(sel[sel >= 0], minlength=p.P), FC.INT32_MAX)
    assert np.array_equal(loads, q - snap.q64)
    # different seeds per call do change the picks
    same = FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap,
                                            [(reqs, 1000)], W)[0][0]
    assert not np.array_equal(same, got)


def check_classtab_equals_port(records, calls_rng, window):
    p = pack_pod_metrics([golden_to_podmetrics(r) for r in records])
    names = sorted(p.adapter_ids, key=p.adapter_ids.get)
    R = 400
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["adapter_id"] = calls_rng.integers(0, p.A + 2, R)
    reqs["flags"] = calls_rng.integers(0, 2, R) * N.LIG_REQ_CRITICAL
    reqs["rand_key"] = calls_rng.integers(0, 1 << 63, R, dtype=np.uint64)
    bounds = FC.random_split(R, calls_rng, window)
    calls = [(c, 11 + k % 2) for k, (c, _) in enumerate(FC.split_calls(reqs, bounds, 0))]
    a, la = FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, p.q.astype(np.int64), p.n_active, p.max_active, p.bitmap,
                                             calls, window)
    b, lb = FC.schedule_batch_feedback_chain_port(records, names, "never-loaded", calls, window)
    assert all(np.array_equal(x, y) for x, y in zip(a, b)) and np.array_equal(la, lb)
    return la


def test_classtab_chain_equals_port_on_golden_pools(golden):
    rng = np.random.default_rng(7)
    for case in golden["TestFilter"]:
        records = case["input"] or []
        for window in (1, 3, 50):
            check_classtab_equals_port(records, rng, window)


def test_classtab_chain_equals_port_on_adversarial_pools():
    rng = np.random.default_rng(8)
    moved = 0
    for _ in range(60):
        loads = check_classtab_equals_port(random_pool(rng), rng, int(rng.choice([1, 2, 5, 17, 64])))
        moved += int(loads.sum() > 0)
    assert moved > 30
