"""Retries under the load-feedback chain (lig_schedule_batch_feedback_chain_excluding) without a GPU: the
definition (feedback_chain_retry_ref.py) against run_chain for rows that exclude nothing, against the
resident retry while no window has closed, split invariance, a window closing inside a retry call, a
retry whose load moves a pod across a queue threshold, and the C ABI's exports and refusals."""
import dataclasses
import os
import re

import numpy as np
import pytest

import feedback_chain_ref as FC
import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import retry_ref as RR
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, pack_columns
from oracle import binding as B
from test_retry_cpu import random_reqs, random_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x0C4A_1E7B_5EED


@pytest.fixture(scope="module")
def c2():
    c = WL.CONFIGS["C2"]
    return c, WL.make_snapshot(c["P"], c["A"], seed=41)


def nothing_rows(R, P, width, rng):
    """Rows of -1 and out-of-range entries only."""
    return rng.choice(np.array([-1, P, P + 7, 32767, -32768], dtype=np.int16), size=(R, width))


@pytest.mark.parametrize("window", [1, 5, 64, 4096])
def test_rows_that_exclude_nothing_are_the_plain_chain(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window)
    reqs = WL.make_requests(700 if window == 1 else 2000, c["A"], seed=window)
    bounds = FC.random_split(len(reqs), rng, window)
    plain = FC.split_calls(reqs, bounds, SEED)
    retry = [CR.retry_call(x, nothing_rows(len(x), p.P, int(rng.integers(1, 33)), rng), s) for x, s in plain]
    want, want_loads = FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap,
                                                        plain, window)
    got, loads = CR.chain_retry(p, retry, window)
    assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
    assert np.array_equal(loads, want_loads) and loads.sum() > 0


def test_no_closed_window_is_the_resident_retry(c2):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(3)
    reqs = random_reqs(rng, 1500, p.A)
    rows = random_rows(rng, len(reqs), p.P, 9)
    bounds = FC.random_split(len(reqs), rng, 200)
    calls = [CR.retry_call(reqs[a:b], rows[a:b], SEED) for a, b in zip(bounds[:-1], bounds[1:])]
    got, _ = CR.chain_retry(p, calls, window=len(reqs) + 1)
    want = RR.retry_batch(p, reqs, rows, SEED)
    assert np.concatenate(got).tobytes() == want.tobytes()


@pytest.mark.parametrize("window", [1, 16, 300])
def test_split_invariance(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window + 9)
    reqs = random_reqs(rng, 1200, p.A)
    rows = random_rows(rng, len(reqs), p.P, 5)
    whole, whole_loads = CR.chain_retry(p, [CR.retry_call(reqs, rows, SEED)], window)
    bounds = FC.random_split(len(reqs), rng, window)
    parts, loads = CR.chain_retry(p, [CR.retry_call(reqs[a:b], rows[a:b], SEED)
                                      for a, b in zip(bounds[:-1], bounds[1:])], window)
    assert np.concatenate(parts).tobytes() == whole[0].tobytes()
    assert np.array_equal(loads, whole_loads)


def test_a_window_closing_inside_a_retry_call_loads_the_rest_of_it(c2):
    """Window 100 closes at request 100 of a 250-request retry call: requests 100.. are scheduled on q
    plus the picks of the first 100, and the definition equals two resident retries on those pools."""
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(17)
    reqs = random_reqs(rng, 250, p.A)
    rows = random_rows(rng, 250, p.P, 4)
    (got,), loads = CR.chain_retry(p, [CR.retry_call(reqs, rows, SEED)], 100)
    first = RR.retry_batch(p, reqs[:100], rows[:100], SEED)
    hist = np.bincount(first["pod_idx"][first["pod_idx"] >= 0], minlength=p.P)
    q1 = dataclasses.replace(p, q=(p.q.astype(np.int64) + hist).astype(np.int32))
    second = RR.retry_batch(q1, reqs[100:200], rows[100:200], SEED)
    assert got[:100].tobytes() == first.tobytes() and got[100:200].tobytes() == second.tobytes()
    ok = got["status"] == N.LIG_OK
    assert loads.sum() == ok.sum()
    assert np.array_equal(loads, np.bincount(got["pod_idx"][ok], minlength=p.P))


def test_a_retry_pushes_a_pod_across_the_queue_threshold():
    """Four idle pods, q = 0, 0, 0, 3: a critical request keeps q < queueingThresholdLoRA (5), pods 0-2
    tie on the least queue.  Retries that exclude pods 0 and 1 all land on pod 2; once the window
    closes pod 2's q is past the threshold, so a later plain critical call's survivor set changes."""
    P = 4
    snap = pack_columns(np.zeros(P), np.array([0, 0, 0, 3]), np.zeros(P, np.int64), np.full(P, 4, np.int64),
                        np.zeros((1, 1), np.uint32), {"a": 0}, [WL.Pod(f"p{i}", f"10.0.0.{i}") for i in range(P)])
    reqs = np.zeros(6, dtype=REQ_DTYPE)
    reqs["adapter_id"] = 1
    reqs["flags"] = 1
    reqs["rand_key"] = np.arange(6, dtype=np.uint64)
    rows = np.tile(np.array([0, 1], dtype=np.int16), (6, 1))
    plain = reqs.copy()
    plain["rand_key"] += 100
    retry_then_plain = [CR.retry_call(reqs, rows, SEED), (plain, SEED)]
    outs, loads = CR.chain_retry(snap, retry_then_plain, window=6)
    assert (outs[0]["pod_idx"] == 2).all() and loads[2] == 6
    before = B.ClassTable(P, 1, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap).klass(True, 1)
    after = B.ClassTable(P, 1, snap.kv, np.array([0, 0, 6, 3], np.int32), snap.n_active, snap.max_active,
                         snap.bitmap).klass(True, 1)
    assert sorted(before[2]) == [0, 1, 2] and sorted(after[2]) == [0, 1]
    assert set(outs[1]["pod_idx"].tolist()) <= {0, 1}
    # the same plain call without the retries before it still sees pod 2
    alone, _ = CR.chain_retry(snap, [(plain, SEED)], window=6)
    assert 2 in set(alone[0]["pod_idx"].tolist())


def test_mixed_kinds_in_one_chain(c2):
    """Plain, model-id, fallback and retry calls in one sequence: the plain and model-id calls and the
    fallback picks are the mixed chain's, with the retry calls' picks counted like theirs."""
    c, snap = c2
    p = snap.packed
    models = WL.make_models(c["A"])
    mo = B.Models(WL.model_records(models))
    rng = np.random.default_rng(23)
    reqs = WL.make_requests(1600, c["A"], seed=23)
    bounds = FC.random_split(len(reqs), rng, 48)
    calls, ks, ref_calls = [], [], []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        kind = k % 4
        if kind == 1:
            call = MC.model_call(mo, p.adapter_id, rng.integers(0, len(models) + 2, b - a).astype(np.uint32), 7, a)
            calls.append(call)
            ref_calls.append(call)
        elif kind == 3:
            calls.append(CR.retry_call(x, nothing_rows(b - a, p.P, 3, rng), 7))
            ref_calls.append((x, 7))
        else:
            calls.append((x, 7))
            ref_calls.append((x, 7))
        ks.append(2 if kind == 2 else 0)
    outs, rows, loads = CR.run_chain_retries(p, calls, 48, ks)
    want, want_loads = MC.schedule_chain(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap, ref_calls, 48)
    assert all(o.tobytes() == w.tobytes() for o, w in zip(outs, want))
    assert np.array_equal(loads, want_loads)
    assert any(r.shape[1] == 2 for r in rows)


NAMES = ("lig_schedule_batch_feedback_chain_excluding", "lig_schedule_batch_feedback_chain_excluding_device")


def test_symbols_are_declared():
    lib = N.load()
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    for name in NAMES:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\bint " + name + r"\(", header), name
    assert lib.lig_abi_version() == 7


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    out = np.zeros(4, dtype=PICK_DTYPE)
    rows = np.zeros((4, 32), dtype=np.int16)
    loads = np.zeros(4, dtype=np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    for nx, win in ((0, 8), (1, 8), (32, 8), (33, 8), (-1, 8), (4, 0)):
        assert lib.lig_schedule_batch_feedback_chain_excluding(None, 1, 2, p(reqs), 4, p(rows), nx, p(out), win,
                                                               p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_feedback_chain_excluding_device(None, 1, 2, p(reqs), 4, p(rows), nx, p(out),
                                                                      win, p(loads), None) == N.LIG_ERR_INVALID
    assert b"chain_excluding" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0) and np.all(loads == 0)
