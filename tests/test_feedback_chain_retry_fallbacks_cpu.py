"""Retries with fallback rows under the load-feedback chain
(lig_schedule_batch_feedback_chain_excluding_fallbacks) without a GPU: the definition
(feedback_chain_retry_fallbacks_ref.py) against the chain retry's picks and loads for every k, against the
chain fallback call for rows that exclude nothing, against the resident retry with rows while no window
has closed; its properties (prefix rows, distinct entries, no excluded entry), split invariance, a window
closing inside a call, a retry whose load moves a pod across a queue threshold, mixed call kinds, and the
C ABI's exports and refusals."""
import dataclasses
import os
import re

import numpy as np
import pytest

import feedback_chain_fallbacks_ref as FR
import feedback_chain_ref as FC
import feedback_chain_retry_fallbacks_ref as CRF
import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import retry_fallbacks_ref as RF
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, pack_columns
from oracle import binding as B
from test_feedback_chain_retry_cpu import nothing_rows
from test_retry_cpu import random_reqs, random_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = N.LIG_MAX_FALLBACKS
SEED = 0x0C4A_F00D_5EED


@pytest.fixture(scope="module")
def c2():
    c = WL.CONFIGS["C2"]
    return c, WL.make_snapshot(c["P"], c["A"], seed=41)


def split_retry_calls(reqs, rows, bounds, seed):
    return [CR.retry_call(reqs[a:b], rows[a:b], seed) for a, b in zip(bounds[:-1], bounds[1:])]


@pytest.mark.parametrize("window", [1, 7, 300])
def test_picks_and_loads_are_the_chain_retry_for_every_k(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window + 1)
    reqs = random_reqs(rng, 900, p.A)
    rows = random_rows(rng, len(reqs), p.P, 9)
    calls = split_retry_calls(reqs, rows, FC.random_split(len(reqs), rng, window), SEED)
    want, want_loads = CR.chain_retry(p, calls, window)
    for k in range(1, K + 1):
        got, got_rows, loads = CRF.chain_retry_fallbacks(p, calls, window, k)
        assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want)), k
        assert np.array_equal(loads, want_loads), k
        assert all(r.shape == (len(x), k) for r, (x, _) in zip(got_rows, calls))


@pytest.mark.parametrize("window", [1, 5, 64, 4096])
def test_rows_that_exclude_nothing_are_the_chain_fallback_call(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window)
    reqs = WL.make_requests(700 if window == 1 else 1500, c["A"], seed=window)
    plain = FC.split_calls(reqs, FC.random_split(len(reqs), rng, window), SEED)
    retry = [CR.retry_call(x, nothing_rows(len(x), p.P, int(rng.integers(1, 33)), rng), s) for x, s in plain]
    for k in (1, 3, K):
        want, want_rows, want_loads = FR.schedule_chain_fallbacks(p.P, p.A, p.kv, p.q, p.n_active, p.max_active,
                                                                  p.bitmap, plain, [k] * len(plain), window)
        got, rows, loads = CRF.chain_retry_fallbacks(p, retry, window, k)
        assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
        assert all(np.array_equal(r, w) for r, w in zip(rows, want_rows)), k
        assert np.array_equal(loads, want_loads) and loads.sum() > 0


def test_no_closed_window_is_the_resident_retry_with_rows(c2):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(3)
    reqs = random_reqs(rng, 1500, p.A)
    rows = random_rows(rng, len(reqs), p.P, 9)
    calls = split_retry_calls(reqs, rows, FC.random_split(len(reqs), rng, 200), SEED)
    got, got_rows, _ = CRF.chain_retry_fallbacks(p, calls, len(reqs) + 1, 5)
    want, want_rows = RF.retry_fallback_batch(p, reqs, rows, SEED, 5)
    assert np.concatenate(got).tobytes() == want.tobytes()
    assert np.array_equal(np.concatenate(got_rows), want_rows)
    assert ((want["status"] == N.LIG_OK).sum() > 500) and (want_rows[:, 0] >= 0).sum() > 100


@pytest.mark.parametrize("window", [3, 100])
def test_prefix_distinct_and_no_excluded_entry(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window + 77)
    reqs = random_reqs(rng, 600, p.A)
    ex = random_rows(rng, len(reqs), p.P, 32)
    calls = [CR.retry_call(reqs, ex, SEED)]
    (pk,), (full,), _ = CRF.chain_retry_fallbacks(p, calls, window, K)
    for k in (1, 2, 5):
        (_,), (r,), _ = CRF.chain_retry_fallbacks(p, calls, window, k)
        assert np.array_equal(r, full[:, :k])
    ok = pk["status"] == N.LIG_OK
    assert np.all(full[~ok] == -1)
    for i in np.flatnonzero(ok):
        entries = [int(pk["pod_idx"][i])] + [int(e) for e in full[i] if e >= 0]
        assert len(set(entries)) == len(entries)
        assert not set(entries) & {int(e) for e in ex[i]}
        assert all(e == -1 for e in full[i][len(entries) - 1:])
    assert (full[ok] >= 0).sum() > 20


@pytest.mark.parametrize("window", [1, 16, 300])
def test_split_invariance(c2, window):
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(window + 9)
    reqs = random_reqs(rng, 1200, p.A)
    rows = random_rows(rng, len(reqs), p.P, 5)
    whole, whole_rows, whole_loads = CRF.chain_retry_fallbacks(p, [CR.retry_call(reqs, rows, SEED)], window, 4)
    parts, part_rows, loads = CRF.chain_retry_fallbacks(
        p, split_retry_calls(reqs, rows, FC.random_split(len(reqs), rng, window), SEED), window, 4)
    assert np.concatenate(parts).tobytes() == whole[0].tobytes()
    assert np.array_equal(np.concatenate(part_rows), whole_rows[0])
    assert np.array_equal(loads, whole_loads)


def test_a_window_closing_inside_a_call_ranks_the_rest_on_the_loaded_pool(c2):
    """Window 100 closes at request 100 of a 250-request call: requests 100.. are picked and ranked on q
    plus the picks of the first 100, as two resident retries with rows on those pools."""
    c, snap = c2
    p = snap.packed
    rng = np.random.default_rng(17)
    reqs = random_reqs(rng, 250, p.A)
    rows = random_rows(rng, 250, p.P, 4)
    (got,), (got_rows,), loads = CRF.chain_retry_fallbacks(p, [CR.retry_call(reqs, rows, SEED)], 100, 6)
    first, first_rows = RF.retry_fallback_batch(p, reqs[:100], rows[:100], SEED, 6)
    hist = np.bincount(first["pod_idx"][first["pod_idx"] >= 0], minlength=p.P)
    q1 = dataclasses.replace(p, q=(p.q.astype(np.int64) + hist).astype(np.int32))
    second, second_rows = RF.retry_fallback_batch(q1, reqs[100:200], rows[100:200], SEED, 6)
    assert got[:100].tobytes() == first.tobytes() and got[100:200].tobytes() == second.tobytes()
    assert np.array_equal(got_rows[:100], first_rows) and np.array_equal(got_rows[100:200], second_rows)
    ok = got["status"] == N.LIG_OK
    assert np.array_equal(loads, np.bincount(got["pod_idx"][ok], minlength=p.P))


def test_a_retry_pushes_a_pod_across_the_queue_threshold():
    """Four idle pods, q = 0, 0, 0, 3: critical requests that exclude pods 0 and 1 all land on pod 2 (the
    reduced set is {2}, rows empty).  Once the window closes pod 2's q is past queueingThresholdLoRA, so the
    next retry-with-rows call, excluding pod 0 only, ranks {1} on the chain's copy where E gives {1, 2}."""
    P = 4
    snap = pack_columns(np.zeros(P), np.array([0, 0, 0, 3]), np.zeros(P, np.int64), np.full(P, 4, np.int64),
                        np.zeros((1, 1), np.uint32), {"a": 0}, [WL.Pod(f"p{i}", f"10.0.0.{i}") for i in range(P)])
    reqs = np.zeros(6, dtype=REQ_DTYPE)
    reqs["adapter_id"] = 1
    reqs["flags"] = 1
    reqs["rand_key"] = np.arange(6, dtype=np.uint64)
    later = reqs.copy()
    later["rand_key"] += 100
    calls = [CR.retry_call(reqs, np.tile(np.array([0, 1], np.int16), (6, 1)), SEED),
             CR.retry_call(later, np.tile(np.array([0, -1], np.int16), (6, 1)), SEED)]
    outs, rows, loads = CRF.chain_retry_fallbacks(snap, calls, window=6, k=3)
    assert (outs[0]["pod_idx"] == 2).all() and np.all(rows[0] == -1) and loads[2] == 6
    assert (outs[1]["pod_idx"] == 1).all() and np.all(rows[1] == -1)
    on_e, rows_e = RF.retry_fallback_batch(snap, later, np.tile(np.array([0, -1], np.int16), (6, 1)), SEED, 3)
    assert set(on_e["pod_idx"].tolist()) | set(rows_e[:, 0].tolist()) == {1, 2}


def test_mixed_kinds_in_one_chain(c2):
    """Plain, model-id, fallback, retry and retry-with-rows calls in one sequence: every pick and the loads
    are those of the same chain with the rows dropped, and the fallback calls' rows are unchanged."""
    c, snap = c2
    p = snap.packed
    models = WL.make_models(c["A"])
    mo = B.Models(WL.model_records(models))
    rng = np.random.default_rng(23)
    reqs = WL.make_requests(1600, c["A"], seed=23)
    bounds = FC.random_split(len(reqs), rng, 48)
    calls, ks = [], []
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        kind = i % 5
        if kind == 1:
            calls.append(MC.model_call(mo, p.adapter_id, rng.integers(0, len(models) + 2, b - a).astype(np.uint32),
                                       7, a))
        elif kind in (3, 4):
            calls.append(CR.retry_call(x, random_rows(rng, b - a, p.P, 3), 7))
        else:
            calls.append((x, 7))
        ks.append(2 if kind == 2 else 4 if kind == 4 else 0)
    outs, rows, loads = CRF.run_chain_retry_fallbacks(p, calls, 48, ks)
    want, want_rows, want_loads = CR.run_chain_retries(p, calls, 48, [k if i % 5 == 2 else 0
                                                                      for i, k in enumerate(ks)])
    assert all(o.tobytes() == w.tobytes() for o, w in zip(outs, want))
    assert np.array_equal(loads, want_loads)
    for i, (r, w) in enumerate(zip(rows, want_rows)):
        if i % 5 == 4:
            assert r.shape == (len(calls[i][0]), 4)
        else:
            assert np.array_equal(r, w)
    assert any((r >= 0).any() for i, r in enumerate(rows) if i % 5 == 4)


NAMES = ("lig_schedule_batch_feedback_chain_excluding_fallbacks",
         "lig_schedule_batch_feedback_chain_excluding_fallbacks_device")


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
    ex = np.zeros((4, 32), dtype=np.int16)
    fb = np.zeros((4, K), dtype=np.int16)
    loads = np.zeros(4, dtype=np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    for nx, nf, win in ((0, 2, 8), (1, 2, 8), (32, K, 8), (33, 2, 8), (-1, 2, 8), (4, 0, 8), (4, K + 1, 8),
                        (4, 2, 0)):
        assert lib.lig_schedule_batch_feedback_chain_excluding_fallbacks(
            None, 1, 2, p(reqs), 4, p(ex), nx, p(out), nf, p(fb), win, p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_feedback_chain_excluding_fallbacks_device(
            None, 1, 2, p(reqs), 4, p(ex), nx, p(out), nf, p(fb), win, p(loads), None) == N.LIG_ERR_INVALID
    assert b"chain_excluding_fallbacks" in lib.lig_last_error()
    assert np.all(ex == 0) and np.all(fb == 0) and np.all(out["pod_idx"] == 0) and np.all(loads == 0)
