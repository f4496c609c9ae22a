"""Fallback rows under the load-feedback chain without a GPU: the sequential definition
(feedback_chain_fallbacks_ref) leaves the chain's picks and loads exactly as run_chain makes them for
every n, equals the resident-epoch ranking while no window has closed, gives distinct survivors of the
load-adjusted tables as prefix rows, does not depend on how the requests are split into calls, and
follows the plain Fisher-Yates loop through forced Int31n rejections after a window has closed.  Also
the C ABI's exports and its refusals without a device."""
import os
import re

import numpy as np
import pytest

import feedback_chain_fallbacks_ref as FF
import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
from draw_keys import GAMMA, M64, accept_top, pick_keys, states_for
from fallback_ref import fallback_row, fallback_rows
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = N.LIG_MAX_FALLBACKS


def chain(snap, calls, ks, window, q=None):
    p = snap.packed
    return FF.schedule_chain_fallbacks(p.P, p.A, p.kv, snap.q64 if q is None else q, p.n_active, p.max_active,
                                       p.bitmap, calls, ks, window)


def plain_chain(snap, calls, window):
    p = snap.packed
    return MC.schedule_chain(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap, calls, window)


def table_at(snap, q):
    p = snap.packed
    return B.ClassTable(p.P, p.A, p.kv, np.asarray(q).astype(np.int32), p.n_active, p.max_active, p.bitmap)


@pytest.fixture(scope="module")
def c2():
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=21)
    models = WL.make_models(c["A"])
    return c, snap, B.Models(WL.model_records(models)), len(models)


def mixed_calls(c, snap, mo, n_models, R=3000, seed=5):
    """Descriptor and model-id calls alternating over one sequence (absent models and ids >= n_models
    included), with per-call seeds."""
    p = snap.packed
    reqs = WL.make_requests(R, c["A"], seed=seed)
    ids = np.random.default_rng(seed).integers(0, n_models + 3, R).astype(np.uint32)
    bounds = FC.random_split(R, np.random.default_rng(seed + 1), 64)
    calls, first = [], 1 << 40
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        if k % 2:
            calls.append(MC.model_call(mo, p.adapter_id, np.ascontiguousarray(ids[a:b]), 100 + k, first))
            first += b - a
        else:
            calls.append((np.ascontiguousarray(reqs[a:b]), 100 + k))
    return calls


@pytest.mark.parametrize("window", [1, 7, 64, 4096])
def test_picks_and_loads_are_the_plain_chain_for_every_n(c2, window):
    c, snap, mo, n_models = c2
    calls = mixed_calls(c, snap, mo, n_models, R=900 if window == 1 else 3000)
    want_outs, want_loads = plain_chain(snap, calls, window)
    rng = np.random.default_rng(window)
    for n in list(range(1, K + 1)) + ["mixed"]:
        ks = rng.integers(0, K + 1, len(calls)).tolist() if n == "mixed" else [n] * len(calls)
        outs, rows, loads = chain(snap, calls, ks, window)
        assert all(o.tobytes() == w.tobytes() for o, w in zip(outs, want_outs)), n
        assert np.array_equal(loads, want_loads), n
        assert [r.shape for r in rows] == [(len(cl), k) for (cl, _), k in zip(calls, ks)]
    assert want_loads.sum() > 0


def test_no_closed_window_is_the_resident_ranking(c2):
    c, snap, mo, n_models = c2
    p = snap.packed
    reqs = WL.make_requests(2500, c["A"], seed=31)
    calls = FC.split_calls(reqs, FC.random_split(len(reqs), np.random.default_rng(32), 300), 77)
    outs, rows, _ = chain(snap, calls, [K] * len(calls), window=len(reqs) + 1)
    tab = table_at(snap, snap.q64)
    picks = tab.schedule_batch(reqs, 77)
    ok = picks["status"] == N.LIG_OK
    crit, a = FF.class_of(reqs, p.A)
    lists = {(cr, ai): tab.klass(bool(cr), int(ai))[2] for cr, ai in set(zip(crit.tolist(), a.tolist()))}
    cnt = np.array([len(lists[(cr, ai)]) for cr, ai in zip(crit.tolist(), a.tolist())], dtype=np.int64)
    pods = np.concatenate([np.asarray(lists[(cr, ai)], dtype=np.int64) for cr, ai in zip(crit.tolist(), a.tolist())])
    starts = np.concatenate([[0], np.cumsum(cnt)])[:-1]
    want, _ = fallback_rows(77, reqs["rand_key"], ok, starts, cnt, pods, K)
    assert np.concatenate(outs).tobytes() == picks.tobytes()
    assert np.array_equal(np.concatenate(rows), want)
    assert (want[:, 0] >= 0).sum() > 1000
    # model ids: resolved requests take the same ranking on their resolved class
    ids = np.concatenate([WL.make_model_requests(2000, c["A"], seed=33),
                          np.array([n_models, n_models + 9, 1 << 31], dtype=np.uint32)])
    mcall = MC.model_call(mo, p.adapter_id, ids, 78, (1 << 64) - 5)
    (mo_out,), (mrows,), _ = chain(snap, [mcall], [K], window=5000)
    r = mcall[0]
    sub = np.ascontiguousarray(r["req"])
    sp = tab.schedule_batch(sub, 78)
    sp["status"] = np.where(r["ok"] == 1, sp["status"], MC.LIG_NO_MODEL)
    sp["pod_idx"] = np.where(r["ok"] == 1, sp["pod_idx"], -1)
    mrows_want = FF.segment_rows(sub, sp, 78, K, lambda cr, ai: (0, tab.klass(cr, ai)[2]), p.A)
    assert np.array_equal(mrows, mrows_want)
    assert mo_out.dtype == MC.B.MPICK_DTYPE and (mo_out["status"] == MC.LIG_NO_MODEL).any()


def test_rows_are_distinct_survivors_of_the_current_tables_and_prefixes(c2):
    """Herding micro-batches of one class: after the first closed window the lists change, and every
    row ranks the list of the tables at its own position."""
    c, snap, _, _ = c2
    p = snap.packed
    W = 40
    q0 = np.zeros(p.P, dtype=np.int64)
    reqs = WL.make_requests(1200, c["A"], seed=41)
    reqs["adapter_id"] = np.random.default_rng(41).choice([0, 1, c["A"]], len(reqs))
    calls = FC.split_calls(reqs, list(range(0, 1201, 8)), 43)
    outs, full, loads = chain(snap, calls, [K] * len(calls), W, q=q0)
    picks, rows = np.concatenate(outs), np.concatenate(full)
    # the tables of every window, replayed from the picks
    q = q0.copy()
    changed = 0
    tab0 = table_at(snap, q0)
    for w0 in range(0, len(reqs), W):
        tab = table_at(snap, q)
        seg = slice(w0, w0 + W)
        crit, a = FF.class_of(reqs[seg], p.A)
        for i, (cr, ai) in enumerate(zip(crit.tolist(), a.tolist())):
            st, n, lst = tab.klass(bool(cr), int(ai))
            pk, row = picks[w0 + i], rows[w0 + i].tolist()
            if pk["status"] != N.LIG_OK:
                assert row == [-1] * K
                continue
            m = min(n, 1 + K)
            ranked = [int(pk["pod_idx"])] + [x for x in row if x >= 0]
            assert len(ranked) == m and len(set(ranked)) == m and set(ranked) <= set(lst)
            assert row[m - 1:] == [-1] * (K - m + 1)
            changed += lst != tab0.klass(bool(cr), int(ai))[2]
        hist = np.bincount(picks["pod_idx"][seg][picks["pod_idx"][seg] >= 0], minlength=p.P)
        q = q + hist
    assert changed > 100 and np.array_equal(q - q0, loads)
    for k in range(1, K):
        _, rk, _ = chain(snap, calls, [k] * len(calls), W, q=q0)
        assert np.array_equal(np.concatenate(rk), rows[:, :k]), k


@pytest.mark.parametrize("window", [1, 7, 64, 4096])
def test_split_invariance(c2, window):
    c, snap, _, _ = c2
    R = 700 if window == 1 else max(3000, 5 * window + 300)
    reqs = WL.make_requests(R, c["A"], seed=51)
    (whole,), (whole_rows,), whole_loads = chain(snap, [(reqs, 9)], [K], window)
    rng = np.random.default_rng(window + 50)
    for _ in range(2):
        calls = FC.split_calls(reqs, FC.random_split(R, rng, window), 9)
        outs, rows, loads = chain(snap, calls, [K] * len(calls), window)
        assert np.concatenate(outs).tobytes() == whole.tobytes()
        assert np.array_equal(np.concatenate(rows), whole_rows) and np.array_equal(loads, whole_loads)


def tied_pool():
    """C2's pods with one KV value and empty queues: the least-KV step keeps ties, so the classes
    have many survivors, and a closed window moves them."""
    snap = WL.make_snapshot(64, 32, seed=21)
    snap.packed.kv[:] = 0.1
    return snap, np.zeros(64, dtype=np.int64)


def _class_after_a_window(W, want):
    """A first call of W requests that closes a window, then the tables it leaves: (snap, q0, first
    call, (critical, adapter, list)) for a class whose survivor count satisfies `want` and whose list
    the window changed."""
    snap, q0 = tied_pool()
    p = snap.packed
    first = WL.make_requests(W, p.A, seed=61)
    (_,), _, loads = chain(snap, [(first, 3)], [K], W, q=q0)
    assert loads.sum() == W
    tab0, tab = table_at(snap, q0), table_at(snap, q0 + loads)
    for cr in (0, 1):
        for a in range(p.A + 1):
            st, n, lst = tab.klass(bool(cr), a)
            if st == N.LIG_OK and want(n) and lst != tab0.klass(bool(cr), a)[2]:
                return snap, q0, first, (cr, a, lst)
    raise AssertionError("no class with the wanted survivor count")


def test_forced_rejection_on_the_pick_after_a_closed_window():
    W, seed = 64, 0xFEED
    not_pow2 = lambda n: n >= 3 and n & (n - 1) != 0                       # noqa: E731
    snap, q0, first, (cr, a, lst) = _class_after_a_window(W, not_pow2)
    n = len(lst)
    v = np.random.default_rng(n).integers(accept_top(n), 1 << 31, size=16)
    reqs = np.zeros(16, dtype=REQ_DTYPE)
    reqs["adapter_id"], reqs["flags"], reqs["rand_key"] = a, cr, pick_keys(seed, v)
    outs, rows, _ = chain(snap, [(first, 3), (reqs, seed)], [K, K], W, q=q0)
    _, r0, _, rejects = fallback_rows(seed, reqs["rand_key"], np.ones(16, bool), np.zeros(16, np.int64),
                                      np.full(16, n), np.asarray(lst), K, with_draws=True)
    assert (rejects[:, 0] >= 1).all()
    for i, key in enumerate(reqs["rand_key"].tolist()):
        pick, row = fallback_row(seed, key, lst, K)
        assert outs[1]["pod_idx"][i] == pick and rows[1][i].tolist() == row


def test_forced_rejection_on_a_fallback_step_after_a_closed_window():
    W, seed = 64, 0xBEEF
    snap, q0, first, (cr, a, lst) = _class_after_a_window(W, lambda n: n >= 4 and (n - 1) & (n - 2) != 0)
    n = len(lst)
    v = np.random.default_rng(n).integers(accept_top(n - 1), 1 << 31, size=64)
    with np.errstate(over="ignore"):
        keys = (states_for(v) - np.uint64(GAMMA)) ^ np.uint64(seed & M64)
    reqs = np.zeros(64, dtype=REQ_DTYPE)
    reqs["adapter_id"], reqs["flags"], reqs["rand_key"] = a, cr, keys
    outs, rows, _ = chain(snap, [(first, 3), (reqs, seed)], [K, K], W, q=q0)
    _, _, _, rejects = fallback_rows(seed, keys, np.ones(64, bool), np.zeros(64, np.int64), np.full(64, n),
                                     np.asarray(lst), K, with_draws=True)
    hit = (rejects[:, 0] == 0) & (rejects[:, 1] >= 1)
    assert hit.sum() >= 16
    for i in np.flatnonzero(hit)[:8]:
        pick, row = fallback_row(seed, int(keys[i]), lst, K)
        assert outs[1]["pod_idx"][i] == pick and rows[1][i].tolist() == row


NAMES = ("lig_schedule_batch_feedback_chain_fallbacks", "lig_schedule_batch_feedback_chain_fallbacks_device",
         "lig_schedule_models_batch_feedback_chain_fallbacks",
         "lig_schedule_models_batch_feedback_chain_fallbacks_device")


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
    ids = np.zeros(4, dtype=np.uint32)
    out, mout = np.zeros(4, dtype=PICK_DTYPE), np.zeros(4, dtype=MPICK_DTYPE)
    rows = np.zeros((4, 8), dtype=np.int16)
    loads = np.zeros(4, dtype=np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    for nf, win in ((0, 8), (1, 8), (8, 8), (9, 8), (-1, 8), (4, 0)):
        assert lib.lig_schedule_batch_feedback_chain_fallbacks(None, 1, 2, p(reqs), 4, p(out), nf, p(rows), win,
                                                               p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_feedback_chain_fallbacks_device(None, 1, 2, p(reqs), 4, p(out), nf, p(rows),
                                                                      win, p(loads), None) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_feedback_chain_fallbacks(None, 1, 2, 0, p(ids), 4, p(mout), nf,
                                                                      p(rows), win, p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_feedback_chain_fallbacks_device(
            None, 1, 2, 0, p(ids), 4, p(mout), nf, p(rows), win, p(loads), None) == N.LIG_ERR_INVALID
    assert b"chain_fallbacks" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0) and np.all(loads == 0)
