"""The fallback ranking of include/lig.h without a GPU: the numpy definition (fallback_ref.py) against
the class-table oracle's pick and a plain Fisher-Yates loop, its properties (distinct survivors,
prefix rows, uniform ordered choices), forced Int31n rejections on the pick and on a later step, and
the C ABI's refusals and exports."""
import itertools
import os
import re

import numpy as np
import pytest
from scipy import stats

from draw_keys import GAMMA, M64, accept_top, pick_keys, rejection_heavy_ns, states_for
from fallback_ref import fallback_row, fallback_rows
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_lists(tab, A, reqs):
    """(ok, offsets, pods) of every request's class list in the class-table oracle."""
    crit = (reqs["flags"] & 1).astype(np.int64)
    a = np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)
    cache = {}
    ok = np.zeros(len(reqs), dtype=bool)
    lists = []
    for i, (c, ai) in enumerate(zip(crit, a)):
        key = (int(c), int(ai))
        if key not in cache:
            st, _, lst = tab.klass(bool(c), int(ai))
            cache[key] = (st == N.LIG_OK, lst)
        ok[i], lst = cache[key]
        lists.append(lst if ok[i] else [])
    offsets = np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.int64)
    pods = np.array([p for l in lists for p in l], dtype=np.int64)
    return ok, offsets, pods


@pytest.fixture(scope="module")
def c2():
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=11)
    p = snap.packed
    tab = B.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap)
    reqs = WL.make_requests(4000, c["A"], seed=12)
    return p, tab, reqs


def test_entry_zero_is_the_class_table_pick(c2):
    p, tab, reqs = c2
    seed = 0x1234_5678_9ABC_DEF0
    picks = tab.schedule_batch(reqs, seed)
    ok, offsets, pods = oracle_lists(tab, p.A, reqs)
    assert np.array_equal(ok, picks["status"] == N.LIG_OK)
    assert ok.sum() > 1000
    _, r0 = fallback_rows(seed, reqs["rand_key"], ok, offsets[:-1], np.diff(offsets), pods, 8)
    got = np.where(ok, pods[np.where(ok, offsets[:-1] + r0, 0)], -1)
    assert np.array_equal(got, picks["pod_idx"])


def test_rows_are_distinct_survivors_and_prefixes(c2):
    p, tab, reqs = c2
    seed = 77
    ok, offsets, pods = oracle_lists(tab, p.A, reqs)
    full, r0 = fallback_rows(seed, reqs["rand_key"], ok, offsets[:-1], np.diff(offsets), pods,
                             N.LIG_MAX_FALLBACKS)
    n = offsets[1:] - offsets[:-1]
    for i in range(len(reqs)):
        lst = pods[offsets[i]:offsets[i + 1]].tolist()
        row = full[i].tolist()
        m = min(int(n[i]), 1 + N.LIG_MAX_FALLBACKS) if ok[i] else 0
        ranked = ([lst[r0[i]]] if ok[i] else []) + [x for x in row if x >= 0]
        assert len(ranked) == m and len(set(ranked)) == m and set(ranked) <= set(lst), i
        assert row[max(m - 1, 0):] == [-1] * (N.LIG_MAX_FALLBACKS - max(m - 1, 0)), i
    for k in range(1, N.LIG_MAX_FALLBACKS):
        rows, r0k = fallback_rows(seed, reqs["rand_key"], ok, offsets[:-1], np.diff(offsets), pods, k)
        assert np.array_equal(rows, full[:, :k]) and np.array_equal(r0k, r0), k


def test_vectorised_definition_equals_plain_loop():
    rng = np.random.default_rng(5)
    seed = int(rng.integers(0, 1 << 63))
    for n in list(range(0, 20)) + [31, 32, 33, 63, 64, 65, 1000, 4097, 32768]:
        keys = rng.integers(0, 1 << 64, size=12, dtype=np.uint64)
        L = np.sort(rng.choice(32768, size=n, replace=False)) if n else np.zeros(0, np.int64)
        offsets = np.arange(13, dtype=np.int64) * n
        pods = np.tile(L, 12)
        for k in (1, 3, 8):
            rows, r0 = fallback_rows(seed, keys, np.ones(12, bool), offsets[:-1], np.diff(offsets), pods, k)
            for i, key in enumerate(keys):
                pick, row = fallback_row(seed, int(key), L.tolist(), k)
                assert (L[r0[i]] if n else -1) == pick and rows[i].tolist() == row, (n, k, i)


@pytest.mark.parametrize("n,k", [(4, 2), (5, 8), (7, 2)])
def test_ordered_choices_are_uniform(n, k):
    """Over keys, every ordered choice of m = min(n, 1 + k) distinct survivors is equally likely
    (chi-square at a fixed seed)."""
    m = min(n, 1 + k)
    cells = list(itertools.permutations(range(n), m))
    R = 400 * len(cells)
    keys = np.random.default_rng(n * 100 + k).integers(0, 1 << 64, size=R, dtype=np.uint64)
    offsets = np.arange(R + 1, dtype=np.int64) * n
    pods = np.tile(np.arange(n), R)
    rows, r0 = fallback_rows(99, keys, np.ones(R, bool), offsets[:-1], np.diff(offsets), pods, k)
    ranked = np.concatenate([r0[:, None], rows[:, :m - 1].astype(np.int64)], axis=1)
    index = {c: j for j, c in enumerate(cells)}
    counts = np.bincount([index[tuple(r)] for r in ranked.tolist()], minlength=len(cells))
    assert counts.sum() == R and (counts > 0).all()
    assert stats.chisquare(counts).pvalue > 1e-3, counts


def test_forced_rejection_on_the_pick():
    """Keys whose pick draw is rejected: the stream continues after the redraw."""
    seed = 0xFEED
    for n in rejection_heavy_ns(3, 20000, 4):
        v = np.random.default_rng(n).integers(accept_top(n), 1 << 31, size=16)
        keys = pick_keys(seed, v)
        offsets = np.arange(17, dtype=np.int64) * n
        pods = np.tile(np.arange(n), 16)
        rows, r0, draws, rejects = fallback_rows(seed, keys, np.ones(16, bool), offsets[:-1], np.diff(offsets),
                                                 pods, 8, with_draws=True)
        assert (rejects[:, 0] >= 1).all()
        for i, key in enumerate(keys):
            pick, row = fallback_row(seed, int(key), list(range(n)), 8)
            assert pick == r0[i] and rows[i].tolist() == row


def test_forced_rejection_on_a_fallback_step():
    """Keys whose second value (step 1's first draw when the pick accepts) lands in the rejection
    band of Int31n(n - 1)."""
    seed = 0xBEEF
    for n1 in rejection_heavy_ns(3, 20000, 4):
        n = n1 + 1
        v = np.random.default_rng(n).integers(accept_top(n1), 1 << 31, size=64)
        with np.errstate(over="ignore"):
            keys = (states_for(v) - np.uint64(GAMMA)) ^ np.uint64(seed & M64)
        offsets = np.arange(65, dtype=np.int64) * n
        pods = np.tile(np.arange(n), 64)
        rows, r0, draws, rejects = fallback_rows(seed, keys, np.ones(64, bool), offsets[:-1], np.diff(offsets),
                                                 pods, 8, with_draws=True)
        hit = (rejects[:, 0] == 0) & (rejects[:, 1] >= 1)
        assert hit.sum() >= 32, n
        for i in np.flatnonzero(hit)[:8]:
            pick, row = fallback_row(seed, int(keys[i]), list(range(n)), 8)
            assert pick == r0[i] and rows[i].tolist() == row


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    ids = np.zeros(4, dtype=np.uint32)
    out, mout = np.zeros(4, dtype=PICK_DTYPE), np.zeros(4, dtype=MPICK_DTYPE)
    rows = np.zeros((4, 8), dtype=np.int16)
    p = lambda a: a.ctypes.data
    for nf in (0, 1, 8, 9, -1):
        assert lib.lig_schedule_batch_fallbacks(None, 1, 2, p(reqs), 4, p(out), nf, p(rows)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_fallbacks_device(None, 1, 2, p(reqs), 4, p(out), nf, p(rows), None) == \
            N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_fallbacks(None, 1, 2, 0, p(ids), 4, p(mout), nf, p(rows)) == \
            N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_fallbacks_device(None, 1, 2, 0, p(ids), 4, p(mout), nf, p(rows),
                                                              None) == N.LIG_ERR_INVALID
    assert b"batch_fallbacks" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0)


def test_symbols_and_limit_are_declared():
    lib = N.load()
    names = ("lig_schedule_batch_fallbacks", "lig_schedule_batch_fallbacks_device",
             "lig_schedule_models_batch_fallbacks", "lig_schedule_models_batch_fallbacks_device")
    for name in names:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    assert re.search(r"#define LIG_MAX_FALLBACKS 8\b", header) and N.LIG_MAX_FALLBACKS == 8
    assert lib.lig_abi_version() == 7
