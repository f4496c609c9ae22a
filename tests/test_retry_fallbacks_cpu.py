"""Retry scheduling with fallback rows (lig_schedule_batch_excluding_fallbacks) without a GPU: the
definition (retry_fallbacks_ref.py) against the fallback ranking of the class-table oracle's lists
for rows that exclude nothing, against the retry's pick, against a plain Fisher-Yates loop over the
reduced lists, its properties (no excluded entry, distinct entries, prefix rows), forced Int31n
rejections on the pick and on a ranking step, and the C ABI's refusals and exports."""
import os

import numpy as np
import pytest

import retry_fallbacks_ref as RF
import retry_ref as RR
from draw_keys import GAMMA, M64, accept_top, pick_keys, rejection_heavy_ns, states_for
from fallback_ref import fallback_row, fallback_rows
from filter_tree_ref import random_pool
from test_fallbacks_cpu import oracle_lists
from test_retry_cpu import NAMES, random_reqs, random_rows
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = N.LIG_MAX_FALLBACKS
SEED = 0x5EED_0F_AB_CDEF_0456
KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]


@pytest.mark.parametrize("config", ["C1", "C2"])
def test_rows_that_exclude_nothing_are_the_class_table_rows(config):
    c = WL.CONFIGS[config]
    snap = WL.make_snapshot(c["P"], c["A"], seed=41).packed
    reqs = WL.make_requests(400, c["A"], seed=42)
    P = snap.P
    nothing = np.array([[-1, P, 32767, -32768]] * len(reqs), dtype=np.int16)
    tab = B.ClassTable(P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)
    ok, offsets, pods = oracle_lists(tab, snap.A, reqs)
    want_rows, _ = fallback_rows(SEED, reqs["rand_key"], ok, offsets[:-1], np.diff(offsets), pods, K)
    picks, rows = RF.retry_fallback_batch(snap, reqs, nothing, SEED, K)
    assert picks.tobytes() == tab.schedule_batch(reqs, SEED).tobytes()
    assert np.array_equal(rows, want_rows)
    assert (picks["status"] == N.LIG_OK).sum() > 100


def pools(rng, count):
    for _ in range(count):
        recs = random_pool(rng)
        yield recs, RR.pack_records(recs, NAMES)


@pytest.mark.parametrize("tree", [None, "keep_all"])
def test_entry_zero_is_the_retry_pick_and_rows_rank_the_reduced_list(tree):
    nodes = KEEP_ALL if tree else None
    rng = np.random.default_rng(43)
    ranked = 0
    for recs, snap in pools(rng, 20):
        reqs = random_reqs(rng, 24, len(NAMES))
        rows_ex = random_rows(rng, 24, snap.P, int(rng.choice([1, 9, 32])))
        picks, rows = RF.retry_fallback_batch(snap, reqs, rows_ex, SEED, K, nodes=nodes)
        assert picks.tobytes() == RR.retry_batch(snap, reqs, rows_ex, SEED, nodes=nodes).tobytes()
        for i, r in enumerate(reqs):
            st, lst = RR.survivors(snap, bool(r["flags"] & 1), int(r["adapter_id"]), rows_ex[i], nodes=nodes)
            assert st == picks["status"][i] and len(lst) == picks["n_survivors"][i]
            gone = {int(e) for e in rows_ex[i]}
            if st != N.LIG_OK:
                assert (rows[i] == -1).all()
                continue
            # the plain Fisher-Yates loop of the fallback definition over the reduced list
            pick, row = fallback_row(SEED, int(r["rand_key"]), lst, K)
            assert pick == picks["pod_idx"][i] and rows[i].tolist() == row
            m = min(len(lst), 1 + K)
            entries = [pick] + [int(x) for x in rows[i] if x >= 0]
            assert len(entries) == m and len(set(entries)) == m
            assert not set(entries) & gone and set(entries) <= set(lst)
            ranked += m - 1
    assert ranked > 20


def test_rows_are_prefixes_across_k():
    rng = np.random.default_rng(44)
    for recs, snap in pools(rng, 10):
        reqs = random_reqs(rng, 32, len(NAMES))
        rows_ex = random_rows(rng, 32, snap.P, 9)
        picks, full = RF.retry_fallback_batch(snap, reqs, rows_ex, SEED, K)
        for k in range(1, K):
            pk, rows = RF.retry_fallback_batch(snap, reqs, rows_ex, SEED, k)
            assert pk.tobytes() == picks.tobytes() and np.array_equal(rows, full[:, :k]), k


def test_large_reduced_lists_against_the_plain_loop():
    """A C3 pool with a caller tree that keeps every pod: lists of hundreds of pods, rows always full."""
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=45).packed
    rng = np.random.default_rng(46)
    reqs = random_reqs(rng, 16, snap.A)
    rows_ex = rng.integers(0, snap.P, size=(16, 32)).astype(np.int16)
    picks, rows = RF.retry_fallback_batch(snap, reqs, rows_ex, SEED, K, nodes=KEEP_ALL)
    for i, r in enumerate(reqs):
        kept = RR.kept_pods(snap.P, rows_ex[i]).tolist()
        assert picks["n_survivors"][i] == len(kept)
        pick, row = fallback_row(SEED, int(r["rand_key"]), kept, K)
        assert pick == picks["pod_idx"][i] and rows[i].tolist() == row and min(row) >= 0


def forced_snapshot(n):
    """n + 3 pods; every request's pool is n pods once the row [0, n // 2, n + 2] is taken out."""
    snap = WL.make_snapshot(n + 3, 4, seed=n).packed
    row = np.array([0, (n + 3) // 2, n + 2], dtype=np.int16)
    return snap, row


def test_forced_rejection_on_the_pick():
    for n in rejection_heavy_ns(40, 4000, 2):
        snap, row = forced_snapshot(n)
        rng = np.random.default_rng(n)
        keys = pick_keys(SEED, rng.integers(accept_top(n), 1 << 31, size=16), rng)
        reqs = np.zeros(16, dtype=REQ_DTYPE)
        reqs["rand_key"] = keys
        rows_ex = np.tile(row, (16, 1))
        picks, rows = RF.retry_fallback_batch(snap, reqs, rows_ex, SEED, K, nodes=KEEP_ALL)
        kept = RR.kept_pods(snap.P, row)
        assert (picks["n_survivors"] == n).all()
        _, _, _, rejects = fallback_rows(SEED, keys, np.ones(16, bool), np.zeros(16, np.int64), np.full(16, n),
                                         kept, K, with_draws=True)
        assert (rejects[:, 0] >= 1).all()
        for i in range(16):
            pick, want = fallback_row(SEED, int(keys[i]), kept.tolist(), K)
            assert pick == picks["pod_idx"][i] and rows[i].tolist() == want


def test_forced_rejection_on_a_ranking_step():
    for n1 in rejection_heavy_ns(40, 4000, 2):
        n = n1 + 1
        snap, row = forced_snapshot(n)
        v = np.random.default_rng(n).integers(accept_top(n1), 1 << 31, size=64)
        with np.errstate(over="ignore"):
            keys = (states_for(v) - np.uint64(GAMMA)) ^ np.uint64(SEED & M64)
        kept = RR.kept_pods(snap.P, row)
        _, _, _, rejects = fallback_rows(SEED, keys, np.ones(64, bool), np.zeros(64, np.int64), np.full(64, n),
                                         kept, K, with_draws=True)
        hit = (rejects[:, 0] == 0) & (rejects[:, 1] >= 1)
        assert hit.sum() >= 16, n
        reqs = np.zeros(int(hit.sum()), dtype=REQ_DTYPE)
        reqs["rand_key"] = keys[hit]
        picks, rows = RF.retry_fallback_batch(snap, reqs, np.tile(row, (len(reqs), 1)), SEED, K, nodes=KEEP_ALL)
        for i in range(len(reqs)):
            pick, want = fallback_row(SEED, int(reqs["rand_key"][i]), kept.tolist(), K)
            assert pick == picks["pod_idx"][i] and rows[i].tolist() == want


def test_an_empty_pool_gets_rows_of_minus_one():
    recs = random_pool(np.random.default_rng(3))[:5]
    snap = RR.pack_records(recs, NAMES)
    reqs = np.zeros(2, dtype=REQ_DTYPE)
    reqs["flags"] = [0, 1]
    picks, rows = RF.retry_fallback_batch(snap, reqs, np.tile(np.arange(5, dtype=np.int16), (2, 1)), SEED, 4)
    assert (picks["status"] == N.LIG_DROP).all() and (rows == -1).all()


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    out = np.zeros(4, dtype=PICK_DTYPE)
    ex = np.zeros((4, 33), dtype=np.int16)
    rows = np.zeros((4, 9), dtype=np.int16)
    p = lambda a: a.ctypes.data
    for nx, nf in [(0, 1), (33, 1), (-1, 1), (1, 0), (1, 9), (1, -1), (32, 8), (1, 1), (0, 0)]:
        assert lib.lig_schedule_batch_excluding_fallbacks(None, 1, 2, p(reqs), 4, p(ex), nx, p(out), nf,
                                                          p(rows)) == N.LIG_ERR_INVALID
        assert b"lig_schedule_batch_excluding_fallbacks:" in lib.lig_last_error()
        assert lib.lig_schedule_batch_excluding_fallbacks_device(None, 1, 2, p(reqs), 4, p(ex), nx, p(out), nf,
                                                                 p(rows), None) == N.LIG_ERR_INVALID
        assert b"lig_schedule_batch_excluding_fallbacks_device" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(ex == 0) and out.tobytes() == bytes(out.nbytes)


def test_symbols_are_declared_and_exported():
    lib = N.load()
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    for name in ("lig_schedule_batch_excluding_fallbacks", "lig_schedule_batch_excluding_fallbacks_device"):
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name) and f"int {name}(" in header
    assert lib.lig_abi_version() == 7
