"""Retry scheduling (lig_schedule_batch_excluding) without a GPU: the reference (retry_ref.py) against
the port of the Go scheduler run on the shortened slice, rows that exclude nothing against the
class-table oracle, how excluding pods moves survivor sets, empty pools, row entries that exclude
nothing, and the C ABI's exports and refusals."""
import os
import re

import numpy as np
import pytest

import retry_ref as RR
from filter_tree_ref import random_pool, random_tree
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["a0", "a1", "a2", "a3"]
SEED = 0x5EED_0F_AB_CDEF_0123


def random_rows(rng, R, P, width):
    """Rows mixing in-range pods, duplicates, -1 padding and out-of-range entries."""
    rows = np.full((R, width), -1, dtype=np.int16)
    for i in range(R):
        k = int(rng.integers(0, width + 1))
        cand = rng.integers(0, max(P, 1), size=k)
        cand = np.where(rng.random(k) < 0.1, rng.choice([P, P + 1, 32767, -2, -32768], size=k), cand)
        rows[i, :k] = cand
        if k >= 2 and rng.random() < 0.3:
            rows[i, 1] = rows[i, 0]                       # a duplicate
    return rows


def random_reqs(rng, R, A):
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["adapter_id"] = rng.integers(-1, A + 2, size=R)
    reqs["flags"] = rng.integers(0, 2, size=R)
    reqs["rand_key"] = rng.integers(0, 1 << 64, size=R, dtype=np.uint64)
    return reqs


def go_port(recs, reqs, rows, seed):
    """Schedule of the Go port (oracle/lig_oracle.c) on the slice without each row's pods."""
    out = np.zeros(len(reqs), dtype=PICK_DTYPE)
    for i, r in enumerate(reqs):
        kept = RR.kept_pods(len(recs), rows[i])
        pool = B.Pool([recs[p] for p in kept])
        a = int(r["adapter_id"])
        model = NAMES[a] if 0 <= a < len(NAMES) else WL.UNKNOWN_MODEL
        st, pod, n = pool.schedule(model, bool(r["flags"] & 1), seed, int(r["rand_key"]))
        out[i] = (int(kept[pod]) if pod >= 0 else -1, st, n)
    return out


THRESHOLDS = [(0.8, 5, 50), (0.0, 0, 0), (float("nan"), -(1 << 63), (1 << 63) - 1),
              (float("inf"), (1 << 63) - 1, -(1 << 63))]


@pytest.mark.parametrize("thresholds", THRESHOLDS)
def test_reference_agrees_with_the_go_port(thresholds):
    rng = np.random.default_rng(7)
    B.set_thresholds(*thresholds)
    try:
        for _ in range(25):
            recs = random_pool(rng)
            snap = RR.pack_records(recs, NAMES)
            reqs = random_reqs(rng, 24, len(NAMES))
            rows = random_rows(rng, 24, snap.P, int(rng.choice([1, 9, 32])))
            got = RR.retry_batch(snap, reqs, rows, SEED, thresholds)
            assert np.array_equal(got, go_port(recs, reqs, rows, SEED))
    finally:
        B.set_thresholds()


def test_caller_tree_reference_agrees_with_the_numpy_walker():
    import filter_tree_ref as FT
    rng = np.random.default_rng(8)
    for _ in range(25):
        recs = random_pool(rng)
        nodes = random_tree(rng)
        snap = RR.pack_records(recs, NAMES)
        rows = random_rows(rng, 6, snap.P, 9)
        for row in rows:
            kept = RR.kept_pods(snap.P, row)
            pods = FT.Pods([recs[p] for p in kept])
            for crit in (False, True):
                for a in range(len(NAMES) + 1):
                    model = NAMES[a] if a < len(NAMES) else WL.UNKNOWN_MODEL
                    st, lst = FT.walk(nodes, pods, crit, model)
                    assert RR.survivors(snap, crit, a, row, nodes=nodes) == (st, [int(kept[p]) for p in lst])


@pytest.mark.parametrize("config", ["C1", "C2", "C3"])
def test_rows_that_exclude_nothing_are_the_class_table_picks(config):
    c = WL.CONFIGS[config]
    snap = WL.make_snapshot(c["P"], c["A"], seed=21).packed
    reqs = WL.make_requests(500, c["A"], seed=22)
    P = snap.P
    rows = np.array([[-1, P, 32767, -32768, P + 5]] * len(reqs), dtype=np.int16)
    want = B.ClassTable(P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap).schedule_batch(
        reqs, SEED)
    assert np.array_equal(RR.retry_batch(snap, reqs, rows, SEED), want)
    assert (want["status"] == N.LIG_OK).sum() > 100


@pytest.fixture(scope="module")
def c4():
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=31).packed
    tab = B.ClassTable(snap.P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)
    return snap, tab


def test_excluding_the_survivors_picks_outside_the_old_survivor_set(c4):
    snap, tab = c4
    outside = 0
    for crit, a in [(True, 0), (True, 1), (False, 0), (True, 5), (False, 7), (True, snap.A), (False, snap.A)]:
        st, n, lst = tab.klass(crit, a)
        if st != N.LIG_OK or n > N.LIG_MAX_EXCLUDED:
            continue
        row = np.array(lst, dtype=np.int16)
        st2, lst2 = RR.survivors(snap, crit, a, row)
        assert not set(lst2) & set(lst)
        reqs = np.zeros(8, dtype=REQ_DTYPE)
        reqs["adapter_id"], reqs["flags"] = a, int(crit)
        reqs["rand_key"] = np.arange(8, dtype=np.uint64) * 0x9E3779B97F4A7C15
        got = RR.retry_batch(snap, reqs, np.tile(row, (8, 1)), SEED)
        ok = got["status"] == N.LIG_OK
        assert not set(got["pod_idx"][ok].tolist()) & set(lst)
        outside += int(ok.sum())
    assert outside > 0


def test_excluding_a_non_survivor_moves_a_survivor_set():
    """A pod that survives nowhere still counts in the least-queuing and least-KV ranges: leaving it
    out moves a bucket bound."""
    # every queue >= queueingThresholdLoRA: the critical walk ranges over the whole pool
    recs = [dict(name=f"pod-{i}", address=f"address-{i}", waiting_queue_size=q, kv_cache_usage_percent=0.5,
                 max_active_models=4, active_models=[]) for i, q in enumerate([50, 60, 100, 1000])]
    snap = RR.pack_records(recs, NAMES)
    assert RR.survivors(snap, True, 0, []) == (N.LIG_OK, [0, 1, 2])        # 50 + (1000 - 50) / 4 = 287
    assert RR.survivors(snap, True, 0, [3]) == (N.LIG_OK, [0, 1])          # 50 + (100 - 50) / 3 = 66
    rng = np.random.default_rng(9)
    moved = 0
    for _ in range(40):
        recs = random_pool(rng)
        snap = RR.pack_records(recs, NAMES)
        for crit in (False, True):
            for a in range(len(NAMES) + 1):
                st, lst = RR.survivors(snap, crit, a, [])
                for p in range(snap.P):
                    if p in lst:
                        continue
                    if RR.survivors(snap, crit, a, [p]) != (st, lst):
                        moved += 1
    assert moved > 0


def test_an_empty_pool():
    recs = random_pool(np.random.default_rng(3))[:5]
    snap = RR.pack_records(recs, NAMES)
    row = np.arange(5, dtype=np.int16)
    reqs = np.zeros(2, dtype=REQ_DTYPE)
    reqs["flags"] = [0, 1]
    got = RR.retry_batch(snap, reqs, np.tile(row, (2, 1)), SEED)
    assert got["status"].tolist() == [N.LIG_DROP] * 2 and got["pod_idx"].tolist() == [-1, -1]
    assert got["n_survivors"].tolist() == [0, 0]
    F = N.LigFilterNode
    trees = {N.LIG_NO_PODS_LEFT: [F(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 50, 0.0)],
             N.LIG_DROP: [F(N.LIG_F_LEAST_QUEUING, -1, 1, -1, 0, 0.0), F(N.LIG_F_DROP, -1, -1, -1, 0, 0.0)],
             N.LIG_EMPTY: [F(N.LIG_F_LEAST_KV_CACHE, -1, -1, -1, 0, 0.0)]}
    for status, nodes in trees.items():
        got = RR.retry_batch(snap, reqs, np.tile(row, (2, 1)), SEED, nodes=nodes)
        assert got["status"].tolist() == [status] * 2 and got["pod_idx"].tolist() == [-1, -1]


def test_padding_out_of_range_entries_and_duplicates():
    rng = np.random.default_rng(4)
    recs = random_pool(rng)
    while len(recs) < 12:
        recs = random_pool(rng)
    snap = RR.pack_records(recs, NAMES)
    P = snap.P
    reqs = random_reqs(rng, 64, len(NAMES))
    plain = np.tile(np.array([3, 7], dtype=np.int16), (64, 1))
    noisy = np.tile(np.array([7, -1, 3, 3, P, 32767, -32768, 7, -1], dtype=np.int16), (64, 1))
    assert RR.kept_pods(P, noisy[0]).tolist() == [p for p in range(P) if p not in (3, 7)]
    assert np.array_equal(RR.retry_batch(snap, reqs, plain, SEED), RR.retry_batch(snap, reqs, noisy, SEED))
    nothing = np.full((64, 3), -1, dtype=np.int16)
    full = B.ClassTable(P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)
    assert np.array_equal(RR.retry_batch(snap, reqs, nothing, SEED), full.schedule_batch(reqs, SEED))


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    out = np.zeros(4, dtype=PICK_DTYPE)
    rows = np.zeros((4, 33), dtype=np.int16)
    p = lambda a: a.ctypes.data
    for k in (0, 1, 32, 33, -1):
        assert lib.lig_schedule_batch_excluding(None, 1, 2, p(reqs), 4, p(rows), k, p(out)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_excluding_device(None, 1, 2, p(reqs), 4, p(rows), k, p(out), None) == \
            N.LIG_ERR_INVALID
    assert b"batch_excluding" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0)


def test_symbols_and_limit_are_declared():
    lib = N.load()
    for name in ("lig_schedule_batch_excluding", "lig_schedule_batch_excluding_device"):
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    assert re.search(r"#define LIG_MAX_EXCLUDED 32\b", header) and N.LIG_MAX_EXCLUDED == 32
    assert lib.lig_abi_version() == 7
