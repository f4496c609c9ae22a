"""Outlier ejection (lig_eject_pods) without a GPU: the reference (eject_ref.py) with nothing ejected
against the class-table oracle, no ejected pod in any result, ejecting every pod, retry rows that
also name ejected pods, and the C ABI's export and null-ctx refusal."""
import os

import numpy as np
import pytest

import eject_ref as ER
import feedback_chain_retry_ref as CR
import retry_ref as RR
from filter_tree_ref import random_pool, random_tree
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["a0", "a1", "a2", "a3"]
SEED = 0x0E1E_C7ED_5EED_0042


@pytest.fixture(scope="module")
def c4():
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=41).packed
    return snap, WL.make_requests(400, c["A"], seed=42)


def test_nothing_ejected_is_the_class_table_oracle(c4):
    snap, reqs = c4
    tab = B.ClassTable(snap.P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)
    want = tab.schedule_batch(reqs, SEED)
    assert np.array_equal(ER.schedule_batch(snap, [], reqs, SEED), want)
    assert (want["status"] == N.LIG_OK).sum() > 100
    for crit, a in [(True, 0), (False, 0), (True, 3), (False, snap.A)]:
        st, _, lst = tab.klass(crit, a)
        assert ER.klass(snap, [], crit, a) == (st, list(lst))


def test_no_ejected_pod_appears_in_any_result(c4):
    snap, reqs = c4
    rng = np.random.default_rng(5)
    tab = B.ClassTable(snap.P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)
    base = tab.schedule_batch(reqs, SEED)
    # eject pods that the base picks, so the pool really changes
    ok = base["status"] == N.LIG_OK
    hot = np.unique(base["pod_idx"][ok])
    ejected = sorted(set(rng.choice(hot, size=min(12, len(hot)), replace=False).tolist()))
    gone = set(ejected)
    picks = ER.schedule_batch(snap, ejected, reqs, SEED)
    assert not gone & set(picks["pod_idx"][picks["status"] == N.LIG_OK].tolist())
    assert (picks["status"] == N.LIG_OK).sum() > 100
    assert not np.array_equal(picks, base)
    for crit in (False, True):
        for a in (0, 1, 2, snap.A):
            _, lst = ER.klass(snap, ejected, crit, a)
            assert not gone & set(lst)
    _, rows = ER.fallback_batch(snap, ejected, reqs[:100], SEED, 4)
    assert not gone & set(rows[rows >= 0].tolist())
    retry = ER.retry_batch(snap, ejected, reqs[:100], np.full((100, 2), 7, dtype=np.int16), SEED)
    assert not (gone | {7}) & set(retry["pod_idx"][retry["pod_idx"] >= 0].tolist())
    outs, _, loads = ER.chain(snap, ejected, [(reqs[:150], SEED), (reqs[150:300], SEED + 1)], window=64)
    assert all(not gone & set(o["pod_idx"][o["pod_idx"] >= 0].tolist()) for o in outs)
    assert loads[ejected].sum() == 0 and loads.sum() > 0


def test_ejecting_every_pod_is_the_empty_slice():
    recs = random_pool(np.random.default_rng(3))
    snap = RR.pack_records(recs, NAMES)
    reqs = np.zeros(4, dtype=B.REQ_DTYPE)
    reqs["flags"] = [0, 1, 0, 1]
    reqs["adapter_id"] = [0, 1, 9, -1]
    every = list(range(snap.P))
    got = ER.schedule_batch(snap, every, reqs, SEED)
    assert got["status"].tolist() == [N.LIG_DROP] * 4 and got["pod_idx"].tolist() == [-1] * 4
    assert got["n_survivors"].tolist() == [0] * 4
    assert ER.klass(snap, every, True, 0) == (N.LIG_DROP, [])
    F = N.LigFilterNode
    nodes = [F(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 50, 0.0)]
    got = ER.schedule_batch(snap, every, reqs, SEED, nodes=nodes)
    assert got["status"].tolist() == [N.LIG_NO_PODS_LEFT] * 4


def test_a_retry_row_naming_ejected_pods_excludes_nothing_more():
    rng = np.random.default_rng(8)
    for _ in range(20):
        recs = random_pool(rng)
        if len(recs) < 6:
            continue
        snap = RR.pack_records(recs, NAMES)
        P = snap.P
        ejected = sorted(rng.choice(P, size=2, replace=False).tolist())
        other = [p for p in range(P) if p not in ejected][0]
        reqs = np.zeros(32, dtype=B.REQ_DTYPE)
        reqs["adapter_id"] = rng.integers(-1, len(NAMES) + 1, size=32)
        reqs["flags"] = rng.integers(0, 2, size=32)
        reqs["rand_key"] = rng.integers(0, 1 << 64, size=32, dtype=np.uint64)
        plain = np.tile(np.array([other, -1, -1], dtype=np.int16), (32, 1))
        noisy = np.tile(np.array([other, ejected[0], ejected[1]], dtype=np.int16), (32, 1))
        nodes = random_tree(rng) if rng.random() < 0.5 else None
        assert np.array_equal(ER.retry_batch(snap, ejected, reqs, plain, SEED, nodes=nodes),
                              ER.retry_batch(snap, ejected, reqs, noisy, SEED, nodes=nodes))
        a = ER.retry_fallback_batch(snap, ejected, reqs, plain, SEED, 3, nodes=nodes)
        b = ER.retry_fallback_batch(snap, ejected, reqs, noisy, SEED, 3, nodes=nodes)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        # and a retry on the base whose row names the ejected pods is the same walk
        assert np.array_equal(ER.retry_batch(snap, ejected, reqs, plain, SEED, nodes=nodes),
                              RR.retry_batch(snap, reqs, noisy, SEED, nodes=nodes))
        ca = ER.chain(snap, ejected, [CR.retry_call(reqs, plain, SEED)], window=8, nodes=nodes)
        cb = ER.chain(snap, ejected, [CR.retry_call(reqs, noisy, SEED)], window=8, nodes=nodes)
        assert np.array_equal(ca[0][0], cb[0][0]) and np.array_equal(ca[2], cb[2])


def test_abi_export_and_null_ctx():
    lib = N.load()
    assert "lig_eject_pods" in N.EXPORTED_SYMBOLS and hasattr(lib, "lig_eject_pods")
    idx = np.array([1, 2], dtype=np.int32)
    assert lib.lig_eject_pods(None, 2, 1, idx.ctypes.data, 2) == N.LIG_ERR_INVALID
    assert b"lig_eject_pods" in lib.lig_last_error()
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    assert "int lig_eject_pods(lig_ctx* ctx, uint64_t new_epoch, uint64_t base_epoch, const int32_t* pod_idx, int n);" \
        in header
    assert lib.lig_abi_version() == 7
