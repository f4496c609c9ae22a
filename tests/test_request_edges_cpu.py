"""request_edges_ref.py against the oracles it is built from: its class lists are the oracles' lists, every
out-of-range adapter id is the class of A, and its picks, fallback rows, affinity rows and model resolves
equal the existing definitions, so the GPU edge tests compare the kernels with nothing new."""
import numpy as np
import pytest

import affinity_ref as AR
import eject_ref as ER
import fallback_ref as FR
import models_feedback_chain_ref as MC
import models_retry_ref as MR
import oracle_tree as OT
import request_edges_ref as E
import retry_fallbacks_ref as RF
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from oracle import binding as B

SEED = 0x5EED_ED6E
LORA_ONLY = [N.LigFilterNode(N.LIG_F_LORA_AFFINITY, -1, -1, -1, 0, 0.0)]


def table(snap):
    return B.ClassTable(snap.P, snap.A, snap.kv, snap.q, snap.n_active, snap.max_active, snap.bitmap)


@pytest.mark.parametrize("P,A", [(1, 0), (33, 1), (257, 5), (97, 64)])
def test_lists_are_the_class_table_oracle(P, A):
    snap = WL.make_snapshot(P, A, seed=P + A).packed
    cl, tab = E.ClassLists(snap), table(snap)
    for c in range(2 * (A + 1)):
        st, n, lst = tab.klass(bool(c // (A + 1)), c % (A + 1))
        assert (cl.status[c], cl.n[c], cl.lists[c].tolist()) == (st, n, lst)
    # out-of-range ids: the oracle's class of A, in the oracle and in the helper
    for crit in (False, True):
        for a in E.hostile_adapters(A):
            assert tab.klass(crit, a) == tab.klass(crit, A)
    reqs = E.edge_requests(cl, 2000, SEED, np.random.default_rng(P))
    hostile = ~np.isin(reqs["adapter_id"], np.arange(A))
    assert hostile.any() and (cl.classes(reqs)[hostile] % (A + 1) == A).all()
    as_A = reqs.copy()
    as_A["adapter_id"][hostile] = A
    assert tab.schedule_batch(reqs, SEED).tobytes() == tab.schedule_batch(as_A, SEED).tobytes()
    # the helper's picks are the oracle's, rejection keys and extreme keys included
    assert cl.picks(reqs, SEED).tobytes() == tab.schedule_batch(reqs, SEED).tobytes()


def test_rejecting_keys_reject():
    rng = np.random.default_rng(1)
    for n in (3, 5, 7, 33, 34, 255, 4097):
        for step in (0, 1):
            if (n - step) & (n - step - 1) == 0:       # a power of two never rejects: a random key
                continue
            key = E.rejecting_key(n, SEED, step, rng)
            _, _, draws, rej = FR.fallback_rows(
                SEED, np.array([key], np.uint64), np.array([True]), np.array([0]), np.array([n]),
                np.arange(n), 1, with_draws=True)
            assert rej[0, step] >= 1, (n, step)
            if step == 1:
                assert rej[0, 0] == 0


def test_caller_tree_and_ejected_lists_are_the_oracles():
    syn = WL.make_snapshot(61, 5, seed=3)
    snap = syn.packed
    names = syn.adapter_names() + [WL.UNKNOWN_MODEL]
    for nodes in (LORA_ONLY, S.DEFAULT_FILTER.flatten()):
        cl = E.ClassLists(snap, nodes=nodes)
        OT.set_filter_tree(nodes)
        try:
            pool = OT.Pool(syn.pod_records())
            for c in range(2 * (snap.A + 1)):
                st, lst = pool.filter(names[c % (snap.A + 1)], bool(c // (snap.A + 1)))
                assert (cl.status[c], cl.lists[c].tolist()) == (st, lst), c
            reqs = E.edge_requests(cl, 500, SEED, np.random.default_rng(2))
            want = pool.schedule_batch(syn.adapter_names(), WL.UNKNOWN_MODEL, reqs, SEED)
        finally:
            OT.set_filter_tree(None)
        assert cl.picks(reqs, SEED).tobytes() == want.tobytes()
    assert N.LIG_NO_PODS_LEFT in E.ClassLists(snap, nodes=LORA_ONLY).status
    gone = [0, 5, 6, 60]
    cl = E.ClassLists(snap, ejected=gone)
    reqs = E.edge_requests(cl, 500, SEED, np.random.default_rng(3))
    assert cl.picks(reqs, SEED).tobytes() == ER.schedule_batch(snap, gone, reqs, SEED).tobytes()
    for c in range(2 * (snap.A + 1)):
        assert not np.isin(cl.lists[c], gone).any()


@pytest.mark.parametrize("P,A", [(33, 5), (257, 64)])
def test_feature_expectations_equal_the_existing_refs(P, A):
    """On make_requests inputs: fallback rows equal retry_fallbacks_ref's with nothing excluded (its lists
    come from retry_ref.survivors), affinity rows equal affinity_ref.affinity_row request by request."""
    snap = WL.make_snapshot(P, A, seed=7).packed
    cl = E.ClassLists(snap)
    reqs = WL.make_requests(300, A, seed=8)
    none = np.full((300, 2), -1, dtype=np.int16)
    for k in (1, 8):
        picks, rows = cl.fallbacks(reqs, SEED, k)
        want, want_rows = RF.retry_fallback_batch(snap, reqs, none, SEED, k)
        assert picks.tobytes() == want.tobytes() and np.array_equal(rows, want_rows)
    pod_keys = np.random.default_rng(9).integers(0, 1 << 64, size=P, dtype=np.uint64)
    ok, offsets, pods = cl.csr(reqs)
    pick, rows = AR.affinity_rows(reqs["rand_key"], ok, offsets, pods, pod_keys, 8)
    for i in range(300):
        p, r = AR.affinity_row(int(reqs["rand_key"][i]), pods[offsets[i]:offsets[i + 1]], pod_keys, 8)
        assert (int(pick[i]), rows[i].tolist()) == (p, r)


@pytest.mark.parametrize("A", [0, 1, 5])
def test_hostile_model_tables(A):
    """The raw table's resolve (what the device reads) equals the oracle's on names: every hostile own or
    target id resolves to the class of A; model picks equal the oracle's model scheduler."""
    syn = WL.make_snapshot(40, A, seed=11)
    snap = syn.packed
    recs = E.hostile_models(A)
    pm = E.pack_raw_models(recs, A)
    ids_of = pm.target_adapter_ids.tolist() + pm.self_adapter_ids[pm.present == 1].tolist()
    assert set(E.hostile_adapters(A)) <= set(ids_of)
    assert {int(x) for x in np.diff(pm.target_offsets)} >= {0, 1, 2, 3}
    models = B.Models(recs)
    ids = E.model_ids(pm.n_models, 400, np.random.default_rng(12))
    first = (1 << 64) - 7
    res = MC.resolve_call(models, snap.adapter_id, ids, SEED, first)
    # the fixed-target resolve of models_retry_ref on the raw table, at the targets the oracle drew
    fixed = MR.fixed_resolve(pm, ids, res["target_idx"], first)
    assert np.array_equal(fixed["ok"], res["ok"])
    cl = E.ClassLists(snap)
    ok = res["ok"] == 1
    assert np.array_equal(cl.classes(fixed["req"][ok]), cl.classes(res["req"][ok]))
    assert np.array_equal(fixed["req"]["flags"][ok], res["req"]["flags"][ok])
    picks = cl.picks(np.ascontiguousarray(res["req"]), SEED)
    got = np.zeros(len(ids), dtype=B.MPICK_DTYPE)
    got["pod_idx"] = np.where(ok, picks["pod_idx"], -1)
    got["status"] = np.where(ok, picks["status"], 3)
    got["target_idx"] = res["target_idx"]
    pool = B.Pool(syn.pod_records())
    want = models.schedule_batch(pool, ids, SEED, first)
    assert got.tobytes() == want.tobytes()
