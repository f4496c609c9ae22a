"""The doorbell stream in model-id mode (include/lig.h, lig_stream_submit_models): one round trip
through the resident kernel resolves and picks up to lig_stream_capacity() model ids.

Every check compares the picks byte for byte with lig_schedule_models_batch on the same epoch,
seed and first_index:
* the synthetic model tables of C2, C3 and C4 at n = 0, 1, 31, 4096 (and 4097 refused);
* model-table edges (0, 1 and 255 targets, weights summing to 2^31-1, targets on adapter id A,
  absent models, ids >= n_models, n_models = 0) under the built-in tree and caller trees with
  DROP and "no pods left" leaves;
* submits that alternate with descriptor submits on one open stream;
* model uploads between submits (the next submit resolves against the new table), model tables
  allocated and grown while the stream is open, and a submit that must wait for an enqueued upload;
* refusals, and identical results after close and reopen.
"""
import numpy as np
import pytest

from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import InferenceModel, InferenceModelSpec
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, pack_models
from test_gpu_models_feedback_chain import edge_models, shuffled_models
from test_gpu_snapshot_mutation import drop_and_no_pods_trees, random_state

pytestmark = pytest.mark.gpu

CAP = 4096


def assert_same(got, want, label):
    assert got.dtype == MPICK_DTYPE and want.dtype == MPICK_DTYPE, label
    assert len(got) == len(want), label
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, (label, bad[:5], got[bad[:5]], want[bad[:5]])


def edge_ids(n, A, n_models, seed):
    ids = WL.make_model_requests(n, A, seed=seed)
    if n >= 8:
        ids[:6] = [n_models, n_models + 5, 2**32 - 1, 2**31, A, A + 1]   # absent x4, pass-through, a split model
    return ids


@pytest.mark.parametrize("cfg", ["C2", "C3", "C4"])
def test_doorbell_models_equal_models_batch(cfg, oracle):
    assert N.load().lig_stream_capacity() == CAP
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"], seed=WL.SNAPSHOT_SEED)
    models = WL.make_models(c["A"])
    pm = pack_models(models, snap.packed)
    ids = edge_ids(CAP + 1, c["A"], pm.n_models, seed=11)
    first = (1 << 40) + 3
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=1 << 16) as e:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, pm)
        e.stream_open()
        try:
            for n in (0, 1, 31, CAP):
                for seed in (5, 2**64 - 1):
                    part = np.ascontiguousarray(ids[:n])
                    got = e.stream_submit_models(1, seed, part, first_index=first)
                    assert_same(got, e.schedule_models_batch(1, seed, part, first_index=first), (cfg, n, seed))
            with pytest.raises(N.LigError) as ei:
                e.stream_submit_models(1, 5, ids, first_index=first)
            assert ei.value.code == N.LIG_ERR_INVALID
            got = e.stream_submit_models(1, 7, np.ascontiguousarray(ids[:CAP]), first_index=0)
        finally:
            e.stream_close()
    st = got["status"]
    assert (st == N.LIG_NO_MODEL).sum() >= 4 and (st == N.LIG_OK).any()
    assert ((got["target_idx"] > 0) & (got["target_idx"] < 255)).any()       # a non-first target was drawn
    pool = oracle.Pool(snap.pod_records())
    want = oracle.Models(WL.model_records(models)).schedule_batch(pool, np.ascontiguousarray(ids[:CAP]), 7, 0)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("tree", [None, 0, 1])
def test_doorbell_model_table_edges(tree):
    P, A = 96, 12
    rng = np.random.default_rng(61)
    state = random_state(P, A, seed=62)
    models, absent = edge_models(A, rng)
    packed = state.packed()
    pm = pack_models(models, packed)
    assert [int(pm.present[i]) for i in absent] == [0]                       # zero-sum packed as absent
    ids = rng.integers(0, len(models) + 3, CAP).astype(np.uint32)
    ids[:3] = [2**32 - 1, len(models), 2**31]
    with Engine(0, max_pods=P, max_adapters=A, max_batch=CAP) as e:
        if tree is not None:
            e.set_filter_tree(drop_and_no_pods_trees()[tree])
        e.upload_snapshot(1, packed)
        e.upload_models(1, pm)
        e.stream_open()
        try:
            for n, first in ((CAP, 5), (1000, 1 << 33), (3, 0)):
                part = np.ascontiguousarray(ids[:n])
                got = e.stream_submit_models(1, 77, part, first_index=first)
                assert_same(got, e.schedule_models_batch(1, 77, part, first_index=first), (tree, n))
                if n == CAP:
                    full = got
            # n_models = 0 (a smaller table fits the resident allocation): every id is LIG_NO_MODEL
            e.upload_models(1, pack_models([], packed))
            got0 = e.stream_submit_models(1, 77, ids, first_index=5)
            assert_same(got0, e.schedule_models_batch(1, 77, ids, first_index=5), (tree, "n_models=0"))
        finally:
            e.stream_close()
    assert (got0["status"] == N.LIG_NO_MODEL).all() and (got0["pod_idx"] == -1).all()
    st = full["status"]
    assert (st == N.LIG_NO_MODEL).any() and (st == N.LIG_OK).any()
    assert (st[ids == absent[0]] == N.LIG_NO_MODEL).all()
    if tree is not None:
        assert (st == (N.LIG_DROP if tree == 0 else N.LIG_NO_PODS_LEFT)).any()
    tg = full["target_idx"]
    assert (tg[ids == 4] > 200).any() and (tg[ids == 5] > 200).any()         # late targets of 255 drawn


def test_doorbell_models_alternate_with_descriptors():
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=21)
    pm = pack_models(WL.make_models(c["A"]), snap.packed)
    ids = edge_ids(CAP, c["A"], pm.n_models, seed=22)
    reqs = WL.make_requests(CAP, c["A"], seed=23)
    rng = np.random.default_rng(24)
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=CAP) as e:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, pm)
        e.stream_open()
        try:
            for k in range(300):
                n = int(rng.choice([1, 2, 3, 4, 5, 31, 255, 1023, 1024, 1025, CAP]))
                lo = int(rng.integers(0, CAP - n + 1))
                seed = int(rng.integers(0, 1 << 63))
                if k % 2:
                    part = np.ascontiguousarray(ids[lo:lo + n])
                    got = e.stream_submit_models(1, seed, part, first_index=lo)
                    assert_same(got, e.schedule_models_batch(1, seed, part, first_index=lo), (k, n))
                else:
                    part = np.ascontiguousarray(reqs[lo:lo + n])
                    assert np.array_equal(e.stream_submit(1, seed, part), e.schedule_batch(1, seed, part)), (k, n)
        finally:
            e.stream_close()


def test_doorbell_models_follow_uploads_and_refuse():
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=31)
    snap2 = WL.make_snapshot(c["P"], c["A"], seed=32)
    tabs = [pack_models(WL.make_models(c["A"]) if k == 0 else shuffled_models(c["A"], 40 + k), snap.packed)
            for k in range(3)]
    ids = edge_ids(CAP, c["A"], tabs[0].n_models, seed=33)
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=CAP) as e:
        e.upload_snapshot(1, snap.packed)
        with pytest.raises(N.LigError) as ei:                                 # stream not open
            e.stream_submit_models(1, 3, ids)
        assert ei.value.code == N.LIG_ERR_INVALID
        e.stream_open()
        try:
            with pytest.raises(N.LigError) as ei:                             # no model table
                e.stream_submit_models(1, 3, ids)
            assert ei.value.code == N.LIG_ERR_NO_SNAPSHOT
        finally:
            e.stream_close()
        e.upload_snapshot(2, snap2.packed)
        e.upload_models(2, pack_models(WL.make_models(c["A"]), snap2.packed))
        e.upload_models(1, tabs[0])
        e.stream_open()
        try:
            with pytest.raises(N.LigError) as ei:                             # stale epoch
                e.stream_submit_models(9, 3, ids)
            assert ei.value.code == N.LIG_ERR_STALE_EPOCH
            first = e.stream_submit_models(1, 3, ids, first_index=9)
            assert_same(first, e.schedule_models_batch(1, 3, ids, first_index=9), "table 0")
            # a blocking upload between submits: the next submit resolves against the new table
            e.upload_models(1, tabs[1])
            got = e.stream_submit_models(1, 3, ids, first_index=9)
            assert_same(got, e.schedule_models_batch(1, 3, ids, first_index=9), "table 1")
            assert not np.array_equal(got, first)
            e.upload_models(1, tabs[2], block=False)
            got = e.stream_submit_models(1, 3, ids, first_index=9)
            assert_same(got, e.schedule_models_batch(1, 3, ids, first_index=9), "table 2")
            got2 = e.stream_submit_models(2, 3, ids, first_index=9)
            assert_same(got2, e.schedule_models_batch(2, 3, ids, first_index=9), "epoch 2")
            # a new epoch replaces epoch 1 in its slot and has no model table until one is uploaded
            e.upload_snapshot(3, snap2.packed)
            with pytest.raises(N.LigError) as ei:
                e.stream_submit_models(3, 3, ids)
            assert ei.value.code == N.LIG_ERR_NO_SNAPSHOT
            with pytest.raises(N.LigError) as ei:
                e.stream_submit_models(1, 3, ids)
            assert ei.value.code == N.LIG_ERR_STALE_EPOCH
            e.upload_models(3, pack_models(shuffled_models(c["A"], 50), snap2.packed))
            got3 = e.stream_submit_models(3, 3, ids, first_index=9)
            assert_same(got3, e.schedule_models_batch(3, 3, ids, first_index=9), "epoch 3")
            assert_same(e.stream_submit_models(2, 3, ids, first_index=9), got2, "epoch 2 still resident")
        finally:
            e.stream_close()
        with pytest.raises(N.LigError) as ei:                                 # closed
            e.stream_submit_models(2, 3, ids)
        assert ei.value.code == N.LIG_ERR_INVALID
        e.stream_open()                                                       # reopen: tickets restart
        try:
            assert_same(e.stream_submit_models(2, 3, ids, first_index=9), got2, "reopened")
            assert_same(e.stream_submit_models(3, 3, ids, first_index=9), got3, "reopened, epoch 3")
        finally:
            e.stream_close()


def with_fillers(models, F):
    """F models without targets in front of `models`: the same models at ids + F, in a table whose
    entries for them sit F x 16 bytes into the blob."""
    fill = [InferenceModel(f"filler-{i}", InferenceModelSpec(ModelName=f"filler-{i}", Criticality=None, TargetModels=[]))
            for i in range(F)]
    return fill + list(models)


def test_doorbell_model_tables_allocate_and_grow_while_open():
    """A runtime opens the stream first and uploads model tables later: the first table of a slot,
    and a table larger than the slot's allocation, are allocated while the stream is open.  The
    resident kernel is stopped around the reallocation and relaunched (one more kernel launch); a
    table that fits is written in place with no relaunch."""
    c = WL.CONFIGS["C2"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=71)
    small = pack_models(WL.make_models(c["A"]), snap.packed)
    big_models = with_fillers(WL.make_models(c["A"]), 5000)
    big = pack_models(big_models, snap.packed)
    same = pack_models(with_fillers(shuffled_models(c["A"], 72), 5000), snap.packed)
    ids = edge_ids(CAP, c["A"], small.n_models, seed=73)
    reqs = WL.make_requests(CAP, c["A"], seed=74)
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=CAP) as e:
        e.upload_snapshot(1, snap.packed)
        e.stream_open()
        try:
            steps = [(small, ids, 1, "first table, allocated while open"),
                     (big, ids + np.uint32(5000), 1, "grown past the allocation"),
                     (same, ids + np.uint32(5000), 0, "fits: written in place")]
            for k, (pm, part, relaunches, label) in enumerate(steps):
                before = e.kernel_launches
                e.upload_models(1, pm)
                assert e.kernel_launches - before == relaunches, label
                got = e.stream_submit_models(1, 11 + k, part, first_index=k << 20)
                assert_same(got, e.schedule_models_batch(1, 11 + k, part, first_index=k << 20), label)
                assert (got["status"] == N.LIG_OK).any(), label
                d = e.stream_submit(1, 11 + k, reqs)                          # descriptors after a relaunch
                assert np.array_equal(d, e.schedule_batch(1, 11 + k, reqs)), label
        finally:
            e.stream_close()


def test_doorbell_submit_waits_for_an_enqueued_model_upload():
    """The entries the ids resolve to sit behind 4.8 MB of filler entries, so an enqueued upload's
    copy is still running when the submit rings the doorbell; a submit that did not wait for it would
    resolve (part of) the ids against the previous table, whose picks differ."""
    c = WL.CONFIGS["C3"]
    F = 300_000
    snap = WL.make_snapshot(c["P"], c["A"], seed=81)
    tabs = [pack_models(with_fillers(WL.make_models(c["A"]) if k == 0 else shuffled_models(c["A"], 82 + k), F),
                        snap.packed) for k in range(3)]
    ids = WL.make_model_requests(CAP, c["A"], seed=83) + np.uint32(F)
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=CAP) as e:
        e.upload_snapshot(1, snap.packed)
        e.stream_open()
        try:
            e.upload_models(1, tabs[0])
            prev = e.stream_submit_models(1, 5, ids)
            assert_same(prev, e.schedule_models_batch(1, 5, ids), "table 0")
            for k in (1, 2):
                e.upload_models(1, tabs[k], block=False)
                got = e.stream_submit_models(1, 5, ids)
                want = e.schedule_models_batch(1, 5, ids)
                assert_same(got, want, f"table {k}, enqueued upload")
                assert (got != prev).mean() > 0.25, k                        # the old table gives other picks
                prev = got
        finally:
            e.stream_close()
