"""Model-id retries (lig_schedule_models_batch[_feedback_chain]_excluding[_fallbacks]) without a GPU: every
LIG_NO_MODEL case of the fixed-target resolve, the first call's targets with rows that exclude nothing
against the oracle's model call, the chain definition against the plain model chain and split into
calls every way, and the C ABI's exports and null-ctx refusals."""
import os
import re

import numpy as np
import pytest

import models_feedback_chain_ref as MC
import models_retry_ref as MR
import retry_ref as RR
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import InferenceModel, InferenceModelSpec, TargetModel
from llm_instance_gateway_b200.packer import pack_models
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x5EED_0F_40DE_1D5
NEW = ("lig_schedule_models_batch_excluding", "lig_schedule_models_batch_excluding_device",
       "lig_schedule_models_batch_excluding_fallbacks", "lig_schedule_models_batch_excluding_fallbacks_device",
       "lig_schedule_models_batch_feedback_chain_excluding",
       "lig_schedule_models_batch_feedback_chain_excluding_device",
       "lig_schedule_models_batch_feedback_chain_excluding_fallbacks",
       "lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device")


def setup(P=70, A=12, seed=3):
    syn = WL.make_snapshot(P, A, seed=seed)
    models = WL.make_models(A)
    return syn, models, pack_models(models, syn.packed)


def no_rows(R, width=2):
    return np.full((R, width), -1, dtype=np.int16)


def test_every_no_model_case():
    snap = WL.make_snapshot(8, 3, seed=1).packed
    models = [InferenceModel("own", InferenceModelSpec(ModelName="adapter-1")),
              InferenceModel("one", InferenceModelSpec(ModelName="one", TargetModels=[TargetModel("adapter-2", 5)])),
              InferenceModel("two", InferenceModelSpec(ModelName="two", Criticality="Critical",
                                                       TargetModels=[TargetModel("adapter-0", 1),
                                                                     TargetModel("adapter-1", 2)])),
              InferenceModel("zero", InferenceModelSpec(ModelName="zero", TargetModels=[TargetModel("adapter-0", 0)]))]
    pm = pack_models(models, snap)
    pm.present[0] = 1
    cases = [  # (model id, target, resolves, adapter, critical)
        (0, 255, True, 1, 0), (0, 0, False, 0, 0), (0, 254, False, 0, 0),
        (1, 0, True, 2, 0), (1, 1, False, 0, 0), (1, 255, False, 0, 0),
        (2, 0, True, 0, 1), (2, 1, True, 1, 1), (2, 2, False, 0, 0), (2, 255, False, 0, 0),
        (3, 255, False, 0, 0), (3, 0, False, 0, 0),                 # zero weights: packed as absent
        (4, 255, False, 0, 0), (0xFFFFFFFF, 0, False, 0, 0)]        # ids past the table
    ids = np.array([c[0] for c in cases], dtype=np.uint32)
    tg = np.array([c[1] for c in cases], dtype=np.uint8)
    res = MR.fixed_resolve(pm, ids, tg, first_index=(1 << 64) - 3)
    assert res["ok"].tolist() == [int(c[2]) for c in cases]
    ok = res["ok"] == 1
    assert res["req"]["adapter_id"][ok].tolist() == [c[3] for c in cases if c[2]]
    assert res["req"]["flags"][ok].tolist() == [c[4] for c in cases if c[2]]
    assert res["req"]["rand_key"].tolist() == [((1 << 64) - 3 + i) % (1 << 64) for i in range(len(cases))]
    got = MR.retry_batch(snap, pm, ids, tg, no_rows(len(cases)), SEED)
    assert (got["status"][~ok] == MR.LIG_NO_MODEL).all() and (got["pod_idx"][~ok] == -1).all()
    assert (got["target_idx"][~ok] == 255).all() and (got["target_idx"][ok] == tg[ok]).all()
    _, rows = MR.retry_fallback_batch(snap, pm, ids, tg, no_rows(len(cases)), SEED, 4)
    assert (rows[~ok] == -1).all()


@pytest.mark.parametrize("first_index", [0, 12345, (1 << 64) - 17])
def test_first_calls_targets_reproduce_the_model_call(first_index):
    syn, models, pm = setup()
    ids = np.concatenate([WL.make_model_requests(600, syn.packed.A, seed=5),
                          np.array([pm.n_models, 0xFFFFFFFF], dtype=np.uint32)])
    pool = B.Pool(syn.pod_records())
    first = B.Models(WL.model_records(models)).schedule_batch(pool, ids, SEED, first_index)
    got = MR.retry_batch(syn.packed, pm, ids, first["target_idx"], no_rows(len(ids)), SEED, first_index)
    assert got.tobytes() == first.tobytes()
    assert (first["status"] == MR.LIG_NO_MODEL).any() and (first["target_idx"] >= 2).any()


def test_model_retry_equals_the_descriptor_retry():
    syn, models, pm = setup()
    rng = np.random.default_rng(9)
    R = 300
    ids = WL.make_model_requests(R, syn.packed.A, seed=6)
    first = B.Models(WL.model_records(models)).schedule_batch(B.Pool(syn.pod_records()), ids, SEED, 7)
    rows = rng.integers(-1, syn.packed.P + 2, size=(R, 5)).astype(np.int16)
    got, got_rows = MR.retry_fallback_batch(syn.packed, pm, ids, first["target_idx"], rows, SEED, 3, first_index=7)
    res = MR.fixed_resolve(pm, ids, first["target_idx"], 7)
    ok = res["ok"] == 1
    want = RR.retry_batch(syn.packed, np.ascontiguousarray(res["req"][ok]), rows[ok], SEED)
    assert np.array_equal(got["pod_idx"][ok], want["pod_idx"]) and np.array_equal(got["status"][ok], want["status"])
    assert (got_rows[~ok] == -1).all()
    for i in np.flatnonzero(got["status"] == N.LIG_OK):
        ranked = [int(got["pod_idx"][i])] + [int(x) for x in got_rows[i] if x >= 0]
        assert len(set(ranked)) == len(ranked) and not set(ranked) & set(rows[i].tolist())


def model_chain_calls(syn, models, ids, bounds, first_index=0):
    return MC.split_model_calls(B.Models(WL.model_records(models)), syn.packed.adapter_id, ids, bounds, SEED,
                                first_index)


@pytest.mark.parametrize("window", [1, 7, 64])
def test_chain_model_retry_with_first_targets_is_the_model_chain(window):
    syn, models, pm = setup()
    snap = syn.packed
    ids = WL.make_model_requests(200, snap.A, seed=8)
    bounds = [0, 50, 51, 120, 200]
    plain = model_chain_calls(syn, models, ids, bounds, 3)
    outs, _, loads = MR.run_chain(snap, plain, window)
    targets = np.concatenate([o["target_idx"] for o in outs])
    for k in (0, 4):
        calls = [MR.model_retry_call(pm, ids[a:b], targets[a:b], no_rows(b - a), SEED, 3 + a)
                 for a, b in zip(bounds[:-1], bounds[1:])]
        got, rows, got_loads = MR.run_chain(snap, calls, window, [k] * len(calls))
        assert all(g.tobytes() == o.tobytes() for g, o in zip(got, outs))
        assert np.array_equal(got_loads, loads)
        if k:
            _, want_rows, _ = MR.run_chain(snap, plain, window, [k] * len(plain))
            assert all(np.array_equal(r, w) for r, w in zip(rows, want_rows))


def test_chain_split_invariance_with_every_kind_of_call():
    syn, models, pm = setup()
    snap = syn.packed
    rng = np.random.default_rng(11)
    R, window = 180, 9
    ids = WL.make_model_requests(R, snap.A, seed=12)
    first = B.Models(WL.model_records(models)).schedule_batch(B.Pool(syn.pod_records()), ids, SEED, 0)
    targets = first["target_idx"].copy()
    targets[::17] = 7                      # some targets no model has: LIG_NO_MODEL inside the windows
    rows = rng.integers(-1, snap.P, size=(R, 4)).astype(np.int16)
    reqs = WL.make_requests(40, snap.A, seed=13)
    whole = [(reqs[:20], SEED), MR.model_retry_call(pm, ids, targets, rows, SEED, 0), (reqs[20:], SEED)]
    want, want_rows, want_loads = MR.run_chain(snap, whole, window, [0, 3, 2])
    for trial in range(3):
        cuts = sorted(set([0, R] + rng.integers(1, R, size=4 + trial).tolist()))
        calls = [(reqs[:20], SEED)]
        calls += [MR.model_retry_call(pm, ids[a:b], targets[a:b], rows[a:b], SEED, a) for a, b in zip(cuts, cuts[1:])]
        calls += [(reqs[20:], SEED)]
        ks = [0] + [3] * (len(cuts) - 1) + [2]
        got, got_rows, got_loads = MR.run_chain(snap, calls, window, ks)
        assert np.concatenate(got[1:-1]).tobytes() == want[1].tobytes()
        assert np.array_equal(np.concatenate(got_rows[1:-1]), want_rows[1])
        assert got[0].tobytes() == want[0].tobytes() and got[-1].tobytes() == want[-1].tobytes()
        assert np.array_equal(got_rows[-1], want_rows[-1]) and np.array_equal(got_loads, want_loads)
    # a LIG_NO_MODEL request holds its place in the window and adds no load
    assert (want[1]["status"] == MR.LIG_NO_MODEL).any()
    ok = want[1]["status"] == N.LIG_OK
    assert int(want_loads.sum()) == int(ok.sum()) + int((want[0]["status"] == 0).sum()) + \
        int((want[2]["status"] == 0).sum())


def test_chain_before_any_window_closes_is_the_resident_retry():
    syn, models, pm = setup()
    snap = syn.packed
    ids = WL.make_model_requests(60, snap.A, seed=14)
    tg = B.Models(WL.model_records(models)).schedule_batch(B.Pool(syn.pod_records()), ids, SEED, 0)["target_idx"]
    rows = np.random.default_rng(15).integers(-1, snap.P, size=(60, 3)).astype(np.int16)
    got, got_rows, _ = MR.run_chain(snap, [MR.model_retry_call(pm, ids, tg, rows, SEED, 0)], 61, [4])
    want, want_rows = MR.retry_fallback_batch(snap, pm, ids, tg, rows, SEED, 4)
    assert got[0].tobytes() == want.tobytes() and np.array_equal(got_rows[0], want_rows)


def test_exports_and_header():
    hdr = open(os.path.join(ROOT, "include", "lig.h")).read()
    for name in NEW:
        assert name in N.EXPORTED_SYMBOLS
        assert re.search(r"\bint %s\(" % name, hdr), name


def lib_or_skip():
    try:
        return N.load()
    except ImportError:
        pytest.skip("liblig.so is not built")


def test_null_ctx_refusals():
    lib = lib_or_skip()
    ids = np.zeros(4, dtype=np.uint32)
    tg = np.zeros(4, dtype=np.uint8)
    rows = np.zeros((4, 2), dtype=np.int16)
    out = np.zeros(16, dtype=np.uint8)
    fb = np.zeros((4, 2), dtype=np.int16)
    p = [a.ctypes.data for a in (ids, tg, rows, out, fb)]
    loads = np.zeros(8, dtype=np.int32).ctypes.data
    calls = [
        lambda: lib.lig_schedule_models_batch_excluding(None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3]),
        lambda: lib.lig_schedule_models_batch_excluding_device(None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3], None),
        lambda: lib.lig_schedule_models_batch_excluding_fallbacks(None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3], 2,
                                                                  p[4]),
        lambda: lib.lig_schedule_models_batch_excluding_fallbacks_device(None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3],
                                                                         2, p[4], None),
        lambda: lib.lig_schedule_models_batch_feedback_chain_excluding(None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3], 4,
                                                                       loads),
        lambda: lib.lig_schedule_models_batch_feedback_chain_excluding_device(None, 1, 1, 0, p[0], p[1], 4, p[2], 2,
                                                                              p[3], 4, loads, None),
        lambda: lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks(None, 1, 1, 0, p[0], p[1], 4, p[2],
                                                                                 2, p[3], 2, p[4], 4, loads),
        lambda: lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device(
            None, 1, 1, 0, p[0], p[1], 4, p[2], 2, p[3], 2, p[4], 4, loads, None),
    ]
    for call in calls:
        assert call() == N.LIG_ERR_INVALID
    assert not out.any() and not fb.any()
