"""Session affinity under the load-feedback chain (include/lig.h,
lig_schedule_[models_]batch_feedback_chain_affinity) without a GPU: the sequential definition
(feedback_chain_affinity_ref.py) and its properties, a seeded herd against resident affinity, and the C
ABI's exports and argument refusals."""
import os
import re

import numpy as np
import pytest

import affinity_ref as AR
import feedback_chain_affinity_ref as FA
import feedback_chain_fallbacks_ref as FF
import feedback_chain_ref as FC
import models_feedback_chain_ref as MC
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models
from oracle import binding as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = N.LIG_MAX_FALLBACKS
THR = (0.8, 5, 50)


def pool(P=48, A=6, seed=1, q_max=8):
    p = WL.make_snapshot(P, A, seed=seed).packed
    rng = np.random.default_rng(seed)
    p.q[:] = rng.integers(0, q_max + 1, P)
    p.kv[:] = np.round(rng.random(P) * 0.7, 2)
    return p, rng.integers(0, 1 << 64, size=P, dtype=np.uint64)


def requests(A, R, seed, n_keys=None):
    rng = np.random.default_rng(seed)
    reqs = WL.make_requests(R, A, seed=seed)
    reqs["adapter_id"] = rng.choice([0, 1, 2, A, A + 7], R)
    if n_keys:                                   # sessions: a few keys repeated
        reqs["rand_key"] = AR.mix(rng.integers(1, n_keys + 1, R).astype(np.uint64))
    return reqs


def chain(p, pod_keys, calls, specs, W):
    return FA.schedule_chain_affinity(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap, pod_keys, calls, specs,
                                      W, THR)


def klass_at(p, q):
    tab = B.ClassTable(p.P, p.A, p.kv, np.asarray(q).astype(np.int32), p.n_active, p.max_active, p.bitmap, THR)
    return lambda crit, a: tab.klass(bool(crit), int(a))[2]


def affinity_calls(reqs, bounds, ks):
    return [(np.ascontiguousarray(reqs[a:b]), 0) for a, b in zip(bounds[:-1], bounds[1:])], \
        [("affinity", k) for k in ks]


def test_no_closed_window_is_resident_affinity():
    p, pk = pool()
    reqs = requests(p.A, 700, 2, n_keys=50)
    bounds = FC.random_split(len(reqs), np.random.default_rng(3), 40)
    calls, specs = affinity_calls(reqs, bounds, [K] * (len(bounds) - 1))
    outs, rows, loads = chain(p, pk, calls, specs, 1 << 20)
    got, got_rows = np.concatenate(outs), np.concatenate(rows)
    plain = B.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap, THR).schedule_batch(reqs, 0)
    klass = klass_at(p, p.q)
    crit, a = FF.class_of(reqs, p.A)
    for i in range(len(reqs)):
        assert got["status"][i] == plain["status"][i] and got["n_survivors"][i] == plain["n_survivors"][i]
        if plain["status"][i] != FA.LIG_OK:
            assert got["pod_idx"][i] == -1 and (got_rows[i] == -1).all()
            continue
        pick, row = AR.affinity_row(int(reqs["rand_key"][i]), klass(crit[i], a[i]), pk, K)
        assert got["pod_idx"][i] == pick and got_rows[i].tolist() == row
    ok = got["pod_idx"] >= 0
    assert np.array_equal(loads, np.bincount(got["pod_idx"][ok], minlength=p.P)) and ok.sum() > 300


@pytest.mark.parametrize("W", [1, 7, 64])
def test_split_invariance_loads_and_prefix_rows(W):
    p, pk = pool(seed=W)
    reqs = requests(p.A, 600, W, n_keys=40)
    want = None
    for split_seed in range(3):
        bounds = FC.random_split(len(reqs), np.random.default_rng(split_seed), W)
        calls, specs = affinity_calls(reqs, bounds, [K] * (len(bounds) - 1))
        outs, rows, loads = chain(p, pk, calls, specs, W)
        got = (np.concatenate(outs), np.concatenate(rows), loads)
        ok = got[0]["pod_idx"] >= 0
        assert np.array_equal(loads, np.bincount(got[0]["pod_idx"][ok], minlength=p.P))
        if want is None:
            want = got
            continue
        assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1])
        assert np.array_equal(got[2], want[2])
    for k in (0, 1, 3):
        bounds = [0, 250, 600]
        calls, specs = affinity_calls(reqs, bounds, [k, k])
        outs, rows, loads = chain(p, pk, calls, specs, W)
        assert np.concatenate(outs).tobytes() == want[0].tobytes() and np.array_equal(loads, want[2])
        assert np.array_equal(np.concatenate(rows), want[1][:, :k])
    # rows are distinct members of the load-adjusted list the pick came from
    r = want[1][want[0]["pod_idx"] >= 0]
    for row, pick in zip(r, want[0]["pod_idx"][want[0]["pod_idx"] >= 0]):
        x = [pick] + [v for v in row.tolist() if v >= 0]
        assert len(set(x)) == len(x)


def test_only_keys_whose_top_left_the_list_move():
    """Against resident affinity on E: where the chain's load-adjusted list of a request's class is a
    subset of E's list (loads only took pods out), the request keeps its resident pick while that pod is
    in the list, and otherwise takes the top of the list.  (When the smallest queue rises, pods can also
    come back into a list; then a key may move to a returning pod that outranks its own.)"""
    p, pk = pool(seed=11, q_max=0)
    W = 16
    reqs = requests(p.A, 2400, 12, n_keys=30)
    calls, specs = affinity_calls(reqs, [0, 2400], [0])
    got = chain(p, pk, calls, specs, W)[0][0]
    resident = chain(p, pk, calls, specs, 1 << 20)[0][0]
    crit, a = FF.class_of(reqs, p.A)
    at_e = klass_at(p, p.q)
    q = p.q.astype(np.int64).copy()
    moved = stayed = 0
    for w0 in range(0, len(reqs), W):
        klass = klass_at(p, q)
        for i in range(w0, min(w0 + W, len(reqs))):
            lst = klass(crit[i], a[i])
            if got["status"][i] != FA.LIG_OK or not set(lst) <= set(at_e(crit[i], a[i])):
                continue
            if resident["pod_idx"][i] in lst:
                stayed += 1
                assert got["pod_idx"][i] == resident["pod_idx"][i]
            else:
                moved += 1
                assert got["pod_idx"][i] == AR.ranking(int(reqs["rand_key"][i]), lst, pk)[0]
        seg = got["pod_idx"][w0:w0 + W]
        q = np.minimum(q + np.bincount(seg[seg >= 0], minlength=p.P), FC.INT32_MAX)
    assert moved >= 10 and stayed >= 10, (moved, stayed)


def test_model_resolve_is_affinity_resolve():
    p, pk = pool(P=40, A=8, seed=21)
    models = WL.make_models(p.A)
    pm = pack_models(models, p)
    mo = B.Models(WL.model_records(models))
    ids = np.random.default_rng(22).integers(0, len(models) + 3, 2000).astype(np.uint32)
    keys = np.random.default_rng(23).integers(0, 1 << 64, size=len(ids), dtype=np.uint64)
    call, _ = FA.affinity_model_call(mo, p.adapter_id, ids, keys)
    reqs, ok, target = AR.affinity_resolve(pm, ids, keys)
    assert np.array_equal(call["ok"] == 1, ok) and 0 < ok.sum() < len(ids)
    assert np.array_equal(call["target_idx"], target)
    assert np.array_equal(call["req"][ok], reqs[ok])
    # with no window closed, the model picks are affinity_ref's over the resolved descriptors
    outs, rows, _ = chain(p, pk, [(call, 0)], [("affinity", 2)], 1 << 20)
    d_outs, d_rows, _ = chain(p, pk, [(np.ascontiguousarray(reqs), 0)], [("affinity", 2)], 1 << 20)
    want = AR.as_mpicks(d_outs[0], ok, target, d_outs[0]["pod_idx"])
    assert outs[0].tobytes() == want.tobytes()
    assert np.array_equal(rows[0], np.where(ok[:, None], d_rows[0], -1))


def test_mixed_kinds_share_one_chain():
    """Plain and fallback calls in a chain with affinity calls get what their own references give them on
    the same sequence of tables; the loads are the bincount of every pick."""
    p, pk = pool(seed=31)
    models = WL.make_models(p.A)
    mo = B.Models(WL.model_records(models))
    W = 23
    reqs = requests(p.A, 900, 32, n_keys=60)
    ids = np.random.default_rng(33).integers(0, len(models) + 2, 900).astype(np.uint32)
    bounds = FC.random_split(900, np.random.default_rng(34), W)
    calls, specs = [], []
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        kind = ("plain", "fallbacks", "affinity")[i % 3]
        k = 0 if kind == "plain" else 1 + i % K
        if i % 2:
            calls.append(FA.affinity_model_call(mo, p.adapter_id, ids[a:b], reqs["rand_key"][a:b]) if kind == "affinity"
                         else MC.model_call(mo, p.adapter_id, ids[a:b], 40 + i, 1000 + a))
        else:
            calls.append((np.ascontiguousarray(reqs[a:b]), 0 if kind == "affinity" else 40 + i))
        specs.append((kind, k))
    outs, rows, loads = chain(p, pk, calls, specs, W)
    picks = np.concatenate([o["pod_idx"] for o in outs]).astype(np.int64)
    assert np.array_equal(loads, np.bincount(picks[picks >= 0], minlength=p.P))
    # every call replaced by a plain call: the same windows, so the non-affinity calls before the first
    # affinity call are the plain chain's and the fallback rows are FF's
    first_aff = next(i for i, s in enumerate(specs) if s[0] == "affinity")
    ff_outs, ff_rows, _ = FF.schedule_chain_fallbacks(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap,
                                                      calls[:first_aff], [s[1] for s in specs[:first_aff]], W, THR)
    for i in range(first_aff):
        assert outs[i].tobytes() == ff_outs[i].tobytes() and np.array_equal(rows[i], ff_rows[i])
    assert {s[0] for s in specs} == {"plain", "fallbacks", "affinity"}


def herd(W, R=3000, P=32, seed=5):
    """Zipf-distributed session keys over one scrape window on an idle pool: (max picks on one pod, pods
    used) for the chain with window W (W = None: resident affinity, no window ever closes)."""
    p = WL.make_snapshot(P, 2, seed=seed).packed
    p.q[:] = 0
    p.kv[:] = 0.1
    pk = np.random.default_rng(seed).integers(0, 1 << 64, size=P, dtype=np.uint64)
    rng = np.random.default_rng(seed + 1)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["adapter_id"] = 2                       # no pod lists it: the tree's "no LoRA affinity" branch
    reqs["flags"] = N.LIG_REQ_CRITICAL           # never shed as the queues grow
    reqs["rand_key"] = AR.mix(np.minimum(rng.zipf(1.3, R), 10 ** 6).astype(np.uint64))
    outs, _, loads = chain(p, pk, [(reqs, 0)], [("affinity", 0)], W or (1 << 30))
    assert (outs[0]["status"] == FA.LIG_OK).all()
    return int(loads.max()), int((loads > 0).sum())


def test_herd_is_spread_by_the_chain():
    resident = herd(None)
    figures = {"resident": resident}
    for W in (1, 8, 64):
        figures[f"W={W}"] = herd(W)
    print("herd (max picks on one pod, pods used):", figures)
    assert figures["W=1"][0] < resident[0] and figures["W=8"][0] < resident[0]
    assert figures["W=1"][1] >= resident[1]


NEW = ("lig_schedule_batch_feedback_chain_affinity", "lig_schedule_batch_feedback_chain_affinity_device",
       "lig_schedule_models_batch_feedback_chain_affinity", "lig_schedule_models_batch_feedback_chain_affinity_device")


def test_symbols_are_exported_and_declared():
    lib = N.load()
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    for name in NEW:
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\bint " + name + r"\(", header)
    from llm_instance_gateway_b200 import host as H
    assert hasattr(H.load(), "ligh_scheduler_new_feedback_affinity")


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    ids = np.zeros(4, dtype=np.uint32)
    keys = np.zeros(4, dtype=np.uint64)
    out, mout = np.zeros(4, dtype=PICK_DTYPE), np.zeros(4, dtype=MPICK_DTYPE)
    rows = np.zeros((4, 8), dtype=np.int16)
    loads = np.zeros(4, dtype=np.int32)
    p = lambda a: a.ctypes.data                                              # noqa: E731
    for nf in (0, 1, 8, 9, -1):
        assert lib.lig_schedule_batch_feedback_chain_affinity(None, 1, p(reqs), 4, p(out), nf, p(rows), 4,
                                                              p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_feedback_chain_affinity_device(None, 1, p(reqs), 4, p(out), nf, p(rows), 4,
                                                                     None, None) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_feedback_chain_affinity(None, 1, p(ids), p(keys), 4, p(mout), nf,
                                                                     p(rows), 4, p(loads)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_feedback_chain_affinity_device(None, 1, p(ids), p(keys), 4, p(mout), nf,
                                                                            p(rows), 4, None, None) == \
            N.LIG_ERR_INVALID
    assert b"feedback_chain_affinity" in lib.lig_last_error()
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0) and np.all(mout["pod_idx"] == 0) and np.all(loads == 0)
