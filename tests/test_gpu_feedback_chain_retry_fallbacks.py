"""Retries with fallback rows under the load-feedback chain
(lig_schedule_batch_feedback_chain_excluding_fallbacks[_device]) on the GPU: every pick, every row and the
chain's loads bit for bit against the definition (feedback_chain_retry_fallbacks_ref.py).  Pools at the
bit-word edges, a C4-like pool and one past staged columns; the built-in tree at default and extreme
thresholds and caller trees; a filter-tree change mid-chain; windows closing inside and across calls;
calls interleaved with plain, model-id, fallback and chain retry calls; n_fallbacks 1, 3, 8 and rows of
width 1, 9, 32; every restart rule; refusals; a stale epoch; buffer kinds and two streams; one call at
R = 65536; the launches of its segments; and the Python and C++ schedulers with feedback_retries and
feedback_fallbacks."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

import feedback_chain_ref as FC
import feedback_chain_retry_fallbacks_ref as CRF
import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import retry_ref as RR
from test_gpu_fallbacks import DROP_AND_NO_PODS, splitmix_keys
from test_gpu_feedback_chain import Pinned
from test_gpu_feedback_chain_retry import VersionedProvider, retry_dev
from test_gpu_filter_batch import StaticProvider, dev
from test_gpu_filter_tree import c4_tree, mkpods
from test_gpu_retry import EXTREME, NO_PODS_TREE, UNSTAGED_P, class_reqs, pool_pods, row_templates, rows_for
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, pack_models, pack_pod_metrics
from oracle import binding as B

pytestmark = pytest.mark.gpu

X = N.LIG_MAX_EXCLUDED
K = N.LIG_MAX_FALLBACKS
SEED = 0x7E7_C4A1_F00D
_ep = [13000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=16384, max_adapters=1024, max_batch=1 << 16)
    yield e
    e.close()


def upload(eng, snap, nodes=None):
    ep = next_epoch()
    eng.set_filter_tree(nodes)
    try:
        eng.upload_snapshot(ep, snap)
    finally:
        eng.set_filter_tree(None)
    return ep


def tree_kw(snap, nodes):
    if nodes is None:
        return {}
    return dict(nodes=nodes, records=RR.records(snap), names=RR.adapter_names(snap) + [WL.UNKNOWN_MODEL])


def rf_dev(eng, ep, seed, reqs, ex, k, window, d_loads=0, stream=0):
    """The device form with torch buffers (picks and rows prefilled with junk)."""
    R, m = ex.shape
    d_in = dev(reqs) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_ex = torch.from_numpy(ex.reshape(-1).copy()).cuda() if R else torch.zeros(1, dtype=torch.int16, device="cuda")
    d_out = torch.full((max(R, 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    d_fb = torch.full((max(R * k, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
    eng.schedule_batch_feedback_chain_excluding_fallbacks_device(ep, seed, d_in.data_ptr(), R, d_ex.data_ptr(), m,
                                                                 d_out.data_ptr(), k, d_fb.data_ptr(), window,
                                                                 d_loads, stream)
    return d_in, d_ex, d_out, d_fb


def host_call(eng, ep, x, seed, k, window):
    """One chain call of any descriptor kind through the host forms: (picks, rows (R, k))."""
    if CR.is_retry(x):
        req, ex = np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"])
        if k:
            return eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, seed, req, ex, k, window)
        return eng.schedule_batch_feedback_chain_excluding(ep, seed, req, ex, window), np.zeros((len(x), 0), np.int16)
    if k:
        return eng.schedule_batch_feedback_chain_fallbacks(ep, seed, x, k, window)
    return eng.schedule_batch_feedback_chain(ep, seed, x, window), np.zeros((len(x), 0), np.int16)


def read_loads(eng, ep, window, P):
    loads = np.zeros(max(P, 1), np.int32)
    eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, 0, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16),
                                                          1, window, loads)
    return loads[:P]


def run(eng, ep, calls, ks, window, P, device=False):
    """The chain of `calls` through the host forms, or with its retry calls through the device forms:
    (outs, rows, loads)."""
    eng.feedback_chain_reset()
    outs, rows, keep = [], [], []
    for (x, seed), k in zip(calls, ks):
        if not (device and CR.is_retry(x)):
            o, r = host_call(eng, ep, x, seed, k, window)
            outs.append(o)
            rows.append(r)
            continue
        req, ex = np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"])
        if k:
            bufs = rf_dev(eng, ep, seed, req, ex, k, window)
        else:
            bufs = retry_dev(eng, ep, seed, req, ex, window)
        torch.cuda.synchronize()
        outs.append(bufs[2].cpu().numpy()[: len(x) * 8].view(PICK_DTYPE))
        rows.append(bufs[3].cpu().numpy()[: len(x) * k].reshape(len(x), k) if k else np.zeros((len(x), 0), np.int16))
        keep.append(bufs)
    if device:
        d_loads = torch.zeros(max(P, 1), dtype=torch.int32, device="cuda")
        rf_dev(eng, ep, 1, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16), 1, window, d_loads.data_ptr())
        torch.cuda.synchronize()
        return outs, rows, d_loads.cpu().numpy()[:P]
    return outs, rows, read_loads(eng, ep, window, P)


def check(eng, ep, snap, calls, ks, window, thresholds=(0.8, 5, 50), nodes=None, device=True):
    want, want_rows, want_loads = CRF.run_chain_retry_fallbacks(snap, calls, window, ks, thresholds=thresholds,
                                                                **tree_kw(snap, nodes))
    for form in (False, True) if device else (False,):
        got, rows, loads = run(eng, ep, calls, ks, window, snap.P, device=form)
        assert [g.tobytes() for g in got] == [w.tobytes() for w in want], form
        assert [r.tobytes() for r in rows] == [w.tobytes() for w in want_rows], form
        assert np.array_equal(loads, want_loads), form
    return want, want_rows, want_loads


def mixed(eng, ep, snap, rng, R=600, window=7, widths=(1, 9, 32), fbs=(1, 3, K), nodes=None, seed=SEED):
    """Retry-with-rows calls alternating with plain, chain retry and chain fallback calls: (calls, ks)."""
    tpl = row_templates(eng, ep, snap, rng, nodes)
    reqs = class_reqs(snap.A, R, rng)
    bounds = FC.random_split(R, rng, window)
    calls, ks = [], []
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        kind = i % 5
        if kind == 1:
            calls.append((x, seed + i))
            ks.append(0)
        elif kind == 2:
            calls.append((x, seed + i))
            ks.append(2)
        elif kind == 3:
            calls.append(CR.retry_call(x, rows_for(tpl, b - a, widths[i % len(widths)], rng), seed + i))
            ks.append(0)
        else:
            calls.append(CR.retry_call(x, rows_for(tpl, b - a, widths[i % len(widths)], rng), seed + i))
            ks.append(fbs[i % len(fbs)])
    return calls, ks


# ---- pools, thresholds and trees ------------------------------------------------------------------------
@pytest.mark.parametrize("P,A", [(1, 4), (31, 4), (33, 4), (64, 32), (512, 256), (4096, 1024), (UNSTAGED_P, 16)])
def test_pools_built_in_tree(P, A, eng):
    rng = np.random.default_rng(P)
    snap = WL.make_snapshot(P, A, seed=P + 3).packed
    ep = upload(eng, snap)
    calls, ks = mixed(eng, ep, snap, rng, R=150 if P == 4096 else 300 if P == UNSTAGED_P else 600)
    _, rows, loads = check(eng, ep, snap, calls, ks, 7)
    assert loads.sum() > 0
    if P >= 512:
        assert any((r >= 0).any() for r, (x, _), k in zip(rows, calls, ks) if k and CR.is_retry(x))


@pytest.mark.parametrize("thresholds", [(0.8, 5, 50)] + EXTREME)
def test_thresholds(thresholds, eng):
    rng = np.random.default_rng(5)
    snap = WL.make_snapshot(200, 16, seed=13).packed
    eng.set_thresholds(*thresholds)
    try:
        ep = upload(eng, snap)
        calls, ks = mixed(eng, ep, snap, rng, R=400, window=16)
        check(eng, ep, snap, calls, ks, 16, thresholds)
    finally:
        eng.set_thresholds()


@pytest.mark.parametrize("P,A", [(33, 4), (512, 256), (UNSTAGED_P, 16)])
@pytest.mark.parametrize("tree", ["drop_and_no_pods", "no_pods", "c4"])
def test_caller_trees(P, A, tree, eng):
    nodes = {"drop_and_no_pods": DROP_AND_NO_PODS, "no_pods": NO_PODS_TREE, "c4": c4_tree().flatten()}[tree]
    rng = np.random.default_rng(P + 1)
    snap = WL.make_snapshot(P, A, seed=P + 4).packed
    ep = upload(eng, snap, nodes)
    eng.set_filter_tree(nodes)                 # the chain takes the tree in force when it starts
    try:
        calls, ks = mixed(eng, ep, snap, rng, R=200 if P == UNSTAGED_P else 400, window=9, nodes=nodes)
        check(eng, ep, snap, calls, ks, 9, nodes=nodes)
    finally:
        eng.set_filter_tree(None)


def test_filter_tree_and_thresholds_set_mid_chain_do_not_change_the_walk(eng):
    nodes = c4_tree().flatten()
    rng = np.random.default_rng(8)
    snap = WL.make_snapshot(300, 32, seed=9).packed
    ep = upload(eng, snap, nodes)
    calls, ks = mixed(eng, ep, snap, rng, R=500, window=11, nodes=nodes)
    want, want_rows, want_loads = CRF.run_chain_retry_fallbacks(snap, calls, 11, ks, **tree_kw(snap, nodes))
    eng.set_filter_tree(nodes)
    eng.feedback_chain_reset()
    got = []
    try:
        for i, ((x, seed), k) in enumerate(zip(calls, ks)):
            if i == 2:
                eng.set_filter_tree(NO_PODS_TREE)
                eng.set_thresholds(0.0, 0, 0)
            got.append(host_call(eng, ep, x, seed, k, 11))
    finally:
        eng.set_filter_tree(None)
        eng.set_thresholds()
    assert [g.tobytes() for g, _ in got] == [w.tobytes() for w in want]
    assert [r.tobytes() for _, r in got] == [w.tobytes() for w in want_rows]
    assert np.array_equal(read_loads(eng, ep, 11, snap.P), want_loads)


# ---- windows and interleaving ------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [1, 5, 64, 1000])
def test_windows_inside_and_across_calls(window, eng):
    rng = np.random.default_rng(window)
    snap = WL.make_snapshot(128, 16, seed=window).packed
    ep = upload(eng, snap)
    tpl = row_templates(eng, ep, snap, rng)
    reqs = class_reqs(snap.A, 900, rng)
    rows = rows_for(tpl, 900, 9, rng)
    bounds = FC.random_split(900, rng, window)
    calls = [CR.retry_call(reqs[a:b], rows[a:b], SEED) for a, b in zip(bounds[:-1], bounds[1:])]
    want, want_rows, _ = check(eng, ep, snap, calls, [4] * len(calls), window)
    whole, whole_rows, _ = CRF.chain_retry_fallbacks(snap, [CR.retry_call(reqs, rows, SEED)], window, 4)
    assert np.concatenate(want).tobytes() == whole[0].tobytes()
    assert np.concatenate(want_rows).tobytes() == whole_rows[0].tobytes()


def test_interleaved_with_plain_model_fallback_and_retry_calls(eng):
    c = WL.CONFIGS["C2"]
    ws = WL.make_snapshot(c["P"], c["A"], seed=31)
    snap = ws.packed
    models = WL.make_models(c["A"])
    mo = B.Models(WL.model_records(models))
    ep = upload(eng, snap)
    eng.upload_models(ep, pack_models(models, snap))
    rng = np.random.default_rng(32)
    tpl = row_templates(eng, ep, snap, rng)
    reqs = WL.make_requests(2400, c["A"], seed=33)
    bounds = FC.random_split(len(reqs), rng, 40)
    calls, ks, first = [], [], 1 << 33
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        kind = i % 5
        if kind == 1:
            ids = rng.integers(0, len(models) + 2, b - a).astype(np.uint32)
            calls.append(MC.model_call(mo, snap.adapter_id, ids, 50 + i, first) + (ids, first))
            first += b - a
        elif kind in (3, 4):
            calls.append(CR.retry_call(x, rows_for(tpl, b - a, 5, rng), 50 + i))
        else:
            calls.append((x, 50 + i))
        ks.append(3 if kind == 2 else (1, 3, K)[i % 3] if kind == 4 else 0)
    want, want_rows, want_loads = CRF.run_chain_retry_fallbacks(snap, [c_[:2] for c_ in calls], 40, ks)
    eng.feedback_chain_reset()
    for call, k, w, wr in zip(calls, ks, want, want_rows):
        x, seed = call[:2]
        if x.dtype == MC.MREQ_DTYPE:
            got = eng.schedule_models_batch_feedback_chain(ep, seed, call[2], 40, first_index=call[3])
        else:
            got, rows = host_call(eng, ep, x, seed, k, 40)
            assert rows.tobytes() == wr.tobytes()
        assert got.tobytes() == w.tobytes()
    assert np.array_equal(read_loads(eng, ep, 40, snap.P), want_loads)


def test_rows_that_exclude_nothing_are_the_chain_fallback_call(eng):
    rng = np.random.default_rng(44)
    snap = WL.make_snapshot(256, 32, seed=44).packed
    ep = upload(eng, snap)
    reqs = class_reqs(snap.A, 500, rng)
    nothing = np.tile(np.array([-1, snap.P, 32767, -32768], np.int16), (500, 1))
    bounds = FC.random_split(500, rng, 13)
    for k in (1, 3, K):
        eng.feedback_chain_reset()
        a_out, a_rows = zip(*[host_call(eng, ep, np.ascontiguousarray(reqs[a:b]), SEED, k, 13)
                              for a, b in zip(bounds[:-1], bounds[1:])])
        a_loads = read_loads(eng, ep, 13, snap.P)
        eng.feedback_chain_reset()
        b_out, b_rows = zip(*[host_call(eng, ep, CR.retry_call(reqs[a:b], nothing[a:b], SEED)[0], SEED, k, 13)
                              for a, b in zip(bounds[:-1], bounds[1:])])
        assert np.concatenate(a_out).tobytes() == np.concatenate(b_out).tobytes()
        assert np.concatenate(a_rows).tobytes() == np.concatenate(b_rows).tobytes()
        assert np.array_equal(read_loads(eng, ep, 13, snap.P), a_loads)


def test_no_closed_window_is_the_resident_retry_with_rows(eng):
    rng = np.random.default_rng(45)
    snap = WL.make_snapshot(300, 32, seed=45).packed
    ep = upload(eng, snap)
    tpl = row_templates(eng, ep, snap, rng)
    reqs = class_reqs(snap.A, 400, rng)
    ex = rows_for(tpl, 400, 9, rng)
    eng.feedback_chain_reset()
    got, rows = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED, reqs, ex, K, 401)
    want, want_rows = eng.schedule_batch_excluding_fallbacks(ep, SEED, reqs, ex, K)
    assert got.tobytes() == want.tobytes() and rows.tobytes() == want_rows.tobytes()


# ---- restarts, refusals, buffers -------------------------------------------------------------------------
@pytest.mark.parametrize("rule", ["epoch", "reupload", "window", "reset", "in_batch"])
def test_restart_rules(rule, eng):
    rng = np.random.default_rng(sum(map(ord, rule)))
    snap = WL.make_snapshot(96, 8, seed=4).packed
    ep = upload(eng, snap)
    calls, ks = mixed(eng, ep, snap, rng, R=300, window=8)
    run(eng, ep, calls, ks, 8, snap.P)                     # a chain with closed windows
    W, ep2 = 8, ep
    if rule == "epoch":
        ep2 = upload(eng, snap)
    elif rule == "reupload":
        eng.upload_snapshot(ep, snap)
    elif rule == "window":
        W = 9
    elif rule == "reset":
        eng.feedback_chain_reset()
    else:
        d = dev(class_reqs(snap.A, 32, rng))
        o = torch.zeros(32 * 8, dtype=torch.uint8, device="cuda")
        eng.schedule_batch_feedback_device(ep, 3, d.data_ptr(), 32, o.data_ptr(), 4)
        torch.cuda.synchronize()
    after, aks = mixed(eng, ep2, snap, rng, R=200, window=W)
    want, want_rows, want_loads = CRF.run_chain_retry_fallbacks(snap, after, W, aks)
    got = [host_call(eng, ep2, x, s, k, W) for (x, s), k in zip(after, aks)]
    assert [g.tobytes() for g, _ in got] == [w.tobytes() for w in want]
    assert [r.tobytes() for _, r in got] == [w.tobytes() for w in want_rows]
    assert np.array_equal(read_loads(eng, ep2, W, snap.P), want_loads)


def test_refused_calls_leave_the_chain_as_it_was(eng):
    rng = np.random.default_rng(77)
    snap = WL.make_snapshot(64, 8, seed=7).packed
    ep = upload(eng, snap)
    small = Engine(0, max_pods=64, max_adapters=8, max_batch=64)
    calls, ks = mixed(eng, ep, snap, rng, R=120, window=6)
    want, want_rows, want_loads = CRF.run_chain_retry_fallbacks(snap, calls, 6, ks)
    lib = N.load()
    fn, fn_dev = (lib.lig_schedule_batch_feedback_chain_excluding_fallbacks,
                  lib.lig_schedule_batch_feedback_chain_excluding_fallbacks_device)
    reqs = class_reqs(snap.A, 20, rng)
    ex = np.full((20, 4), -1, np.int16)
    out = np.zeros(20, PICK_DTYPE)
    fb = np.zeros((20, K), np.int16)
    d_in, d_ex = dev(reqs), torch.zeros(128, dtype=torch.int16, device="cuda")
    d_out = torch.zeros(20 * 8 + 8, dtype=torch.uint8, device="cuda")
    d_fb = torch.zeros(20 * K + 1, dtype=torch.int16, device="cuda")
    p = lambda a: a.ctypes.data                                              # noqa: E731
    try:
        small.upload_snapshot(1, snap)
        for eng_ in (eng, small):
            e_ep = ep if eng_ is eng else 1
            eng_.feedback_chain_reset()
            got = []
            for i, ((x, seed), k) in enumerate(zip(calls, ks)):
                if i == 2:                                      # refusals in the middle of the chain
                    ctx = eng_._ctx
                    for nx, nf, win in ((0, 2, 6), (X + 1, 2, 6), (4, 0, 6), (4, K + 1, 6), (4, 2, 0)):
                        assert fn(ctx, e_ep, 1, p(reqs), 20, p(ex), nx, p(out), nf, p(fb), win,
                                  None) == N.LIG_ERR_INVALID
                        assert fn_dev(ctx, e_ep, 1, d_in.data_ptr(), 20, d_ex.data_ptr(), nx, d_out.data_ptr(), nf,
                                      d_fb.data_ptr(), win, None, None) == N.LIG_ERR_INVALID
                    assert fn(ctx, e_ep, 1, p(reqs), 20, None, 4, p(out), 2, p(fb), 6, None) == N.LIG_ERR_INVALID
                    assert fn(ctx, e_ep, 1, p(reqs), 20, p(ex), 4, p(out), 2, None, 6, None) == N.LIG_ERR_INVALID
                    assert fn(ctx, e_ep, 1, p(reqs), 20, p(ex), 4, None, 2, p(fb), 6, None) == N.LIG_ERR_INVALID
                    if eng_ is small:                       # R > max_batch on the host form
                        big = class_reqs(snap.A, 65, rng)
                        assert fn(ctx, e_ep, 1, p(big), 65, p(np.full((65, 1), -1, np.int16)), 1,
                                  p(np.zeros(65, PICK_DTYPE)), 2, p(np.zeros((65, 2), np.int16)), 6,
                                  None) == N.LIG_ERR_INVALID
                    for din, de, do, df in ((d_in.data_ptr() + 8, d_ex.data_ptr(), d_out.data_ptr(), d_fb.data_ptr()),
                                            (d_in.data_ptr(), d_ex.data_ptr() + 1, d_out.data_ptr(), d_fb.data_ptr()),
                                            (d_in.data_ptr(), d_ex.data_ptr(), d_out.data_ptr() + 4, d_fb.data_ptr()),
                                            (d_in.data_ptr(), d_ex.data_ptr(), d_out.data_ptr(), d_fb.data_ptr() + 1)):
                        assert fn_dev(ctx, e_ep, 1, din, 20, de, 4, do, 2, df, 6, None, None) == N.LIG_ERR_INVALID
                    assert fn(ctx, 999_999, 1, p(reqs), 20, p(ex), 4, p(out), 2, p(fb), 6, None) < 0  # missing epoch
                got.append(host_call(eng_, e_ep, x, seed, k, 6))
            assert [g.tobytes() for g, _ in got] == [w.tobytes() for w in want]
            assert [r.tobytes() for _, r in got] == [w.tobytes() for w in want_rows]
            assert np.array_equal(read_loads(eng_, e_ep, 6, snap.P), want_loads)
        torch.cuda.synchronize()
        assert not out.view(np.uint8).any() and not fb.any() and not d_out.any() and not d_fb.any()
    finally:
        small.close()


def test_stale_epoch_is_refused(eng):
    rng = np.random.default_rng(12)
    snap = WL.make_snapshot(40, 4, seed=12).packed
    ep = upload(eng, snap)
    eng.feedback_chain_reset()
    eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED, class_reqs(4, 5, rng), np.full((5, 2), -1, np.int16),
                                                          3, 5)
    upload(eng, snap)
    upload(eng, snap)                                      # two newer uploads evict ep
    with pytest.raises(N.LigError) as e:
        eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED, class_reqs(4, 3, rng),
                                                              np.full((3, 1), -1, np.int16), 3, 5)
    assert e.value.code == N.LIG_ERR_STALE_EPOCH


def test_buffer_kinds_and_two_streams(eng):
    rng = np.random.default_rng(19)
    snap = WL.make_snapshot(300, 32, seed=19).packed
    ep = upload(eng, snap)
    tpl = row_templates(eng, ep, snap, rng)
    R, W, M, F = 160, 24, 7, 3
    calls = [CR.retry_call(class_reqs(snap.A, R, rng), rows_for(tpl, R, M, rng), SEED + k) for k in range(7)]
    want, want_rows, want_loads = CRF.chain_retry_fallbacks(snap, calls, W, F)
    lib = N.load()
    eng.feedback_chain_reset()
    for k, ((x, seed), w, wr) in enumerate(zip(calls, want, want_rows)):
        reqs, ex = np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"])
        if k in (0, 1, 2):                     # page-locked in place; then misaligned excluded rows, fallback rows
            pr, po = Pinned(lib, R, REQ_DTYPE), Pinned(lib, R, PICK_DTYPE)
            pe, pf = Pinned(lib, R * M + 1, np.int16), Pinned(lib, R * F + 1, np.int16)
            pr.a[:] = reqs
            oe, of = (1 if k == 1 else 0), (1 if k == 2 else 0)
            raw = np.ctypeslib.as_array((C.c_uint8 * ((R * M + 1) * 2)).from_address(pe.ptr))
            raw[oe:oe + R * M * 2] = ex.view(np.uint8).reshape(-1)
            eng.schedule_batch_feedback_chain_excluding_fallbacks_ptr(ep, seed, pr.ptr, R, pe.ptr + oe, M, po.ptr, F,
                                                                      pf.ptr + of, W)
            got = po.a.copy()
            rows = np.ctypeslib.as_array((C.c_uint8 * ((R * F + 1) * 2)).from_address(pf.ptr))[
                of:of + R * F * 2].copy().view(np.int16).reshape(R, F)
            for b in (pr, po, pe, pf):
                b.free()
        elif k == 3:                           # pageable everything, requests at an odd 8 bytes
            buf = np.zeros(R * 16 + 8, np.uint8)
            buf[8:] = reqs.view(np.uint8)
            out = np.zeros(R * 8 + 4, np.uint8)
            rbuf = np.zeros(R * F * 2 + 1, np.uint8)
            eng.schedule_batch_feedback_chain_excluding_fallbacks_ptr(ep, seed, buf.ctypes.data + 8, R, ex.ctypes.data,
                                                                      M, out.ctypes.data + 4, F, rbuf.ctypes.data + 1,
                                                                      W)
            got = out[4:].view(PICK_DTYPE)
            rows = rbuf[1:].copy().view(np.int16).reshape(R, F)
        elif k == 4:
            got, rows = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, seed, reqs, ex, F, W)
        elif k == 5:                           # device form on a stream of its own ...
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                bufs = rf_dev(eng, ep, seed, reqs, ex, F, W, stream=s.cuda_stream)
            s.synchronize()
            got = bufs[2].cpu().numpy()[: R * 8].view(PICK_DTYPE)
            rows = bufs[3].cpu().numpy().reshape(R, F)
        else:                                  # ... then on the legacy default stream
            bufs = rf_dev(eng, ep, seed, reqs, ex, F, W)
            torch.cuda.synchronize()
            got = bufs[2].cpu().numpy()[: R * 8].view(PICK_DTYPE)
            rows = bufs[3].cpu().numpy().reshape(R, F)
        assert got.tobytes() == w.tobytes(), k
        assert rows.tobytes() == wr.tobytes(), k
    d_loads = torch.zeros(snap.P, dtype=torch.int32, device="cuda")
    rf_dev(eng, ep, 0, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16), 1, W, d_loads.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(d_loads.cpu().numpy(), want_loads)


def test_one_call_of_65536(eng):
    c = WL.CONFIGS["C4"] if "C4" in WL.CONFIGS else {"P": 1024, "A": 256}
    P, A = min(c["P"], 2048), min(c["A"], 1024)
    snap = WL.make_snapshot(P, A, seed=65).packed
    ep = upload(eng, snap)
    rng = np.random.default_rng(65)
    distinct = np.full((6, 9), -1, np.int16)
    for i in range(1, 6):
        distinct[i, :2 * i - 1] = rng.choice(P, 2 * i - 1, replace=False)
    R = 1 << 16
    reqs = class_reqs(A, R, rng)
    rows = distinct[rng.integers(0, 6, R)]
    want, want_rows, want_loads = CRF.chain_retry_fallbacks(snap, [CR.retry_call(reqs, rows, SEED)], 4096, K)
    eng.feedback_chain_reset()
    d_loads = torch.zeros(P, dtype=torch.int32, device="cuda")
    bufs = rf_dev(eng, ep, SEED, reqs, rows, K, 4096, d_loads.data_ptr())
    torch.cuda.synchronize()
    assert bufs[2].cpu().numpy().view(PICK_DTYPE).tobytes() == want[0].tobytes()
    assert bufs[3].cpu().numpy().tobytes() == want_rows[0].tobytes()
    assert np.array_equal(d_loads.cpu().numpy(), want_loads)


def test_segments_after_a_close_launch_no_class_build(eng):
    snap = WL.make_snapshot(256, 16, seed=3).packed
    ep = upload(eng, snap)
    rng = np.random.default_rng(3)
    W = 8
    reqs = class_reqs(snap.A, 4 * W, rng)
    rows = np.full((W, 2), -1, np.int16)

    def delta(fn):
        before = eng.kernel_launches
        fn()
        return eng.kernel_launches - before

    plain = lambda r: eng.schedule_batch_feedback_chain(ep, 1, r, W)                              # noqa: E731
    rf = lambda r: eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, 1, r, rows[:len(r)], 3, W)  # noqa: E731
    eng.feedback_chain_reset()
    plain(reqs[:W])                                             # builds, picks, closes the window
    first_after_close = delta(lambda: plain(reqs[:1]))          # build + pick
    eng.feedback_chain_reset()
    plain(reqs[:W])
    assert delta(lambda: rf(reqs[W:2 * W])) == 2                # walk + row + count, close: no build
    assert delta(lambda: rf(reqs[:W])) == 2
    assert delta(lambda: plain(reqs[:1])) == first_after_close  # the stale tables are built once
    assert delta(lambda: rf(reqs[:1])) == 1


# ---- schedulers ------------------------------------------------------------------------------------------
def tried_rows(pods, tried_lists):
    rows = [[p for p, pm in enumerate(pods) if pm.Pod in set(t)] for t in tried_lists]
    ex = np.full((len(rows), max([1] + [len(r) for r in rows])), -1, np.int16)
    for i, r in enumerate(rows):
        ex[i, :len(r)] = r
    return ex


def test_python_scheduler_both_opt_ins():
    pods = pool_pods()
    W, seed, n = 4, 11, 3
    sched = S.NewScheduler(VersionedProvider(pods), load_feedback_window=W, feedback_retries=True,
                           feedback_fallbacks=True, max_pods=64, max_adapters=8, max_batch=256, seed=seed)
    keys = random.Random(seed)
    keys.getrandbits(64)
    snap = pack_pod_metrics(pods)
    calls, ks, got = [], [], []
    try:
        r_rng = np.random.default_rng(seed)
        for i in range(30):
            reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=bool(c))
                    for m, c in zip(r_rng.choice(["a", "b", "zz"], 3), r_rng.integers(0, 2, 3))]
            arr = np.zeros(len(reqs), REQ_DTYPE)
            for j, r in enumerate(reqs):
                arr[j] = (snap.adapter_id(r.ResolvedTargetModel), int(r.Critical), keys.getrandbits(64))
            tried = [[pm.Pod for pm in pods[j:j + int(r_rng.integers(0, 6))]] for j in range(len(reqs))]
            if i % 3 == 0:
                got.append([([p] if p else [], e) for p, e in sched.ScheduleBatch(reqs)])
                calls.append((arr, sched._seed))
                ks.append(0)
            elif i % 3 == 1:
                got.append([([p] if p else [], e) for p, e in sched.ScheduleBatchRetry(reqs, tried)])
                calls.append(CR.retry_call(arr, tried_rows(pods, tried), sched._seed))
                ks.append(0)
            else:
                got.append(sched.ScheduleBatchRetryWithFallbacks(reqs, tried, n))
                calls.append(CR.retry_call(arr, tried_rows(pods, tried), sched._seed))
                ks.append(n)
        want, want_rows, loads = CRF.run_chain_retry_fallbacks(snap, calls, W, ks)
        for g, w, wr in zip(got, want, want_rows):
            expect = [[snap.pods[int(x)]] + [snap.pods[int(p)] for p in row if p >= 0] if s == N.LIG_OK else []
                      for x, s, row in zip(w["pod_idx"], w["status"], wr)]
            assert [pods_ for pods_, _ in g] == expect
            assert [e is None for _, e in g] == [s == N.LIG_OK for s in w["status"]]
        assert any(len(pods_) > 1 for g in got for pods_, _ in g)
        mine = np.zeros(snap.P, np.int32)
        sched._engine.schedule_batch_feedback_chain(sched._epoch, sched._seed, np.zeros(0, REQ_DTYPE), W, mine)
        assert np.array_equal(mine, loads) and loads.sum() > 0
    finally:
        sched.close()


def test_only_feedback_fallbacks_is_refused_in_both_schedulers():
    from llm_instance_gateway_b200 import host as H
    pods = pool_pods()
    sched = S.NewScheduler(StaticProvider(pods), load_feedback_window=4, feedback_fallbacks=True, max_pods=64,
                           max_adapters=8, seed=5)
    try:
        with pytest.raises(ValueError, match="load_feedback_window"):
            sched.ScheduleRetryWithFallbacks(S.LLMRequest(ResolvedTargetModel="a"), [], 2)
    finally:
        sched.close()
    prov = H.HostProvider(pods)
    try:
        hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=5, load_feedback_window=8,
                             feedback_fallbacks=True)
        try:
            code, names, err = hs.ScheduleRetryWithFallbacks("a", False, [], 2)
            assert code == 3 and names == [] and "load_feedback_window" in err
            assert hs.stats()["retry_scheduled"] == 0
        finally:
            hs.close()
    finally:
        prov.close()


def test_cpp_runtime_both_opt_ins():
    """Sequential callers of every kind: each retry with rows gets the definition's pick and row, the
    other calls' picks are unchanged, and the windows count every request once."""
    from llm_instance_gateway_b200 import host as H
    pods = pool_pods()
    W, seed = 4, 0x5151
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=W,
                         feedback_retries=True, feedback_fallbacks=True)
    snap = pack_pod_metrics(pods)
    keys = splitmix_keys(seed, 64)
    calls, ks, got = [], [], []
    try:
        rng = np.random.default_rng(3)
        for i in range(40):
            model, crit = ["a", "b", "zz"][i % 3], bool(i % 2)
            arr = np.zeros(1, REQ_DTYPE)
            arr[0] = (snap.adapter_id(model), int(crit), int(keys[i]))
            tried = [pm.Pod for pm in pods[int(rng.integers(0, 30)):][:int(rng.integers(0, 9))]]
            if i % 4 == 0:
                code, pod, _ = hs.Schedule("m", model, crit)
                calls.append((arr, seed))
                ks.append(0)
                got.append([pod.Name] if pod else [])
            elif i % 4 == 1:
                code, pod, _ = hs.ScheduleRetry(model, crit, tried)
                calls.append(CR.retry_call(arr, tried_rows(pods, [tried]), seed))
                ks.append(0)
                got.append([pod.Name] if pod else [])
            else:
                n = 1 + i % K
                code, names, _ = hs.ScheduleRetryWithFallbacks(model, crit, tried, n)
                calls.append(CR.retry_call(arr, tried_rows(pods, [tried]), seed))
                ks.append(n)
                got.append(names)
                assert not {p.Name for p in tried} & set(names)
        want, want_rows, _ = CRF.run_chain_retry_fallbacks(snap, calls, W, ks)
        expect = [([snap.pods[int(w["pod_idx"][0])].Name] + [snap.pods[int(p)].Name for p in wr[0] if p >= 0])
                  if w["status"][0] == N.LIG_OK else [] for w, wr in zip(want, want_rows)]
        assert got == expect
        assert any(len(g) > 1 for g in got)
        st = hs.stats()
        assert st["retry_scheduled"] == sum(1 for i in range(40) if i % 4) and st["feedback_windows"] == 40 // W
    finally:
        hs.close()
        prov.close()


def test_cpp_runtime_host_refused_waiter_adds_no_load():
    """A tried pod listed 33 times in the provider's slice matches more than LIG_MAX_EXCLUDED pods: the
    ScheduleRetryWithFallbacks waiter is refused on the host, takes its rand_key, and loads no pod."""
    from llm_instance_gateway_b200 import host as H
    base = pool_pods(8)
    pods = base + [base[0]] * 33
    W, seed = 2, 0x99
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=W,
                         feedback_retries=True, feedback_fallbacks=True)
    snap = pack_pod_metrics(pods)
    keys = splitmix_keys(seed, 16)
    try:
        calls, ks, got = [], [], []
        for i in range(9):
            arr = np.zeros(1, REQ_DTYPE)
            arr[0] = (snap.adapter_id("a"), 1, int(keys[i]))
            if i == 3:
                code, names, err = hs.ScheduleRetryWithFallbacks("a", True, [base[0].Pod], 4)
                assert code == 3 and names == [] and str(X) in err
                continue
            if i == 6:
                code, names, _ = hs.ScheduleRetryWithFallbacks("a", True, [base[1].Pod], 4)
                calls.append(CR.retry_call(arr, tried_rows(pods, [[base[1].Pod]]), seed))
                ks.append(4)
                got.append(names)
                continue
            code, pod, _ = hs.Schedule("m", "a", True)
            calls.append((arr, seed))
            ks.append(0)
            got.append([pod.Name] if pod else [])
        want, want_rows, _ = CRF.run_chain_retry_fallbacks(snap, calls, W, ks)
        assert got == [([snap.pods[int(w["pod_idx"][0])].Name] + [snap.pods[int(p)].Name for p in wr[0] if p >= 0])
                       if w["status"][0] == N.LIG_OK else [] for w, wr in zip(want, want_rows)]
        assert hs.stats()["feedback_windows"] == 8 // W
    finally:
        hs.close()
        prov.close()


def test_cpp_runtime_concurrent_retry_and_retry_with_fallbacks_callers():
    """Concurrent callers folded into shared flushes under the chain: every caller's pick is one request
    of the chain's sequence (one key each, in flush order), its pods are a prefix of that key's row, and
    the windows count every caller once whatever n it asked for."""
    from llm_instance_gateway_b200 import host as H
    P, W = 64, 8
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)], [4] * P, [["a"]] * P)
    tried = [pm.Pod for pm in pods[:3]]
    seed = 0x2468
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200,
                         seed=seed, load_feedback_window=W, feedback_retries=True, feedback_fallbacks=True)
    results, lock = [], threading.Lock()

    def caller(t):
        mine = []
        for j in range(40):
            n = (t + j) % 9           # 0: ScheduleRetry
            if n == 0:
                code, pod, _ = hs.ScheduleRetry("a", True, tried)
                mine.append((0, code, [pod.Name] if pod else []))
            else:
                code, names, _ = hs.ScheduleRetryWithFallbacks("a", True, tried, n)
                mine.append((n, code, names))
        with lock:
            results.extend(mine)

    try:
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(12)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        total = len(results)
        assert total == 480 and all(code == H.GRPC_OK for _, code, _ in results)
        st = hs.stats()
        assert st["retry_scheduled"] == total and st["feedback_windows"] == total // W
        assert st["batches"] < total                   # callers were folded into shared flushes
        snap = pack_pod_metrics(pods)
        reqs = np.zeros(total, dtype=REQ_DTYPE)
        reqs["rand_key"] = splitmix_keys(seed, total)
        reqs["adapter_id"] = snap.adapter_id("a")
        reqs["flags"] = 1
        ex = np.tile(np.arange(3, dtype=np.int16), (total, 1))
        (picks,), (fb,), _ = CRF.chain_retry_fallbacks(snap, [CR.retry_call(reqs, ex, seed)], W, K)
        assert (picks["status"] == N.LIG_OK).all()
        expect = [[f"pod-{picks['pod_idx'][j]}"] + [f"pod-{p}" for p in fb[j] if p >= 0] for j in range(total)]
        assert sorted(r[2][0] for r in results) == sorted(x[0] for x in expect)
        prefixes = {tuple(x[:m]) for x in expect for m in range(1, K + 2)}
        for n, _, names in results:
            assert len(names) <= n + 1 and tuple(names) in prefixes
            assert not {"pod-0", "pod-1", "pod-2"} & set(names)
        assert len({r[2][0] for r in results}) > 3                 # the load moved the picks around
    finally:
        hs.close()
        prov.close()
