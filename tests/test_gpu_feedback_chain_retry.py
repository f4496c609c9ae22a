"""Retries under the load-feedback chain (lig_schedule_batch_feedback_chain_excluding[_device]) on the GPU:
every result and the chain's loads bit for bit against the definition (feedback_chain_retry_ref.py).
Pools at the bit-word edges and one past staged columns; the built-in tree at default and extreme
thresholds and caller trees with DROP and "no pods left" leaves; a filter-tree change mid-chain; a herd;
windows closing inside and across retry calls; retry calls interleaved with plain, model-id and fallback
chain calls; every restart rule; refusals; buffer kinds and two streams; R = 0 with loads; one call at
R = 65536; the launches of retry segments; and the Python and C++ schedulers with feedback_retries."""
import ctypes as C
import random
import threading

import numpy as np
import pytest
import torch

import feedback_chain_ref as FC
import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import retry_ref as RR
from test_gpu_fallbacks import DROP_AND_NO_PODS, KEEP_ALL, splitmix_keys
from test_gpu_feedback_chain import Pinned
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
SEED = 0x7E7_C4A1_5EED
_ep = [9000]


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


def retry_dev(eng, ep, seed, reqs, rows, window, d_loads=0, stream=0):
    R, k = rows.shape
    d_in = dev(reqs) if R else torch.zeros(16, dtype=torch.uint8, device="cuda")
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda() if R else torch.zeros(1, dtype=torch.int16,
                                                                                     device="cuda")
    d_out = torch.full((max(R, 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    eng.schedule_batch_feedback_chain_excluding_device(ep, seed, d_in.data_ptr(), R, d_rows.data_ptr(), k,
                                                       d_out.data_ptr(), window, d_loads, stream)
    return d_in, d_rows, d_out


def run(eng, ep, calls, window, P, device=False):
    """The chain of `calls` (descriptor and retry calls) through the host or the device forms: (outs, loads)."""
    eng.feedback_chain_reset()
    outs, keep = [], []
    for x, seed in calls:
        retry = CR.is_retry(x)
        if not device:
            outs.append(eng.schedule_batch_feedback_chain_excluding(ep, seed, np.ascontiguousarray(x["req"]),
                                                                    np.ascontiguousarray(x["excluded"]), window)
                        if retry else eng.schedule_batch_feedback_chain(ep, seed, x, window))
            continue
        if retry:
            bufs = retry_dev(eng, ep, seed, np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"]),
                             window)
            d_out = bufs[2]
        else:
            d_in = dev(x) if len(x) else torch.zeros(16, dtype=torch.uint8, device="cuda")
            d_out = torch.full((max(len(x), 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
            eng.schedule_batch_feedback_chain_device(ep, seed, d_in.data_ptr(), len(x), d_out.data_ptr(), window)
            bufs = (d_in, d_out)
        keep.append(bufs)
        outs.append((d_out, len(x)))
    loads = np.zeros(max(P, 1), dtype=np.int32)
    if device:
        d_loads = torch.zeros(max(P, 1), dtype=torch.int32, device="cuda")
        retry_dev(eng, ep, 1, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16), window, d_loads.data_ptr())
        torch.cuda.synchronize()
        loads = d_loads.cpu().numpy()
        outs = [o.cpu().numpy()[: n * 8].view(PICK_DTYPE) for o, n in outs]
    else:
        eng.schedule_batch_feedback_chain_excluding(ep, 1, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16),
                                                    window, loads)
    return outs, loads[:P]


def check(eng, ep, snap, calls, window, thresholds=(0.8, 5, 50), nodes=None, device=True):
    want, want_loads = CR.chain_retry(snap, calls, window, thresholds=thresholds, **tree_kw(snap, nodes))
    for form in (False, True) if device else (False,):
        got, loads = run(eng, ep, calls, window, snap.P, device=form)
        assert [g.tobytes() for g in got] == [w.tobytes() for w in want], form
        assert np.array_equal(loads, want_loads), form
    return want, want_loads


def mixed(eng, ep, snap, rng, R=600, window=7, widths=(1, 9, 32), nodes=None, seed=SEED):
    """Plain and retry calls alternating over one sequence, at sizes around the window."""
    tpl = row_templates(eng, ep, snap, rng, nodes)
    reqs = class_reqs(snap.A, R, rng)
    bounds = FC.random_split(R, rng, window)
    calls = []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        if k % 3 == 1:
            calls.append((x, seed + k))
        else:
            calls.append(CR.retry_call(x, rows_for(tpl, b - a, widths[k % len(widths)], rng), seed + k))
    return calls


# ---- pools, thresholds and trees ------------------------------------------------------------------------
@pytest.mark.parametrize("P,A", [(1, 4), (31, 4), (32, 4), (33, 4), (64, 32), (512, 256), (4097, 64),
                                 (UNSTAGED_P, 16)])
def test_pools_built_in_tree(P, A, eng):
    rng = np.random.default_rng(P)
    snap = WL.make_snapshot(P, A, seed=P + 3).packed
    ep = upload(eng, snap)
    _, loads = check(eng, ep, snap, mixed(eng, ep, snap, rng, R=300 if P == UNSTAGED_P else 600), 7)
    assert loads.sum() > 0


@pytest.mark.parametrize("thresholds", [(0.8, 5, 50)] + EXTREME)
def test_thresholds(thresholds, eng):
    rng = np.random.default_rng(5)
    snap = WL.make_snapshot(200, 16, seed=13).packed
    eng.set_thresholds(*thresholds)
    try:
        ep = upload(eng, snap)
        check(eng, ep, snap, mixed(eng, ep, snap, rng, R=400, window=16), 16, thresholds)
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
        check(eng, ep, snap, mixed(eng, ep, snap, rng, R=200 if P == UNSTAGED_P else 400, window=9, nodes=nodes),
              9, nodes=nodes)
    finally:
        eng.set_filter_tree(None)


def test_filter_tree_and_thresholds_set_mid_chain_do_not_change_the_walk(eng):
    nodes = c4_tree().flatten()
    rng = np.random.default_rng(8)
    snap = WL.make_snapshot(300, 32, seed=9).packed
    ep = upload(eng, snap, nodes)
    calls = mixed(eng, ep, snap, rng, R=500, window=11, nodes=nodes)
    want, want_loads = CR.chain_retry(snap, calls, 11, **tree_kw(snap, nodes))
    eng.set_filter_tree(nodes)
    eng.feedback_chain_reset()
    got = []
    try:
        for k, (x, seed) in enumerate(calls):
            if k == 2:
                eng.set_filter_tree(NO_PODS_TREE)
                eng.set_thresholds(0.0, 0, 0)
            got.append(eng.schedule_batch_feedback_chain_excluding(ep, seed, np.ascontiguousarray(x["req"]),
                                                                   np.ascontiguousarray(x["excluded"]), 11)
                       if CR.is_retry(x) else eng.schedule_batch_feedback_chain(ep, seed, x, 11))
    finally:
        eng.set_filter_tree(None)
        eng.set_thresholds()
    assert [g.tobytes() for g in got] == [w.tobytes() for w in want]


# ---- load ------------------------------------------------------------------------------------------------
def test_herd_moves_retries_away_from_the_resident_retry(eng):
    P, A, R, W = 16, 4, 512, 16
    snap = WL.make_snapshot(P, A, seed=2).packed
    ep = upload(eng, snap)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["flags"] = 1
    reqs["rand_key"] = np.random.default_rng(1).integers(0, 1 << 64, R, dtype=np.uint64)
    rows = np.tile(np.array([0, 1, -1], np.int16), (R, 1))
    calls = [CR.retry_call(reqs[a:a + 100], rows[a:a + 100], SEED) for a in range(0, R, 100)]
    want, loads = check(eng, ep, snap, calls, W)
    resident = eng.schedule_batch_excluding(ep, SEED, reqs, rows)
    got = np.concatenate(want)
    assert (got["pod_idx"] != resident["pod_idx"]).any()
    assert got[:W].tobytes() == resident[:W].tobytes()          # the first window sees the epoch as it is
    ok = got["status"] == N.LIG_OK
    assert loads.sum() == ok.sum() and not np.isin(got["pod_idx"][ok], [0, 1]).any()


@pytest.mark.parametrize("window", [1, 5, 64, 1000])
def test_windows_inside_and_across_retry_calls(window, eng):
    rng = np.random.default_rng(window)
    snap = WL.make_snapshot(128, 16, seed=window).packed
    ep = upload(eng, snap)
    tpl = row_templates(eng, ep, snap, rng)
    reqs = class_reqs(snap.A, 900, rng)
    rows = rows_for(tpl, 900, 9, rng)
    bounds = FC.random_split(900, rng, window)
    calls = [CR.retry_call(reqs[a:b], rows[a:b], SEED) for a, b in zip(bounds[:-1], bounds[1:])]
    want, loads = check(eng, ep, snap, calls, window)
    whole, _ = CR.chain_retry(snap, [CR.retry_call(reqs, rows, SEED)], window)
    assert np.concatenate(want).tobytes() == whole[0].tobytes()


def test_interleaved_with_plain_model_and_fallback_calls(eng):
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
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        x = np.ascontiguousarray(reqs[a:b])
        kind = k % 4
        if kind == 1:
            ids = rng.integers(0, len(models) + 2, b - a).astype(np.uint32)
            calls.append(MC.model_call(mo, snap.adapter_id, ids, 50 + k, first) + (ids, first))
            first += b - a
        elif kind == 3:
            calls.append(CR.retry_call(x, rows_for(tpl, b - a, 5, rng), 50 + k))
        else:
            calls.append((x, 50 + k))
        ks.append(3 if kind == 2 else 0)
    ref = [c_[:2] for c_ in calls]
    want, want_rows, want_loads = CR.run_chain_retries(snap, ref, 40, ks)
    eng.feedback_chain_reset()
    for (call, k, w, wr) in zip(calls, ks, want, want_rows):
        x, seed = call[:2]
        if x.dtype == MC.MREQ_DTYPE:
            got = eng.schedule_models_batch_feedback_chain(ep, seed, call[2], 40, first_index=call[3])
        elif CR.is_retry(x):
            got = eng.schedule_batch_feedback_chain_excluding(ep, seed, np.ascontiguousarray(x["req"]),
                                                              np.ascontiguousarray(x["excluded"]), 40)
        elif k:
            got, rows = eng.schedule_batch_feedback_chain_fallbacks(ep, seed, x, k, 40)
            assert rows.tobytes() == wr.tobytes()
        else:
            got = eng.schedule_batch_feedback_chain(ep, seed, x, 40)
        assert got.tobytes() == w.tobytes()
    loads = np.zeros(snap.P, np.int32)
    eng.schedule_batch_feedback_chain(ep, 0, np.zeros(0, REQ_DTYPE), 40, loads)
    assert np.array_equal(loads, want_loads)


# ---- restarts, refusals, buffers -------------------------------------------------------------------------
@pytest.mark.parametrize("rule", ["epoch", "reupload", "window", "reset", "in_batch"])
def test_restart_rules(rule, eng):
    rng = np.random.default_rng(sum(map(ord, rule)))
    snap = WL.make_snapshot(96, 8, seed=4).packed
    ep = upload(eng, snap)
    calls = mixed(eng, ep, snap, rng, R=300, window=8)
    run(eng, ep, calls, 8, snap.P)                         # a chain with closed windows
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
    after = mixed(eng, ep2, snap, rng, R=200, window=W)
    want, want_loads = CR.chain_retry(snap, after, W)
    got = [eng.schedule_batch_feedback_chain_excluding(ep2, s, np.ascontiguousarray(x["req"]),
                                                       np.ascontiguousarray(x["excluded"]), W)
           if CR.is_retry(x) else eng.schedule_batch_feedback_chain(ep2, s, x, W) for x, s in after]
    loads = np.zeros(snap.P, np.int32)
    eng.schedule_batch_feedback_chain(ep2, 0, np.zeros(0, REQ_DTYPE), W, loads)
    assert [g.tobytes() for g in got] == [w.tobytes() for w in want] and np.array_equal(loads, want_loads)


def test_refused_calls_leave_the_chain_as_it_was(eng):
    rng = np.random.default_rng(77)
    snap = WL.make_snapshot(64, 8, seed=7).packed
    ep = upload(eng, snap)
    small = Engine(0, max_pods=64, max_adapters=8, max_batch=64)
    calls = mixed(eng, ep, snap, rng, R=120, window=6)
    want, want_loads = CR.chain_retry(snap, calls, 6)
    lib = N.load()
    reqs = class_reqs(snap.A, 20, rng)
    rows = np.full((20, 4), -1, np.int16)
    out = np.zeros(20, PICK_DTYPE)
    d_in, d_rows, d_out = dev(reqs), torch.zeros(64, dtype=torch.int16, device="cuda"), torch.zeros(
        20 * 8 + 8, dtype=torch.uint8, device="cuda")
    p = lambda a: a.ctypes.data                                              # noqa: E731
    try:
        small.upload_snapshot(1, snap)
        for eng_ in (eng, small):
            e_ep = ep if eng_ is eng else 1
            eng_.feedback_chain_reset()
            got = []
            for k, (x, seed) in enumerate(calls):
                if k == 2:                                      # refusals in the middle of the chain
                    ctx = eng_._ctx
                    for nx in (0, X + 1):
                        assert lib.lig_schedule_batch_feedback_chain_excluding(
                            ctx, e_ep, 1, p(reqs), 20, p(rows), nx, p(out), 6, None) == N.LIG_ERR_INVALID
                    assert lib.lig_schedule_batch_feedback_chain_excluding(
                        ctx, e_ep, 1, p(reqs), 20, None, 4, p(out), 6, None) == N.LIG_ERR_INVALID
                    if eng_ is small:                       # R > max_batch on the host form
                        big = class_reqs(snap.A, 65, rng)
                        assert lib.lig_schedule_batch_feedback_chain_excluding(
                            ctx, e_ep, 1, p(big), 65, p(np.full((65, 1), -1, np.int16)), 1,
                            p(np.zeros(65, PICK_DTYPE)), 6, None) == N.LIG_ERR_INVALID
                    for din, dr, do in ((d_in.data_ptr() + 8, d_rows.data_ptr(), d_out.data_ptr()),
                                        (d_in.data_ptr(), d_rows.data_ptr() + 1, d_out.data_ptr()),
                                        (d_in.data_ptr(), d_rows.data_ptr(), d_out.data_ptr() + 4)):
                        assert lib.lig_schedule_batch_feedback_chain_excluding_device(
                            ctx, e_ep, 1, din, 20, dr, 4, do, 6, None, None) == N.LIG_ERR_INVALID
                    assert lib.lig_schedule_batch_feedback_chain_excluding(
                        ctx, 999_999, 1, p(reqs), 20, p(rows), 4, p(out), 6, None) < 0       # missing epoch
                if CR.is_retry(x):
                    got.append(eng_.schedule_batch_feedback_chain_excluding(
                        e_ep, seed, np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"]), 6))
                else:
                    got.append(eng_.schedule_batch_feedback_chain(e_ep, seed, x, 6))
            loads = np.zeros(snap.P, np.int32)
            eng_.schedule_batch_feedback_chain(e_ep, 0, np.zeros(0, REQ_DTYPE), 6, loads)
            assert [g.tobytes() for g in got] == [w.tobytes() for w in want]
            assert np.array_equal(loads, want_loads)
        torch.cuda.synchronize()
        assert not out.view(np.uint8).any() and not d_out.any()
    finally:
        small.close()


def test_stale_epoch_is_refused(eng):
    rng = np.random.default_rng(12)
    snap = WL.make_snapshot(40, 4, seed=12).packed
    ep = upload(eng, snap)
    calls = mixed(eng, ep, snap, rng, R=60, window=5)
    eng.feedback_chain_reset()
    eng.schedule_batch_feedback_chain_excluding(ep, SEED, np.ascontiguousarray(calls[0][0]["req"]),
                                                np.ascontiguousarray(calls[0][0]["excluded"]), 5)
    upload(eng, snap)
    upload(eng, snap)                                      # two newer uploads evict ep
    with pytest.raises(N.LigError) as e:
        eng.schedule_batch_feedback_chain_excluding(ep, SEED, class_reqs(4, 3, rng), np.full((3, 1), -1, np.int16), 5)
    assert e.value.code == N.LIG_ERR_STALE_EPOCH


def test_buffer_kinds_and_two_streams(eng):
    rng = np.random.default_rng(19)
    snap = WL.make_snapshot(300, 32, seed=19).packed
    ep = upload(eng, snap)
    tpl = row_templates(eng, ep, snap, rng)
    R, W = 160, 24
    calls = [CR.retry_call(class_reqs(snap.A, R, rng), rows_for(tpl, R, 7, rng), SEED + k) for k in range(6)]
    want, want_loads = CR.chain_retry(snap, calls, W)
    lib = N.load()
    eng.feedback_chain_reset()
    for k, ((x, seed), w) in enumerate(zip(calls, want)):
        reqs, rows = np.ascontiguousarray(x["req"]), np.ascontiguousarray(x["excluded"])
        if k in (0, 1):                                   # page-locked in place; then pinned, misaligned rows
            pr, po, pw = Pinned(lib, R, REQ_DTYPE), Pinned(lib, R, PICK_DTYPE), Pinned(lib, R * 7 + 1, np.int16)
            pr.a[:] = reqs
            raw = np.ctypeslib.as_array((C.c_uint8 * ((R * 7 + 1) * 2)).from_address(pw.ptr))
            off = 0 if k == 0 else 1
            raw[off:off + R * 14] = rows.view(np.uint8).reshape(-1)
            eng.schedule_batch_feedback_chain_excluding_ptr(ep, seed, pr.ptr, R, pw.ptr + off, 7, po.ptr, W)
            got = po.a.copy()
            for b in (pr, po, pw):
                b.free()
        elif k == 2:                                      # pageable requests at an odd 8 bytes
            buf = np.zeros(R * 16 + 8, np.uint8)
            buf[8:] = reqs.view(np.uint8)
            out = np.zeros(R * 8 + 4, np.uint8)
            eng.schedule_batch_feedback_chain_excluding_ptr(ep, seed, buf.ctypes.data + 8, R, rows.ctypes.data, 7,
                                                            out.ctypes.data + 4, W)
            got = out[4:].view(PICK_DTYPE)
        elif k == 3:
            got = eng.schedule_batch_feedback_chain_excluding(ep, seed, reqs, rows, W)
        elif k == 4:                                      # device form on a stream of its own ...
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                bufs = retry_dev(eng, ep, seed, reqs, rows, W, stream=s.cuda_stream)
            s.synchronize()
            got = bufs[2].cpu().numpy()[: R * 8].view(PICK_DTYPE)
        else:                                             # ... then on the legacy default stream
            bufs = retry_dev(eng, ep, seed, reqs, rows, W)
            torch.cuda.synchronize()
            got = bufs[2].cpu().numpy()[: R * 8].view(PICK_DTYPE)
        assert got.tobytes() == w.tobytes(), k
    d_loads = torch.zeros(snap.P, dtype=torch.int32, device="cuda")
    retry_dev(eng, ep, 0, np.zeros(0, REQ_DTYPE), np.zeros((0, 1), np.int16), W, d_loads.data_ptr())
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
    want, want_loads = CR.chain_retry(snap, [CR.retry_call(reqs, rows, SEED)], 4096)
    eng.feedback_chain_reset()
    d_loads = torch.zeros(P, dtype=torch.int32, device="cuda")
    bufs = retry_dev(eng, ep, SEED, reqs, rows, 4096, d_loads.data_ptr())
    torch.cuda.synchronize()
    assert bufs[2].cpu().numpy().view(PICK_DTYPE).tobytes() == want[0].tobytes()
    assert np.array_equal(d_loads.cpu().numpy(), want_loads)


def test_retry_segments_launch_no_class_build(eng):
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
    retry = lambda r: eng.schedule_batch_feedback_chain_excluding(ep, 1, r, rows[:len(r)], W)     # noqa: E731
    eng.feedback_chain_reset()
    plain(reqs[:W])                                             # builds, picks, closes the window
    closing_plain = delta(lambda: plain(reqs[W:2 * W]))         # build + pick + close
    first_after_close = delta(lambda: plain(reqs[:1]))          # build + pick
    eng.feedback_chain_reset()
    plain(reqs[:W])
    assert delta(lambda: retry(reqs[W:2 * W])) == 2             # retry walk + close: no build
    assert delta(lambda: retry(reqs[:W])) == 2
    assert delta(lambda: plain(reqs[:1])) == first_after_close  # the stale tables are built once
    assert delta(lambda: retry(reqs[:1])) == 1
    assert closing_plain == first_after_close + 1


# ---- schedulers ------------------------------------------------------------------------------------------
class VersionedProvider(StaticProvider):
    """One provider version: the scheduler packs the slice once, so every call joins one chain."""

    def Version(self):  # noqa: N802
        return 1


def test_python_scheduler_feedback_retries():
    pods = pool_pods()
    W, seed = 4, 11
    sched = S.NewScheduler(VersionedProvider(pods), load_feedback_window=W, feedback_retries=True, max_pods=64,
                           max_adapters=8, max_batch=256, seed=seed)
    keys = random.Random(seed)
    keys.getrandbits(64)
    snap = pack_pod_metrics(pods)
    calls, got = [], []
    try:
        r_rng = np.random.default_rng(seed)
        for k in range(30):
            reqs = [S.LLMRequest(ResolvedTargetModel=m, Critical=bool(c))
                    for m, c in zip(r_rng.choice(["a", "b", "zz"], 3), r_rng.integers(0, 2, 3))]
            arr = np.zeros(len(reqs), REQ_DTYPE)
            for i, r in enumerate(reqs):
                arr[i] = (snap.adapter_id(r.ResolvedTargetModel), int(r.Critical), keys.getrandbits(64))
            if k % 2:
                tried = [[pm.Pod for pm in pods[j:j + int(r_rng.integers(0, 6))]] for j in range(len(reqs))]
                rows = [[p for p, pm in enumerate(pods) if pm.Pod in set(t)] for t in tried]
                width = max([1] + [len(r) for r in rows])
                ex = np.full((len(reqs), width), -1, np.int16)
                for i, r in enumerate(rows):
                    ex[i, :len(r)] = r
                got.append(sched.ScheduleBatchRetry(reqs, tried))
                calls.append(CR.retry_call(arr, ex, sched._seed))
            else:
                got.append(sched.ScheduleBatch(reqs))
                calls.append((arr, sched._seed))
        want, loads = CR.chain_retry(snap, calls, W)
        for g, w in zip(got, want):
            assert [p for p, _ in g] == [snap.pods[int(x)] if s == N.LIG_OK else None
                                         for x, s in zip(w["pod_idx"], w["status"])]
        mine = np.zeros(snap.P, np.int32)
        sched._engine.schedule_batch_feedback_chain(sched._epoch, sched._seed, np.zeros(0, REQ_DTYPE), W, mine)
        assert np.array_equal(mine, loads) and loads.sum() > 0
    finally:
        sched.close()


def test_cpp_runtime_feedback_retries():
    from llm_instance_gateway_b200 import host as H
    pods = pool_pods()
    W, seed = 4, 0x5151
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=W,
                         feedback_retries=True)
    snap = pack_pod_metrics(pods)
    keys = splitmix_keys(seed, 64)
    calls, got = [], []
    try:
        rng = np.random.default_rng(3)
        for k in range(40):
            model, crit = ["a", "b", "zz"][k % 3], bool(k % 2)
            arr = np.zeros(1, REQ_DTYPE)
            arr[0] = (snap.adapter_id(model), int(crit), int(keys[k]))
            if k % 3:
                tried = [pm.Pod for pm in pods[int(rng.integers(0, 30)):][:int(rng.integers(0, 9))]]
                code, pod, _ = hs.ScheduleRetry(model, crit, tried)
                row = [p for p, pm in enumerate(pods) if pm.Pod in set(tried)] or [-1]
                calls.append(CR.retry_call(arr, np.array([row], np.int16), seed))
                assert pod is None or pod not in tried
            else:
                code, pod, _ = hs.Schedule("m", model, crit)
                calls.append((arr, seed))
            got.append(pod)
        want, _ = CR.chain_retry(snap, calls, W)
        assert got == [snap.pods[int(w["pod_idx"][0])] if w["status"][0] == N.LIG_OK else None for w in want]
        st = hs.stats()
        assert st["retry_scheduled"] == sum(1 for k in range(40) if k % 3) and st["feedback_windows"] == 40 // W
    finally:
        hs.close()
        prov.close()


def test_cpp_runtime_host_refused_retry_adds_no_load():
    """A tried pod listed 33 times in the provider's slice matches more than LIG_MAX_EXCLUDED pods: the
    waiter is refused on the host, takes its rand_key, and loads no pod."""
    from llm_instance_gateway_b200 import host as H
    base = pool_pods(8)
    pods = base + [base[0]] * 33
    W, seed = 2, 0x99
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=64, max_adapters=8, max_batch=4096, seed=seed, load_feedback_window=W,
                         feedback_retries=True)
    snap = pack_pod_metrics(pods)
    keys = splitmix_keys(seed, 16)
    try:
        calls, got = [], []
        for k in range(9):
            arr = np.zeros(1, REQ_DTYPE)
            arr[0] = (snap.adapter_id("a"), 1, int(keys[k]))
            if k == 3:
                code, pod, err = hs.ScheduleRetry("a", True, [base[0].Pod])
                assert code == 3 and pod is None and str(X) in err
                continue
            code, pod, _ = hs.Schedule("m", "a", True)
            calls.append((arr, seed))
            got.append(pod)
        want, _ = CR.chain_retry(snap, calls, W)
        assert got == [snap.pods[int(w["pod_idx"][0])] if w["status"][0] == N.LIG_OK else None for w in want]
        assert hs.stats()["feedback_windows"] == 8 // W
    finally:
        hs.close()
        prov.close()


def test_cpp_runtime_concurrent_retries():
    from llm_instance_gateway_b200 import host as H
    P, W = 32, 8
    pods = mkpods(list(range(P)), [0.01 * i for i in range(P)], [4] * P, [["a"]] * P)
    prov = H.HostProvider(pods)
    hs = H.HostScheduler(prov, max_pods=P, max_adapters=8, max_batch=4096, flush_size=64, batch_window_us=200,
                         seed=3, filter=KEEP_ALL, load_feedback_window=W, feedback_retries=True)
    results, lock = [], threading.Lock()

    def caller(t):
        rng = random.Random(t)
        mine = []
        for _ in range(40):
            tried = [pm.Pod for pm in rng.sample(pods, rng.randint(0, 6))]
            code, pod, _ = hs.ScheduleRetry("a", False, tried)
            mine.append((code, pod, tried))
        with lock:
            results.extend(mine)
    try:
        threads = [threading.Thread(target=caller, args=(t,)) for t in range(8)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert len(results) == 320 and all(c == H.GRPC_OK and p not in t for c, p, t in results)
        st = hs.stats()
        assert st["retry_scheduled"] == 320 and st["feedback_windows"] == 320 // W
    finally:
        hs.close()
        prov.close()
