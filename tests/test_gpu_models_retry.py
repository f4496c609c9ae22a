"""Model-id retries on the GPU (lig_schedule_models_batch[_feedback_chain]_excluding[_fallbacks]), byte for byte
against their definition (models_retry_ref.py): all eight entry points, the built-in tree and caller trees,
staged and unstaged pod columns, ejected epochs, models with 0, 1 and >= 2 targets, the first call's
targets reproducing the model call (resident and chain), chains mixing every kind of call with windows
closing inside model-retry calls, a model-table re-upload with new adapter ids between the first call and
its retry, page-locked, pageable and misaligned host buffers, and every refusal, which leaves the chain
as it was."""
import numpy as np
import pytest
import torch

import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import models_retry_ref as MR
from test_gpu_filter_batch import Pinned, dev
from test_gpu_retry import NO_PODS_TREE, UNSTAGED_P
from test_gpu_fallbacks import KEEP_ALL
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, pack_models
from oracle import binding as B

pytestmark = pytest.mark.gpu

K = N.LIG_MAX_FALLBACKS
SEED = 0x40DE_1_2E72
_ep = [12000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=UNSTAGED_P, max_adapters=256, max_batch=1 << 14)
    yield e
    e.close()


def upload(eng, P, A, seed, ejected=None):
    syn = WL.make_snapshot(P, A, seed=seed)
    models = WL.make_models(A)
    pm = pack_models(models, syn.packed)
    ep = next_epoch()
    eng.upload_snapshot(ep, syn.packed)
    if ejected is not None:
        base, ep = ep, next_epoch()
        eng.eject_pods(ep, base, np.asarray(ejected, dtype=np.int32))
    eng.upload_models(ep, pm)
    return syn, models, pm, ep


def requests(syn, models, R, rng, first_index=0):
    """Model ids of every kind, the targets the oracle's model call drew for them (0, 1 and >= 2 target
    models, ids past the table), some targets no model has, and rows of excluded pods."""
    ids = WL.make_model_requests(R, syn.packed.A, seed=int(rng.integers(1 << 30)))
    ids[rng.random(R) < 0.02] = 0xFFFFFFFF       # ids past the table
    first = B.Models(WL.model_records(models)).schedule_batch(B.Pool(syn.pod_records()), ids, SEED, first_index)
    tg = first["target_idx"].copy()
    bad = rng.random(R) < 0.05
    tg[bad] = rng.choice([0, 1, 3, 254, 255], size=int(bad.sum()))
    width = int(rng.integers(1, N.LIG_MAX_EXCLUDED + 1))
    rows = np.full((R, width), -1, dtype=np.int16)
    P = syn.packed.P
    for i in range(R):
        k = int(rng.integers(0, width + 1))
        rows[i, :k] = rng.integers(-1, P + 2, size=k)
    return ids, tg, rows


def device_models(eng, ep, seed, fi, ids, tg, rows, k=0, window=0, stream=0):
    R, w = rows.shape
    d_ids, d_tg = dev(ids), torch.from_numpy(tg.copy()).cuda()
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda()
    d_out = torch.full((max(R, 1),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    d_fb = torch.full((max(R * k, 1),), 0x5A5A, dtype=torch.int16, device="cuda")
    if window and k:
        eng.schedule_models_batch_feedback_chain_excluding_fallbacks_device(
            ep, seed, fi, d_ids.data_ptr(), d_tg.data_ptr(), R, d_rows.data_ptr(), w, d_out.data_ptr(), k,
            d_fb.data_ptr(), window, 0, stream)
    elif window:
        eng.schedule_models_batch_feedback_chain_excluding_device(ep, seed, fi, d_ids.data_ptr(), d_tg.data_ptr(), R,
                                                                  d_rows.data_ptr(), w, d_out.data_ptr(), window, 0,
                                                                  stream)
    elif k:
        eng.schedule_models_batch_excluding_fallbacks_device(ep, seed, fi, d_ids.data_ptr(), d_tg.data_ptr(), R,
                                                             d_rows.data_ptr(), w, d_out.data_ptr(), k,
                                                             d_fb.data_ptr(), stream)
    else:
        eng.schedule_models_batch_excluding_device(ep, seed, fi, d_ids.data_ptr(), d_tg.data_ptr(), R,
                                                   d_rows.data_ptr(), w, d_out.data_ptr(), stream)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()[:R].view(MPICK_DTYPE)
    return (out, d_fb.cpu().numpy()[: R * k].reshape(R, k)) if k else out


def check_resident(eng, ep, syn, pm, ids, tg, rows, fi, thresholds=(0.8, 5, 50), nodes=None, ejected=None):
    want, want_rows = MR.retry_fallback_batch(syn.packed, pm, ids, tg, rows, SEED, K, fi, thresholds, nodes, ejected)
    got = eng.schedule_models_batch_excluding(ep, SEED, ids, tg, rows, fi)
    assert got.tobytes() == want.tobytes()
    assert device_models(eng, ep, SEED, fi, ids, tg, rows).tobytes() == want.tobytes()
    for k in (1, 3, K):
        g, r = eng.schedule_models_batch_excluding_fallbacks(ep, SEED, ids, tg, rows, k, fi)
        assert g.tobytes() == want.tobytes() and np.array_equal(r, want_rows[:, :k]), k
        g, r = device_models(eng, ep, SEED, fi, ids, tg, rows, k)
        assert g.tobytes() == want.tobytes() and np.array_equal(r, want_rows[:, :k]), k
    return want


# ---- resident forms ------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,A", [(1, 4), (33, 8), (512, 64), (4097, 32), (UNSTAGED_P, 16)])
def test_resident_built_in_tree(P, A, eng):
    rng = np.random.default_rng(P)
    syn, models, pm, ep = upload(eng, P, A, seed=P + 1)
    R = 400 if P < UNSTAGED_P else 96
    fi = int(rng.integers(0, 1 << 64, dtype=np.uint64))
    ids, tg, rows = requests(syn, models, R, rng, fi)
    want = check_resident(eng, ep, syn, pm, ids, tg, rows, fi)
    assert (want["status"] == MR.LIG_NO_MODEL).any() and (want["status"] == N.LIG_OK).any()


@pytest.mark.parametrize("P", [33, 700, UNSTAGED_P])
@pytest.mark.parametrize("tree", ["default_filter", "keep_all", "no_pods"])
def test_resident_caller_trees(P, tree, eng):
    nodes = {"default_filter": S.DEFAULT_FILTER.flatten(), "keep_all": KEEP_ALL, "no_pods": NO_PODS_TREE}[tree]
    rng = np.random.default_rng(P + 5)
    eng.set_filter_tree(nodes)
    try:
        syn, models, pm, ep = upload(eng, P, 8, seed=P + 2)
    finally:
        eng.set_filter_tree(None)
    ids, tg, rows = requests(syn, models, 200 if P < UNSTAGED_P else 64, rng)
    check_resident(eng, ep, syn, pm, ids, tg, rows, 0, nodes=nodes)


@pytest.mark.parametrize("P", [40, 3000])
def test_resident_ejected_epoch(P, eng):
    rng = np.random.default_rng(P + 9)
    ejected = sorted(set(rng.integers(0, P, size=P // 4).tolist()))
    syn, models, pm, ep = upload(eng, P, 16, seed=P + 3, ejected=ejected)
    ids, tg, rows = requests(syn, models, 300, rng)
    check_resident(eng, ep, syn, pm, ids, tg, rows, 77, ejected=ejected)


def test_first_calls_targets_reproduce_the_model_calls(eng):
    rng = np.random.default_rng(21)
    syn, models, pm, ep = upload(eng, 300, 32, seed=22)
    ids = WL.make_model_requests(2000, 32, seed=23)
    none = np.full((len(ids), 3), -1, dtype=np.int16)
    for fi in (0, int(rng.integers(0, 1 << 63)), (1 << 64) - 700):
        first = eng.schedule_models_batch(ep, SEED, ids, fi)
        assert (first["target_idx"] >= 2).any() and (first["target_idx"] == 255).any()
        got = eng.schedule_models_batch_excluding(ep, SEED, ids, np.ascontiguousarray(first["target_idx"]), none, fi)
        assert got.tobytes() == first.tobytes()
        plain, plain_rows = eng.schedule_models_batch_fallbacks(ep, SEED, ids, 5, fi)
        g, r = eng.schedule_models_batch_excluding_fallbacks(ep, SEED, ids, np.ascontiguousarray(plain["target_idx"]),
                                                             none, 5, fi)
        assert g.tobytes() == plain.tobytes() and np.array_equal(r, plain_rows)


def test_retry_after_a_refresh_with_new_adapter_ids(eng):
    """The first call on one epoch, a refresh that adds adapters (every adapter id moves), the retry of the
    drawn targets on the new epoch: it resolves the same target names against the new table."""
    rng = np.random.default_rng(31)
    syn, models, pm, ep = upload(eng, 200, 12, seed=32)
    ids = WL.make_model_requests(500, 12, seed=33)
    first = eng.schedule_models_batch(ep, SEED, ids, 0)
    tg = np.ascontiguousarray(first["target_idx"])
    syn2 = WL.make_snapshot(200, 20, seed=34)
    ren = list(reversed(range(20)))        # the same names, other dense ids
    names = {WL.adapter_name(a): ren[a] for a in range(20)}
    snap2 = syn2.packed
    bitmap = np.zeros_like(snap2.bitmap)
    for a in range(20):
        bitmap[ren[a]] = snap2.bitmap[a]
    from llm_instance_gateway_b200.packer import pack_columns
    snap2 = pack_columns(snap2.kv, snap2.q.astype(np.int64), snap2.n_active.astype(np.int64),
                         snap2.max_active.astype(np.int64), bitmap, names, snap2.pods)
    pm2 = pack_models(models, snap2)
    ep2 = next_epoch()
    eng.upload_snapshot(ep2, snap2)
    eng.upload_models(ep2, pm2)
    rows = np.stack([np.where(first["pod_idx"] >= 0, first["pod_idx"], -1).astype(np.int16),
                     rng.integers(-1, 200, size=len(ids)).astype(np.int16)], axis=1)
    want, want_rows = MR.retry_fallback_batch(snap2, pm2, ids, tg, rows, SEED, 4, 0)
    assert eng.schedule_models_batch_excluding(ep2, SEED, ids, tg, rows, 0).tobytes() == want.tobytes()
    g, r = eng.schedule_models_batch_excluding_fallbacks(ep2, SEED, ids, tg, rows, 4, 0)
    assert g.tobytes() == want.tobytes() and np.array_equal(r, want_rows)
    # the retry read the new table: a resolved request's adapter is the new id of its target's name
    res = MR.fixed_resolve(pm2, ids, tg, 0)
    m = int(np.flatnonzero((res["ok"] == 1) & (ids < 12))[0])
    assert res["req"]["adapter_id"][m] == ren[int(ids[m])]


def test_model_table_reupload_between_calls(eng):
    rng = np.random.default_rng(41)
    syn, models, pm, ep = upload(eng, 150, 10, seed=42)
    ids, tg, rows = requests(syn, models, 300, rng)
    check_resident(eng, ep, syn, pm, ids, tg, rows, 5)
    flipped = WL.make_models(10)[::-1]     # other ids, targets and criticality for the same names
    pm2 = pack_models(flipped, syn.packed)
    eng.upload_models(ep, pm2)
    want = MR.retry_batch(syn.packed, pm2, ids, tg, rows, SEED, 5)
    assert eng.schedule_models_batch_excluding(ep, SEED, ids, tg, rows, 5).tobytes() == want.tobytes()


def test_host_buffer_kinds(eng):
    rng = np.random.default_rng(51)
    syn, models, pm, ep = upload(eng, 120, 8, seed=52)
    ids, tg, rows = requests(syn, models, 257, rng)
    R, w = rows.shape
    want, want_rows = MR.retry_fallback_batch(syn.packed, pm, ids, tg, rows, SEED, 3, 9)
    # pinned, aligned: used in place
    bufs = [Pinned(R, np.uint32), Pinned(R, np.uint8), Pinned(R * w, np.int16), Pinned(R, MPICK_DTYPE),
            Pinned(R * 3, np.int16)]
    try:
        bufs[0].a[:] = ids
        bufs[1].a[:] = tg
        bufs[2].a[:] = rows.reshape(-1)
        eng.schedule_models_batch_excluding_fallbacks_ptr(ep, SEED, 9, bufs[0].ptr, bufs[1].ptr, R, bufs[2].ptr, w,
                                                          bufs[3].ptr, 3, bufs[4].ptr)
        assert bufs[3].a.tobytes() == want.tobytes() and np.array_equal(bufs[4].a.reshape(R, 3), want_rows)
    finally:
        for b in bufs:
            b.free()
    # pageable and misaligned by one element's worth of bytes: staged
    raw = [np.zeros(R * 4 + 8, np.uint8), np.zeros(R + 8, np.uint8), np.zeros(R * w * 2 + 8, np.uint8),
           np.zeros(R * 4 + 8, np.uint8), np.zeros(R * 6 + 8, np.uint8)]
    for off in (0, 1, 2):
        views = [r[off:] for r in raw]
        views[0][: R * 4] = ids.view(np.uint8)
        views[1][:R] = tg
        views[2][: R * w * 2] = rows.reshape(-1).view(np.uint8)
        ptrs = [v.ctypes.data for v in views]
        eng.schedule_models_batch_excluding_fallbacks_ptr(ep, SEED, 9, ptrs[0], ptrs[1], R, ptrs[2], w, ptrs[3], 3,
                                                          ptrs[4])
        assert views[3][: R * 4].tobytes() == want.tobytes()
        assert np.array_equal(views[4][: R * 6].copy().view(np.int16).reshape(R, 3), want_rows)
        eng.schedule_models_batch_excluding_ptr(ep, SEED, 9, ptrs[0], ptrs[1], R, ptrs[2], w, ptrs[3])
        assert views[3][: R * 4].tobytes() == want.tobytes()


# ---- chain forms ---------------------------------------------------------------------------------------
def run_calls(eng, ep, calls, window, ks, raw, device=False):
    """Make each call on the GPU chain; raw[i] = the host arrays behind calls[i] (None for descriptor calls)."""
    outs, rows = [], []
    for (c, seed), k, r in zip(calls, ks, raw):
        kind = r[0]
        if kind == "model_retry":
            _, ids, tg, ex, fi = r
            if device:
                got = device_models(eng, ep, seed, fi, ids, tg, ex, k, window)
                o, rw = got if k else (got, np.zeros((len(ids), 0), np.int16))
            elif k:
                o, rw = eng.schedule_models_batch_feedback_chain_excluding_fallbacks(ep, seed, ids, tg, ex, k, window, fi)
            else:
                o = eng.schedule_models_batch_feedback_chain_excluding(ep, seed, ids, tg, ex, window, fi)
                rw = np.zeros((len(ids), 0), np.int16)
        elif kind == "retry":
            _, reqs, ex = r
            if k:
                o, rw = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, seed, reqs, ex, k, window)
            else:
                o = eng.schedule_batch_feedback_chain_excluding(ep, seed, reqs, ex, window)
                rw = np.zeros((len(reqs), 0), np.int16)
        elif kind == "model":
            _, ids, fi = r
            o = eng.schedule_models_batch_feedback_chain(ep, seed, ids, window, fi)
            rw = np.zeros((len(ids), 0), np.int16)
        else:
            o = eng.schedule_batch_feedback_chain(ep, seed, c, window)
            rw = np.zeros((len(c), 0), np.int16)
        outs.append(o)
        rows.append(rw)
    return outs, rows


def chain_loads(eng, ep, window, P):
    loads = np.zeros(P, dtype=np.int32)
    eng.schedule_batch_feedback_chain(ep, SEED, np.zeros(0, dtype=B.REQ_DTYPE), window, loads=loads)
    return loads


@pytest.mark.parametrize("nodes_kind", ["built_in", "caller_tree"])
@pytest.mark.parametrize("device", [False, True])
def test_chain_mixes_every_kind_of_call(nodes_kind, device, eng):
    nodes = S.DEFAULT_FILTER.flatten() if nodes_kind == "caller_tree" else None
    rng = np.random.default_rng(61 + device)
    if nodes is not None:
        eng.set_filter_tree(nodes)
    try:
        syn, models, pm, ep = upload(eng, 90, 12, seed=62)
        snap = syn.packed
        window = 13
        calls, raw, ks = [], [], []
        fi = 0
        for j in range(8):
            R = int(rng.integers(1, 40))
            kind = ["model_retry", "retry", "model", "plain"][j % 4] if j < 6 else "model_retry"
            k = int(rng.integers(0, 4)) if kind in ("model_retry", "retry") else 0
            if kind == "model_retry":
                ids, tg, ex = requests(syn, models, R, rng, fi)
                calls.append(MR.model_retry_call(pm, ids, tg, ex, SEED + j, fi))
                raw.append(("model_retry", ids, tg, ex, fi))
                fi += R
            elif kind == "retry":
                reqs = WL.make_requests(R, snap.A, seed=j)
                ex = rng.integers(-1, snap.P, size=(R, 3)).astype(np.int16)
                calls.append(CR.retry_call(reqs, ex, SEED + j))
                raw.append(("retry", reqs, ex))
            elif kind == "model":
                ids = WL.make_model_requests(R, snap.A, seed=j)
                calls.append(MC.model_call(B.Models(WL.model_records(models)), snap.adapter_id, ids, SEED + j, fi))
                raw.append(("model", ids, fi))
                fi += R
            else:
                reqs = WL.make_requests(R, snap.A, seed=100 + j)
                calls.append((reqs, SEED + j))
                raw.append(("plain",))
            ks.append(k)
        want, want_rows, want_loads = MR.run_chain_snapshot(snap, calls, window, ks, nodes=nodes)
        eng.feedback_chain_reset()
        # device=True: model retries take their device forms, the other calls their host forms
        got, got_rows = run_calls(eng, ep, calls, window, ks, raw, device)
        loads = chain_loads(eng, ep, window, snap.P)
    finally:
        if nodes is not None:
            eng.set_filter_tree(None)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.tobytes() == w.tobytes(), (i, raw[i][0])
        if ks[i]:
            assert np.array_equal(got_rows[i], want_rows[i]), i
    assert np.array_equal(loads, want_loads)


def test_chain_first_targets_reproduce_the_model_chain(eng):
    syn, models, pm, ep = upload(eng, 160, 16, seed=71)
    ids = WL.make_model_requests(700, 16, seed=72)
    window, bounds = 37, [0, 100, 101, 450, 700]
    none = np.full((700, 2), -1, dtype=np.int16)
    eng.feedback_chain_reset()
    plain = [eng.schedule_models_batch_feedback_chain(ep, SEED, np.ascontiguousarray(ids[a:b]), window, a)
             for a, b in zip(bounds[:-1], bounds[1:])]
    loads = chain_loads(eng, ep, window, 160)
    tg = np.concatenate([p["target_idx"] for p in plain])
    for k in (0, 4):
        eng.feedback_chain_reset()
        got = []
        for a, b in zip(bounds[:-1], bounds[1:]):
            args = (ep, SEED, np.ascontiguousarray(ids[a:b]), np.ascontiguousarray(tg[a:b]), none[a:b])
            if k:
                got.append(eng.schedule_models_batch_feedback_chain_excluding_fallbacks(*args, k, window, a)[0])
            else:
                got.append(eng.schedule_models_batch_feedback_chain_excluding(*args, window, a))
        assert all(g.tobytes() == p.tobytes() for g, p in zip(got, plain)), k
        assert np.array_equal(chain_loads(eng, ep, window, 160), loads), k


def test_chain_on_an_ejected_epoch(eng):
    rng = np.random.default_rng(81)
    ejected = [0, 5, 6, 40, 41, 42, 99]
    syn, models, pm, ep = upload(eng, 100, 8, seed=82, ejected=ejected)
    calls, raw = [], []
    fi = 0
    for j in range(4):
        ids, tg, ex = requests(syn, models, int(rng.integers(5, 60)), rng, fi)
        calls.append(MR.model_retry_call(pm, ids, tg, ex, SEED, fi))
        raw.append(("model_retry", ids, tg, ex, fi))
        fi += len(ids)
    ks = [0, 2, 0, 5]
    want, want_rows, want_loads = MR.run_chain_snapshot(syn.packed, calls, 11, ks, ejected=ejected)
    eng.feedback_chain_reset()
    got, got_rows = run_calls(eng, ep, calls, 11, ks, raw)
    assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
    assert all(np.array_equal(g, w) for g, w, k in zip(got_rows, want_rows, ks) if k)
    assert np.array_equal(chain_loads(eng, ep, 11, 100), want_loads)


# ---- refusals ------------------------------------------------------------------------------------------
def test_refusals_leave_buffers_and_the_chain_untouched(eng):
    rng = np.random.default_rng(91)
    syn, models, pm, ep = upload(eng, 64, 8, seed=92)
    ids, tg, rows = requests(syn, models, 40, rng)
    R, w = rows.shape
    lib, ctx = N.load(), eng._ctx
    window = 7
    eng.feedback_chain_reset()
    first = eng.schedule_models_batch_feedback_chain_excluding(ep, SEED, ids[:10], tg[:10], rows[:10], window, 0)
    before = chain_loads(eng, ep, window, 64)
    out = np.full(R, 0x77, dtype=np.uint32)
    fb = np.full((R, 2), 0x55, dtype=np.int16)
    loads = np.zeros(64, dtype=np.int32)
    p_ids, p_tg, p_rows, p_out, p_fb = (a.ctypes.data for a in (ids, tg, rows, out, fb))
    no_models_ep = next_epoch()
    eng.upload_snapshot(no_models_ep, syn.packed)
    cases = [  # (rc wanted, call)
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, p_ids, None, R, p_rows, w,
                                                                            p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, None, p_tg, R, p_rows, w,
                                                                            p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, 0,
                                                                            p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, 33,
                                                                            p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, p_ids, p_tg, -1, p_rows, w,
                                                                            p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding_fallbacks(
            ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, w, p_out, 0, p_fb)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding_fallbacks(
            ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, w, p_out, 2, None)),
        (N.LIG_ERR_NO_SNAPSHOT, lambda: lib.lig_schedule_models_batch_excluding(ctx, no_models_ep, 1, 0, p_ids, p_tg,
                                                                                R, p_rows, w, p_out)),
        (N.LIG_ERR_STALE_EPOCH, lambda: lib.lig_schedule_models_batch_excluding(ctx, 999999, 1, 0, p_ids, p_tg, R,
                                                                                p_rows, w, p_out)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_feedback_chain_excluding(
            ctx, ep, 1, 0, p_ids, None, R, p_rows, w, p_out, window, loads.ctypes.data)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_feedback_chain_excluding(
            ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, w, p_out, 0, loads.ctypes.data)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks(
            ctx, ep, 1, 0, p_ids, p_tg, R, p_rows, w, p_out, 9, p_fb, window, loads.ctypes.data)),
        (N.LIG_ERR_NO_SNAPSHOT, lambda: lib.lig_schedule_models_batch_feedback_chain_excluding(
            ctx, no_models_ep, 1, 0, p_ids, p_tg, R, p_rows, w, p_out, window, loads.ctypes.data)),
        (N.LIG_ERR_INVALID, lambda: lib.lig_schedule_models_batch_excluding(ctx, ep, 1, 0, p_ids, p_tg, (1 << 14) + 1,
                                                                            p_rows, w, p_out)),
    ]
    for i, (rc, call) in enumerate(cases):
        assert call() == rc, i
    assert (out == 0x77).all() and (fb == 0x55).all() and not loads.any()
    # device forms: buffers not aligned to their element
    d_ids, d_tg = dev(ids), torch.from_numpy(tg.copy()).cuda()
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda()
    d_out = torch.zeros(R + 1, dtype=torch.int32, device="cuda")
    d_fb = torch.zeros(R * 2 + 1, dtype=torch.int16, device="cuda")
    a = [d_ids.data_ptr(), d_tg.data_ptr(), d_rows.data_ptr(), d_out.data_ptr(), d_fb.data_ptr()]
    for bad in ((a[0] + 2, a[2], a[3], a[4]), (a[0], a[2] + 1, a[3], a[4]), (a[0], a[2], a[3] + 2, a[4]),
                (a[0], a[2], a[3], a[4] + 1)):
        assert lib.lig_schedule_models_batch_excluding_fallbacks_device(
            ctx, ep, 1, 0, bad[0], a[1], R, bad[1], w, bad[2], 2, bad[3], None) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device(
            ctx, ep, 1, 0, bad[0], a[1], R, bad[1], w, bad[2], 2, bad[3], window, None, None) == N.LIG_ERR_INVALID
    # the chain is as it was: its loads, and the next call continues the sequence
    assert np.array_equal(chain_loads(eng, ep, window, 64), before)
    rest = eng.schedule_models_batch_feedback_chain_excluding(ep, SEED, ids[10:], tg[10:], rows[10:], window, 10)
    whole = MR.run_chain_snapshot(syn.packed, [MR.model_retry_call(pm, ids, tg, rows, SEED, 0)], window)[0][0]
    assert np.concatenate([first, rest]).tobytes() == whole.tobytes()


@pytest.mark.parametrize("rows_k", [0, 4])
def test_chain_unstaged_pod_columns(rows_k, eng):
    """The chain forms whose pod columns do not fit shared memory (kStaged = false, kCount), windows closing
    inside the calls, host and device forms alternating."""
    rng = np.random.default_rng(101 + rows_k)
    syn, models, pm, ep = upload(eng, UNSTAGED_P, 16, seed=102)
    calls, raw = [], []
    fi = 0
    for j in range(3):
        ids, tg, ex = requests(syn, models, 40, rng, fi)
        calls.append(MR.model_retry_call(pm, ids, tg, ex, SEED + j, fi))
        raw.append(("model_retry", ids, tg, ex, fi))
        fi += len(ids)
    ks = [rows_k] * 3
    want, want_rows, want_loads = MR.run_chain_snapshot(syn.packed, calls, 17, ks)
    eng.feedback_chain_reset()
    got, got_rows = [], []
    for i, ((c, seed), r) in enumerate(zip(calls, raw)):
        o, rw = run_calls(eng, ep, [(c, seed)], 17, [rows_k], [r], device=bool(i % 2))
        got += o
        got_rows += rw
    assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
    if rows_k:
        assert all(np.array_equal(g, w) for g, w in zip(got_rows, want_rows))
    assert np.array_equal(chain_loads(eng, ep, 17, UNSTAGED_P), want_loads)
