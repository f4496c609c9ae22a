"""Ejected epochs (lig_eject_pods) at the shapes where the pool forms of the kernels differ, against the
definition (eject_ref.py), byte for byte.

* Every descriptor pool form of lig_schedule_excluding_kernel with a non-empty pool: with and without
  rows, with and without the chain's count, staged (P <= 12224) and unstaged, under the
  built-in tree and caller trees, at P in {33, 4096, 5000, 13000, 32768}.  The ejected sets are hot
  pods, the last pod with pods of the last word, one whole 32-pod word, one whole 1024-pod group in
  the middle (so a warp-cooperative select skips an empty group) and every pod but one.  Rows name
  ejected pods, kept pods, the pick, padding and out-of-range entries, and one row removes the last
  survivors of a class.
* Feedback chains and the in-batch feedback call on derived epochs through the general staged and
  unstaged builds, caller-tree builds and the fast build with several classes per build warp: the
  scratch tables are rebuilt from the pool after every closed window.
* The lifecycle past the fast build: a derive from a derived epoch, deltas under a caller tree and at
  unstaged P, threshold rebuilds, an eject under another tree than its base's, and an eject right
  after an asynchronous upload.
"""
import contextlib

import numpy as np
import pytest
import torch

import eject_ref as ER
import feedback_chain_retry_ref as CR
from draw_keys import accept_top, pick_keys
from test_gpu_build_shapes import build_geometry, resolve_A, sm  # noqa: F401  (sm: fixture)
from test_gpu_eject import hot_pods
from test_gpu_fallbacks import DROP_AND_NO_PODS, KEEP_ALL
from test_gpu_filter_batch import dev
from test_gpu_filter_tree import c4_tree
from test_gpu_retry import UNSTAGED_P, class_reqs
from test_gpu_retry_fallbacks import WIDEST_P
from test_gpu_kernel_variants import VARIANTS, make_engine
from test_gpu_snapshot_mutation import SMEM_OPTIN, build_variant
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, pack_models

pytestmark = pytest.mark.gpu

SEED = 0xE1EC_7000_5A9E_0001
GENERIC_P = 5000            # past the fast build's 4096 pods, staged general build
TREES = {"built_in": None, "c4": "c4", "drop_and_no_pods": DROP_AND_NO_PODS, "keep_all": KEEP_ALL}
SETS = ("hot", "tail", "word", "group", "all_but_one")

_ep = [19000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=WIDEST_P, max_adapters=2048, max_batch=1 << 16)
    yield e
    e.close()


def nodes_of(tree):
    t = TREES[tree]
    return c4_tree().flatten() if t == "c4" else t


def walk_staged(P):
    """staged_fits (lig.cu): the retry walks and the caller-tree build stage the pod columns when 96 B
    of scratch and 512 B of columns per 32 pods fit the opt-in shared memory.  The retry launches
    record no launch info, so the form is asserted through this rule, not observed."""
    W = (P + 31) // 32
    return P > 0 and 608 * W <= SMEM_OPTIN


def ejected_set(kind, snap, reqs, rng, nodes):
    P = snap.P
    if kind == "hot":
        return hot_pods(snap, reqs, 6, rng, nodes=nodes)
    if kind == "tail":                                   # the last pod and pods of the (ragged) last word
        last = (P - 1) // 32 * 32
        return sorted({P - 1, last} | set(rng.integers(last, P, size=2).tolist()))
    if kind == "word":
        w = (P // 32) // 2
        return list(range(32 * w, 32 * w + 32))
    if kind == "group":                                  # one whole group of 32 words in the middle
        g = (P // 1024) // 2
        return list(range(1024 * g, 1024 * (g + 1)))
    keep = int(rng.integers(0, P))                       # every pod but one
    return [p for p in range(P) if p != keep]


def derived(eng, snap, ejected, nodes, base_nodes="same", block=True):
    """Upload snap under base_nodes (default: nodes) and derive an epoch without `ejected` under nodes."""
    base, ep = next_epoch(), next_epoch()
    eng.set_filter_tree(nodes if base_nodes == "same" else base_nodes)
    try:
        eng.upload_snapshot(base, snap, block=block)
        eng.set_filter_tree(nodes)
        eng.eject_pods(ep, base, ejected)
    finally:
        eng.set_filter_tree(None)
    return base, ep


@contextlib.contextmanager
def tree_in_force(eng, nodes):
    """The chain and the in-batch feedback call walk the tree in force when they start."""
    eng.set_filter_tree(nodes)
    try:
        yield
    finally:
        eng.set_filter_tree(None)


def retry_rows(snap, ejected, reqs, rng, nodes, width=6):
    """At most 8 distinct rows: nothing, ejected + kept + out-of-range entries, the pick, kept pods
    and the last survivors of one class (its requests get an empty reduced pool)."""
    P = snap.P
    ej = list(ejected)
    kept = np.setdiff1d(np.arange(P), ej)
    oor = P + 3 if P + 3 <= 32767 else -7
    tpl = [[], [ej[0], int(kept[0]), oor, -1, ej[-1]], [int(kept[-1]), ej[len(ej) // 2], 32767, -32768],
           [int(p) for p in rng.choice(kept, size=min(4, len(kept)), replace=False)] + [oor]]
    rows = np.full((len(reqs), width), -1, dtype=np.int16)
    for i in range(len(reqs)):
        t = tpl[i % len(tpl)][:width]
        rows[i, :len(t)] = t
    # three requests (none a multiple of 3) exclude their own pick
    own = [i for i in (2, 7, 17) if i < len(reqs)]
    picks = ER.schedule_batch(snap, ejected, np.ascontiguousarray(reqs[own]), SEED, nodes=nodes)["pod_idx"]
    rows[own] = -1
    rows[own, 0] = picks
    # a class whose survivors all fit one row: every third request of it removes them all
    for crit in (True, False):
        for a in (0, 1, snap.A):
            st, lst = ER.klass(snap, ejected, crit, a, nodes=nodes)
            if st == N.LIG_OK and 0 < len(lst) <= width:
                reqs[::3]["adapter_id"] = a
                reqs[::3]["flags"] = int(crit)
                rows[::3] = -1
                rows[::3, :len(lst)] = lst
                return rows, True
    return rows, False


CASES = [(P, tree, kind) for P in (33, 4096, GENERIC_P, UNSTAGED_P, WIDEST_P) for tree in TREES for kind in SETS
         if not (kind == "group" and P < 2048)
         and not (P == WIDEST_P and tree in ("c4", "drop_and_no_pods"))        # as test_gpu_retry_fallbacks
         and not (P >= UNSTAGED_P and tree != "built_in" and kind in ("tail", "word"))
         and not (P >= UNSTAGED_P and tree != "built_in" and kind == "hot")]


@pytest.mark.parametrize("P,tree,kind", CASES, ids=[f"P={p}-{t}-{k}" for p, t, k in CASES])
def test_every_pool_retry_kernel(eng, P, tree, kind):
    """The four pool retry kernels in the form the case claims (staged below 12224 pods, the tree in
    force at the eject), each against the definition."""
    rng = np.random.default_rng(P * 31 + len(kind) + len(tree))
    nodes = nodes_of(tree)
    A = 4 if P < 64 else 8
    snap = WL.make_snapshot(P, A, seed=P + 13).packed
    R = 48 if P < UNSTAGED_P else 16
    reqs = class_reqs(A, R, rng)
    ejected = ejected_set(kind, snap, reqs, rng, nodes)
    assert 0 < len(ejected) < P
    assert walk_staged(P) == (P < UNSTAGED_P)
    _, ep = derived(eng, snap, ejected, nodes)
    rows, emptied = retry_rows(snap, ejected, reqs, rng, nodes)
    assert emptied or kind != "all_but_one" or tree in ("c4", "drop_and_no_pods")   # their leaves may drop it
    assert len({r.tobytes() for r in rows}) <= 8
    want = ER.retry_batch(snap, ejected, reqs, rows, SEED, nodes=nodes)
    if nodes is not None and kind != "all_but_one":      # the caller tree is the one in force
        assert want.tobytes() != ER.retry_batch(snap, ejected, reqs, rows, SEED).tobytes()
    assert eng.schedule_batch_excluding(ep, SEED, reqs, rows).tobytes() == want.tobytes()
    assert not set(ejected) & set(want["pod_idx"][want["pod_idx"] >= 0].tolist())
    for n in (1, 8):
        p, fb = eng.schedule_batch_excluding_fallbacks(ep, SEED + n, reqs, rows, n)
        wp, wf = ER.retry_fallback_batch(snap, ejected, reqs, rows, SEED + n, n, nodes=nodes)
        assert p.tobytes() == wp.tobytes() and np.array_equal(fb, wf), n
        assert not set(ejected) & set(wf[wf >= 0].ravel().tolist())
    # the chain forms: windows small enough that several close within each call
    window = max(1, R // 5)
    h = R // 2
    a, b = np.ascontiguousarray(reqs[:h]), np.ascontiguousarray(reqs[h:])
    ra, rb = np.ascontiguousarray(rows[:h]), np.ascontiguousarray(rows[h:])
    loads = np.zeros(P, dtype=np.int32)
    with tree_in_force(eng, nodes):
        eng.feedback_chain_reset()
        o1 = eng.schedule_batch_feedback_chain_excluding(ep, SEED + 5, a, ra, window, loads)
        o2, r2 = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED + 6, b, rb, 3, window, loads)
    wouts, wrows, wloads = ER.chain(snap, ejected, [CR.retry_call(a, ra, SEED + 5), CR.retry_call(b, rb, SEED + 6)],
                                    window, [0, 3], nodes=nodes)
    assert o1.tobytes() == wouts[0].tobytes() and o2.tobytes() == wouts[1].tobytes()
    assert np.array_equal(r2, wrows[1])
    assert np.array_equal(loads.astype(np.int64), wloads) and loads[ejected].sum() == 0


# ---- chains and the in-batch feedback call through every build form -------------------------------------
CHAIN_SHAPES = [("general_staged", GENERIC_P, 24, None), ("general_unstaged", UNSTAGED_P, 12, None),
                ("tree_staged", 300, 12, "c4"), ("tree_unstaged", UNSTAGED_P, 12, "c4"),
                ("fast_many_per_warp", 1000, "8s+17", None)]


CHAIN_CASES = [(s, w) for s in CHAIN_SHAPES for w in (1, 7, 256) if not (s[0] == "tree_unstaged" and w == 1)]


@pytest.mark.parametrize("shape,P,A_spec,tree,window", [s + (w,) for s, w in CHAIN_CASES],
                         ids=[f"{s[0]}-{w}" for s, w in CHAIN_CASES])
def test_chain_rebuilds_on_derived_epochs(eng, shape, P, A_spec, tree, window, sm):
    """Plain, fallback, model-id (built-in tree), retry and retry-with-rows chain calls in one chain,
    then the in-batch feedback call over 320 requests: every window that closes rebuilds the scratch
    tables with the pool form of the epoch's build.  At window 256 the chain closes one window at the
    staged shapes and none at the unstaged ones (a control); the in-batch call closes one everywhere."""
    A = resolve_A(A_spec, sm) if isinstance(A_spec, str) else A_spec
    if shape == "fast_many_per_warp":
        kind, grid, per_warp = build_geometry(P, A, sm)
        assert kind == "fast" and per_warp >= 2 and A > 8 * sm, (kind, grid, per_warp)
    elif tree is None:                                  # lig_class_build_kernel<staged, pool>
        assert build_variant(P) == shape.split("_")[1], (shape, build_variant(P))
    else:                                               # lig_class_build_tree_kernel<staged, pool>
        assert walk_staged(P) == (shape == "tree_staged"), shape
    nodes = c4_tree().flatten() if tree else None
    rng = np.random.default_rng(P + window + A)
    snap = WL.make_snapshot(P, A, seed=P + 29).packed
    R = 96 if P < UNSTAGED_P else 40
    reqs = WL.make_requests(2 * R + 320, A, seed=P + 30)
    ejected = hot_pods(snap, reqs, 8, rng, nodes=nodes)
    _, ep = derived(eng, snap, ejected, nodes)
    rreqs = class_reqs(A, 2 * R, rng)
    rows, _ = retry_rows(snap, ejected, rreqs, rng, nodes, width=4)
    a, b = reqs[:R], reqs[R:2 * R]
    if tree is None:                                     # model ids that all resolve, in the same chain
        eng.upload_models(ep, pack_models(WL.make_models(A), snap))
        ids = WL.make_model_requests(R, A, seed=P + 31)
        dreqs, res = eng.resolve_models(ep, SEED + 4, ids)
        present = res["status"] != N.LIG_NO_MODEL
        ids = np.ascontiguousarray(np.where(present, ids, ids[present][0]).astype(np.uint32))
        dreqs, res = eng.resolve_models(ep, SEED + 4, ids)
        assert (res["status"] != N.LIG_NO_MODEL).all()
    c, d = np.ascontiguousarray(rreqs[:R]), np.ascontiguousarray(rreqs[R:])
    ec, ed = np.ascontiguousarray(rows[:R]), np.ascontiguousarray(rows[R:])
    loads = np.zeros(P, dtype=np.int32)
    outs, rws = [], {}
    with tree_in_force(eng, nodes):
        eng.feedback_chain_reset()
        outs.append(eng.schedule_batch_feedback_chain(ep, SEED, a, window, loads))
        o, r = eng.schedule_batch_feedback_chain_fallbacks(ep, SEED + 1, b, 4, window, loads)
        outs.append(o); rws[1] = r
        outs.append(eng.schedule_batch_feedback_chain_excluding(ep, SEED + 2, c, ec, window, loads))
        o, r = eng.schedule_batch_feedback_chain_excluding_fallbacks(ep, SEED + 3, d, ed, 2, window, loads)
        outs.append(o); rws[3] = r
        if tree is None:                                 # model ids, resolved on the device
            mo = eng.schedule_models_batch_feedback_chain(ep, SEED + 4, ids, window, loads=loads)
    calls = [(a, SEED), (b, SEED + 1), CR.retry_call(c, ec, SEED + 2), CR.retry_call(d, ed, SEED + 3)]
    ks = [0, 4, 0, 2]
    if tree is None:
        calls.append((dreqs, SEED + 4))
        ks.append(0)
    wouts, wrows, wloads = ER.chain(snap, ejected, calls, window, ks, nodes=nodes)
    if tree is None:
        w = wouts.pop()
        assert np.array_equal(mo["pod_idx"], w["pod_idx"]) and np.array_equal(mo["status"], w["status"])
    for i, (g, w) in enumerate(zip(outs, wouts)):
        assert g.tobytes() == w.tobytes(), i
    for i, r in rws.items():
        assert np.array_equal(r, wrows[i]), i
    assert np.array_equal(loads.astype(np.int64), wloads) and loads[ejected].sum() == 0
    # the in-batch feedback call: one call, windows of `window` requests
    breqs = reqs[2 * R:]
    d_in = dev(breqs)
    d_out = torch.zeros(len(breqs) * 8, dtype=torch.uint8, device="cuda")
    d_hist = torch.zeros(P, dtype=torch.int32, device="cuda")
    with tree_in_force(eng, nodes):
        eng.schedule_batch_feedback_device(ep, SEED + 9, d_in.data_ptr(), len(breqs), d_out.data_ptr(), window, 0,
                                           d_hist.data_ptr())
        torch.cuda.synchronize()
    wouts, _, wloads = ER.chain(snap, ejected, [(breqs, SEED + 9)], window, nodes=nodes)
    assert d_out.cpu().numpy().tobytes() == wouts[0].tobytes()
    hist = d_hist.cpu().numpy().astype(np.int64)
    assert np.array_equal(hist, wloads) and hist[ejected].sum() == 0


# ---- the lifecycle past the fast build ------------------------------------------------------------------
@pytest.mark.parametrize("P,tree", [(GENERIC_P, None), (UNSTAGED_P, None), (300, "c4"), (UNSTAGED_P, "c4")])
def test_lifecycle_past_the_fast_build(eng, P, tree):
    nodes = c4_tree().flatten() if tree else None
    rng = np.random.default_rng(P + 71)
    A = 12
    snap = WL.make_snapshot(P, A, seed=P + 72).packed
    reqs = WL.make_requests(300, A, seed=P + 73)
    first = hot_pods(snap, reqs, 6, rng, nodes=nodes)
    second = sorted(set(hot_pods(snap, reqs, 6, rng, nodes=nodes)) - set(first[:3]) | {P - 1})
    _, ep = derived(eng, snap, first, nodes)
    with tree_in_force(eng, nodes):                      # ejects and deltas build with the tree in force
        lifecycle(eng, snap, reqs, ep, first, second, nodes, tree)


def lifecycle(eng, snap, reqs, ep, first, second, nodes, tree):
    def same(e, ejected, s=snap, thresholds=(0.8, 5, 50)):
        want = ER.schedule_batch(s, ejected, reqs, SEED, thresholds, nodes)
        assert eng.schedule_batch(e, SEED, reqs).tobytes() == want.tobytes()
        rows = np.full((len(reqs), 2), -1, dtype=np.int16)
        rows[::2, 0] = ejected[0] if ejected else 0
        rows[1::4, 1] = want["pod_idx"][1::4]
        assert eng.schedule_batch_excluding(e, SEED, reqs, rows).tobytes() == \
            ER.retry_batch(s, ejected, reqs, rows, SEED, thresholds, nodes).tobytes()
    same(ep, first)
    # a derive from a derived epoch: the new set replaces the old one, it does not add to it
    other = next_epoch()
    eng.eject_pods(other, ep, second)
    same(other, second)
    again = next_epoch()
    eng.eject_pods(again, other, second)                 # the same set once more
    same(again, second)
    # a delta from the derived epoch keeps its set
    d = next_epoch()
    moved = 8 if second[0] == 7 else 7
    dirty = np.array([second[0], moved], dtype=np.int32)
    kv = np.array([0.02, 0.97]); q = np.array([0, 3], dtype=np.int32)
    na = np.array([0, 1], dtype=np.uint16); ma = np.array([4, 4], dtype=np.uint16)
    eng.update_snapshot(d, again, dirty, kv, q, na, ma, np.array([0, 0, 1], dtype=np.int32),
                        np.array([2], dtype=np.int32))
    snap_d = ER.RR.reduce_snapshot(snap, np.arange(snap.P))
    snap_d.kv[dirty] = kv
    snap_d.q[dirty] = q
    snap_d.n_active[dirty] = na
    snap_d.max_active[dirty] = ma
    for p in dirty:
        snap_d.bitmap[:, p >> 5] &= np.uint32(~(1 << (int(p) & 31)) & 0xFFFFFFFF)
    snap_d.bitmap[2, moved >> 5] |= np.uint32(1 << (moved & 31))
    same(d, second, snap_d)
    if tree is None:                                     # a threshold rebuild keeps the set
        try:
            eng.set_thresholds(0.5, 3, 20)
            same(d, second, snap_d, (0.5, 3, 20))
        finally:
            eng.set_thresholds()


@pytest.mark.parametrize("P", [GENERIC_P, UNSTAGED_P])
def test_eject_follows_the_tree_in_force(eng, P):
    """The derived epoch builds with the tree in force at the eject, whatever its base was built with."""
    snap = WL.make_snapshot(P, 10, seed=P + 81).packed
    reqs = WL.make_requests(256, 10, seed=P + 82)
    c4 = c4_tree().flatten()
    ejected = hot_pods(snap, reqs, 6, np.random.default_rng(P + 83))
    for base_nodes, nodes in ((None, c4), (c4, None)):
        _, ep = derived(eng, snap, ejected, nodes, base_nodes=base_nodes)
        want = ER.schedule_batch(snap, ejected, reqs, SEED, nodes=nodes)
        assert want.tobytes() != ER.schedule_batch(snap, ejected, reqs, SEED, nodes=base_nodes).tobytes()
        assert eng.schedule_batch(ep, SEED, reqs).tobytes() == want.tobytes()


@pytest.mark.parametrize("P", [300, GENERIC_P, UNSTAGED_P])
def test_eject_right_after_an_async_upload(eng, P):
    snap = WL.make_snapshot(P, 10, seed=P + 91).packed
    reqs = WL.make_requests(256, 10, seed=P + 92)
    ejected = hot_pods(snap, reqs, 6, np.random.default_rng(P + 93))
    _, ep = derived(eng, snap, ejected, None, block=False)
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == ER.schedule_batch(snap, ejected, reqs, SEED).tobytes()


# ---- model-id paths on a derived epoch at a general-build shape -----------------------------------------
@pytest.fixture(scope="module")
def generic():
    snap = WL.make_snapshot(GENERIC_P, 40, seed=101).packed
    reqs = WL.make_requests(512, 40, seed=102)
    ejected = hot_pods(snap, reqs, 10, np.random.default_rng(103))
    models = pack_models(WL.make_models(snap.A), snap)
    ids = WL.make_model_requests(1500, snap.A, seed=104)
    return snap, ejected, models, ids


def resolved_want(e, ep, snap, ejected, ids, seed):
    """(requests that resolve, the descriptor picks of the device-resolved requests)."""
    dreqs, res = e.resolve_models(ep, seed, ids)
    present = res["status"] != N.LIG_NO_MODEL
    assert present.sum() > len(ids) // 2
    return present, dreqs, ER.schedule_batch(snap, ejected, np.ascontiguousarray(dreqs[present]), seed)


def assert_mpicks(got, present, want):
    assert np.array_equal(got["pod_idx"][present], want["pod_idx"])
    assert np.array_equal(got["status"][present], want["status"])


def test_model_id_filter_and_doorbell(eng, generic):
    snap, ejected, models, ids = generic
    assert build_variant(snap.P) == "staged"
    _, ep = derived(eng, snap, ejected, None)
    eng.upload_models(ep, models)
    present, dreqs, want = resolved_want(eng, ep, snap, ejected, ids, SEED)
    picks, offsets, pods = eng.filter_models_batch(ep, SEED, ids)
    assert_mpicks(picks, present, want)
    for i in np.nonzero(present)[0][::11]:
        r = dreqs[i]
        a = int(r["adapter_id"])
        st, lst = ER.klass(snap, ejected, bool(r["flags"] & 1), a if 0 <= a < snap.A else snap.A)
        assert pods[offsets[i]:offsets[i + 1]].tolist() == (lst if st == N.LIG_OK else []), i
    eng.stream_open()
    try:
        n = min(len(ids), N.load().lig_stream_capacity())
        got = eng.stream_submit_models(ep, SEED, np.ascontiguousarray(ids[:n]))
    finally:
        eng.stream_close()
    assert_mpicks(got, present[:n], want[:int(present[:n].sum())])


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_model_queue_kernel_variants(variant, generic, monkeypatch):
    snap, ejected, models, ids = generic
    e = make_engine(VARIANTS[variant], monkeypatch, max_pods=snap.P, max_adapters=snap.A, max_batch=1 << 12)
    try:
        _, ep = derived(e, snap, ejected, None)
        e.upload_models(ep, models)
        d_in = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        outs = [torch.zeros(len(ids) * 4, dtype=torch.uint8, device="cuda") for _ in range(2)]
        e.schedule_models_batches_device(ep, SEED, 0, [d_in.data_ptr()] * 2, len(ids), [o.data_ptr() for o in outs])
        torch.cuda.synchronize()
        for b, o in enumerate(outs):
            present, _, want = resolved_want(e, ep, snap, ejected, ids, SEED + b)
            assert_mpicks(o.cpu().numpy().view(MPICK_DTYPE), present, want)
    finally:
        e.close()


# ---- forced Int31n rejections against the reduced class size ---------------------------------------------
def reject_cases():
    """(P, ejected count, draws): KEEP_ALL keeps every pod, so a class holds n = P pods on the base
    and n' = P - ejected on the derived epoch.  Draws rejected for n' and accepted for n, and the
    reverse, with n' a power of two while n is not, and the reverse."""
    out = [(1000, 488, "n_only"), (1024, 24, "n_prime_only")]       # n' = 512; n' = 1000
    n = GENERIC_P                                                   # n' with a lower accept bound than n
    n2 = max(range(n // 2, n), key=lambda m: accept_top(n) - accept_top(m))
    assert accept_top(n2) < accept_top(n)
    out.append((n, n - n2, "n_prime_only"))
    return out


@pytest.mark.parametrize("P,k,where", reject_cases())
def test_forced_rejections_use_the_reduced_class_size(eng, P, k, where):
    """where = n_prime_only: every first draw is rejected for n' (and accepted for n); n_only: the
    reverse.  A pool kernel that bounded Int31n by the base's n would pick differently."""
    rng = np.random.default_rng(P + k)
    snap = WL.make_snapshot(P, 4, seed=P + 111).packed
    ejected = sorted(rng.choice(P, size=k, replace=False).tolist())
    n, n2 = P, P - k
    lo, hi = (accept_top(n2), accept_top(n)) if where == "n_prime_only" else (accept_top(n), accept_top(n2))
    assert lo < hi
    R = 64
    reqs = class_reqs(4, R, rng)
    reqs["rand_key"] = pick_keys(SEED, rng.integers(lo, hi, size=R), rng)
    _, ep = derived(eng, snap, ejected, KEEP_ALL)
    want = ER.schedule_batch(snap, ejected, reqs, SEED, nodes=KEEP_ALL)
    assert (want["n_survivors"] == n2).all()
    assert eng.schedule_batch(ep, SEED, reqs).tobytes() == want.tobytes()
    rows = np.full((R, 1), -1, dtype=np.int16)
    assert eng.schedule_batch_excluding(ep, SEED, reqs, rows).tobytes() == want.tobytes()
    p, fb = eng.schedule_batch_excluding_fallbacks(ep, SEED, reqs, rows, 8)
    wp, wf = ER.retry_fallback_batch(snap, ejected, reqs, rows, SEED, 8, nodes=KEEP_ALL)
    assert p.tobytes() == want.tobytes() and np.array_equal(fb, wf)
    p, fb = eng.schedule_batch_fallbacks(ep, SEED, reqs, 8)
    assert p.tobytes() == want.tobytes() and np.array_equal(fb, wf)
