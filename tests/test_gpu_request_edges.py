"""Every request entry point against the CPU at the request fields' edges: adapter ids -1, A, A+1, 2^31-1 and
INT32_MIN in requests and in uploaded model tables, model ids n_models and 2^32-1, model-retry targets 255,
254, nt and nt-1, rand_keys 0, 2^64-1 and keys that force Int31n rejections on the pick and on fallback
step 1, affinity keys on a duplicated pod key and on a pod's own hash, and batch sizes with partial warps
and CTAs.  Each entry point is one row of FORMS, run with pageable, page-locked and device buffers where
it has them; `out` and every row are compared byte for byte with request_edges_ref.py and the existing
definitions, none of which reads a device result.  The model tables keep ids outside [0, A): they are
the adapter no pod lists, as for lig_req."""
import numpy as np
import pytest
import torch

import affinity_ref as AR
import eject_ref as ER
import feedback_chain_retry_ref as CR
import models_feedback_chain_ref as MC
import models_retry_ref as MR
import request_edges_ref as E
import retry_fallbacks_ref as RF
import retry_ref as RR
from test_gpu_filter_batch import Pinned
from test_gpu_retry import NO_PODS_TREE, rows_for
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_columns
from oracle import binding as B

pytestmark = pytest.mark.gpu

SEED = 0xED6E_5EED_0BAD_F00D
K = N.LIG_MAX_FALLBACKS
BATCHES = (1, 31, 33, 255, 257, 4099)
GRID = [(P, A) for P in (1, 31, 32, 33, 257, 4097) for A in (0, 1, 5, 64)]
FEATURE_POOLS = [(1, 0), (33, 1), (257, 5), (4097, 64)]
FIRST = (1 << 64) - 7          # model rand_keys wrap to 0 inside a batch
_ep = [31000]


def next_epoch():
    _ep[0] += 1
    return _ep[0]


@pytest.fixture(scope="module")
def eng():
    e = Engine(0, max_pods=4097, max_adapters=1024, max_batch=1 << 14)
    yield e
    e.close()


# ---- pools ---------------------------------------------------------------------------------------------
class Epoch:
    """A resident epoch and its CPU lists: snap, nodes (caller tree or None), ejected pods, class lists,
    the raw hostile model table and its oracle twin."""

    def __init__(self, eng, snap, nodes=None, ejected=None):
        self.snap, self.nodes, self.ejected = snap, nodes, ejected
        self.ep = next_epoch()
        eng.set_filter_tree(nodes)
        try:
            eng.upload_snapshot(self.ep, snap)
        finally:
            eng.set_filter_tree(None)
        if ejected is not None:
            base, self.ep = self.ep, next_epoch()
            eng.eject_pods(self.ep, base, np.asarray(ejected, dtype=np.int32))
        self.cl = E.ClassLists(snap, nodes, ejected)
        self.recs = E.hostile_models(snap.A)
        self.pm = E.pack_raw_models(self.recs, snap.A)
        self.models = B.Models(self.recs)
        eng.upload_models(self.ep, self.pm)


def bench_pool(P, A):
    return WL.make_snapshot(P, A, seed=1000 * P + A).packed


def mixed_pool():
    """Idle pods with equal KV: adapter 0 on every pod (a list of 257), adapter 1 on 40, 2 on 3, 3 on one,
    4 on none: per-thread and per-warp affinity lists side by side in one warp."""
    P, A = 257, 5
    W = (P + 31) // 32
    member = np.zeros((A, P), dtype=bool)
    member[0] = True
    member[1, :40] = True
    member[2, [5, 100, 256]] = True
    member[3, 128] = True
    bitmap = np.zeros((A, W), dtype=np.uint32)
    for a, p in zip(*np.nonzero(member)):
        bitmap[a, p >> 5] |= np.uint32(1 << (p & 31))
    return pack_columns(np.full(P, 0.25), np.zeros(P, np.int64), member.sum(0).astype(np.int64),
                        np.full(P, 8, np.int64), bitmap, {WL.adapter_name(a): a for a in range(A)},
                        [WL.Pod(f"pod-{i}", f"address-{i}") for i in range(P)])


def overflow_pool():
    P, A = 4096, 1024
    W = P // 32
    return pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.full(P, 1, np.int64), np.full(P, 2, np.int64),
                        np.full((A, W), 0xFFFFFFFF, dtype=np.uint32), {WL.adapter_name(a): a for a in range(A)},
                        [WL.Pod(f"pod-{i}", f"address-{i}") for i in range(P)])


SPECIAL = {
    "mixed": lambda eng: Epoch(eng, mixed_pool()),
    "overflow": lambda eng: Epoch(eng, overflow_pool()),
    "ejected": lambda eng: Epoch(eng, bench_pool(257, 5), ejected=[0, 31, 32, 33, 100, 256]),
    "no_pods_tree": lambda eng: Epoch(eng, bench_pool(257, 5), nodes=NO_PODS_TREE),
}


# ---- buffers and forms -----------------------------------------------------------------------------------
class In:
    def __init__(self, a):
        self.a = np.ascontiguousarray(a)


class Out:
    def __init__(self, dtype, shape):
        self.dtype, self.shape = np.dtype(dtype), shape


def call(eng, fn, args, form):
    """eng.<fn>(*args) with every In / Out placed in pageable, page-locked or device memory (Outs start
    as junk); returns the Outs as numpy arrays."""
    keep, outs, real = [], [], []
    for x in args:
        if not isinstance(x, (In, Out)):
            real.append(x)
            continue
        nbytes = x.a.nbytes if isinstance(x, In) else int(np.prod(x.shape)) * x.dtype.itemsize
        if form == "device":
            t = torch.full((max(nbytes, 16),), 0xAB, dtype=torch.uint8, device="cuda")
            if isinstance(x, In) and nbytes:
                t[:nbytes] = torch.from_numpy(x.a.view(np.uint8).reshape(-1).copy()).cuda()
            keep.append(t)
            real.append(t.data_ptr())
            if isinstance(x, Out):
                outs.append((x, lambda t=t, n=nbytes: t.cpu().numpy()[:n]))
        else:
            if form == "pinned":
                b = Pinned(max(nbytes, 16), np.uint8)
                buf, ptr = b.a, b.ptr
            else:
                buf = np.empty(max(nbytes, 16), np.uint8)
                ptr = buf.ctypes.data
            buf[:] = 0xAB
            if isinstance(x, In):
                buf[:nbytes] = x.a.view(np.uint8).reshape(-1)
            keep.append(b if form == "pinned" else buf)
            real.append(ptr)
            if isinstance(x, Out):
                outs.append((x, lambda buf=buf, n=nbytes: buf[:n].copy()))
    try:
        getattr(eng, fn)(*real)
        if form == "device":
            torch.cuda.synchronize()
        return [get().view(x.dtype).reshape(x.shape) for x, get in outs]
    finally:
        for b in keep:
            if isinstance(b, Pinned):
                b.free()


# A row: entry point -> (host-pointer method or None, device method or None, args(a) built from the
# request dict a).  Host methods run with pageable and page-locked buffers, device methods with device ones;
# the argument lists are the same but for the device methods' trailing stream.
def _reqs(a):
    return In(a["reqs"])


def _pick(a):
    return Out(PICK_DTYPE, (a["R"],))


def _mpick(a):
    return Out(MPICK_DTYPE, (a["R"],))


def _rows(a):
    return Out(np.int16, (a["R"], a["k"]))


def _ex(a):
    return In(a["ex"])


FORMS = {
    "plain": {
        "schedule_batch": ("schedule_batch_ptr", "schedule_batch_device",
                           lambda a: [a["ep"], a["seed"], _reqs(a), a["R"], _pick(a)]),
        "schedule_scan": (None, "schedule_scan_device", lambda a: [a["ep"], a["seed"], _reqs(a), a["R"], _pick(a), 0]),
    },
    "fallbacks": {
        "schedule_batch_fallbacks": ("schedule_batch_fallbacks_ptr", "schedule_batch_fallbacks_device",
                                     lambda a: [a["ep"], a["seed"], _reqs(a), a["R"], _pick(a), a["k"], _rows(a)]),
    },
    "affinity": {
        "schedule_batch_affinity": ("schedule_batch_affinity_ptr", "schedule_batch_affinity_device",
                                    lambda a: [a["ep"], _reqs(a), a["R"], _pick(a), a["k"],
                                               _rows(a) if a["k"] else 0]),
    },
    "models": {
        "schedule_models_batch": ("schedule_models_batch_ptr", None,
                                  lambda a: [a["ep"], a["seed"], a["fi"], In(a["ids"]), a["R"], _mpick(a)]),
    },
    "models_fallbacks": {
        "schedule_models_batch_fallbacks": (
            "schedule_models_batch_fallbacks_ptr", "schedule_models_batch_fallbacks_device",
            lambda a: [a["ep"], a["seed"], a["fi"], In(a["ids"]), a["R"], _mpick(a), a["k"], _rows(a)]),
    },
    "models_affinity": {
        "schedule_models_batch_affinity": (
            "schedule_models_batch_affinity_ptr", "schedule_models_batch_affinity_device",
            lambda a: [a["ep"], In(a["ids"]), In(a["keys"]), a["R"], _mpick(a), a["k"], _rows(a) if a["k"] else 0]),
    },
    "retry": {
        "schedule_batch_excluding": ("schedule_batch_excluding_ptr", "schedule_batch_excluding_device",
                                     lambda a: [a["ep"], a["seed"], _reqs(a), a["R"], _ex(a), a["w"], _pick(a)]),
    },
    "retry_fallbacks": {
        "schedule_batch_excluding_fallbacks": (
            "schedule_batch_excluding_fallbacks_ptr", "schedule_batch_excluding_fallbacks_device",
            lambda a: [a["ep"], a["seed"], _reqs(a), a["R"], _ex(a), a["w"], _pick(a), a["k"], _rows(a)]),
    },
    "model_retry": {
        "schedule_models_batch_excluding": (
            "schedule_models_batch_excluding_ptr", "schedule_models_batch_excluding_device",
            lambda a: [a["ep"], a["seed"], a["fi"], In(a["ids"]), In(a["tg"]), a["R"], _ex(a), a["w"], _mpick(a)]),
    },
    "model_retry_fallbacks": {
        "schedule_models_batch_excluding_fallbacks": (
            "schedule_models_batch_excluding_fallbacks_ptr", "schedule_models_batch_excluding_fallbacks_device",
            lambda a: [a["ep"], a["seed"], a["fi"], In(a["ids"]), In(a["tg"]), a["R"], _ex(a), a["w"], _mpick(a),
                       a["k"], _rows(a)]),
    },
}


def run_family(eng, family, a, want, want_rows=None):
    """Every form of every entry point of `family` against (want, want_rows)."""
    for name, (host, device, args) in FORMS[family].items():
        for form, fn in (("pageable", host), ("pinned", host), ("device", device)):
            if fn is None:
                continue
            got = call(eng, fn, args(a), form)
            assert got[0].tobytes() == want.tobytes(), (name, form, a["R"])
            if len(got) > 1:
                assert got[1].tobytes() == want_rows[:, :a["k"]].tobytes(), (name, form, a["R"], a["k"])


def mpicks(res, picks):
    out = np.zeros(len(res), dtype=MPICK_DTYPE)
    ok = res["ok"] == 1
    out["pod_idx"] = np.where(ok, picks["pod_idx"], -1)
    out["status"] = np.where(ok, picks["status"], MC.LIG_NO_MODEL)
    out["target_idx"] = res["target_idx"]
    return out


# ---- the plain pick and the survivor lists: the whole grid -------------------------------------------------
def check_plain(eng, p, R, rng):
    cl = p.cl
    reqs = E.edge_requests(cl, R, SEED, rng)
    want = cl.picks(reqs, SEED)
    a = dict(ep=p.ep, seed=SEED, reqs=reqs, R=R)
    forms = dict(FORMS["plain"])
    if p.nodes is not None or p.ejected is not None:
        forms.pop("schedule_scan")            # the direct scan restates the built-in tree on a full pool
    for name, (host, device, args) in forms.items():
        for form, fn in (("pageable", host), ("pinned", host), ("device", device)):
            if fn is not None:
                assert call(eng, fn, args(a), form)[0].tobytes() == want.tobytes(), (name, form, R)
    if p.nodes is None and p.ejected is None:
        assert eng.schedule_scan(p.ep, SEED, reqs, want_masks=False)[0].tobytes() == want.tobytes()
    # two resident batches back to back, batch b with seed + b
    d_in = [torch.from_numpy(reqs.view(np.uint8).copy()).cuda() for _ in range(2)]
    d_out = [torch.full((R * 8,), 0xAB, dtype=torch.uint8, device="cuda") for _ in range(2)]
    eng.schedule_batches_device(p.ep, SEED, [t.data_ptr() for t in d_in], R, [t.data_ptr() for t in d_out])
    torch.cuda.synchronize()
    assert d_out[0].cpu().numpy().tobytes() == want.tobytes()
    assert d_out[1].cpu().numpy().tobytes() == cl.picks(reqs, SEED + 1).tobytes()
    # lig_schedule_batch_async on page-locked buffers
    b_in, b_out = Pinned(R, REQ_DTYPE), Pinned(R, PICK_DTYPE)
    try:
        b_in.a[:] = reqs
        eng.schedule_wait(eng.schedule_batch_async(p.ep, SEED, b_in.ptr, R, b_out.ptr))
        assert b_out.a.tobytes() == want.tobytes()
    finally:
        b_in.free()
        b_out.free()
    # the survivor lists
    ok, offsets, pods = cl.csr(reqs)
    out, off, got = eng.filter_batch(p.ep, SEED, reqs)
    assert out.tobytes() == want.tobytes()
    assert np.array_equal(off, offsets) and np.array_equal(got.astype(np.int64), pods)
    cap = int(offsets[-1]) + 1
    o = call(eng, "filter_batch_device", [p.ep, SEED, _reqs(a), R, _pick(a), Out(np.int64, (R + 1,)),
                                          Out(np.uint16, (cap,)), cap], "device")
    assert o[0].tobytes() == want.tobytes() and np.array_equal(o[1], offsets)
    assert np.array_equal(o[2][: offsets[-1]].astype(np.int64), pods)
    return reqs, want


@pytest.mark.parametrize("P,A", GRID)
def test_plain_pick_and_lists_over_the_grid(P, A, eng):
    p = Epoch(eng, bench_pool(P, A))
    rng = np.random.default_rng(P * 131 + A)
    for R in BATCHES:
        done = check_plain(eng, p, R, rng)
        if R <= 4096:                         # the doorbell's capacity
            reqs, want = done
    eng.stream_open()
    try:
        assert eng.stream_submit(p.ep, SEED, reqs).tobytes() == want.tobytes()
    finally:
        eng.stream_close()


@pytest.mark.parametrize("pool", sorted(SPECIAL))
def test_plain_pick_and_lists_on_special_pools(pool, eng):
    p = SPECIAL[pool](eng)
    if pool == "overflow":
        assert eng.pick_kernel_info(p.ep)["table_bytes"] == 0
    if pool == "no_pods_tree":
        assert N.LIG_NO_PODS_LEFT in p.cl.status
    rng = np.random.default_rng(len(pool))
    for R in (33, 4099):
        check_plain(eng, p, R, rng)


# ---- model ids -------------------------------------------------------------------------------------------
def check_models(eng, p, R, rng, fi):
    ids = E.model_ids(p.pm.n_models, R, rng)
    res = MC.resolve_call(p.models, p.snap.adapter_id, ids, SEED, fi)
    picks, rows = p.cl.fallbacks(np.ascontiguousarray(res["req"]), SEED, K, keep=res["ok"] == 1)
    want = mpicks(res, picks)
    a = dict(ep=p.ep, seed=SEED, fi=fi, ids=ids, R=R)
    run_family(eng, "models", a, want)
    for k in (1, K):
        run_family(eng, "models_fallbacks", dict(a, k=k), want, rows)
    # lig_schedule_models_batches_device: batch b with seed + b
    res1 = MC.resolve_call(p.models, p.snap.adapter_id, ids, SEED + 1, fi)
    want1 = mpicks(res1, p.cl.picks(np.ascontiguousarray(res1["req"]), SEED + 1))
    d_in = [torch.from_numpy(ids.view(np.uint8).copy()).cuda() for _ in range(2)]
    d_out = [torch.full((R * 4,), 0xAB, dtype=torch.uint8, device="cuda") for _ in range(2)]
    eng.schedule_models_batches_device(p.ep, SEED, fi, [t.data_ptr() for t in d_in], R, [t.data_ptr() for t in d_out])
    torch.cuda.synchronize()
    assert d_out[0].cpu().numpy().tobytes() == want.tobytes()
    assert d_out[1].cpu().numpy().tobytes() == want1.tobytes()
    # lig_resolve_models: the descriptors name the oracle's class (ids outside [0, A) are A's)
    reqs, out = eng.resolve_models(p.ep, SEED, ids, fi)
    ok = res["ok"] == 1
    assert np.array_equal(out["status"] == MC.LIG_NO_MODEL, ~ok)
    assert np.array_equal(out["target_idx"], res["target_idx"])
    assert np.array_equal(p.cl.classes(reqs[ok]), p.cl.classes(res["req"][ok]))
    assert np.array_equal(reqs["rand_key"][ok], res["req"]["rand_key"][ok])
    # the survivor lists of the resolved requests
    _, offsets, pods = p.cl.csr(np.ascontiguousarray(res["req"]), keep=ok)
    got, off, gp = eng.filter_models_batch(p.ep, SEED, ids, fi)
    assert got.tobytes() == want.tobytes()
    assert np.array_equal(off, offsets) and np.array_equal(gp.astype(np.int64), pods)
    cap = int(offsets[-1]) + 1
    o = call(eng, "filter_models_batch_device", [p.ep, SEED, fi, In(ids), R, _mpick(a), Out(np.int64, (R + 1,)),
                                                 Out(np.uint16, (cap,)), cap], "device")
    assert o[0].tobytes() == want.tobytes() and np.array_equal(o[1], offsets)
    assert np.array_equal(o[2][: offsets[-1]].astype(np.int64), pods)
    return ids, want


@pytest.mark.parametrize("pool", [f"{P}x{A}" for P, A in FEATURE_POOLS] + ["ejected", "no_pods_tree"])
def test_model_ids_with_hostile_tables(pool, eng):
    if pool in SPECIAL:
        p = SPECIAL[pool](eng)
    else:
        p = Epoch(eng, bench_pool(*map(int, pool.split("x"))))
    rng = np.random.default_rng(7 + len(pool))
    for R, fi in zip(BATCHES, (0, FIRST, 5, FIRST, 0, FIRST)):
        done = check_models(eng, p, R, rng, fi)
        if R <= 4096:                         # the doorbell's capacity
            ids = done[0]
    eng.stream_open()
    try:
        res = MC.resolve_call(p.models, p.snap.adapter_id, ids, SEED, FIRST)
        want = mpicks(res, p.cl.picks(np.ascontiguousarray(res["req"]), SEED))
        assert eng.stream_submit_models(p.ep, SEED, ids, FIRST).tobytes() == want.tobytes()
    finally:
        eng.stream_close()


# ---- fallback rows and affinity -----------------------------------------------------------------------------
@pytest.mark.parametrize("pool", [f"{P}x{A}" for P, A in FEATURE_POOLS] + sorted(SPECIAL))
def test_fallback_rows(pool, eng):
    p = SPECIAL[pool](eng) if pool in SPECIAL else Epoch(eng, bench_pool(*map(int, pool.split("x"))))
    rng = np.random.default_rng(17 + len(pool))
    for R in (1, 31, 257, 4099):
        reqs = E.edge_requests(p.cl, R, SEED, rng)
        want, rows = p.cl.fallbacks(reqs, SEED, K)
        for k in (1, K):
            run_family(eng, "fallbacks", dict(ep=p.ep, seed=SEED, reqs=reqs, R=R, k=k), want, rows)


def affinity_pod_keys(P, rng):
    """Random pod keys with one duplicated pair (a tie broken to the lower pod)."""
    keys = rng.integers(0, 1 << 64, size=P, dtype=np.uint64)
    if P >= 2:
        keys[P - 1] = keys[P // 3]
    return keys


def affinity_keys(p, reqs, pod_keys, rng):
    """Keys 0, 2^64-1, a pod's own hash h_p (its score is 0) and random ones."""
    keys = reqs["rand_key"].copy()
    kind = rng.integers(0, 4, len(keys))
    keys[kind == 0] = 0
    keys[kind == 1] = np.uint64(E.M64)
    h = AR.mix(pod_keys)
    keys[kind == 2] = h[rng.integers(0, len(h), int((kind == 2).sum()))]
    return keys


@pytest.mark.parametrize("pool", ["33x1", "4097x64"] + sorted(SPECIAL))
def test_affinity(pool, eng):
    p = SPECIAL[pool](eng) if pool in SPECIAL else Epoch(eng, bench_pool(*map(int, pool.split("x"))))
    rng = np.random.default_rng(23 + len(pool))
    pod_keys = affinity_pod_keys(p.snap.P, rng)
    eng.upload_pod_keys(p.ep, pod_keys)
    long_in_tail = False
    for R in (1, 33, 257, 4099):
        reqs = E.edge_requests(p.cl, R, SEED, rng)
        reqs["rand_key"] = affinity_keys(p, reqs, pod_keys, rng)
        if pool == "mixed":
            # the batch's last request, alone in the last partial warp, takes the 257-pod list
            reqs["adapter_id"][-1], reqs["flags"][-1] = 0, 0
        ok, offsets, pods = p.cl.csr(reqs)
        n = np.diff(offsets)
        long_in_tail |= bool(R % 32 and (n[R - R % 32:] > 32).any())
        if pool == "mixed" and R >= 33:
            assert (n > 32).any() and ((n > 0) & (n <= 32)).any()
        pick, rows = AR.affinity_rows(reqs["rand_key"], ok, offsets, pods, pod_keys, K)
        want = p.cl.picks(reqs, SEED)
        want["pod_idx"] = np.where(ok, pick, -1)
        for k in (0, 1, K):
            run_family(eng, "affinity", dict(ep=p.ep, reqs=reqs, R=R, k=k), want, rows)
        # model ids at affinity keys
        ids = E.model_ids(p.pm.n_models, R, rng)
        mreqs, resolved, target = AR.affinity_resolve(p.pm, ids, reqs["rand_key"])
        mok, moff, mpods = p.cl.csr(mreqs, keep=resolved)
        mpick, mrows = AR.affinity_rows(mreqs["rand_key"], mok, moff, mpods, pod_keys, K)
        mwant = AR.as_mpicks(p.cl.picks(mreqs, 0), resolved, target, mpick)
        for k in (0, 1, K):
            run_family(eng, "models_affinity", dict(ep=p.ep, ids=ids, keys=reqs["rand_key"], R=R, k=k), mwant, mrows)
    if pool == "mixed":
        assert long_in_tail


# ---- retries ---------------------------------------------------------------------------------------------
def retry_rows(p, R, rng):
    """The tried-pod rows of test_gpu_retry (every kind), with templates from the CPU lists."""
    P = p.snap.P
    t = [[], [-1, P, 32767, -32768], [int(np.argmax(p.snap.q))], [31, 32, P - 1], [0]]
    for k in (1, 9, 32):
        r = rng.integers(0, P, size=k).tolist()
        if k > 2:
            r[1] = r[0]
            r[-1] = P + 3
        t.append(r)
    t += [lst.tolist() for lst in p.cl.lists if 0 < len(lst) <= N.LIG_MAX_EXCLUDED][:3]
    return rows_for(t, R, 5, rng)


def retry_targets(p, ids, rng):
    """Targets 255, 254, nt, nt-1 and ones the model has."""
    nt = np.array([int(p.pm.target_offsets[m + 1] - p.pm.target_offsets[m]) if m < p.pm.n_models else 3
                   for m in ids.tolist()], dtype=np.int64)
    pick = rng.integers(0, 5, len(ids))
    tg = np.where(pick == 0, 255, np.where(pick == 1, 254, np.where(pick == 2, nt, np.where(
        pick == 3, nt - 1, rng.integers(0, np.maximum(nt, 1))))))
    return np.ascontiguousarray(np.clip(tg, 0, 255).astype(np.uint8))


@pytest.mark.parametrize("pool", ["1x0", "33x1", "4097x64", "ejected", "no_pods_tree"])
def test_retries(pool, eng):
    p = SPECIAL[pool](eng) if pool in SPECIAL else Epoch(eng, bench_pool(*map(int, pool.split("x"))))
    rng = np.random.default_rng(29 + len(pool))
    kw = dict(nodes=p.nodes)
    for R in (1, 33, 257) + ((4099,) if p.snap.P <= 257 else ()):
        reqs = E.edge_requests(p.cl, R, SEED, rng)
        ex = retry_rows(p, R, rng)
        a = dict(ep=p.ep, seed=SEED, reqs=reqs, R=R, ex=ex, w=ex.shape[1])
        if p.ejected is None:
            want = RR.retry_batch(p.snap, reqs, ex, SEED, **kw)
            want_f, rows = RF.retry_fallback_batch(p.snap, reqs, ex, SEED, K, **kw)
        else:
            want = ER.retry_batch(p.snap, p.ejected, reqs, ex, SEED, **kw)
            want_f, rows = ER.retry_fallback_batch(p.snap, p.ejected, reqs, ex, SEED, K, **kw)
        assert want_f.tobytes() == want.tobytes()
        run_family(eng, "retry", a, want)
        for k in (1, K):
            run_family(eng, "retry_fallbacks", dict(a, k=k), want, rows)
        # model-id retries on the hostile table
        ids = E.model_ids(p.pm.n_models, R, rng)
        tg = retry_targets(p, ids, rng)
        fi = FIRST if R & 1 else 0
        mwant, mrows = MR.retry_fallback_batch(p.snap, p.pm, ids, tg, ex, SEED, K, fi, nodes=p.nodes,
                                               ejected=p.ejected)
        m = dict(a, ids=ids, tg=tg, fi=fi)
        run_family(eng, "model_retry", m, mwant)
        for k in (1, K):
            run_family(eng, "model_retry_fallbacks", dict(m, k=k), mwant, mrows)


# ---- in-batch feedback and the feedback chain --------------------------------------------------------------
@pytest.mark.parametrize("pool", ["33x5", "257x64", "ejected", "no_pods_tree"])
def test_feedback_and_chain(pool, eng):
    p = SPECIAL[pool](eng) if pool in SPECIAL else Epoch(eng, bench_pool(*map(int, pool.split("x"))))
    rng = np.random.default_rng(37 + len(pool))
    eng.set_filter_tree(p.nodes)             # the tree in force rebuilds the windows' tables
    try:
        check_feedback_and_chain(eng, p, rng)
    finally:
        eng.set_filter_tree(None)


def check_feedback_and_chain(eng, p, rng):
    snap = p.snap
    window = 37
    # in-batch feedback: one chain call with window = sub_batch; the batch ends mid-window on a partial warp
    reqs = E.edge_requests(p.cl, 257, SEED, rng)
    want = MR.run_chain_snapshot(snap, [(reqs, SEED)], window, nodes=p.nodes, ejected=p.ejected)[0][0]
    d_in = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
    d_out = torch.full((257 * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    eng.schedule_batch_feedback_device(p.ep, SEED, d_in.data_ptr(), 257, d_out.data_ptr(), window)
    torch.cuda.synchronize()
    assert d_out.cpu().numpy().tobytes() == want.tobytes()
    # a chain of every kind of call, windows crossing call boundaries, the last call ending mid-window
    calls, raw, ks = [], [], []
    fi = FIRST
    for j, (kind, R) in enumerate([("plain", 31), ("model", 33), ("retry", 1), ("model_retry", 40),
                                   ("plain", 255), ("model", 31), ("retry", 33), ("model_retry", 257)]):
        k = [0, 1, K][j % 3]
        s = SEED + j
        if kind in ("plain", "retry"):
            r = E.edge_requests(p.cl, R, s, rng)
            if kind == "plain":
                calls.append((r, s))
                raw.append((kind, r))
            else:
                ex = retry_rows(p, R, rng)
                calls.append(CR.retry_call(r, ex, s))
                raw.append((kind, r, ex))
        else:
            ids = E.model_ids(p.pm.n_models, R, rng)
            if kind == "model":
                calls.append(MC.model_call(p.models, snap.adapter_id, ids, s, fi))
                raw.append((kind, ids, fi))
            else:
                tg, ex = retry_targets(p, ids, rng), retry_rows(p, R, rng)
                calls.append(MR.model_retry_call(p.pm, ids, tg, ex, s, fi))
                raw.append((kind, ids, tg, ex, fi))
            fi = (fi + R) & E.M64
        ks.append(k)
    assert sum(len(c) for c, _ in calls) % window and sum(len(c) for c, _ in calls) % 32
    want, want_rows, want_loads = MR.run_chain_snapshot(snap, calls, window, ks, nodes=p.nodes, ejected=p.ejected)
    for device in (False, True):
        eng.feedback_chain_reset()
        for i, ((c, s), k, r) in enumerate(zip(calls, ks, raw)):
            got, rows = chain_call(eng, p.ep, s, r, k, window, device)
            assert got.tobytes() == want[i].tobytes(), (i, r[0], k, device)
            if k:
                assert rows.tobytes() == want_rows[i].tobytes(), (i, r[0], k, device)
        loads = np.zeros(snap.P, dtype=np.int32)
        eng.schedule_batch_feedback_chain(p.ep, SEED, np.zeros(0, dtype=REQ_DTYPE), window, loads=loads)
        assert np.array_equal(loads, want_loads), device


def chain_call(eng, ep, seed, r, k, window, device):
    """One chain call of kind r[0]: host (pageable) or device buffers; (out, rows or None)."""
    kind = r[0]
    form = "device" if device else "pageable"
    suffix = "_device" if device else "_ptr"
    if kind in ("plain", "model"):
        if kind == "plain":
            reqs = r[1]
            R = len(reqs)
            head, data, odt = ["schedule_batch_feedback_chain", ep, seed], [In(reqs), R], PICK_DTYPE
        else:
            _, ids, fi = r
            R = len(ids)
            head, data, odt = ["schedule_models_batch_feedback_chain", ep, seed, fi], [In(ids), R], MPICK_DTYPE
        name = head[0] + ("_fallbacks" if k else "") + suffix
        rest = [Out(odt, (R,))] + ([k, Out(np.int16, (R, k))] if k else []) + [window, 0]
        got = call(eng, name, head[1:] + data + rest, form)
    else:
        if kind == "retry":
            _, reqs, ex = r
            R = len(reqs)
            head, data, odt = ["schedule_batch_feedback_chain_excluding", ep, seed], [In(reqs), R], PICK_DTYPE
        else:
            _, ids, tg, ex, fi = r
            R = len(ids)
            head, data, odt = (["schedule_models_batch_feedback_chain_excluding", ep, seed, fi],
                               [In(ids), In(tg), R], MPICK_DTYPE)
        name = head[0] + ("_fallbacks" if k else "") + suffix
        rest = [In(ex), ex.shape[1], Out(odt, (R,))] + ([k, Out(np.int16, (R, k))] if k else []) + [window, 0]
        got = call(eng, name, head[1:] + data + rest, form)
    return got[0], (got[1] if k else None)
