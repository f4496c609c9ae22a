"""The inputs of the class tables that come from outside the library, on the device:

* thresholds at the edges of their Go types (int64 queues, binary64 KV incl. NaN, infinities, signed
  zeros, denormals, one ulp either side of a pod) through all three built-in builds, the caller-tree
  build and every consumer, against the class-table oracle and the port;
* lig_set_thresholds on resident epochs: built-in epochs are rebuilt in place (after an _async upload
  and after a delta, across the compact / strided switch, ordered behind work already queued and
  around an open doorbell stream), caller-tree epochs are left alone;
* junk in the padding pods and the tail of a device blob, which every kernel must ignore;
* host uploads refused before anything is evicted."""
import numpy as np
import pytest
import torch

import threshold_grid as TG
from filter_tree_ref import random_tree
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine, EngineGroup
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, pack_models
from oracle import binding
from test_gpu_filter_tree import ref_tables
from test_gpu_snapshot_mutation import (PodState, build_variant, class_requests, doorbell_picks, model_picks,
                                        queue_picks, random_state, reference)

pytestmark = pytest.mark.gpu

DEFAULTS = (0.8, 5, 50)


@pytest.fixture(autouse=True)
def port_defaults():
    yield
    binding.set_thresholds(*DEFAULTS)


def edge_state(P, A, seed):
    """A random pool with every seventh pod on the edges of the queue and KV types."""
    s = random_state(P, A, seed) if P else PodState(A, [], [], [], [])
    for k, p in enumerate(range(0, P, 7)):
        s.q[p] = TG.Q_POD_EDGE[k % 2]
        s.kv[p] = TG.KV_POD_EDGE[k % len(TG.KV_POD_EDGE)]
    return s


def engine(monkeypatch, P, A, R=1 << 14, env=None):
    with monkeypatch.context() as m:
        for k, v in (env or {}).items():
            m.setenv(k, v)                                   # read at lig_create
        return Engine(0, max_pods=max(P, 1), max_adapters=max(A, 1), max_batch=R)


def classtab(state, thr):
    p = state.packed()
    return binding.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap, thresholds=thr,
                              nthreads=binding.hardware_threads())


def tables(e, ep, A, P):
    return [e.read_class(ep, bool(c), a, P) for c in (0, 1) for a in range(A + 1)]


def as_lists(t):
    return [(st, n, lst.tolist()) for st, n, lst in t]


def klass(reqs, A):
    return (reqs["flags"] & 1).astype(np.int64), np.minimum(reqs["adapter_id"].astype(np.int64) % (1 << 32), A)


def assert_lists(offsets, pods, reqs, out, want_tables, A, label):
    """lig_filter_batch lists: a LIG_OK request's list is its class's survivors, other requests none."""
    crit, a = klass(reqs, A)
    for i in range(len(reqs)):
        st, n, lst = want_tables[int(crit[i]) * (A + 1) + int(a[i])]
        got = pods[offsets[i]:offsets[i + 1]].tolist()
        assert got == (lst if out["status"][i] == N.LIG_OK else []), (label, i)


def consumers(e, ep, seed, reqs, ids, scan, P):
    """Every consumer of the epoch's tables, picks as bytes."""
    out = {"host": e.schedule_batch(ep, seed, reqs)}
    out["queue0"], out["queue1"] = queue_picks(e, ep, reqs, seed)
    out["doorbell"] = doorbell_picks(e, ep, reqs, seed)
    f_out, f_off, f_pods = e.filter_batch(ep, seed, reqs)
    out["filter"], out["filter_lists"] = f_out, (f_off, f_pods)
    if ids is not None:
        out["models"] = model_picks(e, ep, ids, seed)
        out["models_host"] = e.schedule_models_batch(ep, seed, ids)
        n = min(len(ids), N.load().lig_stream_capacity())
        e.stream_open()
        try:
            out["doorbell_models"] = e.stream_submit_models(ep, seed, np.ascontiguousarray(ids[:n]))
        finally:
            e.stream_close()
    if scan:
        out["scan"], out["scan_masks"] = e.schedule_scan(ep, seed, reqs, True, (P + 31) // 32)
    return out


def check_against_oracle(got, state, thr, tab, reqs, ids, seed, label):
    P, A = state.P, state.A
    want_t = [tab.klass(bool(c), a) for c in (0, 1) for a in range(A + 1)]
    host = tab.schedule_batch(reqs, seed)
    assert got["host"].tobytes() == host.tobytes(), label
    for k in ("queue0", "filter"):
        assert got[k].tobytes() == host.tobytes(), (label, k)
    assert got["queue1"].tobytes() == tab.schedule_batch(reqs, seed + 1).tobytes(), label     # batch b: seed + b
    assert got["doorbell"].tobytes() == host[:len(got["doorbell"])].tobytes(), label
    assert_lists(*got["filter_lists"], reqs, host, want_t, A, label)
    binding.set_thresholds(*thr)
    pool = binding.Pool(state.records())
    n = min(len(reqs), 4096)
    want, masks = pool.schedule_batch(state.names()[:-1], WL.UNKNOWN_MODEL, np.ascontiguousarray(reqs[:n]), seed, True)
    assert host[:n].tobytes() == want.tobytes(), label                  # the two references agree here too
    if "scan" in got:
        assert got["scan"].tobytes() == host.tobytes(), label
        assert np.array_equal(got["scan_masks"][:n], masks), label
    if ids is not None:
        wm = binding.Models(WL.model_records(WL.make_models(A))).schedule_batch(pool, ids, seed)
        assert got["models"].tobytes() == wm.tobytes(), label
        assert got["models_host"].tobytes() == wm.tobytes(), label
        assert got["doorbell_models"].tobytes() == wm[:len(got["doorbell_models"])].tobytes(), label
    binding.set_thresholds(*DEFAULTS)
    return want_t


def same_consumers(got, want, label, skip=("scan", "scan_masks")):
    for k in want:
        if k in skip:
            continue
        if k == "filter_lists":
            assert all(np.array_equal(x, y) for x, y in zip(got[k], want[k])), (label, k)
        else:
            assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), (label, k)


# ---- B. thresholds at their edges ------------------------------------------------------------------
SHAPES = [(1, 8, "fast"), (33, 16, "fast"), (1000, 32, "fast"), (33, 0, "fast"), (4097, 24, "staged"),
          (20001, 12, "unstaged")]


class Trio:
    """The built-in tree with tables in shared memory and in global memory, and defaultFilter as a
    caller tree carrying the same thresholds."""

    def __init__(self, monkeypatch, P, A, R=1 << 14):
        self.b = engine(monkeypatch, P, A, R)
        self.g = engine(monkeypatch, P, A, R, {"LIG_TAB_SMEM": "0"})
        self.t = engine(monkeypatch, P, A, R)
        self.ep = 0

    def close(self):
        for e in (self.b, self.g, self.t):
            e.close()

    def upload(self, thr, packed, models):
        self.ep += 1
        for e in (self.b, self.g):
            e.set_thresholds(*thr)
        self.t.set_filter_tree(TG.default_tree(*thr))
        for e in (self.b, self.g, self.t):
            e.upload_snapshot(self.ep, packed)
            if models is not None:
                e.upload_models(self.ep, models)
        return self.ep


def run_grid(trio, state, thr_list, reqs, ids, label):
    P, A = state.P, state.A
    packed = state.packed()
    models = pack_models(WL.make_models(A), packed) if ids is not None else None
    for thr in thr_list:
        lab = (label, thr)
        ep = trio.upload(thr, packed, models)
        tab = classtab(state, thr)
        got = consumers(trio.b, ep, 7, reqs, ids, True, P)
        want_t = check_against_oracle(got, state, thr, tab, reqs, ids, 7, lab)
        assert as_lists(tables(trio.b, ep, A, P)) == [(s, n, lst) for s, n, lst in want_t], lab
        # the caller-tree build gives the same survivor sets and every consumer the same picks
        assert as_lists(tables(trio.t, ep, A, P)) == [(s, n, lst) for s, n, lst in want_t], lab
        same_consumers(consumers(trio.t, ep, 7, reqs, ids, False, P), got, lab + ("caller tree",))
        g_q = queue_picks(trio.g, ep, reqs, 7)
        assert g_q[0].tobytes() == got["queue0"].tobytes() and g_q[1].tobytes() == got["queue1"].tobytes(), lab


@pytest.mark.parametrize("P,A,variant", SHAPES, ids=[f"P={p}-A={a}" for p, a, _ in SHAPES])
def test_builtin_thresholds_at_the_edges(P, A, variant, monkeypatch):
    assert build_variant(P) == variant
    state = edge_state(P, A, seed=P + A)
    rng = np.random.default_rng(P * 31 + A)
    thr_list = TG.triples(state.q, state.kv, 16 if P <= 1000 else 6, rng)
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(3000, A, seed=P)]))
    ids = WL.make_model_requests(3000, A, seed=P + 1) if A else None
    trio = Trio(monkeypatch, P, A)
    try:
        run_grid(trio, state, thr_list, reqs, ids, (P, A))
    finally:
        trio.close()


def test_builtin_thresholds_at_the_edges_C4(monkeypatch):
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=44)
    state = PodState(c["A"], snap.packed.kv, snap.q64, snap.max_active64, snap.active)
    thr_list = [(np.inf, TG.INT64_MAX, TG.INT32_MAX + 1), (np.nan, TG.INT32_MIN - 1, TG.INT64_MAX),
                (-0.0, TG.INT64_MAX, TG.INT64_MIN), (5e-324, 1 << 32, 1 << 32)]
    reqs = WL.make_requests(20000, c["A"], seed=45)
    trio = Trio(monkeypatch, c["P"], c["A"], R=20000)
    try:
        run_grid(trio, state, thr_list, reqs, WL.make_model_requests(20000, c["A"], seed=46), "C4")
    finally:
        trio.close()


@pytest.mark.parametrize("P,A", [(33, 4), (1000, 8)])
def test_caller_trees_with_thresholds_at_the_edges(P, A, monkeypatch):
    """LOW_QUEUEING and NO_QUEUE_AND_LOW_KV nodes with grid thresholds at the root, after each range
    node, on both branches of a predicate, and random trees with grid thresholds."""
    state = edge_state(P, A, seed=5 + P)
    rec, names = state.records(), state.names()
    qs, kvs = TG.q_grid(state.q), TG.kv_grid(state.kv)
    rng = np.random.default_rng(P)
    trees = []
    for q, kv in [(TG.INT64_MAX, np.inf), (TG.INT64_MIN, np.nan), (TG.INT32_MAX + 1, -0.0), (TG.INT32_MIN - 1, 5e-324),
                  (1 << 32, TG.DBL_MAX)]:
        trees += TG.placed_trees(q, kv)
    trees += [TG.with_grid_thresholds(random_tree(rng), rng, qs, kvs) for _ in range(40)]
    reqs = class_requests(A)
    e = engine(monkeypatch, P, A)
    try:
        for i, tree in enumerate(trees):
            e.set_filter_tree(tree)
            e.upload_snapshot(i + 1, state.packed())
            want = ref_tables(tree, rec, names)
            flat = [(st, len(idx), idx) for row in want for st, idx in row]
            assert as_lists(tables(e, i + 1, A, P)) == flat, i
            out, off, pods = e.filter_batch(i + 1, 3, reqs)
            assert_lists(off, pods, reqs, out, flat, A, i)
    finally:
        e.close()


# ---- C. lig_set_thresholds on resident epochs -----------------------------------------------------------
def expect_epoch(e, ep, state, thr, reqs, ids, label):
    got = consumers(e, ep, 11, reqs, ids, True, state.P)
    want_t = check_against_oracle(got, state, thr, classtab(state, thr), reqs, ids, 11, label)
    assert as_lists(tables(e, ep, state.A, state.P)) == want_t, label


def test_set_thresholds_rebuilds_resident_epochs(monkeypatch):
    P, A = 700, 20
    s1, s2 = edge_state(P, A, 1), edge_state(P, A, 2)
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(4000, A, seed=3)]))
    ids = WL.make_model_requests(4000, A, seed=4)
    T1, T2, T3 = (np.inf, TG.INT64_MAX, TG.INT32_MAX + 1), (-0.0, TG.INT32_MIN - 1, TG.INT64_MIN), (0.3, 40, 1 << 32)
    e = engine(monkeypatch, P, A)
    try:
        e.upload_snapshot(1, s1.packed())
        e.upload_models(1, pack_models(WL.make_models(A), s1.packed()))
        e.upload_snapshot(2, s2.packed(), block=False)              # its build may still be pending
        e.upload_models(2, pack_models(WL.make_models(A), s2.packed()), block=False)
        e.set_thresholds(*T1)
        for ep, s in ((1, s1), (2, s2)):
            expect_epoch(e, ep, s, T1, reqs, ids, ("T1", ep))
        # a delta-made epoch (evicts 1), then a rebuild of it and of its base
        s3 = s2.copy()
        dirty = [0, 7, P - 1]
        for p in dirty:
            s3.q[p], s3.kv[p], s3.active[p] = TG.INT32_MIN, np.nan, [1, 2]
        d = dict(pod_idx=dirty, kv=s3.kv[dirty], q=s3.q[dirty].astype(np.int32),
                 n_active=s3.n_active()[dirty].astype(np.uint16), max_active=np.clip(s3.ma[dirty], 0, 65535),
                 adapter_offsets=[0, 2, 4, 6], adapter_ids=[1, 2] * 3)
        e.update_snapshot(3, 2, **d)
        e.upload_models(3, pack_models(WL.make_models(A), s3.packed()))
        e.set_thresholds(*T2)
        for ep, s in ((2, s2), (3, s3)):
            expect_epoch(e, ep, s, T2, reqs, ids, ("T2", ep))
        # a feedback chain on the delta epoch keeps the thresholds it started with
        e.set_thresholds(*T3)
        chain_reqs = WL.make_requests(600, A, seed=9)
        first = e.schedule_batch_feedback_chain(3, 21, np.ascontiguousarray(chain_reqs[:250]), 100)
        e.set_thresholds(*T2)
        second = e.schedule_batch_feedback_chain(3, 21, np.ascontiguousarray(chain_reqs[250:]), 100)
        picks = np.concatenate([first, second])
        want, _, _ = reference(s3, chain_reqs, 21, 100, thresholds=T3)
        assert picks.tobytes() == want.tobytes()
        expect_epoch(e, 3, s3, T2, reqs, ids, ("T2 after chain", 3))
        # a caller-tree epoch keeps its tables byte for byte; the built-in epoch beside it is rebuilt
        tree = TG.placed_trees(30, 0.5)[3]
        e.set_filter_tree(tree)
        e.upload_snapshot(4, s1.packed())                           # evicts 2
        before = as_lists(tables(e, 4, A, P))
        e.set_thresholds(*T1)
        assert as_lists(tables(e, 4, A, P)) == before
        e.set_filter_tree(None)
        expect_epoch(e, 3, s3, T1, reqs, ids, ("T1 beside a caller tree", 3))
    finally:
        e.close()


def test_set_thresholds_switches_compact_and_strided_tables(monkeypatch):
    """4096 identical pods with room that all hold all 1024 adapters, queues of 100: at the default
    thresholds every critical class shares the default list and every sheddable one drops; with
    queueingThresholdLoRA = INT64_MAX every critical class takes the affinity branch and owns a list of
    all 4096 pods, 8 MB of lists, past the 4 MB compact pool."""
    P, A = 4096, 1024
    state = PodState(A, np.full(P, 0.5), np.full(P, 100), np.full(P, 65535), [list(range(A))] * P)
    packed = state.packed()
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A, copies=1), WL.make_requests(20000, A, seed=1)]))
    ids = WL.make_model_requests(20000, A, seed=2)
    e = engine(monkeypatch, P, A, R=1 << 15)
    try:
        e.upload_snapshot(1, packed)
        e.upload_models(1, pack_models(WL.make_models(A), packed))
        infos = []
        for thr in (DEFAULTS, (np.inf, TG.INT64_MAX, TG.INT64_MAX), DEFAULTS):
            e.set_thresholds(*thr)
            info = e.pick_kernel_info(1)
            infos.append(info)
            expect_epoch(e, 1, state, thr, reqs, ids, thr)
        assert infos[0]["table_bytes"] > 0 and infos[0]["tables_in_smem"], infos
        assert infos[1]["table_bytes"] == 0 and not infos[1]["tables_in_smem"], infos
        assert infos[2] == infos[0], infos
    finally:
        e.close()


def test_set_thresholds_waits_for_queued_readers(monkeypatch):
    """Work enqueued on a held stream before the call sees the old thresholds' tables, work enqueued
    after it the new ones.  The pool has no KV of -Inf, which would leave every least-KV stage empty
    at any thresholds."""
    P, A, R = 900, 16, 5000
    state = random_state(P, A, 12)
    packed = state.packed()
    reqs = WL.make_requests(R, A, seed=13)
    ids = WL.make_model_requests(R, A, seed=14)
    T_new = (np.inf, TG.INT64_MAX, TG.INT64_MIN)
    e = engine(monkeypatch, P, A, R)
    try:
        e.upload_snapshot(1, packed)
        e.upload_models(1, pack_models(WL.make_models(A), packed))
        old = (e.schedule_batch(1, 5, reqs), e.schedule_models_batch(1, 5, ids), e.filter_batch(1, 5, reqs))
        d_reqs = torch.from_numpy(reqs.view(np.uint8).reshape(-1).copy()).cuda()
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()

        def enqueue(stream):
            d_out = torch.zeros(R * 8, dtype=torch.uint8, device="cuda")
            d_m = torch.zeros(R * 4, dtype=torch.uint8, device="cuda")
            d_f = torch.zeros(R * 8, dtype=torch.uint8, device="cuda")
            d_off = torch.zeros(R + 1, dtype=torch.int64, device="cuda")
            cap = R * P
            d_pods = torch.zeros(cap, dtype=torch.int16, device="cuda")
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(100_000_000)
            e.schedule_batch_device(1, 5, d_reqs.data_ptr(), R, d_out.data_ptr(), stream.cuda_stream)
            e.schedule_models_batches_device(1, 5, 0, [d_ids.data_ptr()], R, [d_m.data_ptr()], stream.cuda_stream)
            e.filter_batch_device(1, 5, d_reqs.data_ptr(), R, d_f.data_ptr(), d_off.data_ptr(), d_pods.data_ptr(),
                                  cap, stream.cuda_stream)
            return d_out, d_m, d_f, d_off, d_pods

        def read(bufs):
            torch.cuda.synchronize()
            d_out, d_m, d_f, d_off, d_pods = bufs
            off = d_off.cpu().numpy()
            return (d_out.cpu().numpy().view(PICK_DTYPE), d_m.cpu().numpy().view(MPICK_DTYPE),
                    (d_f.cpu().numpy().view(PICK_DTYPE), off, d_pods[: int(off[-1])].cpu().numpy().view(np.uint16)))

        held = torch.cuda.Stream()
        before = enqueue(held)
        assert not held.query()
        e.set_thresholds(*T_new)                 # returns after the held stream's readers drained
        assert held.query()
        got = read(before)
        assert got[0].tobytes() == old[0].tobytes() and got[1].tobytes() == old[1].tobytes()
        assert all(np.array_equal(x, y) for x, y in zip(got[2], old[2]))
        expect_epoch(e, 1, state, T_new, np.ascontiguousarray(reqs[:2000]), ids[:2000], "after")
        after = read(enqueue(torch.cuda.Stream()))
        assert after[0].tobytes() == e.schedule_batch(1, 5, reqs).tobytes()
        assert after[1].tobytes() == e.schedule_models_batch(1, 5, ids).tobytes()
        assert after[0].tobytes() != old[0].tobytes()
    finally:
        e.close()


def test_set_thresholds_with_an_open_doorbell(monkeypatch):
    P, A = 300, 12
    state = random_state(P, A, 22)
    packed = state.packed()
    n = N.load().lig_stream_capacity()
    reqs = WL.make_requests(n, A, seed=23)
    ids = WL.make_model_requests(n, A, seed=24)
    T_new = (-np.inf, TG.INT64_MIN, TG.INT64_MAX)
    e = engine(monkeypatch, P, A, n)
    try:
        e.upload_snapshot(1, packed)
        e.upload_models(1, pack_models(WL.make_models(A), packed))
        old = (e.schedule_batch(1, 8, reqs), e.schedule_models_batch(1, 8, ids))
        e.stream_open()
        try:
            b = (e.stream_submit(1, 8, reqs), e.stream_submit_models(1, 8, ids))
            e.set_thresholds(*T_new)
            a = (e.stream_submit(1, 8, reqs), e.stream_submit_models(1, 8, ids))
        finally:
            e.stream_close()
        assert b[0].tobytes() == old[0].tobytes() and b[1].tobytes() == old[1].tobytes()
        tab = classtab(state, T_new)
        assert a[0].tobytes() == tab.schedule_batch(reqs, 8).tobytes()
        assert a[0].tobytes() != old[0].tobytes()
        assert a[1].tobytes() == e.schedule_models_batch(1, 8, ids).tobytes()
    finally:
        e.close()


def test_group_set_thresholds_rebuilds_the_member(monkeypatch):
    P, A = 500, 10
    state = edge_state(P, A, 31)
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(3000, A, seed=32)]))
    thr = (5e-324, TG.INT32_MAX + 1, TG.INT32_MIN - 1)
    try:
        g = EngineGroup([0], max_pods=P, max_adapters=A, max_batch=1 << 14)
    except N.LigError as err:
        pytest.skip(f"no NCCL: {err}")
    with g:
        g.upload_snapshot(1, state.packed())
        g.set_thresholds(*thr)
        tab = classtab(state, thr)
        assert g.schedule_batch(1, 4, reqs).tobytes() == tab.schedule_batch(reqs, 4).tobytes()
        assert as_lists(tables(g.member(0), 1, A, P)) == [tab.klass(bool(c), a) for c in (0, 1) for a in range(A + 1)]


# ---- D. junk in the padding of a device blob ------------------------------------------------------------
def poison(blob, P, A, kv_val, q_val):
    """The blob with junk in every padding pod, every tail bit set and 0xFF after the bitmap."""
    b = blob.copy()
    W = (P + 31) // 32
    Ppad = 32 * W
    b[0: 8 * Ppad].view(np.float64)[P:] = kv_val
    b[8 * Ppad: 12 * Ppad].view(np.int32)[P:] = q_val
    b[12 * Ppad: 14 * Ppad].view(np.uint16)[P:] = 0
    b[14 * Ppad: 16 * Ppad].view(np.uint16)[P:] = 65535
    end = 16 * Ppad + 4 * A * W
    if A and P & 31:
        bm = b[16 * Ppad: end].view(np.uint32).reshape(A, W)
        bm[:, W - 1] |= np.uint32(~((1 << (P & 31)) - 1) & 0xFFFFFFFF)
    b[end:] = 0xFF
    return b


POISONS = [(np.nan, TG.INT32_MIN), (-np.inf, 0), (-0.0, TG.INT32_MIN), (0.0, 0)]
JUNK_SHAPES = [(P, A) for P in (0, 1, 31, 32, 33, 4095, 4097, 20001) for A in (0, 1, 64)]


def one_node_trees():
    F = N.LigFilterNode
    out = [[F(k, -1, -1, -1, 0, 0.8)] for k in range(9)]
    out.append([F(N.LIG_F_LOW_QUEUEING, -1, -1, -1, TG.INT64_MAX, 0.0)])       # keeps every pod
    rng = np.random.default_rng(3)
    out += [random_tree(rng) for _ in range(2)]
    return out


def epoch_results(e, ep, P, A, reqs, ids, scan):
    out = consumers(e, ep, 13, reqs, ids, scan, P)
    out["tables"] = tables(e, ep, A, P)
    return out


def same_results(got, want, label):
    assert as_lists(got["tables"]) == as_lists(want["tables"]), label
    same_consumers({k: v for k, v in got.items() if k != "tables"},
                   {k: v for k, v in want.items() if k != "tables"}, label, skip=())


def upload_blob(e, ep, P, A, blob, comm=False):
    d = torch.from_numpy(blob).cuda()
    torch.cuda.synchronize()
    if comm:
        e.comm_upload_snapshot_device(ep, P, A, d.data_ptr(), 0, 0)
    else:
        e.upload_snapshot_device(ep, P, A, d.data_ptr(), 0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("P,A", JUNK_SHAPES, ids=[f"P={p}-A={a}" for p, a in JUNK_SHAPES])
def test_padding_junk_is_ignored(P, A, monkeypatch):
    state = edge_state(P, A, seed=7 * P + A)
    packed = state.packed()
    clean = packed.blob()
    assert len(clean) == N.load().lig_snapshot_bytes(P, A)
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(2000, A, seed=P)]))
    ids = WL.make_model_requests(2000, A, seed=A) if A else None
    models = pack_models(WL.make_models(A), packed) if A else None
    e = engine(monkeypatch, P, A)
    ep = 0

    def put(blob):
        nonlocal ep
        ep += 1
        upload_blob(e, ep, P, A, blob)
        if models is not None:
            e.upload_models(ep, models)
        return ep

    try:
        # built-in tree: every consumer, in-batch feedback and a feedback chain
        want = epoch_results(e, put(clean), P, A, reqs, ids, True)
        fb_want = e.schedule_batch_feedback_chain(ep, 3, reqs, 64)
        e.feedback_chain_reset()
        for kv, q in POISONS:
            label = (P, A, kv, q)
            bad = poison(clean, P, A, kv, q)
            assert P % 32 == 0 or A == 0 or not np.array_equal(bad, clean)
            got = epoch_results(e, put(bad), P, A, reqs, ids, True)
            same_results(got, want, label)
            fb = e.schedule_batch_feedback_chain(ep, 3, reqs, 64)
            e.feedback_chain_reset()
            assert fb.tobytes() == fb_want.tobytes(), label
        # in-batch feedback on the poisoned epoch against its sequential definition on the clean pool
        if P:
            from test_gpu_snapshot_mutation import assert_feedback, run_feedback
            assert_feedback(run_feedback(e, ep, 5, reqs, P, 50), reference(state, reqs, 5, 50)[:2], (P, A, "feedback"))
        # caller trees: one-node trees of every kind, LOW_QUEUEING that keeps everything, random trees
        for i, tree in enumerate(one_node_trees()):
            e.set_filter_tree(tree)
            kv, q = POISONS[i % len(POISONS)]
            w = epoch_results(e, put(clean), P, A, reqs, ids, False)
            g = epoch_results(e, put(poison(clean, P, A, kv, q)), P, A, reqs, ids, False)
            same_results(g, w, (P, A, "tree", i))
        e.set_filter_tree(None)
        # a delta on the poisoned base equals the same delta on the clean base
        if P:
            delta = dict(pod_idx=[P - 1], kv=[0.25], q=[3], n_active=[min(A, 2)], max_active=[4],
                         adapter_offsets=[0, min(A, 2)], adapter_ids=list(range(min(A, 2))))
            base = put(clean)
            e.update_snapshot(base + 1, base, **delta)
            ep = base + 1
            if models is not None:
                e.upload_models(ep, models)
            w = epoch_results(e, ep, P, A, reqs, ids, True)
            base = put(poison(clean, P, A, np.nan, TG.INT32_MIN))
            e.update_snapshot(base + 1, base, **delta)
            ep = base + 1
            if models is not None:
                e.upload_models(ep, models)
            same_results(epoch_results(e, ep, P, A, reqs, ids, True), w, (P, A, "delta"))
    finally:
        e.close()


@pytest.mark.parametrize("P,A", [(33, 64), (4097, 1), (20001, 64)])
def test_padding_junk_is_ignored_after_a_broadcast(P, A, monkeypatch):
    state = edge_state(P, A, seed=P)
    clean = state.packed().blob()
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(2000, A, seed=P)]))
    e = engine(monkeypatch, P, A)
    try:
        try:
            e.comm_init_rank(1, 0, e.comm_unique_id())
        except N.LigError as err:
            pytest.skip(f"no NCCL: {err}")
        upload_blob(e, 1, P, A, clean, comm=True)
        want = epoch_results(e, 1, P, A, reqs, None, True)
        for i, (kv, q) in enumerate(POISONS):
            upload_blob(e, 2 + i, P, A, poison(clean, P, A, kv, q), comm=True)
            same_results(epoch_results(e, 2 + i, P, A, reqs, None, True), want, (P, A, kv, q))
    finally:
        e.close()


# ---- E. refused host uploads evict nothing ----------------------------------------------------------------
def raw_upload(e, block, epoch, P, A, cols):
    lib = N.load()
    fn = lib.lig_upload_snapshot if block else lib.lig_upload_snapshot_async
    p = lambda a: None if a is None else a.ctypes.data
    return fn(e._ctx, epoch, P, A, *[p(a) for a in cols])


def refusals(packed, max_pods, max_adapters):
    cols = [packed.kv, packed.q, packed.n_active, packed.max_active, np.ascontiguousarray(packed.bitmap)]
    out = []
    for k, name in enumerate(("kv", "q", "n_active", "max_active", "bitmap")):
        c = list(cols)
        c[k] = None
        out.append((f"null {name}", packed.P, packed.A, c, N.LIG_ERR_INVALID))
    for pod in (0, packed.P - 1):
        c = list(cols)
        c[2] = packed.n_active.copy()
        c[2][pod] = 65535
        out.append((f"n_active 65535 at pod {pod}", packed.P, packed.A, c, N.LIG_ERR_RANGE))
    grown = [np.resize(a, max_pods + 1) for a in cols[:4]] + [np.zeros((packed.A, (max_pods + 32) // 32), np.uint32)]
    out.append(("P > max_pods", max_pods + 1, packed.A, grown, N.LIG_ERR_INVALID))
    out.append(("A > max_adapters", packed.P, max_adapters + 1, cols, N.LIG_ERR_INVALID))
    return out


@pytest.mark.parametrize("block", [True, False], ids=["blocking", "async"])
def test_refused_uploads_evict_nothing(block, monkeypatch):
    P, A = 200, 9
    s1, s2 = edge_state(P, A, 41), edge_state(P, A, 42)
    reqs = np.ascontiguousarray(np.concatenate([class_requests(A), WL.make_requests(1000, A, seed=43)]))
    ids = WL.make_model_requests(1000, A, seed=44)
    e = engine(monkeypatch, P, A)
    try:
        for ep, s in ((1, s1), (2, s2)):
            e.upload_snapshot(ep, s.packed())
            e.upload_models(ep, pack_models(WL.make_models(A), s.packed()))

        def state_of():
            return {ep: (as_lists(tables(e, ep, A, P)), e.schedule_batch(ep, 6, reqs).tobytes(),
                         e.schedule_models_batch(ep, 6, ids).tobytes()) for ep in (1, 2)}

        before = state_of()
        for label, Pb, Ab, cols, code in refusals(s1.packed(), P, A):
            for target in (1, 2, 99):
                rc = raw_upload(e, block, target, Pb, Ab, cols)
                assert rc == code, (label, target, rc, N.load().lig_last_error())
                assert state_of() == before, (label, target)
        # and the ctx still takes uploads: a good one evicts the older epoch as always
        e.upload_snapshot(3, s1.packed(), block=block)
        with pytest.raises(N.LigError) as ei:
            e.schedule_batch(1, 6, reqs)
        assert ei.value.code == N.LIG_ERR_STALE_EPOCH
        assert e.schedule_batch(3, 6, reqs).tobytes() == before[1][1]
    finally:
        e.close()


def test_refused_delta_with_n_active_65535(monkeypatch):
    P, A = 64, 4
    s = edge_state(P, A, 51)
    e = engine(monkeypatch, P, A)
    try:
        e.upload_snapshot(1, s.packed())
        reqs = class_requests(A)
        want = e.schedule_batch(1, 2, reqs).tobytes()
        with pytest.raises(N.LigError) as ei:
            e.update_snapshot(2, 1, [3, 5], [0.1, 0.2], [1, 2], [1, 65535], [4, 4], [0, 1, 1], [0])
        assert ei.value.code == N.LIG_ERR_RANGE
        assert e.schedule_batch(1, 2, reqs).tobytes() == want
        e.update_snapshot(2, 1, [3, 5], [0.1, 0.2], [1, 2], [1, 65534], [4, 65535], [0, 1, 1], [0])
    finally:
        e.close()
