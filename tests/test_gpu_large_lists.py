"""Large survivor lists, crafted draws and the ABI's size limits on the device.

The other parity suites compare picks bit for bit, but their classes keep a handful of pods, so
Int31n's division magic for large non-power-of-two n and its rejection loop (a draw is rejected with
probability (2^31 mod n) / 2^31) were never exercised on the device.  Here every class's list is
known by construction (adapter a is held by exactly n_a random pods and every pod ties on queue and
KV, as in an idle, freshly scaled pool), and the request keys are crafted (tests/draw_keys.py) so
that the first draw is each accept / reject boundary of Int31n(n).  Each pick path is compared with
the construction, not with another path.
"""
import numpy as np
import pytest

import draw_keys as DK
import filter_tree_ref as FR
from helpers import np_int31n
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, PackedModels, pack_columns
from test_gpu_parity import QUEUE_MODES

pytestmark = pytest.mark.gpu

P_MAX = N.LIG_MAX_PODS
SEED = 0x5EED
TOP31 = 1 << 31


# ---- construction ---------------------------------------------------------------------------------
class Snap:
    """Columns + bitmap of a snapshot whose class lists are known: holders[a] (sorted) holds adapter a."""

    def __init__(self, P, holders, q, kv, max_active):
        self.P, self.A = P, len(holders)
        W = (P + 31) // 32
        member = np.zeros((max(self.A, 1), W * 32), dtype=bool)
        for a, h in enumerate(holders):
            member[a, h] = True
        member = member[: self.A]
        self.holders = holders
        self.n_active = member.sum(axis=0)[:P].astype(np.int64)
        bitmap = np.packbits(member.reshape(self.A, W * 4, 8), axis=-1, bitorder="little").reshape(self.A, W * 4)
        bitmap = np.ascontiguousarray(bitmap).view(np.uint32).reshape(self.A, W)
        self.q, self.kv, self.max_active = q, kv, max_active
        self.packed = pack_columns(kv, q, self.n_active, max_active, bitmap)
        self.bitmap = bitmap

    def ref_pods(self):
        """filter_tree_ref.Pods over the columns (affinity read from the bitmap)."""
        pods = FR.Pods([])
        pods.P, pods.q, pods.kv = self.P, self.q.astype(np.int64), self.kv
        pods.room = self.n_active < self.max_active
        bm = self.bitmap

        def affinity(model):
            a = int(model)
            if a >= self.A:
                return np.zeros(self.P, dtype=bool)
            bits = np.unpackbits(bm[a].view(np.uint8), bitorder="little")[: self.P]
            return bits.astype(bool)
        pods.affinity = affinity
        return pods


def idle_snapshot(ns, rng, P=P_MAX):
    """Every pod q = 0, kv = 0.5, MaxActiveModels = 0: both classes of adapter a keep exactly its
    holders, an unheld adapter keeps all P pods."""
    holders = [np.sort(rng.choice(P, int(n), replace=False)).astype(np.int64) for n in ns]
    return Snap(P, holders, np.zeros(P, dtype=np.int64), np.full(P, 0.5), np.zeros(P, dtype=np.int64))


def crafted_values(n):
    """First draws at Int31n(n)'s edges: 0, n-1, n, n+1, top-n-1, top-n, top-1 (last accepted),
    top (first rejected), 2^31-1, with top = floor(2^31/n)*n."""
    top = DK.accept_top(n)
    vs = {0, n - 1, n, n + 1, top - n - 1, top - n, top - 1, TOP31 - 1}
    if top < TOP31:
        vs.add(top)
    return sorted(v for v in vs if 0 <= v < TOP31)


class Requests:
    """Crafted requests of a class table: ids, flags, initial states, expected pick."""

    def __init__(self, classes, rng, extra_states=None):
        """classes: list of (adapter_id, critical, sorted list); extra_states: {class index: states}."""
        ids, flags, states, cls = [], [], [], []
        for ci, (a, crit, lst) in enumerate(classes):
            n = len(lst)
            vs = crafted_values(n)
            st = DK.states_for(vs, rng)
            if extra_states and ci in extra_states:
                st = np.concatenate([st, extra_states[ci]])
            ids += [a] * len(st)
            flags += [int(crit)] * len(st)
            states.append(st)
            cls += [ci] * len(st)
        self.states = np.concatenate(states)
        self.cls = np.array(cls)
        self.ids = np.array(ids, dtype=np.int64)
        self.flags = np.array(flags, dtype=np.uint32)
        self.n = np.array([len(classes[c][2]) for c in range(len(classes))], dtype=np.int64)[self.cls]
        flat = np.concatenate([np.asarray(c[2], dtype=np.int64) for c in classes])
        self.off = np.concatenate([[0], np.cumsum([len(c[2]) for c in classes])])[self.cls]
        self.flat = flat
        d = DK.first_draws(self.states, 2)
        top = np.array([DK.accept_top(int(n)) for n in self.n], dtype=np.int64)
        self.rejected = d[:, 0] >= top
        self.rejected2 = self.rejected & (d[:, 1] >= top)

    def reqs(self, seed):
        r = np.zeros(len(self.ids), dtype=REQ_DTYPE)
        r["adapter_id"] = self.ids
        r["flags"] = self.flags
        r["rand_key"] = self.states ^ np.uint64(seed)
        return r

    def expected_pods(self, seed):
        k = np_int31n(seed, self.states ^ np.uint64(seed), self.n)
        return self.flat[self.off + k]


def check(got, rq, seed, label, sel=None, want_double=True):
    """Every pick equals the construction; the subset served includes rejected first draws."""
    sel = np.arange(len(rq.ids)) if sel is None else sel
    want = rq.expected_pods(seed)[sel]
    assert (got["status"] == N.LIG_OK).all(), (label, np.unique(got["status"]))
    assert np.array_equal(got["n_survivors"].astype(np.int64), rq.n[sel]), label
    bad = np.nonzero(got["pod_idx"] != want)[0]
    assert bad.size == 0, (label, bad[:5], got[bad[:5]], want[bad[:5]], rq.n[sel][bad[:5]])
    assert rq.rejected[sel].sum() > 0, f"{label}: no request had its first draw rejected"
    if want_double:
        assert rq.rejected2[sel].sum() > 0, f"{label}: no request had its first two draws rejected"


def run_queue(eng, ep, batches, seed):
    """schedule_batches_device over host request arrays; batch b runs with seed + b."""
    import torch
    d_in = [torch.from_numpy(b.view(np.uint8).reshape(-1)).cuda() for b in batches]
    d_out = [torch.zeros(len(b) * 8, dtype=torch.uint8, device="cuda") for b in batches]
    torch.cuda.synchronize()
    eng.schedule_batches_device(ep, seed, [t.data_ptr() for t in d_in], len(batches[0]),
                                [t.data_ptr() for t in d_out], 0)
    torch.cuda.synchronize()
    return [t.cpu().numpy().view(PICK_DTYPE) for t in d_out]


def make_engine(env, monkeypatch, **kw):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)               # the knobs are read at lig_create
        return Engine(0, **kw)


# ---- part 2: every survivor count 2..32768 through every pick path ---------------------------------
N_SNAPSHOTS, A_PER = 8, 4096


def test_every_survivor_count_through_every_pick_path(monkeypatch):
    rng = np.random.default_rng(2026)
    kw = dict(max_pods=P_MAX, max_adapters=A_PER, max_batch=1 << 17)
    engines = {mode: make_engine(env, monkeypatch, **kw) for mode, env in QUEUE_MODES.items()}
    tree = Engine(0, **kw)
    tree.set_filter_tree(S.DEFAULT_FILTER)
    base = engines["tma"]
    nodes = S.DEFAULT_FILTER.flatten()
    served_heavy = set()
    try:
        for s in range(N_SNAPSHOTS):
            ns = np.arange(2 + s * A_PER, min(2 + (s + 1) * A_PER, P_MAX + 1))
            snap = idle_snapshot(ns, rng)
            A = snap.A
            everyone = np.arange(P_MAX)
            classes = []
            for crit in (0, 1):
                classes += [(a, crit, snap.holders[a]) for a in range(A)]
                classes += [(A, crit, everyone)]
            extra = {}
            for n in DK.rejection_heavy_ns(int(ns[0]), int(ns[-1]), 4):
                st = DK.double_reject_states(n, 4, rng)
                assert st.size == 4, n
                extra[n - ns[0]] = st[:2]                      # sheddable class of that adapter
                extra[A + 1 + n - ns[0]] = st[2:]              # critical class
                served_heavy.add(n)
            rq = Requests(classes, rng, extra)
            ep = 10 + s
            for e in list(engines.values()) + [tree]:
                e.upload_snapshot(ep, snap.packed)
            info = base.pick_kernel_info(ep)
            assert info["table_bytes"] == 0 and not info["tables_in_smem"], info   # the compact pool overflowed
            # the construction itself, on a sample of classes: the reference tree walk and lig_read_class
            pods = snap.ref_pods()
            for ci in rng.choice(len(classes), 6, replace=False).tolist() + [A, 2 * A + 1]:
                a, crit, lst = classes[ci]
                st_ref, idx = FR.walk(nodes, pods, bool(crit), str(a))
                assert st_ref == N.LIG_OK and np.array_equal(idx, lst), (s, ci)
                for e in (base, tree):
                    st, n, got = e.read_class(ep, bool(crit), a, P_MAX)
                    assert st == N.LIG_OK and n == len(lst) and np.array_equal(got, lst), (s, ci)
            reqs = rq.reqs(SEED)
            check(base.schedule_batch(ep, SEED, reqs), rq, SEED, f"schedule_batch s={s}")
            # the model queue on the overflowed pool: a single-target model per long list
            big = [a for a in range(A) if snap.holders[a].size & (snap.holders[a].size - 1)][-2:]
            base.upload_models(ep, single_target_models(*big))
            for mi, a in enumerate(big):
                check_model_queue(base, ep, snap.holders[a], rng, f"models overflowed s={s} n={snap.holders[a].size}", model=mi)
            check(tree.schedule_batch(ep, SEED, reqs), rq, SEED, f"caller tree s={s}")
            for mode, e in engines.items():
                got = run_queue(e, ep, [reqs, rq.reqs(SEED + 1)], SEED)
                check(got[0], rq, SEED, f"{mode} s={s}")
                check(got[1], rq, SEED + 1, f"{mode} batch 1 s={s}")
            got = run_queue(tree, ep, [reqs], SEED)[0]
            check(got, rq, SEED, f"caller tree queue s={s}")
            # the doorbell, in capacity-sized chunks
            cap = N.load().lig_stream_capacity()
            base.stream_open()
            try:
                got = np.concatenate([base.stream_submit(ep, SEED, np.ascontiguousarray(reqs[i:i + cap]))
                                      for i in range(0, len(reqs), cap)])
            finally:
                base.stream_close()
            check(got, rq, SEED, f"doorbell s={s}")
            # the direct scan (its own int31n and k-th-bit walk) on a subsample with every rejection
            sel = np.unique(np.concatenate([np.nonzero(rq.rejected2)[0], np.nonzero(rq.rejected)[0][:600],
                                            rng.choice(len(reqs), 400, replace=False)]))
            got, _ = base.schedule_scan(ep, SEED, np.ascontiguousarray(reqs[sel]), False)
            check(got, rq, SEED, f"scan s={s}", sel=sel)
        assert len(served_heavy) == 4 * N_SNAPSHOTS
    finally:
        for e in engines.values():
            e.close()
        tree.close()


# ---- part 3: table regimes at large n ------------------------------------------------------------------
BUDGET = 72 * 1024


def room_snapshot(m, adapter_ns, rng, P=P_MAX, kv=0.9):
    """q = 0 everywhere, kv = 0.9 (above the 0.8 threshold: every sheddable class is DROPped), exactly
    m pods with room: the critical default list is those m pods, adapter a's critical list its holders.
    With kv = 0.5 and no adapters, the sheddable classes keep the m pods with room as well."""
    holders = [np.sort(rng.choice(P, int(n), replace=False)).astype(np.int64) for n in adapter_ns]
    room = np.sort(rng.choice(P, m, replace=False))
    n_active = np.zeros(P, dtype=np.int64)
    for h in holders:
        n_active[h] += 1
    max_active = np.zeros(P, dtype=np.int64)
    max_active[room] = n_active[room] + 1
    snap = Snap(P, holders, np.zeros(P, dtype=np.int64), np.full(P, kv), max_active)
    return snap, room


def blob_bytes(A, pool_entries):
    return (16 + 16 * 2 * (A + 1) + 2 * pool_entries + 15) // 16 * 16


def mtab_bytes(models):
    """Size of the model blob: header, 16 B per model, 8 B per target of the models with >= 2 targets."""
    nt = np.diff(models.target_offsets)
    return (16 + 16 * models.n_models + 8 * int(nt[nt >= 2].sum()) + 15) // 16 * 16


def regime_classes(snap, room):
    A = snap.A
    return [(a, 1, snap.holders[a]) for a in range(A)] + [(A, 1, room)]


def check_regime(eng, ep, snap, classes, rng, label):
    rq = Requests(classes, rng)
    reqs = rq.reqs(SEED)
    got = run_queue(eng, ep, [reqs], SEED)[0]
    check(got, rq, SEED, label, want_double=False)
    # sheddable requests are dropped with pod -1
    shed = reqs.copy()
    shed["flags"] = 0
    got = run_queue(eng, ep, [shed], SEED)[0]
    assert (got["status"] == N.LIG_DROP).all() and (got["pod_idx"] == -1).all(), label


def single_target_models(adapter, second=0):
    """Two critical models whose only targets are `adapter` and `second` (no draw), for the model queue."""
    return PackedModels(n_models=2, target_offsets=np.array([0, 1, 2], dtype=np.int32),
                        target_adapter_ids=np.array([adapter, second], dtype=np.int32),
                        target_weights=np.array([1, 1], dtype=np.int32), critical=np.array([1, 1], dtype=np.uint8),
                        self_adapter_ids=np.array([0, 0], dtype=np.int32), present=np.array([1, 1], dtype=np.uint8),
                        model_ids={}, target_names=[["t"], ["u"]])


def model_queue(eng, ep, ids, seed, first_index):
    import torch
    d_in = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.uint32).view(np.uint8)).cuda()
    d_out = torch.zeros(len(ids) * 4, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.schedule_models_batches_device(ep, seed, first_index, [d_in.data_ptr()], len(ids), [d_out.data_ptr()], 0)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(MPICK_DTYPE)


def check_model_queue(eng, ep, lst, rng, label, model=0):
    """Requests for `model`, which resolves to the critical class of `lst`: a crafted seed per call
    puts the pick's first draw (request 0, rand_key = first_index) on each edge; R = 4 takes the
    persistent kernel."""
    n = len(lst)
    for v in crafted_values(n):
        fi = int(rng.integers(0, 1 << 40))
        seed = int(DK.states_for([v], rng)[0] ^ np.uint64(fi))
        got = model_queue(eng, ep, np.full(4, model, dtype=np.uint32), seed, fi)
        keys = np.uint64(fi) + np.arange(4, dtype=np.uint64)
        want = lst[np_int31n(seed, keys, np.full(4, n))]
        assert (got["status"] == N.LIG_OK).all(), (label, v)
        assert np.array_equal(got["pod_idx"].astype(np.int64), want), (label, n, v, got, want)


def test_compact_tables_in_shared_memory_at_large_n():
    rng = np.random.default_rng(7)
    primes = [32749, 32719, 30011, 24593, 16411, 12289, 8191, 6151, 4099, 3079, 1543, 769, 389, 193, 97, 53]
    pow2 = [x for k in range(2, 16) for x in ((1 << k) - 1, (1 << k) + 1) if x <= 32767]
    heavy = DK.rejection_heavy_ns(2, 32767, 40)
    ns = sorted(set(primes + pow2 + heavy + [3, 32767, 21846, 10923]))
    e = Engine(0, max_pods=P_MAX, max_adapters=8, max_batch=1 << 16)
    try:
        for i, m in enumerate(ns):
            snap, room = room_snapshot(m, [], rng)
            ep = 100 + i
            e.upload_snapshot(ep, snap.packed)
            e.upload_models(ep, single_target_models(0))
            info = e.pick_kernel_info(ep)
            assert info["tables_in_smem"] and info["table_bytes"] == blob_bytes(0, 1 + m), (m, info)
            check_regime(e, ep, snap, regime_classes(snap, room), rng, f"smem n={m}")
            if i % 8 == 0 or m == 32767:
                check_model_queue(e, ep, room, rng, f"models smem n={m}")
    finally:
        e.close()


def budget_ns(total, m, A=8):
    """Adapter list lengths that, with an m-pod default list, fill `total` compact pool entries."""
    rest = total - 1 - m
    ns = [rest // A] * A
    ns[-1] += rest - sum(ns)
    return ns


@pytest.mark.parametrize("extra", [0, 16])
def test_compact_budget_boundary(extra):
    rng = np.random.default_rng(8 + extra)
    A, m = 8, 4099
    pool = (BUDGET + extra - (16 + 16 * 2 * (A + 1))) // 2
    snap, room = room_snapshot(m, budget_ns(pool, m, A), rng)
    e = Engine(0, max_pods=P_MAX, max_adapters=A, max_batch=1 << 16)
    try:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, single_target_models(A))
        info = e.pick_kernel_info(1)
        assert info["table_bytes"] == blob_bytes(A, pool) == BUDGET + extra, info
        assert info["tables_in_smem"] == (extra == 0), info
        check_regime(e, 1, snap, regime_classes(snap, room), rng, f"budget+{extra}")
        check_model_queue(e, 1, room, rng, f"models budget+{extra}")
        check_model_queue(e, 1, snap.holders[0], rng, f"models budget+{extra} own list", model=1)
    finally:
        e.close()


@pytest.mark.parametrize("extra", [0, 16])
def test_compact_plus_model_table_budget(extra):
    """ctab fits alone; ctab + mtab (64 bytes: two models, one with two targets) is at the budget or
    16 bytes over it, so the model kernel takes its tables from shared memory in the first case and
    from global memory in the second.  The ABI does not report the model kernel's choice, so only the
    table sizes that decide it and the picks are checked: the model queue and the descriptor queue
    give the construction either way."""
    rng = np.random.default_rng(9 + extra)
    A, m = 8, 4099
    mtab = 64
    pool = (BUDGET - mtab + extra - (16 + 16 * 2 * (A + 1))) // 2
    snap, room = room_snapshot(m, budget_ns(pool, m, A), rng)
    models = PackedModels(n_models=2, target_offsets=np.array([0, 1, 3], dtype=np.int32),
                          target_adapter_ids=np.array([A, 0, 1], dtype=np.int32),
                          target_weights=np.array([1, 3, 5], dtype=np.int32), critical=np.array([1, 1], dtype=np.uint8),
                          self_adapter_ids=np.array([0, 0], dtype=np.int32), present=np.array([1, 1], dtype=np.uint8),
                          model_ids={}, target_names=[["x"], ["y", "z"]])
    e = Engine(0, max_pods=P_MAX, max_adapters=A, max_batch=1 << 16)
    try:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, models)
        info = e.pick_kernel_info(1)
        assert info["table_bytes"] == BUDGET - mtab + extra and info["tables_in_smem"], info
        assert info["table_bytes"] + mtab_bytes(models) == BUDGET + extra
        check_regime(e, 1, snap, regime_classes(snap, room), rng, f"ctab+mtab+{extra}")
        check_model_queue(e, 1, room, rng, f"models ctab+mtab+{extra}")
        # the two-target model: the draw picks adapter 0 or 1, then the pick uses that class
        ids = np.ones(4096, dtype=np.uint32)
        got = model_queue(e, 1, ids, 31, 1 << 20)
        keys = np.uint64(1 << 20) + np.arange(4096, dtype=np.uint64)
        draw = np_int31n(31 ^ DK.LIG_DRAW_DOMAIN, keys, np.full(4096, 8))
        tgt = (draw >= 3).astype(np.int64)
        assert np.array_equal(got["target_idx"].astype(np.int64), tgt)
        n = np.array([len(snap.holders[0]), len(snap.holders[1])])[tgt]
        k = np_int31n(31, keys, n)
        want = np.array([snap.holders[t][kk] for t, kk in zip(tgt, k)])
        assert np.array_equal(got["pod_idx"].astype(np.int64), want)
    finally:
        e.close()


# ---- part 4: model draws at the edges -----------------------------------------------------------------
def np_weighted_select(weights, random_val):
    """datastore.go:91-97: for each target, if randomVal < Weight return it; randomVal -= Weight."""
    for k, w in enumerate(weights):
        if random_val < w:
            return k
        random_val -= w
    return len(weights) - 1


EDGE_MODELS = [
    [1 << 29, (1 << 29) + 1],                      # total 2^30+1: about half of all draws rejected
    [1 << 29, 1 << 29, (1 << 29) + 1],             # 3*2^29+1
    [(1 << 30), (1 << 30) - 1],                    # 2^31-1
    [16384, 16385],                                # just above 32768
    [1, 65535, 1],                                 # just above 65536
    [0, 0, 7, 0, 9, 0] + [0] * 248 + [5],          # 255 targets, zero weights first, inside and last-but-one
    [3] * 254 + [0],                               # 255 targets, zero weight last
]


MODEL_REGIMES = {
    # (snapshot, env): "room" = A = 0 and 12289 pods with room, so ctab + mtab fits the shared-memory
    # budget; "large_n" = the classes of adapters held by 2 .. 32767 pods, a compact blob of ~535 KB
    "smem": ("room", {}),
    "smem_1group_2stage": ("room", {"LIG_MODELS_GROUPS": "1", "LIG_MODELS_STAGES": "2"}),
    "tables_global": ("room", {"LIG_TAB_SMEM": "0"}),
    "large_n": ("large_n", {}),
}


@pytest.mark.parametrize("regime", sorted(MODEL_REGIMES))
def test_model_draws_at_the_edges(regime, oracle, monkeypatch):
    rng = np.random.default_rng(11)
    kind, env = MODEL_REGIMES[regime]
    if kind == "room":
        snap, default_list = room_snapshot(12289, [], rng, kv=0.5)
    else:
        snap = idle_snapshot([2, 3, 4097, 12289, 21846, 32767, 30011, 5], rng)
        default_list = np.arange(P_MAX)
    A = snap.A
    tgt_ids, weights, off = [], [], [0]
    for mi, ws in enumerate(EDGE_MODELS):
        tgt_ids += [(mi + k) % (A + 1) for k in range(len(ws))]   # id A: the unheld adapter (all pods)
        weights += ws
        off.append(len(tgt_ids))
    nm = len(EDGE_MODELS)
    models = PackedModels(n_models=nm, target_offsets=np.array(off, dtype=np.int32),
                          target_adapter_ids=np.array(tgt_ids, dtype=np.int32),
                          target_weights=np.array(weights, dtype=np.int32),
                          critical=(np.arange(nm) % 2).astype(np.uint8), self_adapter_ids=np.zeros(nm, dtype=np.int32),
                          present=np.ones(nm, dtype=np.uint8), model_ids={}, target_names=[[]] * nm)
    names = [f"a{a}" for a in range(A)] + ["unheld"]
    mo = oracle.Models([dict(name=f"m{mi}", critical=bool(mi % 2),
                             targets=[(names[tgt_ids[k]], weights[k]) for k in range(off[mi], off[mi + 1])])
                        for mi in range(nm)])
    lists = [snap.holders[a] for a in range(A)] + [default_list]
    e = make_engine(env, monkeypatch, max_pods=P_MAX, max_adapters=max(A, 1), max_batch=1 << 12)
    rejected = 0
    try:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, models)
        info = e.pick_kernel_info(1)
        if kind == "room":
            # the regime the model kernel runs in: both tables fit the shared-memory budget
            assert info["table_bytes"] == blob_bytes(0, 1 + 2 * len(default_list)), info
            assert info["table_bytes"] + mtab_bytes(models) <= BUDGET, (info, mtab_bytes(models))
            assert info["tables_in_smem"] == ("LIG_TAB_SMEM" not in env), info
        else:
            # a compact blob that does not fit the budget: the kernels read the strided tables
            assert info["table_bytes"] > BUDGET and not info["tables_in_smem"], info
        for mi, ws in enumerate(EDGE_MODELS):
            total = sum(ws)
            cum = np.cumsum(ws)
            top = DK.accept_top(total)
            rvals = {0, total - 1} | {int(c) - 1 for c in cum if c > 0} | {int(c) for c in cum if c < total}
            vs = sorted(rvals) + ([top, TOP31 - 1] if top < TOP31 else [])
            for v in vs:
                seed = int(DK.draw_seed([v], 0, rng)[0])
                r = int(np_int31n(seed ^ DK.LIG_DRAW_DOMAIN, np.zeros(1, dtype=np.uint64), np.array([total]))[0])
                assert r == oracle.int31n(seed ^ DK.LIG_DRAW_DOMAIN, total)
                if v < top:
                    assert r == v
                else:
                    rejected += 1
                k = np_weighted_select(ws, r)
                assert k == int(np.searchsorted(cum, r, side="right")) == mo.weighted_select(mi, r)
                assert mo.resolve(mi, seed, 0)[3] == k
                lst = lists[tgt_ids[off[mi] + k]]
                pod = int(lst[np_int31n(seed, np.zeros(1, dtype=np.uint64), np.array([len(lst)]))[0]])
                # the plain kernel (one request), resolve_models and the persistent kernel (R = 4)
                one = e.schedule_models_batch(1, seed, np.array([mi], dtype=np.uint32))
                assert (int(one["status"][0]), int(one["target_idx"][0]), int(one["pod_idx"][0])) == (N.LIG_OK, k, pod), (mi, v)
                reqs, res = e.resolve_models(1, seed, np.array([mi], dtype=np.uint32))
                assert int(res["target_idx"][0]) == k and int(reqs["adapter_id"][0]) == tgt_ids[off[mi] + k]
                assert int(reqs["flags"][0]) == mi % 2
                q = model_queue(e, 1, np.full(4, mi, dtype=np.uint32), seed, 0)
                assert (int(q["target_idx"][0]), int(q["pod_idx"][0])) == (k, pod), (mi, v)
                q5 = model_queue(e, 1, np.full(5, mi, dtype=np.uint32), seed, 0)
                assert np.array_equal(q5[:4], q), (mi, v)
        assert rejected >= 2 * len(EDGE_MODELS) - 1
    finally:
        e.close()


# ---- part 5: the ABI's hard limits ------------------------------------------------------------------------
A_MAX = N.LIG_MAX_ADAPTERS


def limits_snapshot():
    """pod 0: q 0, kv -inf, holds adapter 1; pod 1: q 0, kv 0.5, holds adapter 0; the rest q 100,
    kv 0.9, no adapters; MaxActiveModels 0.  Built-in tree: (sheddable, 0) and (critical, 0) keep
    [1]; every other class ends EMPTY (-inf in least-KV gives a NaN threshold)."""
    P = P_MAX
    q = np.full(P, 100, dtype=np.int64)
    kv = np.full(P, 0.9)
    q[:2] = 0
    kv[0], kv[1] = -np.inf, 0.5
    W = P // 32
    bitmap = np.zeros((A_MAX, W), dtype=np.uint32)
    bitmap[1, 0] = 1
    bitmap[0, 0] = 2
    na = np.zeros(P, dtype=np.int64)
    na[:2] = 1
    return pack_columns(kv, q, na, np.zeros(P, dtype=np.int64), bitmap)


def limits_requests(rng):
    ids = np.concatenate([np.arange(A_MAX + 1), [-1, A_MAX + 9]])
    r = np.zeros(2 * len(ids), dtype=REQ_DTYPE)
    r["adapter_id"] = np.concatenate([ids, ids])
    r["flags"] = np.repeat([0, 1], len(ids))
    r["rand_key"] = rng.integers(0, 1 << 64, len(r), dtype=np.uint64)
    return r


def all_paths(e, ep, reqs, scan):
    out = {"schedule_batch": e.schedule_batch(ep, SEED, reqs)}
    out["queue"] = run_queue(e, ep, [reqs], SEED)[0]
    cap = N.load().lig_stream_capacity()
    e.stream_open()
    try:
        out["doorbell"] = np.concatenate([e.stream_submit(ep, SEED, np.ascontiguousarray(reqs[i:i + cap]))
                                          for i in range(0, len(reqs), cap)])
    finally:
        e.stream_close()
    if scan:
        sel = np.r_[0:64, A_MAX - 8:A_MAX + 70, len(reqs) - 64:len(reqs)]
        got, _ = e.schedule_scan(ep, SEED, np.ascontiguousarray(reqs[sel]), False)
        out["scan"] = (got, sel)
    return out


def test_hard_limits():
    import torch
    free, _ = torch.cuda.mem_get_info()
    need = 19 << 30
    if free < need:
        pytest.skip(f"needs {need >> 30} GiB of free device memory for two slots of strided lists at "
                    f"P = {P_MAX}, A = {A_MAX}; {free / 2**30:.1f} GiB free")
    rng = np.random.default_rng(12)
    packed = limits_snapshot()
    reqs = limits_requests(rng)
    cls_of = lambda r: r["flags"].astype(np.int64) * (A_MAX + 1) + np.minimum(r["adapter_id"].astype(np.int64) % (1 << 32), A_MAX)
    e = Engine(0, max_pods=P_MAX, max_adapters=A_MAX, max_batch=len(reqs))
    try:
        # built-in tree
        e.upload_snapshot(1, packed)
        c = cls_of(reqs)
        ok = (c == 0) | (c == A_MAX + 1)
        for name, got in all_paths(e, 1, reqs, scan=True).items():
            sel = slice(None)
            if name == "scan":
                got, sel = got
            g, okk = got, ok[sel]
            assert (g["pod_idx"][~okk] == -1).all(), (name, g[~okk][g["pod_idx"][~okk] != -1][:5])
            assert (g["status"][~okk] == N.LIG_EMPTY).all(), name
            assert (g["pod_idx"][okk] == 1).all() and (g["status"][okk] == N.LIG_OK).all(), (name, g[okk])
        for crit, a in [(0, 0), (1, 0), (0, 1), (1, 1), (0, A_MAX), (1, A_MAX)] + [(1, a) for a in range(A_MAX - 10, A_MAX)]:
            st, n, lst = e.read_class(1, bool(crit), a, P_MAX)
            assert (st, n, lst.tolist()) == ((N.LIG_OK, 1, [1]) if a == 0 else (N.LIG_EMPTY, 0, [])), (crit, a)
        # a caller tree: sheddable classes keep every pod (q <= 100, kv <= 1), critical ones end
        # in "no pods left"
        e.set_filter_tree([
            N.LigFilterNode(N.LIG_F_CRITICAL_REQUEST, 1, 2, -1, 0, 0.0),
            N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, -(1 << 31), 0.0),
            N.LigFilterNode(N.LIG_F_NO_QUEUE_AND_LOW_KV, -1, -1, -1, 100, 1.0)])
        e.upload_snapshot(2, packed)
        crit = reqs["flags"] == 1
        k = np_int31n(SEED, reqs["rand_key"], np.full(len(reqs), P_MAX))
        for name, got in all_paths(e, 2, reqs, scan=False).items():
            assert (got["pod_idx"][crit] == -1).all() and (got["status"][crit] == N.LIG_NO_PODS_LEFT).all(), \
                (name, got[crit][got["pod_idx"][crit] != -1][:5])
            assert (got["status"][~crit] == N.LIG_OK).all() and (got["n_survivors"][~crit] == P_MAX).all(), name
            assert np.array_equal(got["pod_idx"][~crit], k[~crit]), name
        everyone = np.arange(P_MAX)
        for a in [0, 1, 2, A_MAX - 1, A_MAX]:
            st, n, lst = e.read_class(2, False, a, P_MAX)
            assert st == N.LIG_OK and n == P_MAX and np.array_equal(lst, everyone), a
        for a in list(range(131060 - (A_MAX + 1), A_MAX + 1)):      # classes c >= 131060
            assert e.read_class(2, True, a, P_MAX)[:2] == (N.LIG_NO_PODS_LEFT, 0), a
        e.set_filter_tree(None)
    finally:
        e.close()
