"""The two entry points that change a device snapshot instead of only reading it, at their edges.

* lig_update_snapshot (delta refresh): an epoch built from a resident base by a delta must equal a
  full upload of the modified pool in another ctx — class tables, every pick path and the oracle —
  for every class-build variant, ragged pools, edge values written by the delta, compact-table
  regime changes, the staging growth path, long chains and caller trees.  Malformed deltas
  (duplicate pods, bad offsets, adapter ids outside the table) are refused before anything is
  written.
* lig_schedule_batch_feedback_device (in-batch load feedback): picks and per-pod pick totals equal
  the sequential definition (oracle/feedback.py, or the caller-tree restatement below) at queue
  saturation, threshold crossings, edge pools, every window shape and on two streams at once.

The one test without a GPU pins the caller-tree feedback reference to oracle/feedback.py."""
import math

import numpy as np
import pytest

import oracle_tree
from filter_tree_ref import random_tree
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_columns, pack_models
from oracle import feedback as FB

INT32_MAX, INT32_MIN = (1 << 31) - 1, -(1 << 31)
TAB_BUDGET = 72 * 1024                  # compact tables pulled into shared memory up to this size
SMEM_OPTIN = 227 * 1024                 # H100 opt-in shared memory per block


# ---- pools as the oracle sees them -------------------------------------------------------------------
class PodState:
    """Per-pod columns at Go width; ActiveModels as adapter ids of the table plus `extra` names the
    table does not know (counted by n_active, absent from the bitmap)."""

    def __init__(self, A, kv, q, ma, active, extra=None):
        self.A = A
        self.kv = np.asarray(kv, dtype=np.float64).copy()
        self.q = np.asarray(q, dtype=np.int64).copy()
        self.ma = np.asarray(ma, dtype=np.int64).copy()
        self.active = [sorted(set(int(a) for a in x)) for x in active]
        self.extra = np.zeros(len(self.kv), dtype=np.int64) if extra is None else np.asarray(extra, dtype=np.int64).copy()

    @property
    def P(self):
        return len(self.kv)

    def copy(self):
        return PodState(self.A, self.kv, self.q, self.ma, self.active, self.extra)

    def n_active(self):
        return np.array([len(a) for a in self.active], dtype=np.int64) + self.extra

    def packed(self):
        W = (self.P + 31) // 32
        bm = np.zeros((self.A, W), dtype=np.uint32)
        pods = np.repeat(np.arange(self.P), [len(a) for a in self.active])
        if pods.size:
            ads = np.concatenate([a for a in self.active if a]).astype(np.int64)
            np.bitwise_or.at(bm, (ads, pods >> 5), (np.uint32(1) << (pods & 31).astype(np.uint32)))
        return pack_columns(self.kv, self.q, self.n_active(), self.ma, bm,
                            {WL.adapter_name(a): a for a in range(self.A)})

    def records(self):
        return [dict(name=f"pod-{i}", address=f"address-{i}", waiting_queue_size=int(self.q[i]),
                     kv_cache_usage_percent=float(self.kv[i]), max_active_models=int(self.ma[i]),
                     active_models=[WL.adapter_name(a) for a in self.active[i]] +
                                   [f"unlisted-{i}-{j}" for j in range(int(self.extra[i]))])
                for i in range(self.P)]

    def names(self):
        """Adapter names of ids 0..A-1, then the model no pod lists (id A)."""
        return [WL.adapter_name(a) for a in range(self.A)] + [WL.UNKNOWN_MODEL]


def random_state(P, A, seed):
    snap = WL.make_snapshot(P, A, seed=seed)
    return PodState(A, snap.packed.kv, snap.q64, snap.max_active64, snap.active)


def uniform_state(P, A, held=(), room=True):
    """Identical pods (q 0, kv 0.5, MaxActiveModels 65535 or 0) that all hold the adapters in `held`:
    every list of a class is the whole pool."""
    return PodState(A, np.full(P, 0.5), np.zeros(P), np.full(P, 65535 if room else 0), [list(held)] * P)


KV_EDGE = [math.nan, math.inf, -math.inf, 0.0, -0.0, 5e-324, 1e-310, 2.2250738585072014e-308,
           0.8, float(np.nextafter(0.8, 0.0)), float(np.nextafter(0.8, 1.0)), 0.5, 1.0]
Q_EDGE = [INT32_MIN, INT32_MAX, 5, 6, 49, 50, 0, -1]
MA_EDGE = [0, 65535, 1, 4]


def mutate(state, dirty, rng, edge=True, dup_id=False):
    """A copy of `state` with the pods in `dirty` replaced, and the delta that makes it (entries in
    a shuffled order).  edge=True cycles the dirty pods through the edge values; dup_id repeats one
    adapter id inside a pod's list (legal: the bit is set twice)."""
    new = state.copy()
    dirty = np.asarray(dirty, dtype=np.int64)
    for k, p in enumerate(dirty):
        if edge:
            new.kv[p] = KV_EDGE[k % len(KV_EDGE)]
            new.q[p] = Q_EDGE[(k // 2) % len(Q_EDGE)]
            new.ma[p] = MA_EDGE[(k // 3) % len(MA_EDGE)]
            new.extra[p] = 3 if k % 5 == 4 else 0         # pods that report adapters outside the table
        else:
            new.kv[p] = float(np.round(rng.random(), 3))
            new.q[p] = int(rng.integers(0, 80))
            new.ma[p] = int(rng.choice([0, 4, 8, 16]))
            new.extra[p] = 0
        size = int(rng.integers(0, min(state.A, 6) + 1)) if state.A else 0
        new.active[p] = sorted(rng.choice(state.A, size=size, replace=False).tolist()) if size else []
    order = rng.permutation(len(dirty))
    return new, delta_between(new, dirty[order], dup_id=dup_id)


def delta_between(new, dirty, dup_id=False):
    """The lig_update_snapshot arguments that replace the pods `dirty` (in this order) by theirs in `new`."""
    packed_na = np.minimum(new.n_active(), 65534).astype(np.uint16)
    off = np.zeros(len(dirty) + 1, dtype=np.int32)
    ids = []
    for k, p in enumerate(dirty):
        lst = list(new.active[p])
        if dup_id and lst and k == 0:
            lst.append(lst[0])
        ids.extend(lst)
        off[k + 1] = len(ids)
    dirty = np.asarray(dirty, dtype=np.int64)
    return dict(pod_idx=dirty.astype(np.int32), kv=new.kv[dirty], q=new.q[dirty].astype(np.int32),
                n_active=packed_na[dirty], max_active=np.clip(new.ma[dirty], 0, 65535).astype(np.uint16),
                adapter_offsets=off, adapter_ids=np.array(ids, dtype=np.int32))


def staged_delta_bytes(n_dirty, n_ids):
    """Size of a delta in the ctx's staging (lig_update_snapshot's layout)."""
    o_ids = 8 * n_dirty + 4 * (n_dirty + 1)
    o_kv = (o_ids + 4 * n_ids + 7) & ~7
    return (o_kv + 12 * n_dirty + 15) & ~15, o_kv != o_ids + 4 * n_ids


def initial_delta_capacity(max_pods):
    return max(64 << 10, max_pods // 4 * (24 + 64 * 4) + 4096)


def build_variant(P):
    """Which class build runs for P pods (launch_class_build): the register-resident fast kernel up
    to 128 bitmap words, then the general kernel with the pod columns staged in shared memory while
    they fit, else reading them from global memory."""
    W = (P + 31) // 32
    if P == 0:
        return "empty"
    if W <= 128:
        return "fast"
    fixed = 512 + (7 + 16) * 4 * W                 # block scalars + 7 block masks + 16 warp masks
    return "staged" if fixed + 16 * 32 * W <= SMEM_OPTIN else "unstaged"


def compact_bytes(A, entries):
    return (16 + 16 * 2 * (A + 1) + 2 * entries + 15) // 16 * 16


# ---- running one epoch through every path ------------------------------------------------------------
def class_requests(A, copies=3, seed=3):
    ids = list(range(A + 1)) + [-1, A + 7]
    reqs = np.zeros(2 * len(ids) * copies, dtype=REQ_DTYPE)
    reqs["adapter_id"] = (ids + ids) * copies
    reqs["flags"] = ([0] * len(ids) + [1] * len(ids)) * copies
    reqs["rand_key"] = np.random.default_rng(seed).integers(0, 1 << 64, size=len(reqs), dtype=np.uint64)
    return reqs


def mixed_requests(A, R, seed):
    return np.ascontiguousarray(np.concatenate([class_requests(A, seed=seed), WL.make_requests(R, A, seed=seed + 1)]))


def queue_picks(eng, ep, reqs, seed):
    import torch
    R = len(reqs)
    d_in = torch.from_numpy(reqs.view(np.uint8).reshape(-1).copy()).cuda()
    d_out = [torch.zeros(R * 8, dtype=torch.uint8, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    eng.schedule_batches_device(ep, seed, [d_in.data_ptr()] * 2, R, [t.data_ptr() for t in d_out], 0)
    torch.cuda.synchronize()
    return [t.cpu().numpy().view(PICK_DTYPE) for t in d_out]


def model_picks(eng, ep, ids, seed):
    import torch
    d_in = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(ids) * 4, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.schedule_models_batches_device(ep, seed, 0, [d_in.data_ptr()], len(ids), [d_out.data_ptr()], 0)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(MPICK_DTYPE)


def doorbell_picks(eng, ep, reqs, seed):
    n = min(len(reqs), N.load().lig_stream_capacity())
    eng.stream_open()
    try:
        return eng.stream_submit(ep, seed, np.ascontiguousarray(reqs[:n]))
    finally:
        eng.stream_close()


def all_paths(eng, ep, reqs, seed, ids, scan):
    out = {"host": eng.schedule_batch(ep, seed, reqs)}
    out["queue0"], out["queue1"] = queue_picks(eng, ep, reqs, seed)
    out["models"] = model_picks(eng, ep, ids, seed)
    out["doorbell"] = doorbell_picks(eng, ep, reqs, seed)
    if scan:
        out["scan"] = eng.schedule_scan(ep, seed, reqs, False)[0]
    return out


def read_tables(eng, ep, A, P):
    return [[eng.read_class(ep, bool(crit), a, P) for a in range(A + 1)] for crit in (0, 1)]


def oracle_picks(state, reqs, seed, tree):
    if tree is None:
        from oracle import binding
        want, _ = binding.Pool(state.records()).schedule_batch(state.names()[:-1], WL.UNKNOWN_MODEL, reqs, seed,
                                                               False, binding.hardware_threads())
        return want
    oracle_tree.set_filter_tree(tree)
    try:
        return oracle_tree.Pool(state.records()).schedule_batch(state.names()[:-1], WL.UNKNOWN_MODEL, reqs, seed)
    finally:
        oracle_tree.set_filter_tree(None)


class Rig:
    """Three ctxs: `delta` and `delta_g` (LIG_TAB_SMEM=0) build epochs by deltas, `full` by full
    uploads of the same pools."""

    def __init__(self, monkeypatch, max_pods, max_adapters, max_batch=1 << 15):
        from llm_instance_gateway_b200.engine import Engine
        kw = dict(max_pods=max(max_pods, 1), max_adapters=max(max_adapters, 1), max_batch=max_batch)
        self.delta = Engine(0, **kw)
        with monkeypatch.context() as m:
            m.setenv("LIG_TAB_SMEM", "0")                 # read at lig_create
            self.delta_g = Engine(0, **kw)
        self.full = Engine(0, **kw)
        self.max_pods = kw["max_pods"]

    def close(self):
        for e in (self.delta, self.delta_g, self.full):
            e.close()

    def set_tree(self, nodes):
        for e in (self.delta, self.delta_g, self.full):
            e.set_filter_tree(nodes)

    def upload(self, ep, state):
        packed = state.packed()
        for e in (self.delta, self.delta_g, self.full):
            e.upload_snapshot(ep, packed)

    def update(self, ep, base, state, delta):
        for e in (self.delta, self.delta_g):
            e.update_snapshot(ep, base, **delta)
        self.full.upload_snapshot(ep, state.packed())

    def check(self, ep, state, reqs, seed, tree=None, n_oracle=4096, label=""):
        """The delta epoch `ep` against the full upload `ep`: every class table, every pick path,
        and the oracle on a sample.  Returns the host picks."""
        P, A = state.P, state.A
        got_t, want_t = read_tables(self.delta, ep, A, P), read_tables(self.full, ep, A, P)
        for crit in (0, 1):
            for a in range(A + 1):
                g, w = got_t[crit][a], want_t[crit][a]
                assert g[:2] == w[:2] and np.array_equal(g[2], w[2]), (label, crit, a, g, w)
        packed = state.packed()
        models = pack_models(WL.make_models(A), packed)
        for e in (self.delta, self.full):
            e.upload_models(ep, models)
        ids = WL.make_model_requests(len(reqs), A, seed=seed)
        got = all_paths(self.delta, ep, reqs, seed, ids, tree is None)
        want = all_paths(self.full, ep, reqs, seed, ids, tree is None)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), (label, k)
        assert np.array_equal(want["queue0"], want["host"]), label
        for k, v in zip(("queue0", "queue1"), queue_picks(self.delta_g, ep, reqs, seed)):
            assert v.tobytes() == want[k].tobytes(), (label, "LIG_TAB_SMEM=0", k)
        n = min(len(reqs), n_oracle)
        sub = np.ascontiguousarray(reqs[:n])
        assert np.array_equal(got["host"][:n], oracle_picks(state, sub, seed, tree)), label
        return got["host"]


def dirty_sets(P, rng):
    """0 pods (copy + rebuild), 1, about 1 % (odd), all; each nonempty set holds pod P-1."""
    if P == 0:
        return [np.zeros(0, dtype=np.int64)]
    k = max(3, P // 100) | 1
    few = np.unique(np.concatenate([rng.choice(P, min(k, P), replace=False), [P - 1]]))
    while len(few) > 1 and len(few) % 2 == 0:
        few = few[1:]
    return [np.zeros(0, dtype=np.int64), np.array([P - 1]), few, np.arange(P)]


# ---- 1. delta == full upload ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("P,A", [(0, 0), (1, 0), (1, 3), (33, 5), (1000, 40), (4097, 16), (20000, 8)])
def test_delta_equals_full_upload_pool_shapes(P, A, monkeypatch):
    want_variant = {0: "empty", 1: "fast", 33: "fast", 1000: "fast", 4097: "staged", 20000: "unstaged"}[P]
    assert build_variant(P) == want_variant
    rng = np.random.default_rng(P * 7 + A)
    rig = Rig(monkeypatch, P, A)
    try:
        state = random_state(P, A, seed=P + A)
        rig.upload(1, state)
        reqs = mixed_requests(A, 3000, seed=P)
        seen_odd = False
        for t, dirty in enumerate(dirty_sets(P, rng)):
            new, delta = mutate(state, dirty, rng, edge=(t % 2 == 1))
            if t == 2 and A > 0 and len(delta["adapter_ids"]) % 2 == 0:     # make n_ids odd
                first = int(delta["pod_idx"][0])
                if new.active[first]:
                    delta = delta_between(new, delta["pod_idx"], dup_id=True)
                else:
                    new.active[first] = [0]
                    delta = delta_between(new, delta["pod_idx"])
            n_ids = len(delta["adapter_ids"])
            seen_odd |= len(dirty) % 2 == 1 and n_ids % 2 == 1 and staged_delta_bytes(len(dirty), n_ids)[1]
            before = rig.delta.schedule_batch(t + 1, 7, reqs)
            rig.update(t + 2, t + 1, new, delta)
            assert np.array_equal(rig.delta.schedule_batch(t + 1, 7, reqs), before)   # the base is untouched
            rig.check(t + 2, new, reqs, seed=11 + t, label=f"P={P} A={A} n_dirty={len(dirty)}")
            state = new
        if P >= 33 and A > 0:
            assert seen_odd, "no delta with odd n_dirty and odd n_ids needed the KV column's padding"
    finally:
        rig.close()


@pytest.mark.gpu
def test_delta_chain_of_ticks(monkeypatch):
    """Twelve ticks, epoch k+1 built from epoch k in one ctx, each equal to a full upload; every
    edge value is written by some tick."""
    P, A = 1000, 40
    rng = np.random.default_rng(12)
    rig = Rig(monkeypatch, P, A)
    try:
        state = random_state(P, A, seed=13)
        rig.upload(1, state)
        reqs = mixed_requests(A, 4000, seed=14)
        written_kv, written_q = set(), set()
        for t in range(12):
            k = [0, 1, 13, 101, P][t % 5]
            dirty = np.unique(np.concatenate([rng.choice(P, k, replace=False), [P - 1] if k else []])).astype(np.int64)
            new, delta = mutate(state, dirty, rng, edge=(t % 3 != 2))
            rig.update(t + 2, t + 1, new, delta)
            rig.check(t + 2, new, reqs, seed=100 + t, n_oracle=2048, label=f"tick {t}")
            written_kv |= {repr(float(x)) for x in delta["kv"]}
            written_q |= {int(x) for x in delta["q"]}
            state = new
        assert {repr(x) for x in KV_EDGE} <= written_kv and set(Q_EDGE) <= written_q
    finally:
        rig.close()


@pytest.mark.gpu
def test_delta_moves_classes_between_compact_regimes(monkeypatch):
    """P = 4096 identical pods with room, holding adapters 0..5: the compact tables fit in shared
    memory.  A delta that gives adapter 6 to every pod adds a whole-pool list and pushes them out; a
    delta that takes it away again brings them back."""
    P, A = 4096, 8
    rig = Rig(monkeypatch, P, A)
    try:
        def entries(k):
            # sentinel + the two default lists + the critical list of each held adapter (with room
            # everywhere, a sheddable class with affinity keeps the sheddable default list)
            return 1 + 2 * P + P * k
        s0 = uniform_state(P, A, held=range(6))
        s1 = uniform_state(P, A, held=range(7))
        reqs = mixed_requests(A, 4000, seed=21)
        for ep, k, smem in ((1, 6, True), (2, 7, False), (3, 6, True)):
            if ep == 1:
                rig.upload(1, s0)
            elif ep == 2:
                rig.update(2, 1, s1, delta_between(s1, np.arange(P)))
            else:
                rig.update(3, 2, s0, delta_between(s0, np.arange(P)[::-1]))
            rig.check(ep, s1 if ep == 2 else s0, reqs, seed=ep, label=f"epoch {ep}")
            for e in (rig.delta, rig.full):
                info = e.pick_kernel_info(ep)
                assert info["table_bytes"] == compact_bytes(A, entries(k)), (ep, info)
                assert info["tables_in_smem"] == smem, (ep, info)
            assert (compact_bytes(A, entries(k)) <= TAB_BUDGET) == smem
            assert not rig.delta_g.pick_kernel_info(ep)["tables_in_smem"]
    finally:
        rig.close()


@pytest.mark.gpu
def test_delta_overflows_the_compact_pool_and_grows_its_staging(monkeypatch):
    """P = 20000 identical pods without room.  One delta gives 54 adapters to every pod: 108
    whole-pool lists (both criticalities of each adapter) overflow the compact pool, so the pick
    kernels keep to the strided tables, and the delta, 4.8 MB staged, is larger than the ctx's
    initial staging.  A small delta follows in the grown staging, then one that takes every adapter
    away (the pool fits again)."""
    P, A, k = 20000, 60, 54
    pool_cap = min(2 * (A + 1) * P, 2 * P + 16 + (2 << 20))
    assert 2 * P * k - 10 > pool_cap
    rng = np.random.default_rng(31)
    rig = Rig(monkeypatch, P, A)
    try:
        s0 = uniform_state(P, A, room=False)
        rig.upload(1, s0)
        info = rig.delta.pick_kernel_info(1)
        assert info["table_bytes"] > TAB_BUDGET and not info["tables_in_smem"], info
        reqs = mixed_requests(A, 3000, seed=32)
        s1 = uniform_state(P, A, held=range(k), room=False)
        big = delta_between(s1, rng.permutation(P))
        assert staged_delta_bytes(P, len(big["adapter_ids"]))[0] > initial_delta_capacity(P)
        s2 = s1.copy()
        for p in (3, 7, 11, P - 1, 12345):              # five pods drop their last adapter
            s2.active[p] = list(range(k - 1))
        small = delta_between(s2, [12345, 3, P - 1, 7, 11])
        steps = [(s1, big, True, "overflowed"), (s2, small, True, "small after growth"),
                 (s0, delta_between(s0, np.arange(P)), False, "adapters removed")]
        assert staged_delta_bytes(5, len(small["adapter_ids"]))[0] < initial_delta_capacity(P)
        for ep, (state, delta, overflowed, label) in enumerate(steps, start=2):
            rig.update(ep, ep - 1, state, delta)
            rig.check(ep, state, reqs, seed=ep, n_oracle=2048, label=label)
            for e in (rig.delta, rig.full):
                info = e.pick_kernel_info(ep)
                assert (info["table_bytes"] == 0) == overflowed and not info["tables_in_smem"], (label, info)
    finally:
        rig.close()


def drop_and_no_pods_trees():
    """A tree with DROP leaves on both sides, and one whose last node is a predicate that keeps no
    pod for some classes (LIG_NO_PODS_LEFT)."""
    kv = S.Filter("least KV", S.LEAST_KV_CACHE)
    crit = S.Filter("kv headroom", S.NO_QUEUE_AND_LOW_KV, queue_threshold=40, kv_threshold=0.9,
                    next_on_success=S.Filter("least queuing", S.LEAST_QUEUING, next_on_success_or_failure=kv),
                    next_on_failure=S.Filter("drop", S.DROP))
    shed = S.Filter("affinity", S.LORA_AFFINITY, next_on_success=kv, next_on_failure=S.Filter("drop sheddable", S.DROP))
    drop_tree = S.Filter("critical", S.CRITICAL_REQUEST, next_on_success=crit, next_on_failure=shed).flatten()
    no_pods = S.Filter("low queue", S.LOW_QUEUEING, queue_threshold=50,
                       next_on_success=S.Filter("affinity", S.LORA_AFFINITY)).flatten()
    return [drop_tree, no_pods]


@pytest.mark.gpu
@pytest.mark.parametrize("P,A", [(300, 20), (4097, 12)])
def test_delta_under_caller_trees(P, A, monkeypatch):
    rng = np.random.default_rng(P)
    trees = drop_and_no_pods_trees() + [random_tree(rng) for _ in range(4 if P < 1000 else 2)]
    rig = Rig(monkeypatch, P, A)
    statuses = set()
    try:
        for i, tree in enumerate(trees):
            rig.set_tree(tree)
            state = random_state(P, A, seed=40 + i)
            ep = 10 * i + 1
            rig.upload(ep, state)
            reqs = mixed_requests(A, 2000, seed=41 + i)
            for t, dirty in enumerate(dirty_sets(P, rng)[1:]):
                new, delta = mutate(state, dirty, rng, edge=(t != 1))
                rig.update(ep + 1, ep, new, delta)
                got = rig.check(ep + 1, new, reqs, seed=i + t, tree=tree, label=f"tree {i} n_dirty={len(dirty)}")
                statuses |= set(got["status"].tolist())
                ep += 1
                state = new
        assert {N.LIG_DROP, N.LIG_NO_PODS_LEFT} <= statuses, statuses
    finally:
        rig.close()


@pytest.mark.gpu
def test_malformed_deltas_are_refused_before_anything_is_written():
    """Duplicate pods, offsets that do not start at 0 or decrease, adapter ids outside [0, A): each
    is LIG_ERR_INVALID, and both resident epochs still answer as before.  The malformed offsets stay
    within a few entries of the valid range."""
    from llm_instance_gateway_b200.engine import Engine
    P, A = 100, 6
    rng = np.random.default_rng(50)
    state = random_state(P, A, seed=51)
    reqs = mixed_requests(A, 2000, seed=52)
    with Engine(0, max_pods=128, max_adapters=8, max_batch=1 << 13) as e:
        e.upload_snapshot(1, state.packed())
        new, good = mutate(state, [2, 40, 41, 99], rng, edge=False)
        for p in (2, 40, 41, 99):                        # every pod lists at least one adapter
            new.active[p] = sorted(set(new.active[p]) | {1})
        good = delta_between(new, good["pod_idx"])
        e.update_snapshot(2, 1, **good)
        before = {ep: (e.schedule_batch(ep, 9, reqs), read_tables(e, ep, A, P)) for ep in (1, 2)}

        def with_(**kw):
            d = {k: np.array(v, copy=True) for k, v in good.items()}
            d.update({k: np.asarray(v, dtype=d[k].dtype) for k, v in kw.items()})
            return d

        pods = good["pod_idx"]
        off = good["adapter_offsets"]
        ids = good["adapter_ids"]
        bad = {
            "duplicate pod, adjacent": with_(pod_idx=[pods[0], pods[0], pods[2], pods[3]]),
            "duplicate pod, far apart": with_(pod_idx=[pods[0], pods[1], pods[2], pods[0]]),
            "adapter_offsets[0] = -2": with_(adapter_offsets=np.concatenate([[-2], off[1:]])),
            "decreasing middle offset": with_(adapter_offsets=[off[0], off[2], off[1], off[3], off[4]]),
            "adapter id -1": with_(adapter_ids=np.concatenate([[-1], ids[1:]])),
            "adapter id A": with_(adapter_ids=np.concatenate([ids[:-1], [A]])),
        }
        assert off[2] > off[1] and len(ids) >= 4
        for name, d in bad.items():
            with pytest.raises(N.LigError) as ei:
                e.update_snapshot(3, 2, **d)
            assert ei.value.code == N.LIG_ERR_INVALID, name
            for ep, (picks, tables) in before.items():
                assert np.array_equal(e.schedule_batch(ep, 9, reqs), picks), (name, ep)
                now = read_tables(e, ep, A, P)
                assert all(g[:2] == w[:2] and np.array_equal(g[2], w[2])
                           for rg, rw in zip(now, tables) for g, w in zip(rg, rw)), (name, ep)
        # the same adapter twice in one pod's list is legal: the bit is set twice
        e.update_snapshot(3, 2, **delta_between(new, pods, dup_id=True))
        assert np.array_equal(e.schedule_batch(3, 9, reqs), before[2][0])


# ---- 2. feedback == its sequential definition ---------------------------------------------------------
def tree_feedback_reference(nodes, records, names, reqs, seed, sub_batch, shards=None):
    """oracle/feedback.py's definition with a caller tree: per window, the oracle's port walking
    `nodes` over the pool with the current queue sizes; then add the window's picks, saturating."""
    R, P = len(reqs), len(records)
    shards = shards or [(0, R)]
    q = np.array([r["waiting_queue_size"] for r in records], dtype=np.int64)
    out = np.zeros(R, dtype=PICK_DTYPE)
    total = np.zeros(P, dtype=np.int64)
    n_windows = max((hi - lo + sub_batch - 1) // sub_batch for lo, hi in shards) if R else 0
    oracle_tree.set_filter_tree(nodes)
    try:
        for w in range(n_windows):
            pool = oracle_tree.Pool([dict(r, waiting_queue_size=int(q[i])) for i, r in enumerate(records)])
            hist = np.zeros(P, dtype=np.int64)
            for lo, hi in shards:
                a, b = lo + w * sub_batch, min(lo + (w + 1) * sub_batch, hi)
                if a >= b:
                    continue
                picks = pool.schedule_batch(names[:-1], names[-1], np.ascontiguousarray(reqs[a:b]), seed)
                out[a:b] = picks
                if P:
                    hist += np.bincount(picks["pod_idx"][picks["pod_idx"] >= 0], minlength=P)
            q = np.minimum(q + hist, INT32_MAX)
            total += hist
    finally:
        oracle_tree.set_filter_tree(None)
    return out, total


def reference(state, reqs, seed, sub_batch, thresholds=(0.8, 5, 50)):
    """(picks, totals, queue sizes before each window) of oracle/feedback.py."""
    p = state.packed()
    picks, total, per_window = FB.schedule_batch_feedback(p.P, p.A, p.kv, state.q, p.n_active, p.max_active, p.bitmap,
                                                          reqs, seed, sub_batch, thresholds=thresholds)
    qs = [state.q.copy()]
    for h in per_window:
        qs.append(np.minimum(qs[-1] + h, INT32_MAX))
    return picks, total, qs


def run_feedback(e, ep, seed, reqs, P, sub_batch, n_windows=0, stream=None):
    import torch
    R = len(reqs)
    d_reqs = torch.from_numpy(reqs.view(np.uint8).reshape(-1).copy()).cuda() if R else None
    d_out = torch.full((max(R, 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda")
    d_hist = torch.full((max(P, 1),), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    st = stream or torch.cuda.Stream()
    with torch.cuda.stream(st):
        e.schedule_batch_feedback_device(ep, seed, d_reqs.data_ptr() if R else 0, R, d_out.data_ptr(), sub_batch,
                                         n_windows, d_hist.data_ptr(), st.cuda_stream)
    st.synchronize()
    return d_out[: R * 8].cpu().numpy().view(PICK_DTYPE), d_hist[:P].cpu().numpy().astype(np.int64)


def assert_feedback(got, want, label):
    picks, hist = got
    for f in ("status", "n_survivors", "pod_idx"):
        bad = np.nonzero(picks[f] != want[0][f])[0]
        assert bad.size == 0, (label, f, bad[:5], picks[bad[:5]], want[0][bad[:5]])
    assert np.array_equal(hist, want[1]), label


def feedback_engine(P, A, R=1 << 15):
    from llm_instance_gateway_b200.engine import Engine
    return Engine(0, max_pods=max(P, 1), max_adapters=max(A, 1), max_batch=max(R, 1))


def edge_pool_state(name):
    from test_gpu_parity import EDGE_POOLS
    pods = EDGE_POOLS[name]
    names = sorted({m for p in pods for m in p.Metrics.ActiveModels})
    ids = {m: i for i, m in enumerate(names)}
    return PodState(len(names), [p.Metrics.KVCacheUsagePercent for p in pods], [p.Metrics.WaitingQueueSize for p in pods],
                    [p.Metrics.MaxActiveModels for p in pods], [[ids[m] for m in p.Metrics.ActiveModels] for p in pods])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["all_near_max", "one_at_max", "negative"])
def test_feedback_saturates_at_int32_max(case):
    """Every pod within a few picks of INT32_MAX (the add must clamp), one pod at INT32_MAX among
    low queues (the least-queuing range spans the whole int32 range as the others grow), and
    negative queues down to INT32_MIN."""
    P, A, R, Sb = 33, 4, 3000, 200
    state = random_state(P, A, seed=60)
    if case == "all_near_max":
        state.q[:] = INT32_MAX - np.arange(P) % 7
    elif case == "one_at_max":
        state.q[:] = np.arange(P) % 4
        state.q[17] = INT32_MAX
    else:
        state.q[:] = -(np.arange(P) * 1000)
        state.q[[0, 5, P - 1]] = INT32_MIN
    reqs = WL.make_requests(R, A, seed=61)
    want = reference(state, reqs, 62, Sb)
    qs = np.array(want[2])
    if case == "all_near_max":                   # the saturating add clamped, not just landed on the max
        assert (qs[1:] == INT32_MAX).any() and (state.q + want[1] > INT32_MAX).any()
    elif case == "one_at_max":
        assert (qs[:, 17] == INT32_MAX).all() and want[1][17] == 0 and want[1].sum() > 0
    else:
        assert qs.min() == INT32_MIN and (want[1] > 0).any()
    with feedback_engine(P, A, R) as e:
        e.upload_snapshot(1, state.packed())
        assert_feedback(run_feedback(e, 1, 62, reqs, P, Sb), want, case)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["P=1", "P=33", "P=4097", "P=20000", "edge_pools"])
def test_feedback_pool_shapes(shape):
    from test_gpu_parity import EDGE_POOLS
    if shape == "edge_pools":
        cases = [(name, edge_pool_state(name)) for name in sorted(EDGE_POOLS)]
    else:
        P = int(shape[2:])
        cases = [(shape, random_state(P, 24, seed=P))]
    for label, state in cases:
        R = 6000 if state.P < 4096 else 20000
        Sb = 701 if state.P < 4096 else 4096
        reqs = mixed_requests(state.A, R, seed=state.P)
        want = reference(state, reqs, 70, Sb)
        with feedback_engine(state.P, state.A, len(reqs)) as e:
            e.upload_snapshot(1, state.packed())
            assert_feedback(run_feedback(e, 1, 70, reqs, state.P, Sb), want, label)
        assert want[1].sum() == (want[0]["pod_idx"] >= 0).sum()
        if label == "drop_all":                         # sheddable traffic is dropped and not counted
            assert (want[0]["status"] == N.LIG_DROP).any()
            assert want[1].sum() < len(reqs)


@pytest.mark.gpu
def test_feedback_window_shapes():
    state = random_state(64, 32, seed=80)
    P = state.P
    with feedback_engine(P, 32, 4096) as e:
        e.upload_snapshot(1, state.packed())
        for R, Sb, nw in [(300, 1, 0), (1000, 333, 0), (1000, 1000, 0), (1000, 1005, 0), (1000, 100, 17), (0, 64, 0)]:
            reqs = WL.make_requests(R, 32, seed=R + Sb)
            want = reference(state, reqs, 81, Sb)
            got = run_feedback(e, 1, 81, reqs, P, Sb, nw)
            assert_feedback(got, want, (R, Sb, nw))
            if Sb >= R:                                  # one window: the plain path's picks
                assert np.array_equal(got[0], e.schedule_batch(1, 81, reqs))
                assert np.array_equal(got[1], np.bincount(got[0]["pod_idx"][got[0]["pod_idx"] >= 0], minlength=P))
            if R == 0:
                assert (got[1] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("thresholds", [None, (0.5, 2, 10)])
def test_feedback_herding_crosses_the_queue_thresholds(thresholds):
    """Requests concentrated on three classes: their pods' queues grow past the critical
    `q <= queue_threshold_critical` and the `q < queueing_threshold_lora` predicates during the call."""
    thr = thresholds or (0.8, 5, 50)
    P, A, R, Sb = 48, 8, 4000, 50
    rng = np.random.default_rng(90)
    state = random_state(P, A, seed=91)
    state.q[:] = rng.integers(0, thr[1] + 1, P)
    state.kv[:] = np.round(rng.random(P) * 0.6, 2)
    reqs = WL.make_requests(R, A, seed=92)
    reqs["adapter_id"] = rng.choice([0, 1, A], R)
    want = reference(state, reqs, 93, Sb, thresholds=thr)
    qs = np.array(want[2])
    assert ((qs[:-1] <= thr[1]) & (qs[1:] > thr[1])).any(), "no pod crossed the critical queue threshold"
    assert ((qs[:-1] < thr[2]) & (qs[1:] >= thr[2])).any(), "no pod crossed the LoRA queueing threshold"
    with feedback_engine(P, A, R) as e:
        if thresholds:
            e.set_thresholds(*thresholds)
        e.upload_snapshot(1, state.packed())
        assert_feedback(run_feedback(e, 1, 93, reqs, P, Sb), want, thr)


@pytest.mark.gpu
@pytest.mark.parametrize("P,A,n_trees", [(64, 32, 6), (512, 256, 3), (4097, 16, 2)])
def test_feedback_under_caller_trees(P, A, n_trees):
    rng = np.random.default_rng(P + 1)
    state = random_state(P, A, seed=P + 2)
    records, names = state.records(), state.names()
    R, Sb = (3000, 400) if P < 4096 else (4000, 1000)
    reqs = mixed_requests(A, R, seed=P + 3)
    trees = drop_and_no_pods_trees()[:1] + [random_tree(rng) for _ in range(n_trees - 1)]
    with feedback_engine(P, A, len(reqs)) as e:
        for i, tree in enumerate(trees):
            e.set_filter_tree(tree)
            e.upload_snapshot(i + 1, state.packed())
            want = tree_feedback_reference(tree, records, names, reqs, 5 + i, Sb)
            assert_feedback(run_feedback(e, i + 1, 5 + i, reqs, P, Sb), want, f"tree {i}")


@pytest.mark.gpu
def test_feedback_calls_on_two_streams():
    """Two calls back to back on two streams, no host synchronisation between them: the second
    waits for the first to finish with the ctx's scratch copy."""
    import torch
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=100)
    P = state.P
    reqs = [WL.make_requests(20000, c["A"], seed=101), WL.make_requests(15001, c["A"], seed=102)]
    args = [(5, 2000), (6, 777)]
    wants = [reference(state, r, s, sb) for r, (s, sb) in zip(reqs, args)]
    with feedback_engine(P, c["A"], 20000) as e:
        e.upload_snapshot(1, state.packed())
        plain = e.schedule_batch(1, 5, reqs[0])
        d_in = [torch.from_numpy(r.view(np.uint8).reshape(-1).copy()).cuda() for r in reqs]
        d_out = [torch.zeros(len(r) * 8, dtype=torch.uint8, device="cuda") for r in reqs]
        d_hist = [torch.full((P,), -1, dtype=torch.int32, device="cuda") for _ in reqs]
        torch.cuda.synchronize()
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        for k, st in enumerate(streams):
            with torch.cuda.stream(st):
                e.schedule_batch_feedback_device(1, args[k][0], d_in[k].data_ptr(), len(reqs[k]), d_out[k].data_ptr(),
                                                 args[k][1], 0, d_hist[k].data_ptr(), st.cuda_stream)
        torch.cuda.synchronize()
        for k in range(2):
            got = (d_out[k].cpu().numpy().view(PICK_DTYPE), d_hist[k].cpu().numpy().astype(np.int64))
            assert_feedback(got, wants[k], f"stream {k}")
        assert np.array_equal(e.schedule_batch(1, 5, reqs[0]), plain)      # the resident epoch is untouched


# ---- 3. the caller-tree feedback reference, without a GPU ---------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C5"])
def test_tree_feedback_reference_with_default_filter_equals_the_definition(cfg):
    c = WL.CONFIGS[cfg]
    snap = WL.make_snapshot(c["P"], c["A"], seed=110)
    p = snap.packed
    R = 3000
    reqs = WL.make_requests(R, c["A"], seed=111)
    names = snap.adapter_names() + [WL.UNKNOWN_MODEL]
    for shards in (None, [(0, 1000), (1000, R)], [(0, 1), (1, 1700), (1700, R)]):
        want, want_total, _ = FB.schedule_batch_feedback(p.P, p.A, p.kv, snap.q64, p.n_active, p.max_active, p.bitmap,
                                                         reqs, 5, 256, shards)
        got, total = tree_feedback_reference(S.DEFAULT_FILTER.flatten(), snap.pod_records(), names, reqs, 5, 256, shards)
        assert np.array_equal(got, want) and np.array_equal(total, want_total), shards
    assert want_total.sum() == (want["pod_idx"] >= 0).sum() > 0
