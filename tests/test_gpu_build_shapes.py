"""Class-table builds at large adapter counts, checked exactly against the class-table oracle.

The fast build (pools of up to 4096 pods) runs min(ceil(2(A+1) / 16), SMs) CTAs of 16 warps.  Warp
w of CTA b builds class w * grid + b, then the classes 16 * grid further on, round-robin: from
A = 8 * SMs adapters on, a warp builds several classes one after the other, fetching its bitmap row
again and reusing its scratch mask for each.  The general build and the caller-tree build deal
their classes the same way.  Every shape below states the regime it is meant to reach, derived from
the device's SM count, and asserts it before checking anything; then, for snapshots whose
per-class answers differ from class to class:

* every class table equals oracle/lig_oracle_classtab.c, and the general build's tables equal the
  fast build's;
* every pick path (host call, persistent queue with and without tables in shared memory, doorbell,
  model queue, direct scan with masks) equals the oracle;
* the built-in tree restated as a caller tree builds the same tables;
* delta epochs equal full uploads at A = 8 * SMs + 17 and A = LIG_MAX_ADAPTERS;
* in-batch load feedback equals its sequential definition while every window rebuild deals several
  classes to a warp."""
import numpy as np
import pytest

from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import pack_models
from test_gpu_snapshot_mutation import (TAB_BUDGET, PodState, Rig, assert_feedback, build_variant, class_requests,
                                        delta_between, doorbell_picks, model_picks, queue_picks, reference,
                                        run_feedback)

pytestmark = pytest.mark.gpu

BUILD_WARPS = 16                # warps per CTA of the built-in builds (kBuildWarps)
TREE_WARPS = 8                  # warps per CTA of the caller-tree build (kWarpsPerCta)
MAX_THREADS_PER_SM = 2048
FAMILIES = ("low", "no_low", "no_shed", "no_room")
Q_LORA, Q_CRIT, KV_THR = 50, 5, 0.8     # the default thresholds


# ---- launch geometry (launch_class_build) --------------------------------------------------------------
def build_geometry(P, A, sm):
    """(build variant, CTAs, most classes one warp builds) of the built-in build: the fast kernel
    runs one CTA per 16 classes, the general one per 32, both capped at one CTA per SM."""
    n = 2 * (A + 1)
    kind = build_variant(P)
    per_cta = BUILD_WARPS if kind == "fast" else 2 * BUILD_WARPS
    grid = max(1, min(-(-n // per_cta), sm))
    return kind, grid, -(-n // (BUILD_WARPS * grid))


def tree_min_classes_per_warp(A, sm):
    """A lower bound on the classes some warp of the caller-tree build takes: its grid is capped
    at SMs x resident 256-thread CTAs per SM, at most 2048 / 256."""
    return -(-2 * (A + 1) // (TREE_WARPS * sm * (MAX_THREADS_PER_SM // (TREE_WARPS * 32))))


def entries_bytes(A):
    """The compact blob's header and class entries alone."""
    return 16 + 16 * 2 * (A + 1)


def strided_slot_bytes(P, A):
    return 2 * (A + 1) * P * 2


def free_device_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def need_bytes(P, A, n_ctx):
    """Device memory for n_ctx ctxs of two slots of strided lists each, plus 2 GiB for the rest."""
    return n_ctx * 2 * strided_slot_bytes(P, A) + (2 << 30)


def skip_unless_memory(P, A, n_ctx):
    free, need = free_device_bytes(), need_bytes(P, A, n_ctx)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory for {n_ctx} ctxs with two slots of "
                    f"strided lists at P = {P}, A = {A}; {free / 2**30:.1f} GiB free")


@pytest.fixture(scope="module")
def sm():
    from llm_instance_gateway_b200.engine import Engine
    with Engine(0, max_pods=1, max_adapters=1, max_batch=1) as e:
        return e.sm_count


# ---- snapshots whose classes differ -------------------------------------------------------------------
def family_state(P, A, family, seed):
    """Every pod holds 8 to 64 adapters, dealt from successive permutations of [0, A) so that every
    adapter has about the same number of holders; queues and KV vary per pod.
      low      about half the pods below the LoRA queueing threshold, room mixed
      no_low   every queue at or above it (the critical side goes through the room mask)
      no_shed  no pod with q <= 5 and kv <= 0.8 (every sheddable class is DROP)
      no_room  n_active >= MaxActiveModels everywhere"""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(8, 65, P)
    deck = np.concatenate([rng.permutation(A) for _ in range(-(-int(sizes.sum()) // A))])
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    active = [deck[cuts[i]:cuts[i + 1]] for i in range(P)]
    n_active = np.array([len(set(a.tolist())) for a in active])
    low = rng.random(P) < 0.5
    q = np.where(low, rng.integers(1, Q_LORA, P), rng.integers(Q_LORA, 4 * Q_LORA, P))
    kv = np.round(rng.random(P), 2)
    ma = np.maximum(n_active + rng.integers(-8, 9, P), 0)
    # pod 0 alone has the shortest queue and is above the KV threshold: from a few hundred pods on
    # the critical default list is [0], which no sheddable list holds
    q[0], kv[0], ma[0] = 0, 0.85, n_active[0] + 8
    if family == "no_low":
        # half the pods share the shortest queue; the ones with room have the higher KV, so the
        # least-KV stage keeps adapter holders over room
        q = np.where(low, Q_LORA, rng.integers(Q_LORA + 1, 4 * Q_LORA, P))
        room = n_active < ma
        kv = np.round(np.where(room, 0.5 + 0.5 * rng.random(P), 0.5 * rng.random(P)), 2)
    elif family == "no_shed":
        shed = (q <= Q_CRIT) & (kv <= KV_THR)
        kv[shed] = np.round(KV_THR + 0.01 + rng.random(int(shed.sum())) * 0.19, 2)
    elif family == "no_room":
        ma = rng.integers(0, n_active + 1)
    return PodState(A, kv, q, ma, active)


def family_holds(state, family):
    q, kv, room = state.q, state.kv, state.n_active() < state.ma
    if family == "low":
        assert 0.3 * state.P <= (q < Q_LORA).sum() <= 0.7 * state.P and 0 < room.sum() < state.P
    elif family == "no_low":
        assert (q >= Q_LORA).all()
    elif family == "no_shed":
        assert not ((q <= Q_CRIT) & (kv <= KV_THR)).any() and (q < Q_LORA).any()
    else:
        assert not room.any()


def expected_tables(state):
    from oracle import binding
    p = state.packed()
    return binding.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap,
                              nthreads=binding.hardware_threads())


def klass_of(c, A):
    return (c >= A + 1, c - (A + 1) if c >= A + 1 else c)


def assert_round_robin_pairs_differ(tab, A, grid, rng, family):
    """The classes a warp builds one after the other (c and c + 16 * grid) must have different
    answers, else a stale row or scratch word would go unseen.  Checked on a sample of pairs with
    a critical class (in no_shed and no_low every sheddable class is DROP): at most half of them
    may agree."""
    step = BUILD_WARPS * grid
    firsts = np.arange(max(0, 2 * (A + 1) - step))
    firsts = firsts[firsts + step >= A + 1]
    assert firsts.size > 0
    sample = rng.choice(firsts, min(256, firsts.size), replace=False)
    same = sum(tab.klass(*klass_of(int(c), A)) == tab.klass(*klass_of(int(c) + step, A)) for c in sample)
    assert same <= sample.size // 2, (family, same, sample.size)


def class_sample(A, grid, rng, n=4096):
    """A random sample of classes plus every class within 40 of a multiple of 16 * grid (where a
    warp's next class starts) and the first and last ones."""
    nc = 2 * (A + 1)
    step = BUILD_WARPS * grid
    near = np.concatenate([np.arange(m - 40, m + 41) for m in range(0, nc + step, step)])
    picked = np.concatenate([rng.choice(nc, min(n, nc), replace=False), near, [0, A, A + 1, nc - 1]])
    return np.unique(picked[(picked >= 0) & (picked < nc)])


def assert_tables(got_engine, ep, want, A, P, classes, label):
    """want: the oracle table, or another engine (compared class by class)."""
    for c in classes:
        crit, a = klass_of(int(c), A)
        st, n, lst = got_engine.read_class(ep, crit, a, P)
        if hasattr(want, "klass"):
            w = want.klass(crit, a)
        else:
            ws, wn, wl = want.read_class(ep, crit, a, P)
            w = (ws, wn, wl.tolist())
        assert (st, n, lst.tolist()) == w, (label, int(c), crit, a, st, n, w[:2])


def requests_for(A, seed, R=20000):
    return np.ascontiguousarray(np.concatenate([class_requests(A, seed=seed), WL.make_requests(R, A, seed=seed + 1)]))


def model_ids_for(A, seed, R=20000):
    """Every model id once (one per adapter, the base model, the splits), then a random batch."""
    n_models = A + 1 + WL.N_SPLIT_MODELS
    return np.ascontiguousarray(np.concatenate([np.arange(n_models, dtype=np.uint32),
                                                WL.make_model_requests(R, A, seed=seed)]))


def pick_paths(e, ep, reqs, seed, ids=None):
    out = {"host": e.schedule_batch(ep, seed, reqs)}
    out["queue0"], out["queue1"] = queue_picks(e, ep, reqs, seed)
    out["doorbell"] = doorbell_picks(e, ep, reqs, seed)
    if ids is not None:
        out["models"] = model_picks(e, ep, ids, seed)
    return out


def assert_picks_equal(got, want, label):
    for f in ("status", "n_survivors", "pod_idx"):
        bad = np.nonzero(got[f] != want[f][:len(got)])[0]
        assert bad.size == 0, (label, f, bad[:5], got[bad[:5]], want[bad[:5]])


def engine_for(monkeypatch, P, A, R, fast=True, tab_smem=True):
    from llm_instance_gateway_b200.engine import Engine
    with monkeypatch.context() as m:
        m.setenv("LIG_FAST_BUILD", "1" if fast else "0")          # both read at lig_create
        m.setenv("LIG_TAB_SMEM", "1" if tab_smem else "0")
        return Engine(0, max_pods=P, max_adapters=A, max_batch=R)


# ---- 1. every shape, every family -----------------------------------------------------------------------
SHAPES = [  # (P, A as a function of the SM count s, regime)
    (1000, "8s-1", "one"), (4096, "8s-1", "one"),
    (33, "8s", "second"), (2049, "8s", "second"), (4096, "8s", "second"),
    (4096, "8s+17", "two_smem"),
    (4096, "3000", "strided"),
    (4095, "16384", "many"), (4096, "16384", "many"),
    (4096, "65534", "max"),
    (4097, "8s", "general"), (4097, "16384", "general"),
]


def resolve_A(spec, s):
    return int(eval(spec.replace("8s", "8*s"), {"s": s}))


def assert_regime(P, A, regime, sm):
    kind, grid, per_warp = build_geometry(P, A, sm)
    n = 2 * (A + 1)
    if regime == "one":
        assert (kind, grid, per_warp) == ("fast", sm, 1) and n == BUILD_WARPS * grid, (P, A, kind, grid, per_warp)
    elif regime == "second":
        assert kind == "fast" and per_warp == 2 and n - BUILD_WARPS * grid == 2, (P, A, kind, grid, per_warp)
    elif regime == "two_smem":
        assert kind == "fast" and per_warp == 2 and entries_bytes(A) <= TAB_BUDGET, (P, A, kind, grid, per_warp)
    elif regime == "strided":
        assert kind == "fast" and 2 <= per_warp <= 3 and entries_bytes(A) > TAB_BUDGET, (P, A, kind, grid, per_warp)
    elif regime == "many":
        assert kind == "fast" and per_warp >= 8 and tree_min_classes_per_warp(A, sm) >= 2, (P, A, grid, per_warp)
    elif regime == "max":
        assert A == N.LIG_MAX_ADAPTERS and kind == "fast" and per_warp >= 32 and tree_min_classes_per_warp(A, sm) >= 2
    else:
        assert kind == "staged" and per_warp >= 2, (P, A, kind, grid, per_warp)
    return grid, per_warp


@pytest.mark.parametrize("P,A_spec,regime", SHAPES, ids=[f"P={p}-A={a}" for p, a, _ in SHAPES])
def test_class_tables_and_picks_at_shape(P, A_spec, regime, sm, monkeypatch):
    from oracle import binding
    A = resolve_A(A_spec, sm)
    grid, per_warp = assert_regime(P, A, regime, sm)
    with_tree = regime in ("many", "max")
    skip_unless_memory(P, A, 3 if with_tree else 2)
    reqs = requests_for(A, seed=P + A)
    R = len(reqs)
    rng = np.random.default_rng(P * 31 + A)
    ctxs = {"fast": engine_for(monkeypatch, P, A, R), "general": engine_for(monkeypatch, P, A, R, fast=False, tab_smem=False)}
    if with_tree:
        ctxs["tree"] = engine_for(monkeypatch, P, A, R)
        ctxs["tree"].set_filter_tree(S.DEFAULT_FILTER.flatten())
    fast, general = ctxs["fast"], ctxs["general"]
    # every table of every ctx at up to 16384 adapters; at LIG_MAX_ADAPTERS the fast build's in
    # full, the others on a sample that holds every warp's change of class
    every = np.arange(2 * (A + 1))
    others = every if A <= 16384 else class_sample(A, grid, rng)
    try:
        for ep, family in enumerate(FAMILIES, start=1):
            label = f"P={P} A={A} {family}"
            state = family_state(P, A, family, seed=1000 * ep + P + A)
            family_holds(state, family)
            tab = expected_tables(state)
            if family == "no_shed":
                assert all(tab.klass(False, a)[0] == N.LIG_DROP for a in (0, A // 2, A - 1, A))
            if per_warp > 1:
                assert_round_robin_pairs_differ(tab, A, grid, rng, family)
            packed = state.packed()
            models = pack_models(WL.make_models(A), packed)
            for e in ctxs.values():
                e.upload_snapshot(ep, packed)
                e.upload_models(ep, models)
            # 1. every class table
            assert_tables(fast, ep, tab, A, P, every, label + " fast")
            assert_tables(general, ep, fast, A, P, others, label + " general")
            # the table regime the picks read
            info = fast.pick_kernel_info(ep)
            in_smem = 0 < info["table_bytes"] <= TAB_BUDGET
            assert info["tables_in_smem"] == in_smem, (label, info)
            if regime == "two_smem":
                assert in_smem, (label, info)
            if entries_bytes(A) > TAB_BUDGET:
                assert not info["tables_in_smem"], (label, info)
            assert not general.pick_kernel_info(ep)["tables_in_smem"]
            # 2. every pick path against the class-table oracle
            seed = 7 + ep                   # the second of two queued batches draws with seed + 1
            want = tab.schedule_batch(reqs, seed, nthreads=binding.hardware_threads())
            want1 = tab.schedule_batch(reqs, seed + 1, nthreads=binding.hardware_threads())
            ids = model_ids_for(A, seed)
            got = {k: pick_paths(e, ep, reqs, seed, ids) for k, e in (("fast", fast), ("general", general))}
            for name in got:
                for k in ("host", "queue0", "doorbell"):
                    assert_picks_equal(got[name][k], want, (label, name, k))
                assert_picks_equal(got[name]["queue1"], want1, (label, name, "queue1"))
            assert got["fast"]["models"].tobytes() == got["general"]["models"].tobytes(), label
            # the model queue, the direct scan with its masks and the port itself on samples
            pool = binding.Pool(state.records())
            n_m = 2048
            sample_ids = np.ascontiguousarray(np.concatenate([ids[:n_m // 2], ids[-n_m // 2:]]))
            m_got = np.concatenate([got["fast"]["models"][:n_m // 2], got["fast"]["models"][-n_m // 2:]])
            m_want = binding.Models(WL.model_records(WL.make_models(A))).schedule_batch(
                pool, sample_ids[:n_m // 2], seed, nthreads=binding.hardware_threads())
            m_want2 = binding.Models(WL.model_records(WL.make_models(A))).schedule_batch(
                pool, sample_ids[n_m // 2:], seed, first_index=len(ids) - n_m // 2, nthreads=binding.hardware_threads())
            assert np.array_equal(m_got, np.concatenate([m_want, m_want2])), label
            sel = np.unique(np.concatenate([rng.choice(R, 3072, replace=False), np.arange(1024) * (R // 1024)]))[:4096]
            sub = np.ascontiguousarray(reqs[sel])
            port, port_masks = pool.schedule_batch(state.names()[:-1], WL.UNKNOWN_MODEL, sub, seed, True,
                                                   binding.hardware_threads())
            assert np.array_equal(port, want[sel]), label
            scan_sel = slice(0, 1024)
            picks, masks = fast.schedule_scan(ep, seed, np.ascontiguousarray(sub[scan_sel]), True, packed.W)
            assert np.array_equal(picks, port[scan_sel]), label
            assert np.array_equal(masks, port_masks[scan_sel]), label
            # 3. the built-in tree as a caller tree: same tables, same picks
            if with_tree:
                tree = ctxs["tree"]
                assert_tables(tree, ep, fast, A, P, others, label + " caller tree")
                t_got = pick_paths(tree, ep, reqs, seed)
                for k in ("host", "queue0", "doorbell"):
                    assert_picks_equal(t_got[k], want, (label, "caller tree", k))
                assert_picks_equal(t_got["queue1"], want1, (label, "caller tree", "queue1"))
            del tab
    finally:
        for e in ctxs.values():
            e.close()


# ---- 2. deltas at large A --------------------------------------------------------------------------------
def redraw(state, dirty, rng, seed):
    """A copy of `state` with the pods in `dirty` redrawn from the `low` family, and among them: the
    first drops all its adapters, the second gains ids A-1 and A-32.  The delta lists the pods in
    a shuffled order and repeats an id in its first pod's list."""
    A = state.A
    fresh = family_state(len(dirty), A, "low", seed)
    new = state.copy()
    for k, p in enumerate(dirty):
        new.kv[p], new.q[p], new.ma[p] = fresh.kv[k], fresh.q[k], fresh.ma[k]
        new.active[p] = fresh.active[k]
    if len(dirty) >= 1:
        new.active[dirty[0]] = []
    if len(dirty) >= 2:
        new.active[dirty[1]] = sorted(set(new.active[dirty[1]]) | {A - 1, A - 32})
    order = rng.permutation(len(dirty))
    if len(dirty) >= 2 and order[0] == 0:                 # the repeated id goes to a pod with adapters
        order = np.roll(order, -1)
    delta = delta_between(new, np.asarray(dirty)[order], dup_id=True)
    return new, delta


def dirty_sets(P, rng):
    """One pod, about 1 % of the pods (an odd count), every pod."""
    k = max(3, P // 100) | 1
    return [np.array([P - 1]), np.sort(rng.choice(P, k, replace=False)), rng.permutation(P)]


@pytest.mark.parametrize("P,A_spec", [(1000, "8s+17"), (4096, "65534")], ids=["P=1000-A=8s+17", "P=4096-A=65534"])
def test_deltas_at_large_adapter_counts(P, A_spec, sm, monkeypatch):
    from oracle import binding
    A = resolve_A(A_spec, sm)
    kind, grid, per_warp = build_geometry(P, A, sm)
    assert kind == "fast" and per_warp >= 2, (P, A, grid, per_warp)
    skip_unless_memory(P, A, 3)
    rng = np.random.default_rng(A)
    reqs = requests_for(A, seed=A)
    rig = Rig(monkeypatch, P, A, max_batch=len(reqs))
    try:
        state = family_state(P, A, "low", seed=5)
        rig.upload(1, state)
        for t, dirty in enumerate(dirty_sets(P, rng)):
            new, delta = redraw(state, dirty, rng, seed=50 + t)
            assert not new.active[dirty[0]]
            if len(dirty) >= 2:
                ids, off = delta["adapter_ids"], delta["adapter_offsets"]
                assert len(np.unique(ids[off[0]:off[1]])) < off[1] - off[0], "the first pod's list repeats an id"
                assert {A - 1, A - 32} <= set(new.active[dirty[1]])
            ep = t + 2
            rig.update(ep, ep - 1, new, delta)
            label = f"P={P} A={A} n_dirty={len(dirty)}"
            if A <= 4096:
                rig.check(ep, new, reqs, seed=11 + t, label=label)
            else:
                # every class through its picks, the tables of a sample holding every warp's change
                # of class, and the class-table oracle on every request
                tab = expected_tables(new)
                classes = class_sample(A, grid, rng)
                assert_tables(rig.delta, ep, tab, A, P, classes, label + " delta")
                assert_tables(rig.full, ep, tab, A, P, classes, label + " full")
                # the second of two queued batches draws with the next seed
                want = {k: tab.schedule_batch(reqs, 11 + t + (k == "queue1"), nthreads=binding.hardware_threads())
                        for k in ("host", "queue1")}
                want["queue0"] = want["doorbell"] = want["host"]
                for name, e in (("delta", rig.delta), ("full", rig.full)):
                    for k, v in pick_paths(e, ep, reqs, 11 + t).items():
                        assert_picks_equal(v, want[k], (label, name, k))
                for k, v in zip(("queue0", "queue1"), queue_picks(rig.delta_g, ep, reqs, 11 + t)):
                    assert_picks_equal(v, want[k], (label, "LIG_TAB_SMEM=0", k))
                del tab
            state = new
    finally:
        rig.close()


# ---- 3. in-batch load feedback --------------------------------------------------------------------------
def test_feedback_with_several_classes_per_warp(sm):
    """One feedback call of six windows at P = 1000, A = 8 * SMs + 17: every window's rebuild runs
    the fast build with two classes on some warps."""
    from llm_instance_gateway_b200.engine import Engine
    P, A = 1000, 8 * sm + 17
    kind, grid, per_warp = build_geometry(P, A, sm)
    assert kind == "fast" and per_warp == 2
    state = family_state(P, A, "low", seed=71)
    reqs = requests_for(A, seed=72, R=3000)
    Sb = -(-len(reqs) // 6)
    want = reference(state, reqs, 73, Sb)
    assert len(want[2]) - 1 >= 4
    with Engine(0, max_pods=P, max_adapters=A, max_batch=len(reqs)) as e:
        e.upload_snapshot(1, state.packed())
        assert_feedback(run_feedback(e, 1, 73, reqs, P, Sb), want, f"P={P} A={A}")
