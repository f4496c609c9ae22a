"""The pool histories of tests/pool_history.py test what they claim to test (no GPU).

tests/test_gpu_runtime_refresh.py drives the C++ runtime through these histories and compares it
with the oracle after every tick.  Here, on the CPU: every history holds every tick kind, every
tick kind changes what it says it changes, and every swap tick and every tick after a refusal
changes at least one class's survivor set in the oracle, so a runtime that missed the change
would answer differently.
"""
import math

import pytest

import pool_history as PH
from test_gpu_snapshot_mutation import drop_and_no_pods_trees

# (id, P, caller tree: None = the built-in tree, 0 = DROP leaves, 1 = a "no pods left" leaf)
CASES = [("p1", 1, None), ("p33", 33, None), ("p1000", 1000, None), ("p4097", 4097, None), ("p5000", 5000, None),
         ("drop_tree", 33, 0), ("no_pods_tree", 33, 1), ("no_pods_tree_p1", 1, 1)]


def case_sets(tree):
    return PH.survivor_sets(None if tree is None else drop_and_no_pods_trees()[tree])


def case_history(P, tree, seed):
    # one pod under the built-in tree: every class is that pod or a drop, whatever it lists, so no
    # swap can show there (the one-pod history under a caller tree's affinity leaf covers names)
    sets = None if (P == 1 and tree is None) else case_sets(tree)
    return PH.make_history(P, seed, sets)


def by_name(pods):
    return {p.Pod.Name: p for p in pods}


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_history_holds_every_kind_and_every_kind_does_its_change(case):
    _, P, tree = case
    hist = case_history(P, tree, seed=P + 7 * (tree or 0))
    kinds = [t.kind for t in hist]
    assert set(kinds) == set(PH.KINDS), set(PH.KINDS) - set(kinds)
    assert kinds[0] == "start" and hist[0].published
    pools = PH.expected_pools(hist)
    for t, tick in enumerate(hist):
        kept = tick.kept()
        assert len(kept) == (P + 1 if tick.kind == "refused" else P - 1 if tick.kind == "unrepresentable" else P)
        assert tick.published == (tick.kind != "refused")
        assert len(PH.names_of(kept)) <= PH.MAX_ADAPTERS
        if t == 0:
            continue
        prev, cur = hist[t - 1].kept(), kept
        if tick.kind in ("qkv_boundary", "qkv_past", "qkv_most"):
            n = sum(1 for a, b in zip(prev, cur)
                    if (a.Metrics.WaitingQueueSize, PH.kv_bits(a.Metrics.KVCacheUsagePercent))
                    != (b.Metrics.WaitingQueueSize, PH.kv_bits(b.Metrics.KVCacheUsagePercent)))
            want = {"qkv_boundary": P // 4, "qkv_past": P // 4 + 1}.get(tick.kind, max(P // 4 + 1, 3 * P // 4))
            assert n == want and all(a.Pod == b.Pod and a.Metrics.ActiveModels == b.Metrics.ActiveModels
                                     for a, b in zip(prev, cur))
        elif tick.kind in ("swap", "after_refusal"):
            # a swap keeps every pod's adapter count and changes at least one pod's names
            base = pools[t - 1]
            assert [p.Pod for p in base] == [p.Pod for p in cur]
            assert all(len(a.Metrics.ActiveModels) == len(b.Metrics.ActiveModels) for a, b in zip(base, cur))
            assert any(a.Metrics.ActiveModels != b.Metrics.ActiveModels for a, b in zip(base, cur))
        elif tick.kind == "rename":
            assert [p.Metrics for p in prev] == [p.Metrics for p in cur]
            assert [p.Pod for p in prev] != [p.Pod for p in cur]
        elif tick.kind == "reorder":
            assert by_name(prev).keys() == by_name(cur).keys()
        elif tick.kind == "join_leave":
            assert by_name(prev).keys() != by_name(cur).keys() and len(prev) == len(cur)
        elif tick.kind == "new_names":
            assert PH.names_of(cur) - PH.names_of(p for tk in hist[:t] for p in tk.kept())
        elif tick.kind == "rebuild":
            assert tick.rebuilt
        elif tick.kind == "kv_bits":
            flips = [(a.Metrics.KVCacheUsagePercent, b.Metrics.KVCacheUsagePercent) for a, b in zip(prev, cur)
                     if PH.kv_bits(a.Metrics.KVCacheUsagePercent) != PH.kv_bits(b.Metrics.KVCacheUsagePercent)]
            assert flips and all(x == y or (math.isnan(x) and math.isnan(y)) for x, y in flips)
        elif tick.kind == "max_active":
            pairs = [(a.Metrics.MaxActiveModels, b.Metrics.MaxActiveModels) for a, b in zip(prev, cur)
                     if a.Metrics.MaxActiveModels != b.Metrics.MaxActiveModels]
            assert pairs and all(min(max(x, 0), 65535) == min(max(y, 0), 65535) for x, y in pairs)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_eject_schedule_holds_every_situation(case):
    """The ejected sets of tests/test_gpu_runtime_refresh.py: across the history, the set in force
    at a rename, reorder, join_leave and unrepresentable tick holds a pod that tick changes; a set
    names a pod that is in no slice; one set is the whole pool, and the empty set lifts it."""
    _, P, tree = case
    hist = case_history(P, tree, seed=P + 7 * (tree or 0))
    pools = PH.expected_pools(hist)
    sched = PH.eject_schedule(hist, seed=P)
    assert sched == PH.eject_schedule(hist, seed=P)
    seen, active = set(), []
    for t, tick in enumerate(hist):
        if t and set(active) & set(PH.affected(hist, t)):
            seen.add(tick.kind)
        if t in sched:
            new = sched[t]
            pool = {p.Pod for p in pools[t]}
            seen |= {"not_in_pool"} if set(new) - pool else set()
            seen |= {"whole_pool"} if pool <= set(new) else set()
            seen |= {"lifted"} if active and not new else set()
            active = new
    want = {"rename", "reorder", "join_leave", "unrepresentable", "not_in_pool", "whole_pool", "lifted"}
    assert seen == (want - {"reorder"} if P == 1 else want), seen      # one pod cannot move


@pytest.mark.parametrize("case", [c for c in CASES if not (c[1] == 1 and c[2] is None)],
                         ids=[c[0] for c in CASES if not (c[1] == 1 and c[2] is None)])
def test_swaps_and_refusals_change_survivor_sets(case):
    """A swap tick, and the tick after a refused one, against the pool the scheduler held before it:
    at least one class's survivor set differs in the oracle."""
    _, P, tree = case
    sets = case_sets(tree)
    hist = case_history(P, tree, seed=P + 7 * (tree or 0))
    pools = PH.expected_pools(hist)
    checked = 0
    for t, tick in enumerate(hist):
        if tick.kind in ("swap", "after_refusal"):
            assert PH.changed_classes(sets, pools[t - 1], pools[t]), (t, tick.kind)
            checked += 1
        if tick.kind == "refused":
            assert pools[t] is pools[t - 1]
    assert checked == 4
