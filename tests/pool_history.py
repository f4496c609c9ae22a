"""Seeded histories of a pod pool for the C++ runtime's refresh tick (test infrastructure).

A history is a list of ticks.  Each tick is the provider's full slice (PodMetrics, in slice order)
and whether Scheduler::Refresh of that slice publishes a new epoch or is refused (more than
max_pods representable pods).  The pool a scheduler must answer for after tick t is the kept pods
(those whose metrics fit the device record) of the last published tick up to t: expected_pools().

Tick kinds (KINDS), one unit or more of each per history, in a seeded order:
  start                the first slice (NewScheduler's refresh)
  qkv_boundary         q and/or KV change on exactly P // 4 pods (dirty * 4 <= P, the largest delta)
  qkv_past             ... on P // 4 + 1 pods (one pod past it: a full upload)
  qkv_most             ... on about three quarters of the pods
  swap                 a few pods swap one adapter name for another already interned name; every
                       pod keeps its adapter count, so only the per-pod name memo sees the change
  add_remove           pods gain or lose a name
  new_names            pods gain names the interning table has never seen
  rebuild              enough fresh names to outgrow max_adapters: the table is rebuilt from scratch
  rebuild_back         every pod goes back to its names from before the rebuild
  reorder              the slice is permuted
  rename               pods are renamed with identical metrics (no pod is dirty, names must follow)
  join_leave           pods leave and new pods join at other positions, P unchanged
  unrepresentable      one pod reports a WaitingQueueSize beyond int32 (excluded from the snapshot)
  representable_again  ... and comes back
  refused              a visible swap plus one extra pod: max_pods + 1 pods, the refresh is refused
  after_refusal        the pool of before the refusal with that tick's swap kept
  kv_bits              KV values change only in the sign of zero or the payload of a NaN
  max_active           MaxActiveModels changes between values that saturate to the same u16
"""
from __future__ import annotations

import dataclasses
import math
import struct
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics

KINDS = ("start", "qkv_boundary", "qkv_past", "qkv_most", "swap", "add_remove", "new_names", "rebuild",
         "rebuild_back", "reorder", "rename", "join_leave", "unrepresentable", "representable_again", "refused",
         "after_refusal", "kv_bits", "max_active")
NEVER_LOADED = "never-loaded"
MAX_ADAPTERS = 16
INT32_MIN, INT32_MAX = -(2 ** 31), 2 ** 31 - 1
SATURATED_HIGH = (65535, 70000, 2 ** 40)       # all pack to MaxActiveModels 65535
SATURATED_LOW = (0, -1, -(2 ** 40))            # all pack to 0


def nan_with_payload(payload: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000000 | payload))[0]


def kv_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def representable(pm: PodMetrics) -> bool:
    """What Scheduler::RefreshImpl keeps in the snapshot (the rest is excluded and counted)."""
    return INT32_MIN <= pm.Metrics.WaitingQueueSize <= INT32_MAX


@dataclasses.dataclass
class Tick:
    kind: str
    pods: List[PodMetrics]     # the provider's slice
    published: bool
    rebuilt: bool = False      # the names of this tick outgrew the interning table (rebuilt from scratch)

    def kept(self) -> List[PodMetrics]:
        return [p for p in self.pods if representable(p)]


def names_of(pods: Sequence[PodMetrics]) -> set:
    return {a for p in pods for a in p.Metrics.ActiveModels}


def records(pods: Sequence[PodMetrics]) -> List[dict]:
    """The oracle's pod records."""
    return [dict(name=p.Pod.Name, address=p.Pod.Address, waiting_queue_size=p.Metrics.WaitingQueueSize,
                 kv_cache_usage_percent=p.Metrics.KVCacheUsagePercent, max_active_models=p.Metrics.MaxActiveModels,
                 active_models=list(p.Metrics.ActiveModels)) for p in pods]


def expected_pools(history: Sequence[Tick]) -> List[List[PodMetrics]]:
    """Per tick, the pool the scheduler answers for: the kept pods of the last published tick."""
    out, last = [], None
    for t in history:
        if t.published:
            last = t.kept()
        assert last is not None, "the first tick must publish"
        out.append(last)
    return out


# (pods, names) -> {(name, critical): (status, [survivor pod names in slice order])}, status numbered as
# include/lig.h (0 OK, 1 DROP, 2 EMPTY, 4 NO_PODS_LEFT)
SurvivorSets = Callable[[Sequence[PodMetrics], Sequence[str]], Dict[Tuple[str, bool], Tuple[int, List[str]]]]


def survivor_sets(nodes=None) -> SurvivorSets:
    """The oracle's survivor sets under the built-in tree (nodes None) or a caller tree."""
    def run(pods, names):
        if nodes is None:
            from oracle import binding
            binding.load()
            pool = binding.Pool(records(pods))
        else:
            import oracle_tree
            oracle_tree.set_filter_tree(nodes)
            pool = oracle_tree.Pool(records(pods))
        out = {}
        for name in names:
            for crit in (False, True):
                rc, idx = pool.filter(name, crit)
                out[(name, crit)] = (rc, [pods[i].Pod.Name for i in idx])
        return out
    return run


def changed_classes(sets: SurvivorSets, before, after) -> List[Tuple[str, bool]]:
    """The classes (name, critical) whose survivor set differs between two pools, over the names of
    both and a never-loaded one."""
    names = sorted(names_of(before) | names_of(after) | {NEVER_LOADED})
    a, b = sets(before, names), sets(after, names)
    return [k for k in a if a[k] != b[k]]


def _pm(name: str, address: str, q: int, kv: float, ma: int, active) -> PodMetrics:
    return PodMetrics(Pod(name, address), Metrics(ActiveModels={a: 1 for a in active}, MaxActiveModels=ma,
                                                  WaitingQueueSize=q, KVCacheUsagePercent=kv))


def _with(pm: PodMetrics, name=None, q=None, kv=None, ma=None, active=None) -> PodMetrics:
    m = pm.Metrics
    return _pm(pm.Pod.Name if name is None else name,
               pm.Pod.Address if name is None else name.replace("pod-", "address-"),
               m.WaitingQueueSize if q is None else q, m.KVCacheUsagePercent if kv is None else kv,
               m.MaxActiveModels if ma is None else ma, list(m.ActiveModels) if active is None else active)


class _Gen:
    def __init__(self, P: int, seed: int, sets: Optional[SurvivorSets]):
        self.P, self.sets = P, sets
        self.rng = np.random.default_rng(seed)
        self.n_names = self.n_pods = 0
        self.live = [self.fresh_name() for _ in range(MAX_ADAPTERS // 2)]
        self.interned: set = set()          # the runtime's grow-only table, as far as the slices decide it
        self.pods = [self.new_pod() for _ in range(P)]
        self.history: List[Tick] = []

    def fresh_name(self) -> str:
        self.n_names += 1
        return f"lora-{self.n_names - 1}"

    def new_pod(self) -> PodMetrics:
        self.n_pods += 1
        r = self.rng
        u, v = r.random(), r.random()
        kv = 0.0 if u < 0.08 else nan_with_payload(1) if u < 0.14 else float(np.round(r.random(), 3))
        ma = int(r.choice(SATURATED_HIGH)) if v < 0.1 else int(r.choice(SATURATED_LOW)) if v < 0.2 else int(r.integers(0, 4))
        small = self.P < 10      # small pools: every pod has a name and a low queue, so names can show
        q = 60 if not small and r.random() < 0.1 else int(r.integers(0, 12))
        k = int(r.integers(1 if small else 0, min(3, len(self.live)) + 1))
        active = [self.live[i] for i in r.choice(len(self.live), size=k, replace=False)]
        return _pm(f"pod-{self.n_pods - 1}", f"address-{self.n_pods - 1}", q, kv, ma, active)

    def emit(self, kind: str, pods: List[PodMetrics], published: Optional[bool] = None):
        kept = [p for p in pods if representable(p)]
        if published is None:
            published = len(kept) <= self.P
        listed = names_of(kept)
        assert len(listed) <= MAX_ADAPTERS
        rebuilt = len(self.interned | listed) > MAX_ADAPTERS
        self.interned = set(listed) if rebuilt else self.interned | listed
        self.history.append(Tick(kind, list(pods), published, rebuilt))

    # ---- per-kind changes; self.pods is always P representable pods between units ----------------
    def new_kv(self, old: float) -> float:
        if math.isnan(old):
            return 0.0
        if old == 0.0:
            return nan_with_payload(1)
        while True:
            kv = float(np.round(self.rng.random(), 3))
            if kv != old:
                return kv

    def qkv(self, kind: str, count: int):
        pods = list(self.pods)
        qmod = 50 if self.P < 10 else 64
        for j, i in enumerate(self.rng.choice(self.P, size=count, replace=False)):
            m = pods[i].Metrics
            q = m.WaitingQueueSize if j % 3 == 1 else (m.WaitingQueueSize + 1 + int(self.rng.integers(0, 20))) % qmod
            kv = m.KVCacheUsagePercent if j % 3 == 0 else self.new_kv(m.KVCacheUsagePercent)
            pods[i] = _with(pods[i], q=q, kv=kv)
        self.pods = pods
        self.emit(kind, pods)

    def swap_once(self, pods: List[PodMetrics], n: int) -> List[PodMetrics]:
        """n pods each trade one listed name for an interned name they do not list.  With survivor
        sets, the pods are taken from the survivors of classes of their names (where a swap shows)."""
        out = list(pods)
        holders = [i for i, p in enumerate(pods) if p.Metrics.ActiveModels]
        if self.sets is not None:
            by_name = {p.Pod.Name: i for i, p in enumerate(pods)}
            names = sorted(names_of(pods))
            sets = self.sets(pods, names)
            cand = sorted({by_name[s] for (a, _), (rc, surv) in sets.items() if rc == 0 for s in surv
                           if a in pods[by_name[s]].Metrics.ActiveModels})
            holders = cand or holders
        for i in self.rng.choice(holders, size=min(n, len(holders)), replace=False):
            have = list(out[i].Metrics.ActiveModels)
            spare = sorted(self.interned - set(have))
            if not spare:
                spare = [self.fresh_name()]
            x = have[int(self.rng.integers(0, len(have)))]
            y = spare[int(self.rng.integers(0, len(spare)))]
            out[i] = _with(out[i], active=[y if a == x else a for a in have])
        return out

    def visible_swap(self, n: int) -> List[PodMetrics]:
        for _ in range(40):
            pods = self.swap_once(self.pods, n)
            if self.sets is None or changed_classes(self.sets, self.pods, pods):
                return pods
        raise AssertionError("no swap changed a survivor set")

    def unit(self, kind: str):
        P, r = self.P, self.rng
        if kind == "qkv_boundary":
            self.qkv(kind, P // 4)
        elif kind == "qkv_past":
            self.qkv(kind, P // 4 + 1)
        elif kind == "qkv_most":
            self.qkv(kind, max(P // 4 + 1, (3 * P) // 4))
        elif kind == "swap":
            self.pods = self.visible_swap(min(3, max(1, P // 8)))
            self.emit(kind, self.pods)
        elif kind == "add_remove":
            pods = list(self.pods)
            for j, i in enumerate(r.choice(P, size=min(P, 4), replace=False)):
                have = list(pods[i].Metrics.ActiveModels)
                if have and (j % 2 or len(have) >= 3):
                    have.pop(int(r.integers(0, len(have))))
                else:
                    spare = [a for a in self.live if a not in have]
                    have.append(spare[int(r.integers(0, len(spare)))] if spare else self.fresh_name())
                pods[i] = _with(pods[i], active=have)
            self.pods = pods
            self.emit(kind, pods)
        elif kind == "new_names":
            pods = list(self.pods)
            for i in r.choice(P, size=min(P, 2), replace=False):
                name = self.fresh_name()
                self.live.append(name)
                pods[i] = _with(pods[i], active=list(pods[i].Metrics.ActiveModels) + [name])
            self.pods = pods
            self.emit(kind, pods)
        elif kind == "rebuild":
            before = self.pods
            fresh = [self.fresh_name() for _ in range(MAX_ADAPTERS - len(self.interned) + 1)]
            remap = {a: fresh[k % len(fresh)] for k, a in enumerate(sorted(names_of(before)))}
            pods = [_with(p, active=sorted({remap[a] for a in p.Metrics.ActiveModels})) for p in before]
            pods[0] = _with(pods[0], active=fresh)             # every fresh name is listed
            self.emit(kind, pods)
            assert self.history[-1].rebuilt
            self.emit("rebuild_back", before)
        elif kind == "reorder":
            self.pods = [self.pods[i] for i in r.permutation(P)]
            self.emit(kind, self.pods)
        elif kind == "rename":
            pods = list(self.pods)
            for i in r.choice(P, size=max(1, P // 10), replace=False):
                self.n_pods += 1
                pods[i] = _with(pods[i], name=f"pod-{self.n_pods - 1}")
            self.pods = pods
            self.emit(kind, pods)
        elif kind == "join_leave":
            k = max(1, P // 20)
            leave = set(r.choice(P, size=k, replace=False).tolist())
            pods = [p for i, p in enumerate(self.pods) if i not in leave]
            for _ in range(k):
                new = self.new_pod()
                if P < 10:
                    new = _with(new, kv=0.0, ma=SATURATED_HIGH[0])
                pods.insert(int(r.integers(0, len(pods) + 1)), new)
            self.pods = pods
            self.emit(kind, pods)
        elif kind == "unrepresentable":
            i = int(r.integers(0, P))
            pods = list(self.pods)
            pods[i] = _with(pods[i], q=INT32_MAX + 1 if r.random() < 0.5 else INT32_MIN - 1)
            self.emit(kind, pods)
            self.emit("representable_again", self.pods)
        elif kind == "refused":
            after = self.visible_swap(1)
            self.emit(kind, after + [self.new_pod()], published=False)
            self.pods = after
            self.emit("after_refusal", after)
        elif kind == "kv_bits":
            pods = list(self.pods)
            for i, p in enumerate(pods):
                kv = p.Metrics.KVCacheUsagePercent
                if math.isnan(kv):
                    pods[i] = _with(p, kv=nan_with_payload(2 if kv_bits(kv) & 0xF == 1 else 1))
                elif kv == 0.0:
                    pods[i] = _with(p, kv=-kv)
            self.pods = pods
            self.emit(kind, pods)
        elif kind == "max_active":
            pods = list(self.pods)
            for i, p in enumerate(pods):
                ma = p.Metrics.MaxActiveModels
                for fam in (SATURATED_HIGH, SATURATED_LOW):
                    if ma in fam:
                        pods[i] = _with(p, ma=fam[(fam.index(ma) + 1) % len(fam)])
            self.pods = pods
            self.emit(kind, pods)
        else:
            raise ValueError(kind)


UNITS = ("qkv_boundary", "qkv_past", "qkv_most", "swap", "add_remove", "new_names", "rebuild", "reorder", "rename",
         "join_leave", "unrepresentable", "refused", "kv_bits", "max_active")


NOT_IN_POOL = Pod("pod-never", "address-never")


def affected(history: Sequence[Tick], t: int) -> List[Pod]:
    """The pods of the slice before tick t that tick t changes by its kind: renamed away (rename),
    at a new index (reorder), gone (join_leave), or no longer representable (unrepresentable)."""
    kind, prev, cur = history[t].kind, history[t - 1].pods, history[t].pods
    now = [p.Pod for p in cur]
    if kind in ("rename", "join_leave"):
        return [p.Pod for p in prev if p.Pod not in now]
    if kind == "reorder":
        return [p.Pod for i, p in enumerate(prev) if now.index(p.Pod) != i]
    if kind == "unrepresentable":
        return [p.Pod for p in cur if not representable(p)]
    return []


def eject_schedule(history: Sequence[Tick], seed: int) -> Dict[int, List[Pod]]:
    """{tick: the complete set Scheduler::EjectPods is called with after that tick's refresh}.

    The set in force at a rename, reorder, join_leave and unrepresentable tick holds up to two of the
    pods that tick changes (ejected the tick before), a kept pod at random and a pod that is in no
    slice.  Once, the whole pool is ejected, and at the next tick the empty set lifts every pod; a
    non-empty set is in force again from the tick after that on, so the sets change across ticks of
    every kind."""
    rng = np.random.default_rng(seed)
    pools = expected_pools(history)
    out: Dict[int, List[Pod]] = {}
    for kind in ("rename", "reorder", "join_leave", "unrepresentable"):
        t = [tk.kind for tk in history].index(kind)
        hit = affected(history, t)
        hit = [hit[i] for i in sorted(rng.choice(len(hit), size=min(2, len(hit)), replace=False))]
        other = pools[t - 1][int(rng.integers(0, len(pools[t - 1])))].Pod
        out[t - 1] = sorted(set(out.get(t - 1, [])) | set(hit) | {other, NOT_IN_POOL}, key=lambda p: p.Name)
    free = [t for t in range(len(history) - 2) if not {t, t + 1, t + 2} & set(out)]
    whole = free[int(rng.integers(0, len(free)))]
    out[whole] = [p.Pod for p in pools[whole]]
    out[whole + 1] = []
    out[whole + 2] = [pools[whole + 2][0].Pod, NOT_IN_POOL]
    return dict(sorted(out.items()))


def make_history(P: int, seed: int, sets: Optional[SurvivorSets] = None) -> List[Tick]:
    """A seeded history over a pool of P pods for a scheduler with max_pods = P and max_adapters =
    MAX_ADAPTERS.  With `sets`, every swap (also the one of a refused tick) changes at least one
    class's survivor set under those survivor sets."""
    g = _Gen(P, seed, sets)
    if P < 10:    # small pools: make sure the kv_bits and max_active ticks have something to flip
        g.pods[-1] = _with(g.pods[-1], kv=0.0, ma=SATURATED_HIGH[0])
    g.emit("start", g.pods)
    units = list(UNITS) + ["qkv_boundary", "swap", "refused", "rename"]
    for i in g.rng.permutation(len(units)):
        g.unit(units[i])
    return g.history
