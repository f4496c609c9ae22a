"""Expected answers of every request entry point at the request fields' edges, from the CPU only (test
infrastructure).

The survivor list of each (critical, adapter) class of a pool comes from an oracle: the class-table
oracle (oracle.binding.ClassTable.klass) for the built-in tree, filter_tree_ref.walk for a caller tree,
and either of them on eject_ref.reduced's snapshot for an ejected epoch, mapped back to the epoch's pod
order.  Requests are turned into a CSR of those lists (offsets, pods: lig_filter_batch's shape) and the
existing definitions rank it: fallback_ref.fallback_rows for the pick and the fallback rows,
affinity_ref.affinity_rows for affinity.  Model ids resolve with oracle.binding.Models (the draw) or
affinity_ref.affinity_resolve (affinity).  Nothing here reads a device result.

An adapter id outside [0, A), whether a request carries it or a model table does, is the class of A:
the adapter no pod lists (include/lig.h, lig_req.adapter_id and lig_upload_models).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

import draw_keys as DK
import eject_ref as ER
import fallback_ref as FR
import filter_tree_ref as FT
import retry_ref as RR
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE, PackedModels
from oracle import binding as B

M64 = (1 << 64) - 1
INT32_MAX, INT32_MIN = (1 << 31) - 1, -(1 << 31)


def hostile_adapters(A: int) -> List[int]:
    """Adapter ids that name no adapter of a pool with A adapters."""
    return [-1, A, A + 1, INT32_MAX, INT32_MIN]


def adapter_name(a: int, A: int) -> str:
    """The name the oracles see for adapter id a: the pool's name, or one no pod lists."""
    return WL.adapter_name(a) if 0 <= a < A else f"unloaded-{a}"


class ClassLists:
    """Survivor lists of every class c = critical * (A + 1) + a, a in [0, A], of one epoch: `snap` built
    with the built-in tree (nodes None, `thresholds`) or the caller tree `nodes`, without the pods
    `ejected` (None: an uploaded epoch).  Pod indices are in `snap`'s order."""

    def __init__(self, snap, nodes=None, ejected: Optional[Sequence[int]] = None, thresholds=(0.8, 5, 50)):
        self.P, self.A = snap.P, snap.A
        small, kept = (snap, np.arange(snap.P, dtype=np.int64)) if ejected is None else ER.reduced(snap, ejected)
        self.status = np.zeros(2 * (self.A + 1), dtype=np.int64)
        self.n = np.zeros(2 * (self.A + 1), dtype=np.int64)
        self.lists: List[np.ndarray] = []
        if nodes is None:
            tab = B.ClassTable(small.P, small.A, small.kv, small.q, small.n_active, small.max_active, small.bitmap,
                               thresholds)
        else:
            pods = FT.Pods(RR.records(small))
        for c in range(2 * (self.A + 1)):
            crit, a = c // (self.A + 1), c % (self.A + 1)
            if nodes is None:
                st, n, lst = tab.klass(bool(crit), a)
            else:
                st, lst = FT.walk(nodes, pods, bool(crit), adapter_name(a, self.A))
                n = len(lst)
            self.status[c], self.n[c] = st, n
            self.lists.append(ER.map_back(kept, np.asarray(lst, dtype=np.int64)))

    def classes(self, reqs: np.ndarray) -> np.ndarray:
        crit = (reqs["flags"] & N.LIG_REQ_CRITICAL).astype(np.int64)
        a = reqs["adapter_id"].astype(np.int64)
        return crit * (self.A + 1) + np.where((a >= 0) & (a < self.A), a, self.A)

    def csr(self, reqs: np.ndarray, keep=None):
        """(LIG_OK mask, int64 offsets[R + 1], int64 pods): request i's survivors are
        pods[offsets[i]:offsets[i + 1]], empty unless it is LIG_OK (and keep[i], when given)."""
        c = self.classes(reqs)
        ok = self.status[c] == N.LIG_OK
        if keep is not None:
            ok &= np.asarray(keep, dtype=bool)
        parts = [self.lists[ci] if o else np.zeros(0, np.int64) for ci, o in zip(c.tolist(), ok.tolist())]
        offsets = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        pods = np.concatenate(parts + [np.zeros(0, np.int64)]).astype(np.int64)
        return ok, offsets, pods

    def fallbacks(self, reqs: np.ndarray, seed: int, k: int, keep=None):
        """(picks PICK_DTYPE, rows (R, k) int16): lig_schedule_batch's picks and the fallback rows, both
        ranked by fallback_ref on the CSR (the pick is ranked entry 0)."""
        ok, offsets, pods = self.csr(reqs, keep)
        c = self.classes(reqs)
        rows, r0 = FR.fallback_rows(seed, reqs["rand_key"], ok, offsets[:-1], np.diff(offsets), pods, k)
        out = np.zeros(len(reqs), dtype=PICK_DTYPE)
        out["pod_idx"] = np.where(ok, pods[np.where(ok, offsets[:-1] + np.maximum(r0, 0), 0)] if len(pods) else -1,
                                  -1)
        out["status"] = self.status[c]
        out["n_survivors"] = self.n[c]
        return out, rows

    def picks(self, reqs: np.ndarray, seed: int) -> np.ndarray:
        return self.fallbacks(reqs, seed, 0)[0]


# ---- model tables --------------------------------------------------------------------------------------
def hostile_models(A: int) -> List[Optional[dict]]:
    """Model records (oracle.binding.Models's input, None = absent) whose own and target adapters include
    every hostile id, with 0, 1 and >= 2 targets, and a weight-1 target beside a large one.  A model's
    name is its own adapter's, so a model without targets resolves to it."""
    bad = hostile_adapters(A)
    ok = [a for a in (0, A - 1, A // 2) if 0 <= a < A] or [A]
    nm = lambda a: adapter_name(a, A)
    recs: List[Optional[dict]] = []
    for i, a in enumerate(bad + ok[:1]):                     # no targets: the own id
        recs.append(dict(name=nm(a), critical=bool(i & 1), targets=[]))
    for i, a in enumerate(bad + ok[-1:]):                    # one target
        recs.append(dict(name=f"single-{i}", critical=not (i & 1), targets=[(nm(a), 1 + 7 * i)]))
    recs.append(None)                                        # absent
    recs.append(dict(name="split-0", critical=True, targets=[(nm(ok[0]), 1), (nm(INT32_MAX), 1_000_000)]))
    recs.append(dict(name="split-1", critical=False, targets=[(nm(INT32_MIN), 5), (nm(A), 7), (nm(ok[-1]), 1)]))
    recs.append(dict(name="split-2", critical=True, targets=[(nm(-1), 1), (nm(ok[0]), 1 << 30), (nm(A + 1), 3),
                                                              (nm(ok[-1]), 2)]))
    recs.append(dict(name="split-3", critical=False, targets=[(nm(a), 1) for a in bad + ok]))
    return recs


def _id_of(name: str, A: int) -> int:
    """The raw id a caller uploads for `name` (the inverse of adapter_name)."""
    if name.startswith("unloaded-"):
        return int(name[len("unloaded-"):])
    return int(name[len("adapter-"):])


def pack_raw_models(recs: Sequence[Optional[dict]], A: int) -> PackedModels:
    """The lig_upload_models arrays of `recs`, adapter ids as given (hostile ones included, unchecked)."""
    n = len(recs)
    off = np.zeros(n + 1, dtype=np.int32)
    ids, wts = [], []
    crit = np.zeros(n, dtype=np.uint8)
    self_ids = np.zeros(n, dtype=np.int32)
    present = np.ones(n, dtype=np.uint8)
    names = []
    for m, r in enumerate(recs):
        if r is None:
            present[m] = 0
            self_ids[m] = INT32_MIN
            names.append([])
        else:
            crit[m] = 1 if r["critical"] else 0
            self_ids[m] = _id_of(r["name"], A) if not r["targets"] else -1
            for t, w in r["targets"]:
                ids.append(_id_of(t, A))
                wts.append(w)
            names.append([t for t, _ in r["targets"]])
        off[m + 1] = len(ids)
    return PackedModels(n_models=n, target_offsets=off, target_adapter_ids=np.array(ids, dtype=np.int32),
                        target_weights=np.array(wts, dtype=np.int32), critical=crit, self_adapter_ids=self_ids,
                        present=present, model_ids={r["name"]: m for m, r in enumerate(recs) if r},
                        target_names=names)


def model_ids(n_models: int, R: int, rng: np.random.Generator) -> np.ndarray:
    """Every id of the table, n_models and 2^32-1, then random ones of the same mix."""
    edge = np.array(list(range(n_models)) + [n_models, (1 << 32) - 1], dtype=np.uint32)
    pool = np.concatenate([edge, edge[-2:]])
    ids = rng.choice(pool, size=R).astype(np.uint32)
    ids[: min(R, len(edge))] = edge[: min(R, len(edge))]
    return np.ascontiguousarray(ids)



# ---- request keys and adapter ids ----------------------------------------------------------------------
def edge_requests(cl: ClassLists, R: int, seed: int, rng: np.random.Generator) -> np.ndarray:
    """R descriptors: valid and hostile adapter ids, critical 0 / 1, and rand_keys 0, 2^64-1, random keys,
    and keys whose pick (under `seed`) or fallback step 1 takes an Int31n rejection at the request's
    survivor count."""
    A = cl.A
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    ids = np.array(hostile_adapters(A) + list(range(A)), dtype=np.int64)
    reqs["adapter_id"] = rng.choice(ids, size=R).astype(np.int32)
    reqs["adapter_id"][: min(R, 5)] = hostile_adapters(A)[: min(R, 5)]
    reqs["flags"] = rng.integers(0, 2, R).astype(np.uint32)
    reqs["rand_key"] = rng.integers(0, 1 << 64, size=R, dtype=np.uint64)
    kind = rng.integers(0, 6, R)
    reqs["rand_key"][kind == 0] = 0
    reqs["rand_key"][kind == 1] = np.uint64(M64)
    c = cl.classes(reqs)
    n = np.where(cl.status[c] == N.LIG_OK, cl.n[c], 0)
    for i in np.flatnonzero(kind >= 4).tolist():
        reqs["rand_key"][i] = rejecting_key(int(n[i]), seed, step=int(kind[i]) - 4, rng=rng)
    return reqs


def rejecting_key(n: int, seed: int, step: int, rng: np.random.Generator) -> int:
    """A rand_key whose pick (step 0) or first fallback step (step 1, Int31n(n - 1) after an accepted
    Int31n(n)) draws a rejected value first; a random key when that bound never rejects."""
    bound = n if step == 0 else n - 1
    if bound < 3 or DK.accept_top(bound) == 1 << 31:
        return int(rng.integers(0, 1 << 64, dtype=np.uint64))
    top = DK.accept_top(bound)
    for _ in range(64):
        v = rng.integers(top, 1 << 31, size=1, dtype=np.int64)
        st = DK.states_for(v, rng)
        if step == 1:                      # the second word is v: start one gamma earlier
            with np.errstate(over="ignore"):
                st = st - np.uint64(DK.GAMMA)
            if DK.first_draws(st, 1)[0, 0] >= DK.accept_top(n):
                continue                   # the pick itself would reject: not the case wanted
        return int(st[0] ^ np.uint64(seed & M64))
    raise AssertionError("no key found")
