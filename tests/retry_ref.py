"""Retry scheduling (lig_schedule_batch_excluding, include/lig.h) by its definition (test infrastructure).

A request's pool is the epoch's pods in their order minus the distinct entries of its row that lie
in [0, P).  The reference builds that pool literally: the kept pods' columns in order and the bitmap
columns of the removed pods dropped.  It then runs Schedule on it, with the class-table oracle for
the built-in tree or the oracle_tree walker for a caller tree, and maps the result back to the
epoch's pod indices.  It never masks a full pool, so it shares no logic with the kernel.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

import oracle_tree as OT
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, PackedSnapshot, pack_columns
from oracle import binding as B

FILLER = "~not-an-adapter-"      # ActiveModels entries that are no adapter of the snapshot


def kept_pods(P: int, row) -> np.ndarray:
    """The request's pool: every pod of [0, P) that no in-range entry of `row` names, in order."""
    gone = {int(e) for e in row if 0 <= int(e) < P}
    return np.array([p for p in range(P) if p not in gone], dtype=np.int64)


def _unpack(bitmap: np.ndarray, P: int) -> np.ndarray:
    A, W = bitmap.shape
    if A == 0 or W == 0:
        return np.zeros((A, P), dtype=bool)
    bits = np.unpackbits(np.ascontiguousarray(bitmap).view(np.uint8).reshape(A, W * 4), axis=1, bitorder="little")
    return bits[:, :P].astype(bool)


def _pack(member: np.ndarray) -> np.ndarray:
    A, P = member.shape
    W = (P + 31) // 32
    padded = np.zeros((A, W * 32), dtype=np.uint8)
    padded[:, :P] = member
    return np.packbits(padded, axis=1, bitorder="little").view(np.uint32).reshape(A, W) if W else \
        np.zeros((A, 0), dtype=np.uint32)


def reduce_snapshot(snap: PackedSnapshot, kept: np.ndarray) -> PackedSnapshot:
    """The snapshot of the pool `kept`: those pods' columns in order, the other bitmap columns dropped."""
    member = _unpack(snap.bitmap, snap.P)[:, kept]
    return pack_columns(snap.kv[kept], snap.q[kept].astype(np.int64), snap.n_active[kept].astype(np.int64),
                        snap.max_active[kept].astype(np.int64), _pack(member), snap.adapter_ids,
                        [snap.pods[int(p)] for p in kept])


def adapter_names(snap: PackedSnapshot) -> List[str]:
    names = [""] * snap.A
    for name, a in snap.adapter_ids.items():
        if 0 <= a < snap.A:
            names[a] = name
    return [n or f"adapter-{a}" for a, n in enumerate(names)]


def records(snap: PackedSnapshot) -> List[dict]:
    """Oracle pod records of a packed snapshot: ActiveModels holds the pod's adapters from the bitmap,
    padded with names of no adapter up to n_active."""
    names = adapter_names(snap)
    member = _unpack(snap.bitmap, snap.P)
    out = []
    for p in range(snap.P):
        act = [names[a] for a in np.nonzero(member[:, p])[0]]
        act += [f"{FILLER}{j}" for j in range(int(snap.n_active[p]) - len(act))]
        out.append(dict(name=snap.pods[p].Name, address=snap.pods[p].Address,
                        waiting_queue_size=int(snap.q[p]), kv_cache_usage_percent=float(snap.kv[p]),
                        max_active_models=int(snap.max_active[p]), active_models=act))
    return out


def pack_records(recs: Sequence[dict], names: Sequence[str]) -> PackedSnapshot:
    """A packed snapshot of oracle records whose adapters are `names` (other ActiveModels entries count
    toward n_active only)."""
    P, A = len(recs), len(names)
    ids = {n: a for a, n in enumerate(names)}
    bitmap = np.zeros((A, (P + 31) // 32), dtype=np.uint32)
    for p, r in enumerate(recs):
        for m in r["active_models"]:
            if m in ids:
                bitmap[ids[m], p >> 5] |= np.uint32(1 << (p & 31))
    return pack_columns(np.array([r["kv_cache_usage_percent"] for r in recs], dtype=np.float64),
                        np.array([r["waiting_queue_size"] for r in recs], dtype=np.int64),
                        np.array([len(r["active_models"]) for r in recs], dtype=np.int64),
                        np.array([r["max_active_models"] for r in recs], dtype=np.int64), bitmap, ids,
                        [WL.Pod(r["name"], r["address"]) for r in recs])


def _groups(P: int, excluded: np.ndarray) -> Dict[Tuple[int, ...], List[int]]:
    groups: Dict[Tuple[int, ...], List[int]] = {}
    for i, row in enumerate(excluded):
        groups.setdefault(tuple(kept_pods(P, row).tolist()), []).append(i)
    return groups


def retry_batch(snap: PackedSnapshot, reqs: np.ndarray, excluded: np.ndarray, seed: int,
                thresholds=(0.8, 5, 50), nodes=None) -> np.ndarray:
    """lig_schedule_batch_excluding by its definition: picks (PICK_DTYPE) with pod_idx in the epoch's
    pod order.  nodes: the caller tree that built the epoch (None = the built-in tree with
    `thresholds`)."""
    excluded = np.asarray(excluded).reshape(len(reqs), -1)
    out = np.zeros(len(reqs), dtype=PICK_DTYPE)
    if nodes is not None:
        OT.set_filter_tree(nodes)
    try:
        for kept_t, idx in _groups(snap.P, excluded).items():
            kept = np.array(kept_t, dtype=np.int64)
            small = reduce_snapshot(snap, kept)
            sub = np.ascontiguousarray(reqs[idx])
            if nodes is None:
                got = B.ClassTable(small.P, small.A, small.kv, small.q, small.n_active, small.max_active,
                                   small.bitmap, thresholds).schedule_batch(sub, seed)
            else:
                got = OT.Pool(records(small)).schedule_batch(adapter_names(small), WL.UNKNOWN_MODEL, sub, seed)
            pod = got["pod_idx"].astype(np.int64)
            got["pod_idx"] = np.where(pod >= 0, kept[np.maximum(pod, 0)] if len(kept) else -1, -1)
            out[idx] = got
    finally:
        if nodes is not None:
            OT.set_filter_tree(None)
    return out


def survivors(snap: PackedSnapshot, critical: bool, adapter: int, row, thresholds=(0.8, 5, 50),
              nodes=None) -> Tuple[int, List[int]]:
    """(status, survivors in the epoch's pod indices) of one request class over the pool without `row`."""
    kept = kept_pods(snap.P, row)
    small = reduce_snapshot(snap, kept)
    if nodes is None:
        st, _, lst = B.ClassTable(small.P, small.A, small.kv, small.q, small.n_active, small.max_active,
                                  small.bitmap, thresholds).klass(critical, adapter if 0 <= adapter < small.A
                                                                  else small.A)
        return st, [int(kept[p]) for p in lst]
    OT.set_filter_tree(nodes)
    try:
        names = adapter_names(small)
        model = names[adapter] if 0 <= adapter < small.A else WL.UNKNOWN_MODEL
        st, lst = OT.Pool(records(small)).filter(model, critical)
    finally:
        OT.set_filter_tree(None)
    return st, [int(kept[p]) for p in lst]
