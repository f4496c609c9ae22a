"""Session affinity (lig_schedule_[models_]batch_affinity, include/lig.h) by its definition (test
infrastructure).

Pod p of an epoch carries h_p = mix(pod_key[p]), mix the SplitMix64 finalizer.  A LIG_OK request with
affinity key k and survivor list L ranks L by the score s(k, p) = mix(k ^ h_p), descending, ties (equal
pod keys only) to the lower pod index.  The pick is ranked entry 0; the row holds entries 1 .. m-1,
m = min(n, 1 + n_fallbacks), padded with -1.  A request that is not LIG_OK picks -1 and gets a row of
-1.  Model ids resolve as lig_schedule_models_batch does, but the target draw's state is
k ^ LIG_DRAW_DOMAIN.  Nothing depends on a seed or on the request's place in the batch.
"""
from __future__ import annotations

import numpy as np

from helpers import np_splitmix_int31
from llm_instance_gateway_b200.packer import MPICK_DTYPE, REQ_DTYPE, PackedModels

M64 = (1 << 64) - 1
LIG_OK, LIG_NO_MODEL = 0, 3
LIG_DRAW_DOMAIN = 0xA0761D6478BD642F
SELF = 255
FNV_OFFSET, FNV_PRIME = 0xCBF29CE484222325, 0x100000001B3


def mix(z):
    """The SplitMix64 finalizer, elementwise on uint64 (a bijection of 64-bit words)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def pod_key(name: str, address: str) -> int:
    """A pod's key in both schedulers: FNV-1a 64 over Name, a zero byte, then Address."""
    h = FNV_OFFSET
    for b in name.encode() + b"\0" + address.encode():
        h = ((h ^ b) * FNV_PRIME) & M64
    return h


def ranking(key: int, survivors, pod_keys) -> list:
    """Every member of `survivors` (pod indices) in descending score for `key`, ties to the lower pod."""
    L = np.asarray(list(survivors), dtype=np.int64)
    if len(L) == 0:
        return []
    s = mix(np.uint64(key & M64) ^ mix(np.asarray(pod_keys, dtype=np.uint64)[L]))
    return L[np.lexsort((L, ~s))].tolist()


def affinity_row(key: int, survivors, pod_keys, k: int):
    """One LIG_OK request: (pick, row of k entries)."""
    r = ranking(key, survivors, pod_keys)
    if not r:
        return -1, [-1] * k
    ranked = r[:1 + k]
    return ranked[0], ranked[1:] + [-1] * (k + 1 - len(ranked))


def affinity_rows(keys, ok, offsets, pods, pod_keys, k: int):
    """(pick int64 (R,), rows int16 (R, k)) for requests whose survivor lists are
    pods[offsets[i]:offsets[i + 1]] (lig_filter_batch's CSR) and LIG_OK mask `ok`."""
    keys = np.asarray(keys, dtype=np.uint64)
    R = len(keys)
    pick = np.full(R, -1, dtype=np.int64)
    rows = np.full((R, k), -1, dtype=np.int16)
    h = mix(np.asarray(pod_keys, dtype=np.uint64))
    pods = np.asarray(pods, dtype=np.int64)
    for i in np.flatnonzero(np.asarray(ok, dtype=bool)):
        L = pods[offsets[i]:offsets[i + 1]]
        if len(L) == 0:
            continue
        s = mix(keys[i] ^ h[L])
        if len(L) > 1 + k:
            keep = ~s <= np.partition(~s, k)[k]   # every score tied with or above the (k+1)-th largest
            L, s = L[keep], s[keep]
        ranked = L[np.lexsort((L, ~s))][:1 + k]
        pick[i] = ranked[0]
        rows[i, :len(ranked) - 1] = ranked[1:]
    return pick, rows


def affinity_resolve(pm: PackedModels, ids, keys) -> np.ndarray:
    """Model ids at their affinity keys -> (descriptors, resolved mask, target_idx): the resolve of
    lig_schedule_models_batch with draw state key ^ LIG_DRAW_DOMAIN.  Descriptors carry rand_key = key."""
    ids = np.asarray(ids, dtype=np.uint32)
    keys = np.asarray(keys, dtype=np.uint64)
    R = len(ids)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["rand_key"] = keys
    ok = np.zeros(R, dtype=bool)
    target = np.full(R, SELF, dtype=np.uint8)
    for i, m in enumerate(ids.tolist()):
        if m >= pm.n_models or not pm.present[m]:
            continue
        lo, hi = int(pm.target_offsets[m]), int(pm.target_offsets[m + 1])
        nt = hi - lo
        if nt == 0:
            adapter = int(pm.self_adapter_ids[m])
        elif nt == 1:
            adapter, target[i] = int(pm.target_adapter_ids[lo]), 0
        else:
            w = pm.target_weights[lo:hi].astype(np.int64)
            r = int31n(int(keys[i]) ^ LIG_DRAW_DOMAIN, int(w.sum()))
            t = int(np.searchsorted(np.cumsum(w), r, side="right"))
            t = min(t, nt - 1)
            adapter, target[i] = int(pm.target_adapter_ids[lo + t]), t
        reqs["adapter_id"][i] = adapter
        reqs["flags"][i] = 1 if pm.critical[m] else 0
        ok[i] = True
    return reqs, ok, target


def int31n(state: int, n: int) -> int:
    """Go 1.22 Int31n(n) on a SplitMix64 stream started at `state`."""
    st = np.array([state & M64], dtype=np.uint64)
    while True:
        st, v = np_splitmix_int31(st)
        v = int(v[0])
        if n & (n - 1) == 0:
            return v & (n - 1)
        if v <= (1 << 31) - 1 - ((1 << 31) % n):
            return v % n


def as_mpicks(plain: np.ndarray, resolved: np.ndarray, target: np.ndarray, pick: np.ndarray) -> np.ndarray:
    """lig_mpick rows: `plain` the descriptor call's picks of the resolved requests."""
    out = np.zeros(len(plain), dtype=MPICK_DTYPE)
    out["pod_idx"] = np.where(resolved, pick, -1)
    out["status"] = np.where(resolved, plain["status"], LIG_NO_MODEL)
    out["target_idx"] = np.where(resolved, target, SELF)
    return out
