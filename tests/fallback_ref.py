"""The fallback ranking of include/lig.h in numpy (test infrastructure).

A LIG_OK request with survivor list L of n pods draws its pick r_0 = Int31n(n) on its stream
(state = seed ^ rand_key), then continues the same stream: step j = 1 .. m-1 (m = min(n, 1 + k))
draws r_j = j + Int31n(n - j), and every step swaps perm[j] and perm[r_j] in a partial Fisher-Yates
shuffle of [0, n).  The row holds L[perm[1]] .. L[perm[m-1]], padded with -1 to k entries.
"""
from __future__ import annotations

import numpy as np

from helpers import np_splitmix_int31


def int31n_step(state: np.ndarray, n: np.ndarray, active: np.ndarray):
    """Go 1.22 Int31n(n) on each active stream, continuing `state`: (new state, value, rejections).
    Inactive streams keep their state and give 0."""
    n = np.where(active, n, 1).astype(np.int64)
    state2, v = np_splitmix_int31(state)
    state = np.where(active, state2, state)
    pow2 = (n & (n - 1)) == 0
    mx = (1 << 31) - 1 - ((1 << 31) % n)
    rejections = np.zeros(len(n), dtype=np.int64)
    pending = active & ~pow2 & (v > mx)
    while pending.any():
        state2, v2 = np_splitmix_int31(state)
        state = np.where(pending, state2, state)
        v = np.where(pending, v2, v)
        rejections += pending
        pending = pending & (v > mx)
    k = np.where(pow2, v & (n - 1), v % n)
    return state, np.where(active, k, 0), rejections


def fallback_rows(seed: int, keys: np.ndarray, ok: np.ndarray, starts: np.ndarray, counts: np.ndarray,
                  pods: np.ndarray, k: int, with_draws: bool = False):
    """Rows (R, k) int16 for requests with rand_key `keys`, LIG_OK mask `ok` and survivor lists
    pods[starts[i]:starts[i] + counts[i]] (a CSR such as lig_filter_batch's, or one list per class
    shared by its requests).  Also returns r_0 per request (the pick's index into its list, -1 where
    not ok); with_draws adds (r, rejections) per step, shape (R, k + 1) each."""
    keys = np.asarray(keys, dtype=np.uint64)
    R = len(keys)
    ok = np.asarray(ok, dtype=bool)
    starts = np.asarray(starts, dtype=np.int64)
    pods = np.asarray(pods).astype(np.int64)
    n = np.where(ok, np.asarray(counts, dtype=np.int64), 0)
    m = np.minimum(n, 1 + k)
    state = np.uint64(seed) ^ keys
    rows = np.full((R, k), -1, dtype=np.int16)
    draws = np.zeros((R, k + 1), dtype=np.int64)
    rejects = np.zeros((R, k + 1), dtype=np.int64)
    state, r0, rej = int31n_step(state, n, n >= 1)
    draws[:, 0], rejects[:, 0] = r0, rej
    # perm as a record of (position, value) writes; the latest write to a position wins
    pos = [r0.copy()]
    val = [np.zeros(R, dtype=np.int64)]
    for j in range(1, k + 1):
        active = j < m
        state, t, rej = int31n_step(state, n - j, active)
        rj = j + t
        a = np.full(R, j, dtype=np.int64)
        b = rj.copy()
        for p, v in zip(pos, val):
            a = np.where(p == j, v, a)
            b = np.where(p == rj, v, b)
        pos.append(np.where(active, rj, -1))
        val.append(a)
        idx = np.where(active, starts + b, 0)
        rows[:, j - 1] = np.where(active, pods[idx] if len(pods) else 0, -1)
        draws[:, j], rejects[:, j] = np.where(active, rj, 0), rej
    r0 = np.where(n >= 1, r0, -1)
    if with_draws:
        return rows, r0, draws, rejects
    return rows, r0


def fallback_row(seed: int, key: int, survivors, k: int):
    """One request: (pick, row) by the definition, written as a plain Fisher-Yates loop."""
    from helpers import np_splitmix_int31 as nxt
    L = list(survivors)
    n = len(L)
    if n == 0:
        return -1, [-1] * k
    state = np.array([(seed ^ key) & ((1 << 64) - 1)], dtype=np.uint64)

    def int31n(bound):
        nonlocal state
        state, v = nxt(state)
        v = int(v[0])
        if bound & (bound - 1) == 0:
            return v & (bound - 1)
        mx = (1 << 31) - 1 - ((1 << 31) % bound)
        while v > mx:
            state, v = nxt(state)
            v = int(v[0])
        return v % bound

    perm = list(range(n))
    ranked = []
    for j in range(min(n, 1 + k)):
        r = j + int31n(n - j)
        perm[j], perm[r] = perm[r], perm[j]
        ranked.append(L[perm[j]])
    return ranked[0], ranked[1:] + [-1] * (k - len(ranked) + 1)
