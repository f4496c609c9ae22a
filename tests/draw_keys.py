"""Request keys that make the first draws of a request's random stream take chosen values.

The stream of a request is SplitMix64 (include/lig.h): state += golden gamma, then an output mix of
xor-shifts and odd multipliers.  Every step of that mix is a bijection of 64-bit words, so for any
31-bit value v the words whose top 31 bits (Int31() = next() >> 33) are v can be inverted back to
the state that produces them.  The state minus the gamma is the stream's initial state
`seed ^ rand_key` (picks) or `seed ^ rand_key ^ LIG_DRAW_DOMAIN` (model draws), which gives the key
or the seed.  The suite uses this to hit Int31n's accept boundaries and rejection loops on purpose.
"""
from __future__ import annotations

import numpy as np

from helpers import np_splitmix_int31

GAMMA = 0x9E3779B97F4A7C15
MUL1 = 0xBF58476D1CE4E5B9
MUL2 = 0x94D049BB133111EB
LIG_DRAW_DOMAIN = 0xA0761D6478BD642F
M64 = (1 << 64) - 1
_INV1 = np.uint64(pow(MUL1, -1, 1 << 64))
_INV2 = np.uint64(pow(MUL2, -1, 1 << 64))


def _unxorshift(y: np.ndarray, k: int) -> np.ndarray:
    """Inverse of x -> x ^ (x >> k) on uint64."""
    x = y.copy()
    s = k
    while s < 64:
        x ^= y >> np.uint64(s)
        s += k
    return x


def states_for(v, rng: np.random.Generator | None = None) -> np.ndarray:
    """Initial states whose first Int31() is v (one per element of v; the free low 33 bits of the
    mixed word are random)."""
    rng = rng if rng is not None else np.random.default_rng(0)
    v = np.asarray(v, dtype=np.uint64).reshape(-1)
    assert (v < np.uint64(1 << 31)).all()
    low = rng.integers(0, 1 << 33, size=v.size, dtype=np.uint64)
    z = (v << np.uint64(33)) | low
    with np.errstate(over="ignore"):
        z = _unxorshift(z, 31)
        z = z * _INV2
        z = _unxorshift(z, 27)
        z = z * _INV1
        s = _unxorshift(z, 30)
        return s - np.uint64(GAMMA)


def pick_keys(seed: int, v, rng: np.random.Generator | None = None) -> np.ndarray:
    """rand_key per element of v such that the pick's first Int31() under `seed` is v."""
    return states_for(v, rng) ^ np.uint64(seed & M64)


def draw_seed(v, key: int = 0, rng: np.random.Generator | None = None) -> np.ndarray:
    """Seeds such that a model request with rand_key `key` draws randomVal's first Int31() = v."""
    return states_for(v, rng) ^ np.uint64(key & M64) ^ np.uint64(LIG_DRAW_DOMAIN)


def first_draws(states: np.ndarray, k: int) -> np.ndarray:
    """The first k Int31() of each initial state, shape (len(states), k)."""
    s = np.asarray(states, dtype=np.uint64).copy()
    out = np.empty((s.size, k), dtype=np.int64)
    for i in range(k):
        s, out[:, i] = np_splitmix_int31(s)
    return out


def accept_top(n: int) -> int:
    """Int31n(n) accepts a draw v iff v < top (Go: v <= 2^31-1-(2^31 % n)); a power of two never rejects."""
    return (1 << 31) if n & (n - 1) == 0 else ((1 << 31) // n) * n


def double_reject_states(n: int, want: int, rng: np.random.Generator, batch: int = 1 << 20,
                         max_batches: int = 64) -> np.ndarray:
    """Up to `want` initial states whose first TWO Int31() are both rejected by Int31n(n): invert
    random rejected first values and keep those whose second draw is rejected as well."""
    top = accept_top(n)
    if top == 1 << 31:
        return np.zeros(0, dtype=np.uint64)
    found = []
    got = 0
    for _ in range(max_batches):
        v1 = rng.integers(top, 1 << 31, size=batch, dtype=np.int64)
        st = states_for(v1, rng)
        d = first_draws(st, 2)
        keep = st[d[:, 1] >= top]
        found.append(keep)
        got += keep.size
        if got >= want:
            break
    return np.concatenate(found)[:want]


def rejection_heavy_ns(lo: int, hi: int, count: int) -> list:
    """The `count` n in [lo, hi] with the widest rejection band (2^31 mod n) / 2^31."""
    n = np.arange(lo, hi + 1, dtype=np.int64)
    r = (1 << 31) % n
    order = np.argsort(-r, kind="stable")[:count]
    return sorted(int(x) for x in n[order])
