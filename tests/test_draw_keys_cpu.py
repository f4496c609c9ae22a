"""The key construction of tests/draw_keys.py: crafted keys really produce the chosen first draws,
checked with the numpy restatement of the stream and with the oracle's Int31n."""
import numpy as np

import draw_keys as DK
from helpers import np_int31n, np_splitmix_int31

EDGE_V = [0, 1, 2, (1 << 30), (1 << 31) - 2, (1 << 31) - 1]


def test_pick_keys_give_the_chosen_first_draw():
    rng = np.random.default_rng(1)
    v = np.concatenate([EDGE_V, rng.integers(0, 1 << 31, 20000)]).astype(np.int64)
    for seed in (0, 1, 0x5EED, (1 << 64) - 1):
        keys = DK.pick_keys(seed, v, rng)
        _, got = np_splitmix_int31(np.uint64(seed) ^ keys)
        assert np.array_equal(got, v)
    # the free low bits are random: the same value gives different keys
    k = DK.pick_keys(7, np.zeros(64, dtype=np.int64), rng)
    assert len(set(k.tolist())) == 64


def test_draw_seed_gives_the_chosen_model_draw():
    rng = np.random.default_rng(2)
    v = np.concatenate([EDGE_V, rng.integers(0, 1 << 31, 2000)]).astype(np.int64)
    for key in (0, 77, 1 << 33):
        seeds = DK.draw_seed(v, key, rng)
        _, got = np_splitmix_int31(seeds ^ np.uint64(key) ^ np.uint64(DK.LIG_DRAW_DOMAIN))
        assert np.array_equal(got, v)


def test_keys_against_the_oracle_int31n(oracle):
    """Accepted draws give v % n, the first rejected one resamples: both agree with the oracle's
    lig_oracle_int31n and with np_int31n."""
    rng = np.random.default_rng(3)
    seed = 0xABCDEF
    for n in (3, 5, 7, 100, 1000, 4097, 12289, 21846, 32767, 32768, 1 << 30 | 1, (1 << 31) - 1):
        top = DK.accept_top(n)
        vs = sorted({0, n - 1, n, n + 1, max(top - n - 1, 0), max(top - n, 0), top - 1} |
                    ({top, (1 << 31) - 1} if top < (1 << 31) else set()))
        vs = [x for x in vs if x < (1 << 31)]
        keys = DK.pick_keys(seed, vs, rng)
        want = np_int31n(seed, keys, np.full(len(vs), n))
        for v, key, w in zip(vs, keys, want):
            assert oracle.int31n(seed ^ int(key), n) == int(w), (n, v)
            if v < top:
                assert int(w) == v % n, (n, v)


def test_double_rejections_are_rejected_twice(oracle):
    rng = np.random.default_rng(4)
    ns = DK.rejection_heavy_ns(2, 32768, 6)
    assert all((1 << 31) % n > n // 2 for n in ns)
    for n in ns:
        st = DK.double_reject_states(n, 4, rng)
        assert st.size >= 1, n
        d = DK.first_draws(st, 3)
        top = DK.accept_top(n)
        assert (d[:, 0] >= top).all() and (d[:, 1] >= top).all()
        keys = st ^ np.uint64(9)
        got = np_int31n(9, keys, np.full(st.size, n))
        # the value is that of the first accepted draw
        for i in range(st.size):
            k = 2
            s = st[i:i + 1].copy()
            draws = DK.first_draws(s, 8)[0]
            while draws[k] >= top:
                k += 1
            assert got[i] == draws[k] % n
            assert oracle.int31n(int(st[i]), n) == int(got[i])
    # a power of two has no rejection band
    assert DK.double_reject_states(4096, 4, rng).size == 0


def test_rejection_heavy_ns():
    ns = DK.rejection_heavy_ns(2, 32768, 40)
    assert len(ns) == 40 and len(set(ns)) == 40
    r = [(1 << 31) % n for n in ns]
    assert min(r) >= sorted(((1 << 31) % n for n in range(2, 32769)), reverse=True)[39]
