"""Session affinity (include/lig.h) without a GPU: the numpy definition (affinity_ref.py), its properties
(distinct scores, independence of pod order, consistency when the survivor set shrinks, uniform picks over
keys, prefix rows), the model-id draw on k ^ LIG_DRAW_DOMAIN against the oracle's draw, the pod-key
function in Python and C++, and the C ABI's refusals and exports."""
import os
import re

import numpy as np
import pytest
from scipy import stats

import affinity_ref as AR
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Pod
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models
from llm_instance_gateway_b200.scheduling import pod_key
from oracle import lig_oracle_py as PY

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rng = np.random.default_rng(2026)


def test_scores_are_distinct_for_distinct_pod_keys():
    pod_keys = np.unique(rng.integers(0, 1 << 64, size=20000, dtype=np.uint64))
    h = AR.mix(pod_keys)
    assert len(np.unique(h)) == len(pod_keys)
    for k in rng.integers(0, 1 << 64, size=16, dtype=np.uint64):
        assert len(np.unique(AR.mix(k ^ h))) == len(pod_keys)


def test_ties_break_to_the_lower_pod():
    keys = np.array([7, 7, 9, 7], dtype=np.uint64)
    r = AR.ranking(123, [0, 1, 2, 3], keys)
    sevens = [p for p in r if p != 2]
    assert sevens == [0, 1, 3]


@pytest.mark.parametrize("n", [1, 4, 31, 33, 300])
def test_pick_and_rows_do_not_depend_on_pod_order(n):
    pod_keys = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    perm = rng.permutation(n)
    inv = np.argsort(perm)
    for key in rng.integers(0, 1 << 64, size=20, dtype=np.uint64).tolist():
        pick, row = AR.affinity_row(key, range(n), pod_keys, 8)
        pick2, row2 = AR.affinity_row(key, range(n), pod_keys[perm], 8)   # pod p of the new order is perm[p]
        assert perm[pick2] == pick
        assert [perm[p] if p >= 0 else -1 for p in row2] == row
        assert inv[pick] == pick2


def test_consistency_when_the_set_shrinks():
    """S' subset of S with pick(S) in S' gives pick(S') = pick(S); removing one pod moves only its keys."""
    P = 64
    pod_keys = rng.integers(0, 1 << 64, size=P, dtype=np.uint64)
    keys = rng.integers(0, 1 << 64, size=2000, dtype=np.uint64).tolist()
    full = [AR.affinity_row(k, range(P), pod_keys, 0)[0] for k in keys]
    for _ in range(10):
        sub = sorted(rng.choice(P, size=int(rng.integers(1, P)), replace=False).tolist())
        for k, p in zip(keys, full):
            if p in sub:
                assert AR.affinity_row(k, sub, pod_keys, 0)[0] == p
    gone = 17
    rest = [p for p in range(P) if p != gone]
    moved = [AR.affinity_row(k, rest, pod_keys, 0)[0] != p for k, p in zip(keys, full)]
    assert moved == [p == gone for p in full]


@pytest.mark.parametrize("n", [2, 4, 7, 33])
def test_pick_is_uniform_over_keys(n):
    pod_keys = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    R = 500 * n
    keys = rng.integers(0, 1 << 64, size=R, dtype=np.uint64)
    offsets = np.arange(R + 1, dtype=np.int64) * n
    pick, _ = AR.affinity_rows(keys, np.ones(R, bool), offsets, np.tile(np.arange(n), R), pod_keys, 0)
    counts = np.bincount(pick, minlength=n)
    assert stats.chisquare(counts).pvalue > 1e-3, counts


def test_rows_are_prefixes_and_match_the_plain_ranking():
    P = 200
    pod_keys = rng.integers(0, 1 << 64, size=P, dtype=np.uint64)
    R = 300
    keys = rng.integers(0, 1 << 64, size=R, dtype=np.uint64)
    lists = [np.sort(rng.choice(P, size=int(rng.integers(0, 40)), replace=False)) for _ in range(R)]
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    pods = np.concatenate(lists).astype(np.int64)
    ok = rng.random(R) < 0.9
    full_pick, full = AR.affinity_rows(keys, ok, offsets, pods, pod_keys, N.LIG_MAX_FALLBACKS)
    for k in range(0, N.LIG_MAX_FALLBACKS):
        pick, rows = AR.affinity_rows(keys, ok, offsets, pods, pod_keys, k)
        assert np.array_equal(pick, full_pick) and np.array_equal(rows, full[:, :k])
    for i in range(R):
        if not ok[i] or len(lists[i]) == 0:
            assert full_pick[i] == -1 and (full[i] == -1).all()
            continue
        r = AR.ranking(int(keys[i]), lists[i].tolist(), pod_keys)
        m = min(len(r), 1 + N.LIG_MAX_FALLBACKS)
        assert [full_pick[i]] + full[i, :m - 1].tolist() == r[:m]
        assert (full[i, m - 1:] == -1).all()


def test_model_draw_is_the_oracle_draw_on_the_key():
    """The target of a model-id affinity request is the reference draw (oracle) on state k ^ LIG_DRAW_DOMAIN."""
    A = 64
    snap = WL.make_snapshot(32, A, seed=3)
    models = WL.make_models(A)
    pm = pack_models(models, snap.packed)
    ids = WL.make_model_requests(3000, A, seed=4)
    keys = rng.integers(0, 1 << 64, size=len(ids), dtype=np.uint64)
    reqs, ok, target = AR.affinity_resolve(pm, ids, keys)
    py_models = [PY.InferenceModel(m.Spec.ModelName, bool(pm.critical[i]),
                                   [PY.TargetModel(t.Name, int(t.Weight)) for t in m.Spec.TargetModels])
                 for i, m in enumerate(models)]
    multi = 0
    for i, (m, k) in enumerate(zip(ids.tolist(), keys.tolist())):
        if not ok[i]:
            continue
        st, name, crit, idx = PY.resolve(py_models, m, 0, k)   # state 0 ^ k ^ DRAW_DOMAIN
        assert st == PY.LIGO_OK and idx == target[i] and crit == bool(reqs["flags"][i])
        multi += len(models[m].Spec.TargetModels) >= 2
    assert ok.sum() > 1000 and multi > 100
    # the key alone picks the target: the same key gives the same target wherever the request sits
    _, _, t2 = AR.affinity_resolve(pm, ids[::-1], keys[::-1])
    assert np.array_equal(t2[::-1], target)


# FNV-1a 64 over Name, a zero byte, then Address: fixed vectors for the Python and C++ key functions
POD_KEY_VECTORS = [
    (("", ""), 0xAF63BD4C8601B7DF),
    (("pod1", ""), 0x49D762352D374465),
    (("pod-0", "address-0"), 0x504BFE0EB6DF4E24),
    (("vllm-0", "10.0.0.1:8000"), 0xF8608833A4D0D0CF),
]


def fnv1a(data: bytes) -> int:
    h = 0xCBF29CE484222325
    for b in data:
        h = ((h ^ b) * 0x100000001B3) % (1 << 64)
    return h


def test_pod_key_vectors():
    assert fnv1a(b"") == 0xCBF29CE484222325 and fnv1a(b"a") == 0xAF63DC4C8601EC8C   # FNV-1a 64 known answers
    for (name, addr), want in POD_KEY_VECTORS:
        got = pod_key(Pod(name, addr))
        assert got == AR.pod_key(name, addr) == fnv1a(name.encode() + b"\0" + addr.encode())
        assert got == want
    assert pod_key(Pod("ab", "c")) != pod_key(Pod("a", "bc"))          # the zero byte separates the fields


def test_pod_key_matches_the_cpp_runtime():
    from llm_instance_gateway_b200 import host as H
    lib = H.load()
    for (name, addr), want in POD_KEY_VECTORS:
        assert lib.ligh_pod_key(name.encode(), addr.encode()) == want
    assert lib.ligh_pod_key(b"ab", b"c") == pod_key(Pod("ab", "c")) != lib.ligh_pod_key(b"a", b"bc")


def test_abi_refusals_without_a_gpu():
    lib = N.load()
    reqs = np.zeros(4, dtype=REQ_DTYPE)
    ids = np.zeros(4, dtype=np.uint32)
    keys = np.zeros(4, dtype=np.uint64)
    out, mout = np.zeros(4, dtype=PICK_DTYPE), np.zeros(4, dtype=MPICK_DTYPE)
    rows = np.zeros((4, 8), dtype=np.int16)
    p = lambda a: a.ctypes.data
    for nf in (0, 1, 8, 9, -1):
        assert lib.lig_schedule_batch_affinity(None, 1, p(reqs), 4, p(out), nf, p(rows)) == N.LIG_ERR_INVALID
        assert lib.lig_schedule_batch_affinity_device(None, 1, p(reqs), 4, p(out), nf, p(rows), None) == \
            N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_affinity(None, 1, p(ids), p(keys), 4, p(mout), nf, p(rows)) == \
            N.LIG_ERR_INVALID
        assert lib.lig_schedule_models_batch_affinity_device(None, 1, p(ids), p(keys), 4, p(mout), nf, p(rows),
                                                             None) == N.LIG_ERR_INVALID
    assert b"affinity" in lib.lig_last_error()
    assert lib.lig_upload_pod_keys(None, 1, 4, p(keys)) == N.LIG_ERR_INVALID
    assert np.all(rows == 0) and np.all(out["pod_idx"] == 0) and np.all(mout["pod_idx"] == 0)


def test_symbols_are_declared():
    lib = N.load()
    header = open(os.path.join(ROOT, "include", "lig.h")).read()
    for name in ("lig_upload_pod_keys", "lig_schedule_batch_affinity", "lig_schedule_batch_affinity_device",
                 "lig_schedule_models_batch_affinity", "lig_schedule_models_batch_affinity_device"):
        assert name in N.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert re.search(r"\bint " + name + r"\(", header)
    assert lib.lig_abi_version() == 7
