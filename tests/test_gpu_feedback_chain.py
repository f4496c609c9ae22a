"""The load-feedback chain on the device (include/lig.h, lig_schedule_batch_feedback_chain[_device]):
load feedback carried across calls against one epoch until the next snapshot.

Every check compares picks byte for byte and the per-pod loads exactly:
* the chain over any split of a request sequence into calls, with one seed, equals ONE in-batch
  feedback call over the concatenation (sub_batch = window) and the chain oracle
  (feedback_chain_ref); with a seed per call it equals the oracle;
* host buffers (page-locked and pageable), device buffers, both mixed, two streams;
* restarts: another epoch (also a delta-made one), back to an older epoch, another window,
  lig_feedback_chain_reset, an in-batch feedback call;
* resident epochs stay untouched; caller trees and thresholds of the chain's start; saturation;
  warp-aggregated counting at 2^20 single-survivor requests; refused calls change nothing;
* the C++ runtime's and the Python scheduler's load_feedback_window option.
"""
import ctypes as C

import numpy as np
import pytest

import feedback_chain_ref as FC
from helpers import golden_to_podmetrics
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE
from test_gpu_snapshot_mutation import (INT32_MAX, INT32_MIN, PodState, drop_and_no_pods_trees, edge_pool_state,
                                        feedback_engine, mixed_requests, random_state, run_feedback, uniform_state)

pytestmark = pytest.mark.gpu


def oracle(state, calls, W, thr=(0.8, 5, 50)):
    p = state.packed()
    return FC.schedule_batch_feedback_chain(p.P, p.A, p.kv, state.q, p.n_active, p.max_active, p.bitmap, calls, W, thr)


def host_chain(e, ep, calls, W, P):
    """Pageable host buffers; loads after every call."""
    outs, loads = [], None
    for reqs, seed in calls:
        loads = np.full(max(P, 1), -7, dtype=np.int32)
        outs.append(e.schedule_batch_feedback_chain(ep, seed, np.ascontiguousarray(reqs), W, loads))
    return outs, loads[:P].astype(np.int64)


class Pinned:
    """A page-locked, device-mapped buffer from lig_host_alloc viewed as a numpy array."""

    def __init__(self, lib, n, dtype):
        self.lib, dtype = lib, np.dtype(dtype)
        nbytes = max(n, 1) * dtype.itemsize
        self.ptr = lib.lig_host_alloc(nbytes)
        assert self.ptr
        self.a = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr)).view(dtype)[:n]

    def free(self):
        self.lib.lig_host_free(self.ptr)


def pinned_chain(e, ep, calls, W, P):
    lib = N.load()
    outs = []
    loads = Pinned(lib, max(P, 1), np.int32)
    try:
        for reqs, seed in calls:
            bi, bo = Pinned(lib, len(reqs), REQ_DTYPE), Pinned(lib, len(reqs), PICK_DTYPE)
            bi.a[:] = reqs
            e.schedule_batch_feedback_chain_ptr(ep, seed, bi.ptr if len(reqs) else 0, len(reqs),
                                                bo.ptr if len(reqs) else 0, W, loads.ptr)
            outs.append(bo.a.copy())
            bi.free()
            bo.free()
        return outs, loads.a[:P].astype(np.int64)
    finally:
        loads.free()


def device_chain(e, ep, calls, W, P, streams=None, sync_between=True):
    """Device buffers; calls round-robin over `streams` (no host synchronisation between them when
    sync_between is False)."""
    import torch
    streams = streams or [torch.cuda.Stream()]
    ins = [torch.from_numpy(r.view(np.uint8).reshape(-1).copy()).cuda() if len(r) else None for r, _ in calls]
    outs = [torch.full((max(len(r), 1) * 8,), 0xAB, dtype=torch.uint8, device="cuda") for r, _ in calls]
    d_loads = torch.full((max(P, 1),), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for k, (r, seed) in enumerate(calls):
        st = streams[k % len(streams)]
        with torch.cuda.stream(st):
            e.schedule_batch_feedback_chain_device(ep, seed, ins[k].data_ptr() if len(r) else 0, len(r),
                                                   outs[k].data_ptr(), W, d_loads.data_ptr(), st.cuda_stream)
        if sync_between:
            st.synchronize()
    torch.cuda.synchronize()
    return ([o[: len(r) * 8].cpu().numpy().view(PICK_DTYPE) for o, (r, _) in zip(outs, calls)],
            d_loads[:P].cpu().numpy().astype(np.int64))


def assert_same(got, want, label):
    outs, loads = got
    assert len(outs) == len(want[0]), label
    for k, (g, w) in enumerate(zip(outs, want[0])):
        for f in ("status", "n_survivors", "pod_idx"):
            bad = np.nonzero(g[f] != w[f])[0]
            assert bad.size == 0, (label, k, f, bad[:5], g[bad[:5]], w[bad[:5]])
    assert np.array_equal(loads, want[1]), (label, np.nonzero(loads != want[1])[0][:5])


def pool_cases(name):
    from test_gpu_parity import EDGE_POOLS
    if name == "edge_pools":
        return [(n, edge_pool_state(n)) for n in sorted(EDGE_POOLS)]
    if name in WL.CONFIGS:
        c = WL.CONFIGS[name]
        return [(name, random_state(c["P"], c["A"], seed=c["P"] + 7))]
    if name == "A=0":
        return [(name, random_state(40, 0, seed=41))]
    P = int(name[2:])
    if P == 0:
        return [(name, uniform_state(0, 4))]
    return [(name, random_state(P, 24, seed=P))]


# ---- 1. split invariance -------------------------------------------------------------------------
@pytest.mark.parametrize("pool", ["C2", "C3", "C5", "edge_pools", "P=0", "P=1", "P=33", "P=4097", "P=20000", "A=0"])
def test_split_invariance(pool):
    for label, state in pool_cases(pool):
        P = state.P
        for W in (1, 7, 64, 4096):
            R = {1: 150, 7: 900, 64: 3000, 4096: 13000}[W]
            if P >= 4096:
                R = min(R, 600) if W < 64 else R
            reqs = mixed_requests(state.A, R, seed=P + W)
            R = len(reqs)
            rng = np.random.default_rng(P * 7 + W)
            bounds = FC.random_split(R, rng, W)
            calls = FC.split_calls(reqs, bounds, 31)
            want = oracle(state, calls, W)
            with feedback_engine(P, state.A, R) as e:
                e.upload_snapshot(1, state.packed())
                whole = run_feedback(e, 1, 31, reqs, P, W)
                assert np.array_equal(whole[0], np.concatenate(want[0])), (label, W)
                assert np.array_equal(whole[1], want[1]), (label, W)
                assert_same(host_chain(e, 1, calls, W, P), want, (label, W, "host"))
                e.feedback_chain_reset()
                assert_same(device_chain(e, 1, calls, W, P), want, (label, W, "device"))
            assert want[1].sum() == (np.concatenate(want[0])["pod_idx"] >= 0).sum()


def test_per_call_seeds():
    state = random_state(256, 64, seed=5)
    reqs = WL.make_requests(6000, 64, seed=6)
    rng = np.random.default_rng(7)
    bounds = FC.random_split(len(reqs), rng, 100)
    calls = [(c, 1000 + 17 * k) for k, (c, _) in enumerate(FC.split_calls(reqs, bounds, 0))]
    want = oracle(state, calls, 100)
    with feedback_engine(256, 64, 6000) as e:
        e.upload_snapshot(1, state.packed())
        assert_same(host_chain(e, 1, calls, 100, 256), want, "per-call seeds")


# ---- 3. buffer forms -----------------------------------------------------------------------------
def test_buffer_forms_and_streams():
    import torch
    c = WL.CONFIGS["C3"]
    state = random_state(c["P"], c["A"], seed=11)
    P, W = state.P, 333
    reqs = WL.make_requests(20000, c["A"], seed=12)
    calls = FC.split_calls(reqs, FC.random_split(len(reqs), np.random.default_rng(13), W), 77)
    want = oracle(state, calls, W)
    with feedback_engine(P, c["A"], 20000) as e:
        e.upload_snapshot(1, state.packed())
        assert_same(pinned_chain(e, 1, calls, W, P), want, "pinned")
        e.feedback_chain_reset()
        assert_same(host_chain(e, 1, calls, W, P), want, "pageable")
        e.feedback_chain_reset()
        assert_same(device_chain(e, 1, calls, W, P), want, "device")
        e.feedback_chain_reset()
        assert_same(device_chain(e, 1, calls, W, P, [torch.cuda.Stream(), torch.cuda.Stream()], sync_between=False),
                    want, "two streams")
        # both forms in one chain: halves alternate between pinned, pageable and device calls
        e.feedback_chain_reset()
        outs = []
        for k, call in enumerate(calls):
            form = (pinned_chain, host_chain, device_chain)[k % 3]
            o, loads = form(e, 1, [call], W, P)
            outs += o
        assert_same((outs, loads), want, "mixed forms")
        # R = 0 with loads reads them without scheduling
        L = np.zeros(P, dtype=np.int32)
        e.schedule_batch_feedback_chain(1, 5, np.zeros(0, dtype=REQ_DTYPE), W, L)
        assert np.array_equal(L, want[1])


# ---- 4. restarts ---------------------------------------------------------------------------------
def test_restarts():
    from test_gpu_snapshot_mutation import delta_between, mutate
    P, A, W = 300, 40, 50
    s1, s2 = random_state(P, A, seed=21), random_state(P, A, seed=22)
    reqs = [WL.make_requests(700, A, seed=23 + k) for k in range(12)]
    call = lambda k: [(reqs[k], 9)]                                          # noqa: E731
    with feedback_engine(P, A, 1000) as e:
        e.upload_snapshot(1, s1.packed())
        e.upload_snapshot(2, s2.packed())
        first = host_chain(e, 1, call(0), W, P)
        assert_same(first, oracle(s1, call(0), W), "E1")
        w01 = oracle(s1, call(0) + call(1), W)
        assert_same(host_chain(e, 1, call(1), W, P), (w01[0][1:], w01[1]), "E1 continued")
        assert_same(host_chain(e, 2, call(2), W, P), oracle(s2, call(2), W), "epoch switch")
        assert_same(host_chain(e, 1, call(3), W, P), oracle(s1, call(3), W), "back to E1: its scrape, zero loads")
        # a delta-made epoch
        s3, delta = mutate(s2, np.arange(0, P, 9), np.random.default_rng(24), edge=False)
        e.update_snapshot(3, 2, **delta)
        assert_same(host_chain(e, 3, call(4), W, P), oracle(s3, call(4), W), "delta epoch")
        # another window size
        assert_same(host_chain(e, 3, call(5), 17, P), oracle(s3, call(5), 17), "window change")
        # reset
        host_chain(e, 3, call(6), 17, P)
        e.feedback_chain_reset()
        assert_same(host_chain(e, 3, call(7), 17, P), oracle(s3, call(7), 17), "reset")
        # an interleaved in-batch feedback call
        host_chain(e, 3, call(8), 17, P)
        run_feedback(e, 3, 9, reqs[9], P, 17)
        assert_same(host_chain(e, 3, call(10), 17, P), oracle(s3, call(10), 17), "in-batch call")
        # the same epoch number uploaded again is a new scrape
        host_chain(e, 3, call(11), 17, P)
        e.upload_snapshot(3, s1.packed())
        assert_same(host_chain(e, 3, call(0), 17, P), oracle(s1, call(0), 17), "epoch re-uploaded")


# ---- 5. resident epochs untouched ----------------------------------------------------------------
def test_resident_epochs_untouched():
    P, A = 64, 8
    state = random_state(P, A, seed=31)
    state.q[:] = 0
    reqs = WL.make_requests(20000, A, seed=32)
    reqs["adapter_id"] = 0                       # one class: a herd without feedback
    with feedback_engine(P, A, 20000) as e:
        e.upload_snapshot(1, state.packed())
        classes = lambda: [e.read_class(1, cr, a, P) for cr in (0, 1) for a in range(A + 1)]   # noqa: E731
        before_cls, before = classes(), e.schedule_batch(1, 3, reqs)
        outs, loads = host_chain(e, 1, FC.split_calls(reqs, list(range(0, 20001, 2500)), 3), 8, P)
        assert loads.max() < np.bincount(before["pod_idx"][before["pod_idx"] >= 0], minlength=P).max()
        after_cls = classes()
        assert all(b[0] == a[0] and b[1] == a[1] and np.array_equal(b[2], a[2]) for b, a in zip(before_cls, after_cls))
        assert np.array_equal(e.schedule_batch(1, 3, reqs), before)


# ---- 6. tree and thresholds ----------------------------------------------------------------------
def test_caller_tree_and_mid_chain_changes():
    P, A, W = 96, 12, 40
    state = random_state(P, A, seed=41)
    records, names = state.records(), state.names()
    reqs = mixed_requests(A, 3000, seed=42)
    calls = FC.split_calls(reqs, FC.random_split(len(reqs), np.random.default_rng(43), W), 5)
    half = len(calls) // 2
    t1, t2 = drop_and_no_pods_trees()
    want = FC.schedule_batch_feedback_chain_tree(t1, records, names, calls, W)
    want2 = FC.schedule_batch_feedback_chain_tree(t2, records, names, calls, W)
    assert (np.concatenate(want[0])["status"] == N.LIG_DROP).any()
    assert (np.concatenate(want2[0])["status"] == N.LIG_NO_PODS_LEFT).any()
    with feedback_engine(P, A, len(reqs)) as e:
        e.set_filter_tree(t1)
        e.upload_snapshot(1, state.packed())
        a = host_chain(e, 1, calls[:half], W, P)
        e.set_filter_tree(t2)                        # mid-chain: not before the next chain start
        b = host_chain(e, 1, calls[half:], W, P)
        assert_same((a[0] + b[0], b[1]), want, "tree set mid-chain")
        e.feedback_chain_reset()
        assert_same(host_chain(e, 1, calls, W, P), want2, "new tree after the restart")
        # thresholds: the built-in tree, set mid-chain
        e.set_filter_tree(None)
        e.upload_snapshot(2, state.packed())
        a = host_chain(e, 2, calls[:half], W, P)
        e.set_thresholds(0.5, 2, 10)
        b = host_chain(e, 2, calls[half:], W, P)
        assert_same((a[0] + b[0], b[1]), oracle(state, calls, W), "thresholds set mid-chain")
        e.feedback_chain_reset()
        assert_same(host_chain(e, 2, calls, W, P), oracle(state, calls, W, (0.5, 2, 10)), "new thresholds")


@pytest.mark.parametrize("thresholds", [None, (0.5, 2, 10)])
def test_herding_crosses_the_queue_thresholds(thresholds):
    thr = thresholds or (0.8, 5, 50)
    P, A, W = 48, 8, 50
    rng = np.random.default_rng(90)
    state = random_state(P, A, seed=91)
    state.q[:] = rng.integers(0, thr[1] + 1, P)
    state.kv[:] = np.round(rng.random(P) * 0.6, 2)
    reqs = WL.make_requests(4000, A, seed=92)
    reqs["adapter_id"] = rng.choice([0, 1, A], len(reqs))
    calls = FC.split_calls(reqs, list(range(0, 4001, 8)), 93)       # micro-batches of 8
    want = oracle(state, calls, W, thr)
    q_end = np.minimum(state.q + want[1], INT32_MAX)
    assert ((state.q <= thr[1]) & (q_end > thr[1])).any() and ((state.q < thr[2]) & (q_end >= thr[2])).any()
    with feedback_engine(P, A, 4000) as e:
        if thresholds:
            e.set_thresholds(*thresholds)
        e.upload_snapshot(1, state.packed())
        assert_same(host_chain(e, 1, calls, W, P), want, thr)


# ---- 7. saturation and negatives -----------------------------------------------------------------
@pytest.mark.parametrize("case", ["all_near_max", "negative"])
def test_saturation_and_negative_queues(case):
    P, A, W = 33, 4, 200
    state = random_state(P, A, seed=60)
    if case == "all_near_max":
        state.q[:] = INT32_MAX - np.arange(P) % 7
    else:
        state.q[:] = -(np.arange(P) * 1000)
        state.q[[0, 5, P - 1]] = INT32_MIN
    reqs = WL.make_requests(3000, A, seed=61)
    calls = FC.split_calls(reqs, FC.random_split(3000, np.random.default_rng(62), W), 62)
    want = oracle(state, calls, W)
    if case == "all_near_max":
        assert (state.q + want[1] > INT32_MAX).any()
    with feedback_engine(P, A, 3000) as e:
        e.upload_snapshot(1, state.packed())
        assert_same(host_chain(e, 1, calls, W, P), want, case)


# ---- 8. warp-aggregated counting -----------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 64])
def test_single_survivor_counts_are_exact(P):
    """2^20 critical requests whose class has exactly one survivor, in one open window: every warp
    counts runs of equal pods with one atomic per pod."""
    R = 1 << 20
    A = max(P, 1)
    state = PodState(A, np.full(P, 0.1), np.zeros(P), np.full(P, 4), [[p] for p in range(P)])
    rng = np.random.default_rng(P)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["adapter_id"] = np.sort(rng.integers(0, A, R)) if P > 1 else 0     # long runs of one pod per warp
    reqs["flags"] = N.LIG_REQ_CRITICAL
    reqs["rand_key"] = rng.integers(0, 1 << 63, R, dtype=np.uint64)
    with feedback_engine(P, A, R) as e:
        e.upload_snapshot(1, state.packed())
        loads = np.zeros(P, dtype=np.int32)
        out = e.schedule_batch_feedback_chain(1, 3, reqs, 1 << 30, loads)
        assert (out["status"] == N.LIG_OK).all() and (out["n_survivors"] == 1).all()
        assert np.array_equal(out["pod_idx"], reqs["adapter_id"])
        assert np.array_equal(loads, np.bincount(reqs["adapter_id"], minlength=P))
        assert np.array_equal(out, e.schedule_batch(1, 3, reqs))


# ---- 9. refusals change nothing ------------------------------------------------------------------
def test_refused_calls_leave_the_chain_untouched():
    P, A, W = 128, 16, 30
    state = random_state(P, A, seed=71)
    reqs = WL.make_requests(2000, A, seed=72)
    calls = FC.split_calls(reqs, FC.random_split(2000, np.random.default_rng(73), W), 74)
    want = oracle(state, calls, W)
    lib = N.load()
    with feedback_engine(P, A, 700) as e:
        e.upload_snapshot(1, state.packed())
        ctx = e._ctx
        junk = WL.make_requests(800, A, seed=75)
        out = np.zeros(800, dtype=PICK_DTYPE)
        refusals = [
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 1, 74, junk.ctypes.data, 10, out.ctypes.data, 0, None),
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 1, 74, junk.ctypes.data, -1, out.ctypes.data, W, None),
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 1, 74, None, 10, out.ctypes.data, W, None),
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 1, 74, junk.ctypes.data, 10, None, W, None),
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 1, 74, junk.ctypes.data, 800, out.ctypes.data, W, None),
            lambda: lib.lig_schedule_batch_feedback_chain(ctx, 9, 74, junk.ctypes.data, 10, out.ctypes.data, W, None),
            lambda: lib.lig_schedule_batch_feedback_chain_device(ctx, 1, 74, None, 10, None, W, None, None),
            lambda: lib.lig_schedule_batch_feedback_chain_device(ctx, 1, 74, None, 0, None, -3, None, None),
        ]
        codes = [N.LIG_ERR_INVALID] * 5 + [N.LIG_ERR_STALE_EPOCH] + [N.LIG_ERR_INVALID] * 2
        outs, loads = [], None
        for k, (r, seed) in enumerate(calls):
            o, loads = host_chain(e, 1, [(r, seed)], W, P)
            outs += o
            f = refusals[k % len(refusals)]
            assert f() == codes[k % len(refusals)], k
        assert_same((outs, loads), want, "refusals interleaved")
    # a doorbell stream open before the scratch exists
    with feedback_engine(P, A, 2000) as e:
        e.upload_snapshot(1, state.packed())
        e.stream_open()
        try:
            with pytest.raises(N.LigError) as ei:
                e.schedule_batch_feedback_chain(1, 74, calls[0][0], W)
            assert ei.value.code == N.LIG_ERR_INVALID and "doorbell" in str(ei.value)
        finally:
            e.stream_close()
        assert_same(host_chain(e, 1, calls, W, P), want, "after the doorbell refusal")
    # a ctx with a (single-rank) communicator
    with feedback_engine(P, A, 2000) as e:
        try:
            e.comm_init_rank(1, 0, e.comm_unique_id())
        except N.LigError as err:
            pytest.skip(f"no NCCL: {err}")
        e.upload_snapshot(1, state.packed())
        with pytest.raises(N.LigError) as ei:
            e.schedule_batch_feedback_chain(1, 74, calls[0][0], W)
        assert ei.value.code == N.LIG_ERR_INVALID and "communicator" in str(ei.value)


# ---- 10-12. the schedulers' load_feedback_window -------------------------------------------------
def runtime_pool(P=64, A=12, seed=81):
    state = random_state(P, A, seed=seed)
    state.q[:] = np.random.default_rng(seed).integers(0, 4, P)
    return state, state.records()


def splitmix_keys(seed, n):
    M = (1 << 64) - 1
    s, out = seed ^ 0xD1B54A32D192ED03, []
    for _ in range(n):
        s = (s + 0x9E3779B97F4A7C15) & M
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        out.append(z ^ (z >> 31))
    return out


def test_cpp_runtime_exact_sequence():
    from llm_instance_gateway_b200.host import HostProvider, HostScheduler
    state, records = runtime_pool()
    names = state.names()
    rng = np.random.default_rng(82)
    n, seed, W = 400, 12345, 8
    models = [names[i] for i in rng.integers(0, len(names), n)]
    crit = rng.integers(0, 2, n).astype(bool)
    prov = HostProvider([golden_to_podmetrics(r) for r in records])
    s = HostScheduler(prov, max_pods=64, max_adapters=16, seed=seed, batch_window_us=20, load_feedback_window=W)
    try:
        got = []
        for m, c in zip(models, crit):
            code, pod, _ = s.Schedule(m, m, bool(c))
            got.append(int(pod.Name.split("-")[1]) if code == 0 else -1)
        st = s.stats()
    finally:
        s.close()
        prov.close()
    reqs = np.zeros(n, dtype=REQ_DTYPE)
    reqs["adapter_id"] = [names.index(m) for m in models]
    reqs["flags"] = crit * N.LIG_REQ_CRITICAL
    reqs["rand_key"] = np.array(splitmix_keys(seed, n), dtype=np.uint64)
    want, loads = FC.schedule_batch_feedback_chain_port(records, names[:-1], names[-1], [(reqs, seed)], W)
    assert got == want[0]["pod_idx"].tolist()
    assert st["feedback_windows"] == n // W and st["feedback_restarts"] == 0
    plain, _ = FC.schedule_batch_feedback_chain_port(records, names[:-1], names[-1], [(reqs, seed)], 1 << 30)
    assert got != plain[0]["pod_idx"].tolist()            # the option changes the outcome


def test_cpp_runtime_concurrent_and_refusals():
    from llm_instance_gateway_b200.host import HostProvider, HostSchedulerError, HostScheduler
    state, records = runtime_pool(P=128, A=8, seed=83)
    names = state.names()
    prov = HostProvider([golden_to_podmetrics(r) for r in records])
    try:
        s = HostScheduler(prov, max_pods=128, max_adapters=16, seed=7, load_feedback_window=16)
        try:
            models = names[:3]
            codes, pods = s.schedule_concurrent(16, 250, models, [True] * 3)
            assert (codes == 0).all() and (pods >= 0).all()
            per_pod = np.bincount(pods, minlength=128)
            assert per_pod.sum() == 4000
            s.Refresh()
            codes, pods = s.schedule_concurrent(16, 250, models, [True] * 3)
            assert (codes == 0).all() and (pods >= 0).all()
            st = s.stats()
            assert st["feedback_restarts"] == 1 and st["scheduled"] == 8000
            assert st["feedback_windows"] <= 8000 // 16
        finally:
            s.close()
        for kw in (dict(devices=[0, 1]), dict(use_doorbell=True)):
            with pytest.raises(HostSchedulerError, match="load_feedback_window"):
                HostScheduler(prov, max_pods=128, max_adapters=16, load_feedback_window=4, **kw)
    finally:
        prov.close()


def test_python_scheduler_load_feedback_window():
    import random

    from llm_instance_gateway_b200 import scheduling as S
    from llm_instance_gateway_b200.packer import pack_pod_metrics
    state, records = runtime_pool(P=96, A=10, seed=91)
    pms = [golden_to_podmetrics(r) for r in records]

    class Provider:
        def AllPodMetrics(self):
            return pms

        def Version(self):
            return 1

    names = state.names()
    rng = np.random.default_rng(92)
    batches = [[S.LLMRequest(Model=m, ResolvedTargetModel=m, Critical=bool(c))
                for m, c in zip([names[i] for i in rng.integers(0, len(names), k)], rng.integers(0, 2, k))]
               for k in (1, 7, 0, 30, 13, 64, 5, 100)]
    W = 9
    sched = S.NewScheduler(Provider(), load_feedback_window=W, seed=2024, max_pods=96, max_adapters=16)
    try:
        got = [sched.ScheduleBatch(b) for b in batches]
    finally:
        sched.close()
    snap = pack_pod_metrics(pms)
    r = random.Random(2024)
    seed = r.getrandbits(64)
    calls = []
    for b in batches:
        reqs = np.zeros(len(b), dtype=REQ_DTYPE)
        for i, q in enumerate(b):
            reqs[i] = (snap.adapter_id(q.ResolvedTargetModel), N.LIG_REQ_CRITICAL if q.Critical else 0, r.getrandbits(64))
        calls.append((reqs, seed))
    want, _ = FC.schedule_batch_feedback_chain(snap.P, snap.A, snap.kv, snap.q.astype(np.int64), snap.n_active,
                                               snap.max_active, snap.bitmap, calls, W)
    for g, w in zip(got, want):
        assert [snap.pods.index(p) if p is not None else -1 for p, _ in g] == w["pod_idx"].tolist()
