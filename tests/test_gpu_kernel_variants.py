"""Every pick-kernel instantiation the LIG_* knobs select, and the edges where the host splits a
queue into several launches, against references computed on the host.

The pick kernels are templates and `lig_create` picks one instantiation per ctx from the knobs, so
each shape a knob can select is part of the library:

  * lig_pick_persistent_kernel<groups, stages, bulk, tab>: 9 (groups, stages) pairs x bulk x tab;
  * lig_pick_loop_kernel<tab> (LIG_PICK_KERNEL=loop);
  * lig_pick_stream_kernel<ppt> / lig_pick_queue_kernel<ppt>, ppt = LIG_PICK_PER_THREAD;
  * lig_pick_models_kernel<groups, stages, tab>: 2 x 3 x tab;
  * host buffers through the TMA ring (LIG_HOST_TMA=1).

No check here compares one device path with another.  Descriptor picks come from the class-table
CPU arm (`oracle.ClassTable`) with the per-batch seed folded into the keys (the pick state is
`seed ^ rand_key`, so batch b with seed s_b is seed 0 with keys `s_b ^ rand_key`; the CPU test
test_seed_folding_cpu.py pins that), or, on the large-n snapshot, from the construction of
test_gpu_large_lists.py.  Model picks come from `oracle.Models`.  Every comparison also asserts that
its inputs produced what they were built to produce (non-OK statuses, rejected first draws, draws
past target 0, LIG_NO_MODEL), so no variant can pass on trivial output.
"""
import ctypes as C

import numpy as np
import pytest

import draw_keys as DK
from helpers import M64, fold, np_int31n
from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import CRITICAL, InferenceModel, InferenceModelSpec, TargetModel
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models, pack_pod_metrics
from test_gpu_large_lists import BUDGET, EDGE_MODELS, P_MAX, Requests, idle_snapshot, mtab_bytes
from test_gpu_parity import EDGE_POOLS

pytestmark = pytest.mark.gpu

C3 = WL.CONFIGS["C3"]
EDGE_POOL = "all_nan_kv"            # sheddable classes DROP, critical ones EMPTY
LARGE_NS = [2, 3, 4097, 12289, 21846, 32767, 30011, 5]
SENTINEL = 0xAB                     # fill byte of every output buffer: an unwritten pick shows


def make_engine(env, monkeypatch, **kw):
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)               # the knobs are read at lig_create
        return Engine(0, **kw)


# ---- descriptor pools and their references --------------------------------------------------------
class OraclePool:
    """A pool whose picks come from the class-table CPU arm; requests are random, with adapter ids
    outside [0, A) (-1, A, 2^31-1, -2^31) mixed in."""

    def __init__(self, name, packed, oracle):
        self.name, self.packed = name, packed
        p = packed
        self.table = oracle.ClassTable(p.P, p.A, p.kv, p.q, p.n_active, p.max_active, p.bitmap)
        self.threads = oracle.hardware_threads()
        self.smem = True

    def requests(self, nb, R, seeds):
        A = self.packed.A
        rng = np.random.default_rng([nb, R, 7])
        r = WL.make_requests(nb * R, A, seed=int(rng.integers(1 << 40)))
        odd = rng.random(nb * R) < 0.05
        r["adapter_id"][odd] = rng.choice(np.array([-1, A, 2**31 - 1, -(2**31)], dtype=np.int32), int(odd.sum()))
        if A == 0:
            r["adapter_id"] = rng.choice(np.array([-1, 0, 1, 2**31 - 1], dtype=np.int32), nb * R)
        return r.reshape(nb, R)

    def want(self, reqs, seeds):
        folded = fold(reqs, np.array(seeds, dtype=np.uint64)[:, None])
        return self.table.schedule_batch(folded.reshape(-1), 0, self.threads).reshape(reqs.shape)

    def assert_nontrivial(self, want, label):
        if self.packed.A == 0:           # the edge pool: DROP and EMPTY, never a pick
            assert (want["status"] == N.LIG_DROP).any() and (want["status"] == N.LIG_EMPTY).any(), label
        else:
            assert (want["status"] == N.LIG_OK).any() and (want["n_survivors"] > 1).any(), label


class LargePool:
    """The idle snapshot of test_gpu_large_lists: adapter a is held by exactly LARGE_NS[a] pods, an
    unheld adapter keeps all 32768.  Its compact blob does not fit the shared-memory budget, so the
    kernels take their tab = 0 form.  Requests carry crafted first draws (every Int31n accept /
    reject edge of every class), rejected ones first, so even a one-request batch rejects."""

    def __init__(self):
        rng = np.random.default_rng(2027)
        self.snap = idle_snapshot(LARGE_NS, rng)
        self.packed = self.snap.packed
        A = self.snap.A
        self.name = "large_n"
        self.smem = False
        everyone = np.arange(P_MAX)
        classes = []                     # class index = critical * (A + 1) + adapter, as on the device
        for crit in (0, 1):
            classes += [(a, crit, self.snap.holders[a]) for a in range(A)] + [(A, crit, everyone)]
        self.rq = Requests(classes, rng)
        self.order = np.argsort(~self.rq.rejected, kind="stable")
        self.n_rejected = int(self.rq.rejected.sum())
        self.top = np.array([DK.accept_top(int(len(c[2]))) for c in classes], dtype=np.int64)
        self.n_cls = np.array([len(c[2]) for c in classes], dtype=np.int64)
        self.off = np.concatenate([[0], np.cumsum(self.n_cls)])[:-1]
        self.flat = self.rq.flat

    def requests(self, nb, R, seeds):
        out = np.empty((nb, R), dtype=REQ_DTYPE)
        k = len(self.order)
        for b, s in enumerate(seeds):
            idx = self.order[np.arange(b * R, (b + 1) * R) % k]
            idx[0] = self.order[b % self.n_rejected]                   # a rejected first draw leads
            out[b] = self.rq.reqs(s & M64)[idx]
        return out

    def klass(self, r):
        A = self.snap.A
        return (r["flags"] & 1).astype(np.int64) * (A + 1) + np.minimum(r["adapter_id"].astype(np.int64) % (1 << 32), A)

    def want(self, reqs, seeds):
        want = np.zeros(reqs.shape, dtype=PICK_DTYPE)
        for b, s in enumerate(seeds):
            c = self.klass(reqs[b])
            k = np_int31n(0, reqs[b]["rand_key"] ^ np.uint64(s & M64), self.n_cls[c])
            want[b]["pod_idx"] = self.flat[self.off[c] + k]
            want[b]["n_survivors"] = self.n_cls[c]
        return want

    def rejected(self, reqs, seeds):
        """Requests whose first draw Int31n(n) rejected."""
        rej = np.zeros(reqs.shape, dtype=bool)
        for b, s in enumerate(seeds):
            st = reqs[b]["rand_key"] ^ np.uint64(s & M64)
            rej[b] = DK.first_draws(st, 1)[:, 0] >= self.top[self.klass(reqs[b])]
        return rej

    def assert_nontrivial(self, want, label):
        assert (want["status"] == N.LIG_OK).all() and (want["n_survivors"] > 4096).any(), label


@pytest.fixture(scope="module")
def pools(oracle):
    c3 = WL.make_snapshot(C3["P"], C3["A"], seed=41)
    return [OraclePool("c3", c3.packed, oracle), OraclePool(EDGE_POOL, pack_pod_metrics(EDGE_POOLS[EDGE_POOL]), oracle),
            LargePool()]


class RefCache:
    """(pool, shape, seed) -> (requests, reference picks), computed once for every variant."""

    def __init__(self):
        self._c = {}

    def get(self, pool, nb, R, seed):
        key = (pool.name, nb, R, seed)
        if key not in self._c:
            seeds = [(seed + b) & M64 for b in range(nb)]
            reqs = pool.requests(nb, R, seeds)
            self._c[key] = (reqs, pool.want(reqs, seeds), seeds)
        return self._c[key]


@pytest.fixture(scope="module")
def refs():
    return RefCache()


def device_queue(eng, ep, reqs, seed, out_off=0):
    """lig_schedule_batches_device over one contiguous request buffer and one contiguous pick buffer
    (batch stride rounded up to 16 bytes, then shifted by out_off bytes); returns picks (nb, R) and
    the launch count of the call."""
    import torch
    nb, R = reqs.shape
    stride = (R + 1) // 2 * 2
    d_in = torch.from_numpy(np.ascontiguousarray(reqs).reshape(-1).view(np.uint8)).cuda()
    d_out = torch.full((nb * stride * 8 + 16,), SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = eng.kernel_launches
    eng.schedule_batches_device(ep, seed & M64, [d_in.data_ptr() + b * R * 16 for b in range(nb)], R,
                                [d_out.data_ptr() + out_off + b * stride * 8 for b in range(nb)], 0)
    torch.cuda.synchronize()
    launches = eng.kernel_launches - before
    raw = d_out.cpu().numpy()[out_off: out_off + nb * stride * 8]
    return raw.view(PICK_DTYPE).reshape(nb, stride)[:, :R], launches


def assert_picks(got, want, label):
    bad = np.argwhere(got != want)
    assert bad.size == 0, (label, bad[:5].tolist(), got[tuple(bad[:5].T)], want[tuple(bad[:5].T)])


def assert_launched(e, label, kernel, **args):
    """The ctx's last pick launch was `kernel` with these template arguments (lig_last_pick_launch):
    the call really ran the instantiation the test means."""
    want = dict(kernel=kernel, groups=0, stages=0, bulk_store=0, tables_in_smem=0, per_thread=0)
    want.update(args)
    got = e.last_pick_launch()
    assert got == want, (label, got, want)


# ---- 1 + 2: the persistent descriptor kernels ---------------------------------------------------------
# (n_batches, R): 1, 2, 7 and 97 batches (97 > 96 uses the device item table); R = 1, 3, one tile
# -1 / exact / +1 (ragged last tiles under bulk stores), 4097 and ~150 000 requests
SHAPES = [(1, 1), (2, 3), (97, 3), (7, 1023), (2, 1024), (97, 1025), (7, 4097), (1, 150_001)]
SEED = M64 - 40                     # the seeds of a 97-batch queue wrap past 2^64
PAIRS = [(1, 2), (1, 3), (1, 4), (1, 6), (2, 2), (2, 4), (2, 6), (3, 3), (3, 6)]
VARIANTS = {f"g{g}s{s}" + ("_bulk" if bulk else ""): {"LIG_TMA_GROUPS": str(g), "LIG_TMA_STAGES": str(s),
                                                      "LIG_TMA_BULK_STORE": str(int(bulk))}
            for g, s in PAIRS for bulk in (False, True)}
VARIANTS["g2s2_ctas1"] = {"LIG_PERSIST_CTAS": "1"}
VARIANTS["loop"] = {"LIG_PICK_KERNEL": "loop"}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_persistent_queue_variants(variant, pools, refs, monkeypatch):
    """Each variant runs a C3 pool and the DROP / EMPTY edge pool with its compact tables in shared
    memory (tab = 1) and the large-n snapshot with the strided tables (tab = 0)."""
    env = VARIANTS[variant]
    groups = int(env.get("LIG_TMA_GROUPS", 2))
    stages = int(env.get("LIG_TMA_STAGES", 2))
    bulk = env.get("LIG_TMA_BULK_STORE") == "1"
    loop = env.get("LIG_PICK_KERNEL") == "loop"
    e = make_engine(env, monkeypatch, max_pods=P_MAX, max_adapters=C3["A"], max_batch=1 << 12)
    statuses = set()
    try:
        for i, pool in enumerate(pools):
            ep = 1 + i
            e.upload_snapshot(ep, pool.packed)
            info = e.pick_kernel_info(ep)
            if loop:
                assert info["kernel"] == "lig_pick_loop_kernel" and info["threads"] == 512, info
            else:
                assert info["kernel"] == "lig_pick_persistent_kernel", info
                assert info["threads"] == 256 * groups + 32, info
            assert info["tables_in_smem"] == pool.smem, (pool.name, info)
            if pool.smem:
                assert 0 < info["table_bytes"] <= BUDGET, info
            else:
                assert info["table_bytes"] > BUDGET, info
            if "LIG_PERSIST_CTAS" in env:
                assert info["grid"] == e.sm_count, info
            rejected = 0

            def launched(label, bulk_store):
                if loop:
                    assert_launched(e, label, N.LIG_KERNEL_LOOP, tables_in_smem=int(pool.smem))
                else:
                    assert_launched(e, label, N.LIG_KERNEL_PERSISTENT, groups=groups, stages=stages,
                                    bulk_store=int(bulk_store), tables_in_smem=int(pool.smem))
            for nb, R in SHAPES:
                reqs, want, seeds = refs.get(pool, nb, R, SEED)
                got, launches = device_queue(e, ep, reqs, SEED)
                label = (variant, pool.name, nb, R)
                assert launches == 1, label
                launched(label, bulk)
                assert_picks(got, want, label)
                if R > 3:
                    pool.assert_nontrivial(want, label)
                statuses |= set(np.unique(want["status"]).tolist())
                if isinstance(pool, LargePool):
                    rej = pool.rejected(reqs, seeds)
                    assert rej[:, 0].all(), label             # every batch's first request is rejected once
                    rejected += int(rej.sum())
                if bulk and pool.smem and R >= 1024:
                    # 8-byte aligned pick buffers: the queue takes the plain-store form
                    got, _ = device_queue(e, ep, reqs, SEED, out_off=8)
                    launched(label + ("out+8",), False)
                    assert_picks(got, want, label + ("out+8",))
            if isinstance(pool, LargePool):
                assert rejected > 1000, rejected
        assert {N.LIG_OK, N.LIG_DROP, N.LIG_EMPTY} <= statuses, statuses
    finally:
        e.close()


# ---- 3: the plain kernels, every LIG_PICK_PER_THREAD ----------------------------------------------------
def host_buffers(lib, reqs):
    n = len(reqs)
    h_in, h_out = lib.lig_host_alloc(n * 16 + 16), lib.lig_host_alloc(n * 8 + 16)
    assert h_in and h_out
    return h_in, h_out


def host_view(addr, n, dtype):
    return np.ctypeslib.as_array((C.c_uint8 * (n * dtype.itemsize)).from_address(addr)).view(dtype)


def host_call(e, ep, seed, reqs, in_off=0, out_off=0):
    """lig_schedule_batch on lig_host_alloc buffers, the requests at in_off and the picks at out_off."""
    lib = N.load()
    h_in, h_out = host_buffers(lib, reqs)
    try:
        host_view(h_in + in_off, len(reqs), REQ_DTYPE)[:] = reqs
        host_view(h_out + out_off, len(reqs), PICK_DTYPE).view(np.uint8)[:] = SENTINEL
        before = e.kernel_launches
        e.schedule_batch_ptr(ep, seed & M64, h_in + in_off, len(reqs), h_out + out_off)
        assert e.kernel_launches - before == 1
        return host_view(h_out + out_off, len(reqs), PICK_DTYPE).copy()
    finally:
        lib.lig_host_free(h_in)
        lib.lig_host_free(h_out)


@pytest.mark.parametrize("ppt", [1, 2, 4, 8, 16])
def test_plain_kernels_every_per_thread_count(ppt, pools, refs, monkeypatch):
    """R = 256 ppt - 1 (one ragged CTA), 256 ppt (one full CTA: the plain or, from 8 on, the
    software-pipelined form), 256 ppt + 1 (full + ragged) through lig_schedule_batch (page-locked
    and pageable), lig_schedule_batch_device, the merged queue and the per-batch mode on 1 and 8
    streams."""
    import torch
    base = {"LIG_PICK_KERNEL": "merged", "LIG_PICK_PER_THREAD": str(ppt)}
    kw = dict(max_pods=P_MAX, max_adapters=C3["A"], max_batch=1 << 13)
    engines = {"merged": make_engine(base, monkeypatch, **kw),
               "per_batch_1": make_engine({**base, "LIG_MERGE_MAX": "0", "LIG_QUEUE_STREAMS": "1"}, monkeypatch, **kw),
               "per_batch_8": make_engine({**base, "LIG_MERGE_MAX": "0", "LIG_QUEUE_STREAMS": "8"}, monkeypatch, **kw)}
    nb = 7
    try:
        for i, pool in enumerate(pools[:2]):
            ep = 1 + i
            for e in engines.values():
                e.upload_snapshot(ep, pool.packed)
                assert e.pick_kernel_info(ep)["kernel"] == "lig_pick_queue_kernel"
            for R in (256 * ppt - 1, 256 * ppt, 256 * ppt + 1):
                reqs, want, seeds = refs.get(pool, nb, R, SEED)
                label = (ppt, pool.name, R)
                pool.assert_nontrivial(want, label)
                for name, e in engines.items():
                    got, launches = device_queue(e, ep, reqs, SEED)
                    assert launches == (1 if name == "merged" else nb), (label, name)
                    assert_launched(e, label + (name,), N.LIG_KERNEL_QUEUE if name == "merged" else N.LIG_KERNEL_PLAIN,
                                    per_thread=ppt)
                    assert_picks(got, want, label + (name,))
                e = engines["merged"]
                b = nb - 1                                           # the batch whose seed wrapped
                for in_off, out_off in ((0, 0), (8, 8)):
                    assert_picks(host_call(e, ep, seeds[b], reqs[b], in_off, out_off), want[b], label + ("pinned", in_off))
                    assert_launched(e, label + ("pinned", in_off), N.LIG_KERNEL_PLAIN, per_thread=ppt)
                assert_picks(e.schedule_batch(ep, seeds[b], np.ascontiguousarray(reqs[b])), want[b], label + ("pageable",))
                d_in = torch.from_numpy(np.ascontiguousarray(reqs[b]).view(np.uint8)).cuda()
                d_out = torch.full((R * 8,), SENTINEL, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                e.schedule_batch_device(ep, seeds[b], d_in.data_ptr(), R, d_out.data_ptr(), 0)
                torch.cuda.synchronize()
                assert_picks(d_out.cpu().numpy().view(PICK_DTYPE), want[b], label + ("device",))
                assert_launched(e, label + ("device",), N.LIG_KERNEL_PLAIN, per_thread=ppt)
    finally:
        for e in engines.values():
            e.close()


# ---- 4: the persistent model kernel --------------------------------------------------------------------
class ModelRefs:
    """The C3 pool with WL.make_models plus the edge models of test_gpu_large_lists (255 targets, a
    weight total of 2^31-1, totals with about half of all draws rejected) and one absent model."""

    def __init__(self, oracle):
        A = C3["A"]
        self.snap = WL.make_snapshot(C3["P"], A, seed=41)
        models = WL.make_models(A)
        names = [WL.adapter_name(a) for a in range(A)] + [WL.UNKNOWN_MODEL]
        self.edge0 = len(models)
        for mi, ws in enumerate(EDGE_MODELS):
            tms = [TargetModel(names[(37 * mi + k) % (A + 1)], w) for k, w in enumerate(ws)]
            models.append(InferenceModel(f"edge-{mi}", InferenceModelSpec(
                ModelName=f"edge-{mi}", Criticality=CRITICAL if mi % 2 else None, TargetModels=tms)))
        models.append(InferenceModel("absent", InferenceModelSpec(ModelName="absent", Criticality=None,
                                                                  TargetModels=[TargetModel(names[0], 0)])))
        self.pm = pack_models(models, self.snap.packed)
        assert self.pm.present[-1] == 0
        recs = WL.model_records(models)
        recs[-1] = None
        self.mo = oracle.Models(recs)
        self.pool = oracle.Pool(self.snap.pod_records())
        self.threads = oracle.hardware_threads()
        self._c = {}

    def ids(self, n, rng):
        nm = self.pm.n_models
        ids = WL.make_model_requests(n, C3["A"], seed=int(rng.integers(1 << 40))).astype(np.int64)
        u = rng.random(n)
        edge = u < 0.25
        ids[edge] = self.edge0 + rng.integers(0, len(EDGE_MODELS), int(edge.sum()))
        ids[(u >= 0.25) & (u < 0.27)] = nm - 1                        # absent
        far = (u >= 0.27) & (u < 0.29)
        ids[far] = rng.choice(np.array([nm, nm + 5, 2**32 - 1]), int(far.sum()))
        return ids.astype(np.uint32)

    def get(self, nb, R, seed, first_index):
        key = (nb, R, seed, first_index)
        if key not in self._c:
            rng = np.random.default_rng([nb, R, 11])
            ids = np.stack([self.ids(R, rng) for _ in range(nb)])
            seeds = [(seed + b) & M64 for b in range(nb)]
            want = np.stack([self.mo.schedule_batch(self.pool, np.ascontiguousarray(ids[b]), seeds[b],
                                                    first_index, self.threads) for b in range(nb)])
            self._c[key] = (ids, want)
        return self._c[key]


@pytest.fixture(scope="module")
def mrefs(oracle):
    return ModelRefs(oracle)


def assert_models_nontrivial(want, label):
    tgt = want["target_idx"]
    assert ((tgt > 0) & (tgt < 255)).any(), label                      # draws past target 0
    assert (want["status"] == N.LIG_NO_MODEL).any(), label
    assert (want["status"] == N.LIG_OK).any(), label


def device_models(e, ep, ids, seed, first_index, ids_off=None, out_off=None):
    """lig_schedule_models_batches_device over contiguous buffers (one 16-byte padded region per
    batch); ids_off / out_off = (batch, bytes) shifts one batch's ids or picks off 16-byte alignment."""
    import torch
    nb, R = ids.shape
    region = (R * 4 + 15) // 16 * 16 + 16
    d_in = torch.zeros(nb * region, dtype=torch.uint8, device="cuda")
    d_out = torch.full((nb * region,), SENTINEL, dtype=torch.uint8, device="cuda")
    in_at = [b * region + (ids_off[1] if ids_off and ids_off[0] == b else 0) for b in range(nb)]
    out_at = [b * region + (out_off[1] if out_off and out_off[0] == b else 0) for b in range(nb)]
    host = np.zeros(nb * region, dtype=np.uint8)
    for b in range(nb):
        host[in_at[b]: in_at[b] + R * 4] = ids[b].view(np.uint8)
    d_in.copy_(torch.from_numpy(host))
    torch.cuda.synchronize()
    before = e.kernel_launches
    e.schedule_models_batches_device(ep, seed & M64, first_index, [d_in.data_ptr() + a for a in in_at], R,
                                     [d_out.data_ptr() + a for a in out_at], 0)
    torch.cuda.synchronize()
    launches = e.kernel_launches - before
    raw = d_out.cpu().numpy()
    got = np.stack([raw[a: a + R * 4].view(MPICK_DTYPE) for a in out_at])
    return got, launches


MSHAPES = [(1, 4), (5, 4), (5, 4096), (5, 4100), (1, 100_000)]
MSEED = M64 - 2                     # batch seeds 2^64-2, 2^64-1, 0, 1, 2


@pytest.mark.parametrize("tab", [True, False], ids=["tab", "notab"])
@pytest.mark.parametrize("stages", [2, 4, 8])
@pytest.mark.parametrize("groups", [1, 2])
def test_model_kernel_variants(groups, stages, tab, mrefs, monkeypatch):
    """first_index = 2^64 - R/2 - 3: the keys wrap inside every batch (and inside a tile)."""
    env = {"LIG_MODELS_GROUPS": str(groups), "LIG_MODELS_STAGES": str(stages)}
    if not tab:
        env["LIG_TAB_SMEM"] = "0"
    e = make_engine(env, monkeypatch, max_pods=C3["P"], max_adapters=C3["A"], max_batch=1 << 12)
    try:
        e.upload_snapshot(1, mrefs.snap.packed)
        e.upload_models(1, mrefs.pm)
        info = e.pick_kernel_info(1)
        assert info["tables_in_smem"] == tab, info
        assert info["table_bytes"] + mtab_bytes(mrefs.pm) <= BUDGET, info     # both tables fit: tab is the knob's
        seen = []
        for nb, R in MSHAPES:
            fi = (M64 + 1 - R // 2 - 3) & M64
            ids, want = mrefs.get(nb, R, MSEED, fi)
            got, launches = device_models(e, 1, ids, MSEED, fi)
            label = (groups, stages, tab, nb, R)
            assert launches == 1, label                                        # one persistent launch
            assert_launched(e, label, N.LIG_KERNEL_MODELS, groups=groups, stages=stages, tables_in_smem=int(tab))
            assert_picks(got, want, label)
            seen.append(want.reshape(-1))
        assert_models_nontrivial(np.concatenate(seen), (groups, stages, tab))
    finally:
        e.close()


# ---- 5: long queues ------------------------------------------------------------------------------------
def test_long_model_queues(mrefs):
    """65 batches = two launches of at most 64 inline batches; 1100 batches = 18 launches, which
    wraps the 16-slot tile-claim counter ring inside one call.  Batch b runs with seed + b from a
    seed that wraps inside the queue, and the keys wrap inside each batch."""
    e = Engine(0, max_pods=C3["P"], max_adapters=C3["A"], max_batch=1 << 12)
    try:
        e.upload_snapshot(1, mrefs.snap.packed)
        e.upload_models(1, mrefs.pm)
        for nb, R, launches_want in ((65, 8, 2), (1100, 4, 18)):
            seed, fi = M64 - 600, M64 - 2
            ids, want = mrefs.get(nb, R, seed, fi)
            got, launches = device_models(e, 1, ids, seed, fi)
            assert launches == launches_want, (nb, launches)
            assert_launched(e, nb, N.LIG_KERNEL_MODELS, groups=2, stages=4, tables_in_smem=1)
            assert_picks(got, want, ("long model queue", nb))
            assert_models_nontrivial(want, nb)
    finally:
        e.close()


LONG = [65_536, 4 * 65_535 + 97]    # two launches; five, whose fifth chunk (97 > 96) wraps the item-table ring


@pytest.mark.parametrize("mode", ["persistent", "loop", "merged"])
def test_long_descriptor_queues(mode, pools, refs, monkeypatch):
    env = {"persistent": {}, "loop": {"LIG_PICK_KERNEL": "loop"}, "merged": {"LIG_PICK_KERNEL": "merged"}}[mode]
    e = make_engine(env, monkeypatch, max_pods=C3["P"], max_adapters=C3["A"], max_batch=1 << 12)
    pool = pools[0]
    try:
        e.upload_snapshot(1, pool.packed)
        for nb in LONG:
            for R in (1, 3):
                seed = M64 - nb // 2                                  # the batch seeds wrap mid-queue
                reqs, want, _ = refs.get(pool, nb, R, seed)
                got, launches = device_queue(e, 1, reqs, seed)
                label = (mode, nb, R)
                assert launches == -(-nb // 65_535), label
                if mode == "persistent":
                    assert_launched(e, label, N.LIG_KERNEL_PERSISTENT, groups=2, stages=2, tables_in_smem=1)
                elif mode == "loop":
                    assert_launched(e, label, N.LIG_KERNEL_LOOP, tables_in_smem=1)
                else:
                    assert_launched(e, label, N.LIG_KERNEL_QUEUE, per_thread=4)
                assert_picks(got, want, label)
                pool.assert_nontrivial(want, label)
    finally:
        e.close()


# ---- 6: model queues with one unaligned buffer -----------------------------------------------------------
def test_model_queue_with_one_unaligned_buffer(mrefs):
    """R % 4 == 0 and every buffer 16-byte aligned but one: the whole queue takes the plain kernel
    (one launch per batch) and still equals the reference."""
    e = Engine(0, max_pods=C3["P"], max_adapters=C3["A"], max_batch=1 << 12)
    try:
        e.upload_snapshot(1, mrefs.snap.packed)
        e.upload_models(1, mrefs.pm)
        nb, R = 5, 4096
        fi = (M64 + 1 - R // 2 - 3) & M64
        ids, want = mrefs.get(nb, R, MSEED, fi)
        got, launches = device_models(e, 1, ids, MSEED, fi)
        assert launches == 1
        assert_launched(e, "aligned", N.LIG_KERNEL_MODELS, groups=2, stages=4, tables_in_smem=1)
        assert_picks(got, want, "aligned")
        for which in ("ids", "out"):
            for off in (4, 8, 12):
                shift = (2, off)
                got, launches = device_models(e, 1, ids, MSEED, fi, **{f"{which}_off": shift})
                assert launches == nb, (which, off)
                assert_launched(e, (which, off), N.LIG_KERNEL_MODELS_PLAIN)
                assert_picks(got, want, (which, off))
        assert_models_nontrivial(want, "mixed")
    finally:
        e.close()


# ---- 7: host buffers through the TMA ring --------------------------------------------------------------------
@pytest.mark.parametrize("bulk", [False, True], ids=["plain_store", "bulk_store"])
def test_host_buffers_through_the_tma_ring(bulk, pools, refs, monkeypatch):
    """LIG_HOST_TMA=1: page-locked host buffers (16-byte aligned, and at +8: requests there are
    staged through the aligned bounce buffer, picks there take the plain stores), pageable buffers
    (the bounce path), and 40 tickets in flight on the 8 lanes, so the 16 tile-claim counters are
    reused across streams.  The async form refuses a request array at +8."""
    env = {"LIG_HOST_TMA": "1", "LIG_TMA_BULK_STORE": str(int(bulk))}
    e = make_engine(env, monkeypatch, max_pods=P_MAX, max_adapters=C3["A"], max_batch=1 << 17)
    lib = N.load()
    try:
        for i, pool in enumerate(pools[:2]):
            ep = 1 + i
            e.upload_snapshot(ep, pool.packed)
            for R in (1, 1023, 1025, 4097, 100_003):
                reqs, want, seeds = refs.get(pool, 1, R, SEED)
                label = (bulk, pool.name, R)
                if R > 3:
                    pool.assert_nontrivial(want, label)
                for in_off, out_off in ((0, 0), (0, 8), (8, 0), (8, 8)):
                    assert_picks(host_call(e, ep, SEED, reqs[0], in_off, out_off), want[0], label + (in_off, out_off))
                    # requests at +8 are staged into the aligned bounce buffer, picks included
                    tma_bulk = bulk and (in_off == 8 or out_off == 0)
                    assert_launched(e, label + (in_off, out_off), N.LIG_KERNEL_PERSISTENT, groups=2, stages=2,
                                    bulk_store=int(tma_bulk), tables_in_smem=1)
                assert_picks(e.schedule_batch(ep, SEED, np.ascontiguousarray(reqs[0])), want[0], label + ("pageable",))
                assert_launched(e, label + ("pageable",), N.LIG_KERNEL_PERSISTENT, groups=2, stages=2,
                                bulk_store=int(bulk), tables_in_smem=1)
            # many tickets in flight at once, each with its own seed
            nt, R = 40, 1025
            reqs, want, seeds = refs.get(pool, nt, R, SEED)
            bufs = [host_buffers(lib, reqs[t]) for t in range(nt)]
            try:
                tickets = []
                for t, (h_in, h_out) in enumerate(bufs):
                    host_view(h_in, R, REQ_DTYPE)[:] = reqs[t]
                    host_view(h_out, R, PICK_DTYPE).view(np.uint8)[:] = SENTINEL
                for t, (h_in, h_out) in enumerate(bufs):
                    tickets.append(e.schedule_batch_async(ep, seeds[t], h_in, R, h_out))
                for t in tickets:
                    e.schedule_wait(t)
                for t, (h_in, h_out) in enumerate(bufs):
                    assert_picks(host_view(h_out, R, PICK_DTYPE), want[t], (bulk, pool.name, "async", t))
                with pytest.raises(N.LigError) as ei:
                    e.schedule_batch_async(ep, SEED, bufs[0][0] + 8, R - 1, bufs[0][1])
                assert ei.value.code == N.LIG_ERR_INVALID
            finally:
                for h_in, h_out in bufs:
                    lib.lig_host_free(h_in)
                    lib.lig_host_free(h_out)
    finally:
        e.close()


def filter_reference(pool, reqs, want):
    """offsets and survivor lists of lig_filter_batch: a request's class list when its pick is OK,
    nothing otherwise (from the class-table CPU arm)."""
    A = pool.packed.A
    lists, parts = {}, []
    for r, w in zip(reqs, want):
        if int(w["status"]) != N.LIG_OK:
            parts.append([])
            continue
        key = (int(r["flags"]) & 1, min(int(r["adapter_id"]) % (1 << 32), A))
        if key not in lists:
            lists[key] = pool.table.klass(bool(key[0]), key[1])[2]
        parts.append(lists[key])
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.int64)
    return offsets, np.array([p for x in parts for p in x], dtype=np.uint16)


def test_host_forms_take_unaligned_request_arrays(pools, refs):
    """The feedback chain's host form and lig_filter_batch stage a page-locked request array at +8
    as they stage pageable memory (every kernel reads a lig_req with one 16-byte load).  With a
    window longer than every call, no window closes and the chain's picks are the plain picks; the
    filter's picks are those picks and its lists the class lists."""
    pool = pools[0]
    e = Engine(0, max_pods=C3["P"], max_adapters=C3["A"], max_batch=1 << 13)
    lib = N.load()
    try:
        e.upload_snapshot(1, pool.packed)
        for R in (1, 1025, 4097):
            reqs, want, _ = refs.get(pool, 1, R, SEED)
            offsets_want, pods_want = filter_reference(pool, reqs[0], want[0])
            assert R == 1 or pods_want.size > R                        # lists of more than one pod
            h_in, h_out = host_buffers(lib, reqs[0])
            try:
                for in_off in (0, 8):
                    label = (R, in_off)
                    host_view(h_in + in_off, R, REQ_DTYPE)[:] = reqs[0]
                    host_view(h_out, R, PICK_DTYPE).view(np.uint8)[:] = SENTINEL
                    e.feedback_chain_reset()
                    e.schedule_batch_feedback_chain_ptr(1, SEED, h_in + in_off, R, h_out, 1 << 20)
                    assert_picks(host_view(h_out, R, PICK_DTYPE), want[0], ("chain",) + label)
                    host_view(h_out, R, PICK_DTYPE).view(np.uint8)[:] = SENTINEL
                    offsets = np.full(R + 1, -1, dtype=np.int64)
                    pods = np.zeros(pods_want.size, dtype=np.uint16)
                    e.filter_batch_ptr(1, SEED, h_in + in_off, R, h_out, offsets.ctypes.data, pods.ctypes.data,
                                       pods.size)
                    assert_picks(host_view(h_out, R, PICK_DTYPE), want[0], ("filter",) + label)
                    assert np.array_equal(offsets, offsets_want), label
                    assert np.array_equal(pods, pods_want), label
            finally:
                lib.lig_host_free(h_in)
                lib.lig_host_free(h_out)
    finally:
        e.close()
