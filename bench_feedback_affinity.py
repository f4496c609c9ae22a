"""Session affinity under the load-feedback chain on one GPU, at C4 (P = 4096, A = 1024, built-in tree).

1. Host-buffer calls with page-locked buffers, R in {1, 16, 256, 4096}, n in {0, 8}, descriptors and
   model ids.  Four calls alternate, one of each per round, --calls rounds after a warm-up, each timed on
   the host clock around the blocking call:
     chain_aff        lig_schedule_[models_]batch_feedback_chain_affinity, W larger than the run (no
                      window closes)
     chain_aff_close  the chain affinity call with W = R on a second context: every call closes one
                      window, and the next call rebuilds the class tables first
     resident_aff     lig_schedule_[models_]batch_affinity on the resident epoch
     chain            the plain chain call lig_schedule_[models_]batch_feedback_chain, no window closes
   Prints median and p99 per call.
2. The device form at R = 2^20, n in {0, 8}: lig_schedule_batch_feedback_chain_affinity_device with W
   larger than the run against lig_schedule_batch_affinity_device and the plain chain device call, CUDA
   events over --iters back-to-back calls, --rounds times, alternating.
3. The herd: Zipf-distributed session keys (s = 1.3) over one scrape window, critical requests for an
   adapter no pod holds, on an idle pool; the largest number of picks on one pod and the pods used, for
   resident affinity and for the chain with W in {1, 8, 64}.  P = 32 with R = 3000 (the CPU test's
   case, so the figures must equal its printout) and the C4 pool with R = 65536.
Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_feedback_affinity.py [--calls 300] [--iters 20] [--rounds 11]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_feedback_fallbacks import Pinned  # noqa: E402
from bench_filter_batch import card, timed  # noqa: E402
from llm_instance_gateway_b200 import _native as N  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models  # noqa: E402

NF = N.LIG_MAX_FALLBACKS
NO_CLOSE = (1 << 31) - 1


def mix(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def c4_engines(n, max_batch):
    c = WL.CONFIGS["C4"]
    P, A = c["P"], c["A"]
    snap = WL.make_snapshot(P, A)
    models = pack_models(WL.make_models(A), snap.packed)
    pod_keys = np.random.default_rng(1).integers(0, 1 << 64, size=P, dtype=np.uint64)
    engines = [Engine(0, max_pods=P, max_adapters=A, max_batch=max_batch) for _ in range(n)]
    for e in engines:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, models)
        e.upload_pod_keys(1, pod_keys)
    return engines, A


def host_part(calls):
    lib = N.load()
    engines, A = c4_engines(2, 4096)
    bufs = []
    try:
        a, b = engines
        for R in (1, 16, 256, 4096):
            for kind in ("descriptors", "model_ids"):
                m = kind == "model_ids"
                data = WL.make_model_requests(R, A) if m else WL.make_requests(R, A)
                keys = np.random.default_rng(R).integers(0, 1 << 64, size=R, dtype=np.uint64)
                pin, pout = Pinned(lib, data.nbytes), Pinned(lib, R * (MPICK_DTYPE if m else PICK_DTYPE).itemsize)
                prows, pkeys = Pinned(lib, R * NF * 2), Pinned(lib, R * 8)
                bufs += [pin, pout, prows, pkeys]
                np.ctypeslib.as_array((C.c_uint8 * data.nbytes).from_address(pin.ptr))[:] = \
                    np.frombuffer(data.tobytes(), np.uint8)
                np.ctypeslib.as_array((C.c_uint8 * keys.nbytes).from_address(pkeys.ptr))[:] = \
                    np.frombuffer(keys.tobytes(), np.uint8)
                for n in (0, NF):
                    rp = prows.ptr if n else 0
                    if m:
                        fns = {"chain_aff": lambda: a.schedule_models_batch_feedback_chain_affinity_ptr(
                                   1, pin.ptr, pkeys.ptr, R, pout.ptr, n, rp, NO_CLOSE),
                               "chain_aff_close": lambda: b.schedule_models_batch_feedback_chain_affinity_ptr(
                                   1, pin.ptr, pkeys.ptr, R, pout.ptr, n, rp, R),
                               "resident_aff": lambda: a.schedule_models_batch_affinity_ptr(1, pin.ptr, pkeys.ptr, R,
                                                                                            pout.ptr, n, rp),
                               "chain": lambda: a.schedule_models_batch_feedback_chain_ptr(1, 5, 0, pin.ptr, R,
                                                                                           pout.ptr, NO_CLOSE)}
                    else:
                        fns = {"chain_aff": lambda: a.schedule_batch_feedback_chain_affinity_ptr(
                                   1, pin.ptr, R, pout.ptr, n, rp, NO_CLOSE),
                               "chain_aff_close": lambda: b.schedule_batch_feedback_chain_affinity_ptr(
                                   1, pin.ptr, R, pout.ptr, n, rp, R),
                               "resident_aff": lambda: a.schedule_batch_affinity_ptr(1, pin.ptr, R, pout.ptr, n, rp),
                               "chain": lambda: a.schedule_batch_feedback_chain_ptr(1, 5, pin.ptr, R, pout.ptr,
                                                                                    NO_CLOSE)}
                    for e in engines:
                        e.feedback_chain_reset()
                    for _ in range(20):                    # warm-up (and the chains' starts)
                        for fn in fns.values():
                            fn()
                    times = {k: [] for k in fns}
                    for r in range(calls):
                        order = list(fns) if r % 2 == 0 else list(fns)[::-1]
                        for k in order:
                            t0 = time.perf_counter()
                            fns[k]()
                            times[k].append((time.perf_counter() - t0) * 1e6)
                    row = {"part": "host", "kind": kind, "R": R, "n": n, "calls": calls}
                    for k, v in times.items():
                        row[k + "_median_us"] = round(float(np.median(v)), 2)
                        row[k + "_p99_us"] = round(float(np.percentile(v, 99)), 2)
                    print(json.dumps(row), flush=True)
    finally:
        for p in bufs:
            p.free()
        for e in engines:
            e.close()


def device_part(iters, rounds):
    R = WL.CONFIGS["C4"]["R"]
    (eng,), A = c4_engines(1, 4096)
    try:
        reqs = WL.make_requests(R, A)
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.empty(R * NF, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        for n in (0, NF):
            rp = d_rows.data_ptr() if n else 0
            fns = {
                "resident_aff": lambda: eng.schedule_batch_affinity_device(1, d_reqs.data_ptr(), R, d_out.data_ptr(),
                                                                           n, rp, st),
                "chain_aff": lambda: eng.schedule_batch_feedback_chain_affinity_device(
                    1, d_reqs.data_ptr(), R, d_out.data_ptr(), n, rp, NO_CLOSE, 0, st),
                "chain": lambda: eng.schedule_batch_feedback_chain_device(1, 7, d_reqs.data_ptr(), R, d_out.data_ptr(),
                                                                          NO_CLOSE, 0, st),
            }
            eng.feedback_chain_reset()
            # NO_CLOSE requests in all would close a window: the run stays far below it
            assert (3 + rounds * iters) * 2 * R < NO_CLOSE
            for _ in range(3):
                for fn in fns.values():
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in fns}
            for r in range(rounds):
                order = list(fns) if r % 2 == 0 else list(fns)[::-1]
                for k in order:
                    times[k].append(timed(fns[k], iters))
            row = {"part": "device", "R": R, "n": n, "iters": iters, "rounds": rounds}
            for k, v in times.items():
                row[k + "_median_us"] = round(float(np.median(v)), 2)
                row[k + "_us_min_max"] = [round(min(v), 2), round(max(v), 2)]
            row["chain_aff_over_resident"] = round(row["chain_aff_median_us"] / row["resident_aff_median_us"], 3)
            print(json.dumps(row), flush=True)
    finally:
        eng.close()


def herd(P, R, snap_seed, seed=5):
    snap = WL.make_snapshot(P, 2 if P == 32 else WL.CONFIGS["C4"]["A"], seed=snap_seed)
    p = snap.packed
    p.q[:] = 0
    p.kv[:] = 0.1
    pod_keys = np.random.default_rng(seed).integers(0, 1 << 64, size=P, dtype=np.uint64)
    rng = np.random.default_rng(seed + 1)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["adapter_id"] = p.A                      # no pod lists it
    reqs["flags"] = N.LIG_REQ_CRITICAL
    reqs["rand_key"] = mix(np.minimum(rng.zipf(1.3, R), 10 ** 6).astype(np.uint64))
    row = {"part": "herd", "P": P, "R": R, "zipf_s": 1.3}
    with Engine(0, max_pods=P, max_adapters=p.A, max_batch=R) as e:
        e.upload_snapshot(1, p)
        e.upload_pod_keys(1, pod_keys)
        out, _ = e.schedule_batch_affinity(1, reqs, 0)
        assert (out["status"] == N.LIG_OK).all()
        loads = np.bincount(out["pod_idx"], minlength=P)
        row["resident"] = [int(loads.max()), int((loads > 0).sum())]
        for W in (1, 8, 64):
            e.feedback_chain_reset()
            L = np.zeros(P, np.int32)
            e.schedule_batch_feedback_chain_affinity(1, reqs, 0, W, loads=L)
            row[f"W={W}"] = [int(L.max()), int((L > 0).sum())]
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=11)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    herd(32, 3000, 5)
    herd(WL.CONFIGS["C4"]["P"], 1 << 16, 1)
    host_part(args.calls)
    device_part(args.iters, args.rounds)


if __name__ == "__main__":
    main()
