"""Outlier ejection on one GPU at C4 (P = 4096, A = 1024, the built-in tree).

1. Writers, blocking wall time (median and p99 over --calls calls each, alternating call by call):
   lig_eject_pods with 16 pods against lig_update_snapshot with 16 dirty pods, and against
   lig_upload_snapshot.  All three leave a new resident epoch with its class tables built.
2. The pick on a derived epoch against its base: one queue of 8 HBM-resident batches of 65536
   requests (lig_schedule_batches_device), CUDA events over --iters queues, alternating --rounds
   times.  Both run the same pick kernels.
3. The pool build kernels against the plain ones: with one plain and one derived epoch (16 pods
   ejected) resident, every lig_set_thresholds call rebuilds both, so the two forms of the build run
   back to back, --iters x --rounds times; their device times are read kernel by kernel from the CUDA
   activity trace (torch.profiler).  The C4 fast build, and the general staged build at P = 8192.

Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_eject.py [--calls 200] [--iters 20] [--rounds 9]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_filter_batch import card, timed  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402


def wall(fn, calls):
    ts = []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e6)
    return float(np.median(ts)), float(np.percentile(ts, 99))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=9)
    a = ap.parse_args()
    print(f"card: {card()}")
    c = WL.CONFIGS["C4"]
    P, A = c["P"], c["A"]
    snap = WL.make_snapshot(P, A, seed=1).packed
    rng = np.random.default_rng(2)
    ejected = np.sort(rng.choice(P, size=16, replace=False)).astype(np.int32)
    dirty = ejected.copy()
    kv, q = snap.kv[dirty].copy(), snap.q[dirty].copy()
    na, ma = snap.n_active[dirty].copy(), snap.max_active[dirty].copy()
    off = np.zeros(len(dirty) + 1, dtype=np.int32)
    ids = np.zeros(0, dtype=np.int32)
    eng = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 16)
    ep = [1]

    def nxt():
        ep[0] += 1
        return ep[0]

    base = 1
    eng.upload_snapshot(base, snap)
    cur = [base]

    def eject():                         # derive from the newest epoch: the base is never the victim
        e = nxt()
        eng.eject_pods(e, cur[0], ejected)
        cur[0] = e

    def update():
        e = nxt()
        eng.update_snapshot(e, cur[0], dirty, kv, q, na, ma, off, ids)
        cur[0] = e

    def upload():
        e = nxt()
        eng.upload_snapshot(e, snap)
        cur[0] = e

    for fn in (eject, update, upload):
        wall(fn, 10)                     # warm-up
    res = {"eject": [], "update": [], "upload": []}
    for _ in range(a.calls):
        for name, fn in (("eject", eject), ("update", update), ("upload", upload)):
            t = time.perf_counter()
            fn()
            res[name].append((time.perf_counter() - t) * 1e6)
    for name, ts in res.items():
        print(json.dumps({"measure": "writer", "call": name, "P": P, "A": A, "n": 16,
                          "median_us": round(float(np.median(ts)), 1), "p99_us": round(float(np.percentile(ts, 99)), 1)}))

    # 2. picks: derived epoch against its base
    base, derived = nxt(), nxt()
    eng.upload_snapshot(base, snap)
    eng.eject_pods(derived, base, ejected)
    R, B = 65536, 8
    reqs = WL.make_requests(R, A, seed=3)
    d_in = torch.from_numpy(reqs.view(np.uint8).reshape(-1).copy()).cuda()
    outs = [torch.zeros(R * 8, dtype=torch.uint8, device="cuda") for _ in range(B)]
    optrs = [o.data_ptr() for o in outs]
    run = {e: (lambda e=e: eng.schedule_batches_device(e, 7, [d_in.data_ptr()] * B, R, optrs)) for e in (base, derived)}
    for e in (base, derived):
        timed(run[e], 3)
    t = {base: [], derived: []}
    for _ in range(a.rounds):
        for e in (base, derived):
            t[e].append(timed(run[e], a.iters))
    for e, name in ((base, "base"), (derived, "derived")):
        us = float(np.median(t[e]))
        print(json.dumps({"measure": "pick_queue", "epoch": name, "R": R, "batches": B, "median_us": round(us, 1),
                          "decisions_per_s": round(R * B / us * 1e6)}))

    # 3. builds: one plain and one derived epoch resident, so each lig_set_thresholds rebuild runs the
    # plain and the pool form of the same build kernel once each; their device times come from the
    # CUDA activity trace (torch.profiler), kernel by kernel
    eng.close()
    for label, bp in (("C4 fast build", P), ("general staged build", 8192)):
        bsnap = snap if bp == P else WL.make_snapshot(bp, A, seed=1).packed
        be = Engine(0, max_pods=bp, max_adapters=A, max_batch=1 << 12)
        be.upload_snapshot(1, bsnap)
        be.eject_pods(2, 1, ejected)
        for _ in range(3):
            be.set_thresholds(0.8, 5, 50)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters * a.rounds):
                be.set_thresholds(0.8, 5, 50)
        torch.cuda.synchronize()
        for ev in prof.key_averages():
            if "lig_class_build" in ev.key:
                us = getattr(ev, "device_time", None)
                us = ev.cuda_time if us is None else us
                form = "pool" if ("<true>" in ev.key or ", true>" in ev.key) else "plain"
                print(json.dumps({"measure": "build_kernel", "build": label, "P": bp, "A": A, "form": form,
                                  "kernel": ev.key.split("(")[0], "launches": ev.count, "mean_us": round(us, 2)}))
        be.close()


if __name__ == "__main__":
    main()
