"""Retries under the load-feedback chain on one GPU: lig_schedule_batch_feedback_chain_excluding against the
calls it is compared with, at C4 (P = 4096, A = 1024) with the built-in tree and 9 excluded pods per
request (the pick and its 8 fallbacks, as a proxy sends them back).

1. The device form at R = 65536 with a window no call fills, CUDA events over --iters back-to-back calls,
   alternating --rounds times with lig_schedule_batch_excluding_device (the resident retry) and
   lig_schedule_batch_feedback_chain_device (the plain chain call) on the same requests.  The retries
   are reported as pod evaluations per second, R x P / time.
2. Blocking host calls with page-locked buffers at R = 1, 16, 256, 4096, alternating call by call with
   lig_schedule_batch_excluding: once with a window no call fills, once with window = R, so that every
   chain call closes a window and the next one runs after a close (a retry segment rebuilds no class
   table).  Median and p99 wall time over --calls calls each.

Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_feedback_retry.py [--calls 400] [--iters 10] [--rounds 9]"""
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
from bench_retry import Pinned  # noqa: E402
from llm_instance_gateway_b200 import _native as N  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import PICK_DTYPE  # noqa: E402

NO_CLOSE = 1 << 30


def host_calls(eng, lib, ep, seed, reqs, rows, window, calls):
    R, k = rows.shape
    bufs = [Pinned(lib, reqs), Pinned(lib, rows), Pinned(lib, np.zeros(R, PICK_DTYPE)), Pinned(lib, np.zeros(R, PICK_DTYPE))]
    pin, prows, pout, pout2 = (b.ptr for b in bufs)
    try:
        resident = lambda: eng.schedule_batch_excluding_ptr(ep, seed, pin, R, prows, k, pout)
        chain = lambda: eng.schedule_batch_feedback_chain_excluding_ptr(ep, seed, pin, R, prows, k, pout2, window)
        eng.feedback_chain_reset()
        for _ in range(20):                  # warm-up
            resident()
            chain()
        tr, tc = [], []
        for i in range(calls):               # alternate which call goes first
            for fn, acc in (((chain, tc), (resident, tr)) if i % 2 else ((resident, tr), (chain, tc))):
                t0 = time.perf_counter()
                fn()
                acc.append((time.perf_counter() - t0) * 1e6)
        return tr, tc
    finally:
        for b in bufs:
            b.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=9)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    c = WL.CONFIGS["C4"]
    P, A, R_dev = c["P"], c["A"], 65536
    snap = WL.make_snapshot(P, A)
    lib = N.load()
    eng = Engine(0, max_pods=P, max_adapters=A, max_batch=R_dev)
    try:
        ep, seed = 1, 0xC0FFEE
        eng.upload_snapshot(ep, snap.packed)
        reqs = WL.make_requests(R_dev, A)
        picks, fb = eng.schedule_batch_fallbacks(ep, seed, reqs, N.LIG_MAX_FALLBACKS)
        rows9 = np.concatenate([np.where(picks["status"] == N.LIG_OK, picks["pod_idx"], -1)[:, None].astype(np.int16),
                                fb], axis=1)
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_rows = torch.from_numpy(rows9.reshape(-1).copy()).cuda()
        d_out = [torch.empty(R_dev * 8, dtype=torch.uint8, device="cuda") for _ in range(3)]
        st = torch.cuda.current_stream().cuda_stream
        k = rows9.shape[1]
        resident = lambda: eng.schedule_batch_excluding_device(ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(),
                                                               k, d_out[0].data_ptr(), st)
        chain = lambda: eng.schedule_batch_feedback_chain_excluding_device(
            ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(), k, d_out[1].data_ptr(), NO_CLOSE, 0, st)
        plain = lambda: eng.schedule_batch_feedback_chain_device(ep, seed, d_reqs.data_ptr(), R_dev,
                                                                 d_out[2].data_ptr(), NO_CLOSE, 0, st)
        eng.feedback_chain_reset()
        for _ in range(3):
            resident()
            chain()
            plain()
        torch.cuda.synchronize()
        same = torch.equal(d_out[0], d_out[1])   # no window closed: the chain retry is the resident one
        times = {"resident": [], "chain": [], "plain_chain": []}
        fns = [("resident", resident), ("chain", chain), ("plain_chain", plain)]
        for r in range(args.rounds):
            for name, fn in fns[r % 3:] + fns[:r % 3]:
                times[name].append(timed(fn, args.iters))
        med = {n: float(np.median(t)) for n, t in times.items()}
        print(json.dumps({"form": "device", "R": R_dev, "excluded": int(k), "chain_equals_resident": bool(same),
                          **{f"{n}_us": round(m, 1) for n, m in med.items()},
                          **{f"{n}_us_min_max": [round(min(t), 1), round(max(t), 1)] for n, t in times.items()},
                          "chain_over_resident": round(med["chain"] / med["resident"], 3),
                          "chain_pod_evals_per_s": round(R_dev * P / (med["chain"] * 1e-6), 0),
                          "resident_pod_evals_per_s": round(R_dev * P / (med["resident"] * 1e-6), 0)}), flush=True)
        for R in (1, 16, 256, 4096):
            for window in (NO_CLOSE, R):
                rows = np.ascontiguousarray(rows9[:R])
                tr, tc = host_calls(eng, lib, ep, seed, np.ascontiguousarray(reqs[:R]), rows, window, args.calls)
                print(json.dumps({"form": "host_pinned", "R": R, "excluded": int(k),
                                  "window": "none closes" if window == NO_CLOSE else "every call closes one",
                                  "chain_us_median": round(float(np.median(tc)), 2),
                                  "chain_us_p99": round(float(np.percentile(tc, 99)), 2),
                                  "resident_us_median": round(float(np.median(tr)), 2),
                                  "resident_us_p99": round(float(np.percentile(tr, 99)), 2)}), flush=True)
        print(json.dumps({"P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
