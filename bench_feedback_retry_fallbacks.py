"""Retries with fallback rows under the load-feedback chain on one GPU:
lig_schedule_batch_feedback_chain_excluding_fallbacks against the calls it is compared with, at C4
(P = 4096, A = 1024) with the built-in tree and 9 excluded pods per request (the pick and its 8 fallbacks,
as a proxy sends them back).

1. The device form at R = 65536 with a window no call fills, at n_fallbacks = 1, 4, 8: CUDA events over
   --iters back-to-back calls, rotating --rounds times with lig_schedule_batch_feedback_chain_excluding_device
   (the chain retry without rows) and lig_schedule_batch_excluding_fallbacks_device (the resident retry
   with rows) on the same requests.  No window closes, so all three must return the same picks, and the
   chain's rows must be the resident rows.
2. Blocking host calls with page-locked buffers at R = 1, 16, 256, 4096 and n_fallbacks = 8, alternating
   call by call with lig_schedule_batch_excluding_fallbacks: once with a window no call fills, once with
   window = R, so that every chain call closes a window.  Median and p99 wall time over --calls calls each.

Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_feedback_retry_fallbacks.py [--calls 400] [--iters 10] [--rounds 9]"""
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


def host_calls(eng, lib, ep, seed, reqs, rows, n, window, calls):
    R, k = rows.shape
    bufs = [Pinned(lib, reqs), Pinned(lib, rows), Pinned(lib, np.zeros(R, PICK_DTYPE)),
            Pinned(lib, np.zeros(R, PICK_DTYPE)), Pinned(lib, np.zeros((R, n), np.int16)),
            Pinned(lib, np.zeros((R, n), np.int16))]
    pin, prows, pout, pout2, pfb, pfb2 = (b.ptr for b in bufs)
    try:
        resident = lambda: eng.schedule_batch_excluding_fallbacks_ptr(ep, seed, pin, R, prows, k, pout, n, pfb)
        chain = lambda: eng.schedule_batch_feedback_chain_excluding_fallbacks_ptr(ep, seed, pin, R, prows, k, pout2, n,
                                                                                  pfb2, window)
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
        d_fb = [torch.empty(R_dev * N.LIG_MAX_FALLBACKS, dtype=torch.int16, device="cuda") for _ in range(2)]
        st = torch.cuda.current_stream().cuda_stream
        k = rows9.shape[1]
        for n in (1, 4, 8):
            chain_rows = lambda: eng.schedule_batch_feedback_chain_excluding_fallbacks_device(  # noqa: E731
                ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(), k, d_out[0].data_ptr(), n, d_fb[0].data_ptr(),
                NO_CLOSE, 0, st)
            chain = lambda: eng.schedule_batch_feedback_chain_excluding_device(  # noqa: E731
                ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(), k, d_out[1].data_ptr(), NO_CLOSE, 0, st)
            resident_rows = lambda: eng.schedule_batch_excluding_fallbacks_device(  # noqa: E731
                ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(), k, d_out[2].data_ptr(), n, d_fb[1].data_ptr(),
                st)
            eng.feedback_chain_reset()
            for _ in range(3):
                chain_rows()
                chain()
                resident_rows()
            torch.cuda.synchronize()
            same = (torch.equal(d_out[0], d_out[1]) and torch.equal(d_out[0], d_out[2])
                    and torch.equal(d_fb[0][:R_dev * n], d_fb[1][:R_dev * n]))
            times = {"chain_rows": [], "chain": [], "resident_rows": []}
            fns = [("chain_rows", chain_rows), ("chain", chain), ("resident_rows", resident_rows)]
            for r in range(args.rounds):
                for name, fn in fns[r % 3:] + fns[:r % 3]:
                    times[name].append(timed(fn, args.iters))
            med = {m: float(np.median(t)) for m, t in times.items()}
            print(json.dumps({"form": "device", "R": R_dev, "excluded": int(k), "n_fallbacks": n,
                              "picks_and_rows_equal": bool(same),
                              **{f"{m}_us": round(v, 1) for m, v in med.items()},
                              **{f"{m}_us_min_max": [round(min(t), 1), round(max(t), 1)] for m, t in times.items()},
                              "chain_rows_over_resident_rows": round(med["chain_rows"] / med["resident_rows"], 3),
                              "chain_rows_over_chain": round(med["chain_rows"] / med["chain"], 3)}), flush=True)
        for R in (1, 16, 256, 4096):
            for window in (NO_CLOSE, R):
                rows = np.ascontiguousarray(rows9[:R])
                tr, tc = host_calls(eng, lib, ep, seed, np.ascontiguousarray(reqs[:R]), rows, 8, window, args.calls)
                print(json.dumps({"form": "host_pinned", "R": R, "excluded": int(k), "n_fallbacks": 8,
                                  "window": "none closes" if window == NO_CLOSE else "every call closes one",
                                  "chain_rows_us_median": round(float(np.median(tc)), 2),
                                  "chain_rows_us_p99": round(float(np.percentile(tc, 99)), 2),
                                  "resident_rows_us_median": round(float(np.median(tr)), 2),
                                  "resident_rows_us_p99": round(float(np.percentile(tr, 99)), 2)}), flush=True)
        print(json.dumps({"P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
