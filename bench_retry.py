"""Retry scheduling on one GPU: lig_schedule_batch_excluding against the calls it is compared with, at C4
(P = 4096, A = 1024) with the built-in tree.

1. Blocking host calls with page-locked buffers at R = 1, 16, 256, 4096 with 1 and 9 excluded pods per
   request (the pick, then the pick and its 8 fallbacks), alternating call by call with
   lig_schedule_batch on the same requests: median and p99 wall time over --calls calls each.
2. The device form at R = 65536 with 9 excluded pods, CUDA events over --iters back-to-back calls,
   alternating --rounds times with lig_schedule_scan_device (the direct scan, no masks) on the same
   requests.  Both walk the tree per request over all P pods, so both are reported as pod evaluations
   per second, R x P / time.

Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_retry.py [--calls 400] [--iters 10] [--rounds 9]"""
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

from bench_filter_batch import card, timed  # noqa: E402
from llm_instance_gateway_b200 import _native as N  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import PICK_DTYPE  # noqa: E402


class Pinned:
    """A page-locked host array (lig_host_alloc)."""

    def __init__(self, lib, arr: np.ndarray):
        self.lib = lib
        self.ptr = lib.lig_host_alloc(max(arr.nbytes, 16))
        assert self.ptr
        self.a = np.ctypeslib.as_array((C.c_uint8 * max(arr.nbytes, 16)).from_address(self.ptr))[: arr.nbytes]
        self.a[:] = np.frombuffer(np.ascontiguousarray(arr).tobytes(), np.uint8)

    def free(self):
        self.lib.lig_host_free(self.ptr)


def host_calls(eng, lib, ep, seed, reqs, rows, calls):
    R, k = rows.shape
    bufs = [Pinned(lib, reqs), Pinned(lib, rows), Pinned(lib, np.zeros(R, PICK_DTYPE)), Pinned(lib, np.zeros(R, PICK_DTYPE))]
    pin, prows, pout, pout2 = (b.ptr for b in bufs)
    try:
        plain = lambda: eng.schedule_batch_ptr(ep, seed, pin, R, pout)
        retry = lambda: eng.schedule_batch_excluding_ptr(ep, seed, pin, R, prows, k, pout2)
        for _ in range(20):                  # warm-up
            plain()
            retry()
        tp, tr = [], []
        for i in range(calls):               # alternate which call goes first
            for fn, acc in (((retry, tr), (plain, tp)) if i % 2 else ((plain, tp), (retry, tr))):
                t0 = time.perf_counter()
                fn()
                acc.append((time.perf_counter() - t0) * 1e6)
        return tp, tr
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
        # the rows a proxy would send back: the pick, or the pick and its 8 fallbacks
        picks, fb = eng.schedule_batch_fallbacks(ep, seed, reqs, N.LIG_MAX_FALLBACKS)
        rows9 = np.concatenate([np.where(picks["status"] == N.LIG_OK, picks["pod_idx"], -1)[:, None].astype(np.int16),
                                fb], axis=1)
        print(json.dumps({"excluded_in_range_per_row_9": round(float((rows9 >= 0).sum(axis=1).mean()), 2)}), flush=True)
        for R in (1, 16, 256, 4096):
            for k in (1, 9):
                rows = np.ascontiguousarray(rows9[:R, :k])
                tp, tr = host_calls(eng, lib, ep, seed, np.ascontiguousarray(reqs[:R]), rows, args.calls)
                print(json.dumps({"form": "host_pinned", "R": R, "excluded": k,
                                  "retry_us_median": round(float(np.median(tr)), 2),
                                  "retry_us_p99": round(float(np.percentile(tr, 99)), 2),
                                  "schedule_us_median": round(float(np.median(tp)), 2),
                                  "schedule_us_p99": round(float(np.percentile(tp, 99)), 2),
                                  "retry_pod_evals_per_s": round(R * P / (float(np.median(tr)) * 1e-6), 0)}), flush=True)
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_rows = torch.from_numpy(rows9.reshape(-1).copy()).cuda()
        d_out = torch.empty(R_dev * 8, dtype=torch.uint8, device="cuda")
        d_out2 = torch.empty(R_dev * 8, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        scan = lambda: eng.schedule_scan_device(ep, seed, d_reqs.data_ptr(), R_dev, d_out.data_ptr(), 0, st)
        retry = lambda: eng.schedule_batch_excluding_device(ep, seed, d_reqs.data_ptr(), R_dev, d_rows.data_ptr(),
                                                            rows9.shape[1], d_out2.data_ptr(), st)
        for _ in range(3):
            scan()
            retry()
        torch.cuda.synchronize()
        ts, tr = [], []
        for r in range(args.rounds):
            if r % 2:
                tr.append(timed(retry, args.iters))
                ts.append(timed(scan, args.iters))
            else:
                ts.append(timed(scan, args.iters))
                tr.append(timed(retry, args.iters))
        ms, mr = float(np.median(ts)), float(np.median(tr))
        print(json.dumps({"form": "device", "R": R_dev, "excluded": int(rows9.shape[1]),
                          "retry_us": round(mr, 1), "scan_us": round(ms, 1), "retry_over_scan": round(mr / ms, 3),
                          "retry_pod_evals_per_s": round(R_dev * P / (mr * 1e-6), 0),
                          "scan_pod_evals_per_s": round(R_dev * P / (ms * 1e-6), 0),
                          "retry_us_min_max": [round(min(tr), 1), round(max(tr), 1)],
                          "scan_us_min_max": [round(min(ts), 1), round(max(ts), 1)]}), flush=True)
        print(json.dumps({"P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
