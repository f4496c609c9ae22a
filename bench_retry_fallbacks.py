"""Retry scheduling with fallback rows on one GPU: lig_schedule_batch_excluding_fallbacks against the plain
retry, lig_schedule_batch_excluding, on the same inputs, at C4 (P = 4096, A = 1024).

Every request excludes 9 pods: a real pick and its 8-entry fallback row (the rows a proxy sends back once
its first row is used up, as bench_retry.py builds them).

1. The device form at R = 65536 and n = 1, 4 and 8, CUDA events over --iters back-to-back calls,
   alternating --rounds times with the plain retry, for the built-in tree and for a one-predicate caller
   tree that keeps every pod (so every row fills and every request makes all n + 1 selects).
2. Blocking host calls with page-locked buffers at R = 1, 16, 256, 4096 (built-in tree, n = 8),
   alternating call by call with the plain retry: median and p99 wall time over --calls calls each.

Each configuration also reports the mean number of in-range row entries per request: the extra
attempts one round trip serves besides the pick.  Prints the card and its power limit first, then one
JSON line per measurement.

Usage: python bench_retry_fallbacks.py [--calls 400] [--iters 10] [--rounds 9]"""
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

K = N.LIG_MAX_FALLBACKS
KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]


def excluded_rows(eng, ep, seed, reqs):
    """The pick and its 8 fallbacks per request, as int16 rows of 9 (-1 where the request is not OK)."""
    picks, fb = eng.schedule_batch_fallbacks(ep, seed, reqs, K)
    pick = np.where(picks["status"] == N.LIG_OK, picks["pod_idx"], -1)[:, None].astype(np.int16)
    return np.ascontiguousarray(np.concatenate([pick, fb], axis=1))


def device_rounds(eng, ep, seed, reqs, rows, k, args):
    R, w = rows.shape
    d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
    d_rows = torch.from_numpy(rows.reshape(-1).copy()).cuda()
    d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
    d_out2 = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
    d_fb = torch.empty(R * k, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    retry = lambda: eng.schedule_batch_excluding_device(ep, seed, d_reqs.data_ptr(), R, d_rows.data_ptr(), w,
                                                        d_out.data_ptr(), st)
    rows_call = lambda: eng.schedule_batch_excluding_fallbacks_device(ep, seed, d_reqs.data_ptr(), R,
                                                                      d_rows.data_ptr(), w, d_out2.data_ptr(), k,
                                                                      d_fb.data_ptr(), st)
    for _ in range(3):
        retry()
        rows_call()
    torch.cuda.synchronize()
    assert torch.equal(d_out, d_out2), "the picks differ from the plain retry's"
    tp, tf = [], []
    for r in range(args.rounds):
        order = ((rows_call, tf), (retry, tp)) if r % 2 else ((retry, tp), (rows_call, tf))
        for fn, acc in order:
            acc.append(timed(fn, args.iters))
    fb = d_fb.cpu().numpy().reshape(R, k)
    return float(np.median(tp)), float(np.median(tf)), tp, tf, fb


def host_calls(eng, lib, ep, seed, reqs, rows, calls):
    R, w = rows.shape
    bufs = [Pinned(lib, reqs), Pinned(lib, rows), Pinned(lib, np.zeros(R, PICK_DTYPE)),
            Pinned(lib, np.zeros(R, PICK_DTYPE)), Pinned(lib, np.zeros((R, K), np.int16))]
    pin, prows, pout, pout2, pfb = (b.ptr for b in bufs)
    try:
        retry = lambda: eng.schedule_batch_excluding_ptr(ep, seed, pin, R, prows, w, pout)
        rows_call = lambda: eng.schedule_batch_excluding_fallbacks_ptr(ep, seed, pin, R, prows, w, pout2, K, pfb)
        for _ in range(20):                  # warm-up
            retry()
            rows_call()
        tp, tf = [], []
        for i in range(calls):               # alternate which call goes first
            for fn, acc in (((rows_call, tf), (retry, tp)) if i % 2 else ((retry, tp), (rows_call, tf))):
                t0 = time.perf_counter()
                fn()
                acc.append((time.perf_counter() - t0) * 1e6)
        assert bufs[2].a.tobytes() == bufs[3].a.tobytes(), "the picks differ from the plain retry's"
        return tp, tf
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
        seed = 0xC0FFEE
        reqs = WL.make_requests(R_dev, A)
        for ep, tree in ((1, None), (2, KEEP_ALL)):
            eng.set_filter_tree(tree)
            eng.upload_snapshot(ep, snap.packed)
            eng.set_filter_tree(None)
            rows = excluded_rows(eng, ep, seed, reqs)
            for k in (1, 4, K):          # n = 1 and 4: what the ranking steps cost beyond the walk and the pick
                mp, mf, tp, tf, fb = device_rounds(eng, ep, seed, reqs, rows, k, args)
                print(json.dumps({"form": "device", "tree": "built-in" if tree is None else "keep_all", "R": R_dev,
                                  "excluded": int(rows.shape[1]), "n_fallbacks": k,
                                  "excluding_fallbacks_us": round(mf, 1), "excluding_us": round(mp, 1),
                                  "ratio": round(mf / mp, 3),
                                  "excluding_fallbacks_us_min_max": [round(min(tf), 1), round(max(tf), 1)],
                                  "excluding_us_min_max": [round(min(tp), 1), round(max(tp), 1)],
                                  "row_entries_per_request": round(float((fb >= 0).sum(axis=1).mean()), 2)}),
                      flush=True)
            if tree is not None:
                continue
            for R in (1, 16, 256, 4096):
                sub_reqs, sub_rows = np.ascontiguousarray(reqs[:R]), np.ascontiguousarray(rows[:R])
                tp, tf = host_calls(eng, lib, ep, seed, sub_reqs, sub_rows, args.calls)
                print(json.dumps({"form": "host_pinned", "tree": "built-in", "R": R, "excluded": int(rows.shape[1]),
                                  "n_fallbacks": K,
                                  "excluding_fallbacks_us_median": round(float(np.median(tf)), 2),
                                  "excluding_fallbacks_us_p99": round(float(np.percentile(tf, 99)), 2),
                                  "excluding_us_median": round(float(np.median(tp)), 2),
                                  "excluding_us_p99": round(float(np.percentile(tp, 99)), 2),
                                  "ratio": round(float(np.median(tf)) / float(np.median(tp)), 3)}), flush=True)
        print(json.dumps({"P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
