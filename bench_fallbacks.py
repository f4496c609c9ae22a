"""Fallback endpoints on one GPU: lig_schedule_batch_fallbacks_device at n = 1, 4, 8 against
lig_schedule_batch_device in the same process, and lig_schedule_models_batch_fallbacks_device against
lig_schedule_models_batches_device with one batch.

C4 (R = 2^20, P = 4096, A = 1024), HBM-resident buffers, one stream; once with the built-in tree
(at most 4 survivors per class after the least-KV stage, so rows are mostly -1) and once with a
caller tree of one predicate node that keeps every pod (full rows).  The two calls of a pair
alternate, each timed with CUDA events over --iters back-to-back calls, --rounds times.  Prints the
card and its power limit first, then one JSON line per (tree, form, n): median time per call, the
spread, and the bytes per call the fallback call moves by the formula
    descriptors  R x (16 B in + 8 B pick + 2 B x n)
    model ids    R x (4 B in + 4 B pick + 2 B x n)
(class tables, the compact pool and the model table are not counted: they stay in L2).

Usage: python bench_fallbacks.py [--iters 20] [--rounds 15]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_filter_batch import card, timed  # noqa: E402
from llm_instance_gateway_b200 import _native as N  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import pack_models  # noqa: E402

KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]


def compare(label, base, fb, iters, rounds, bytes_per_call):
    for _ in range(3):                       # warm-up
        base()
        fb()
    torch.cuda.synchronize()
    tb, tf = [], []
    for r in range(rounds):                  # alternate which call goes first
        if r % 2:
            tf.append(timed(fb, iters))
            tb.append(timed(base, iters))
        else:
            tb.append(timed(base, iters))
            tf.append(timed(fb, iters))
    mf, mb = float(np.median(tf)), float(np.median(tb))
    print(json.dumps({**label, "fallbacks_us": round(mf, 2), "schedule_us": round(mb, 2),
                      "fallbacks_over_schedule": round(mf / mb, 3), "fallbacks_bytes_per_call": bytes_per_call,
                      "fallbacks_gb_per_s": round(bytes_per_call / mf / 1e3, 1),
                      "fallbacks_us_min_max": [round(min(tf), 2), round(max(tf), 2)],
                      "schedule_us_min_max": [round(min(tb), 2), round(max(tb), 2)]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=15)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    c = WL.CONFIGS["C4"]
    R, P, A = c["R"], c["P"], c["A"]
    snap = WL.make_snapshot(P, A)
    eng = Engine(0, max_pods=P, max_adapters=A, max_batch=R)
    try:
        reqs = WL.make_requests(R, A)
        ids = WL.make_model_requests(R, A)
        seed = 0xC0FFEE
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.empty(R * N.LIG_MAX_FALLBACKS, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        for ep, (tree_name, tree) in enumerate((("builtin", None), ("keep_all", KEEP_ALL)), start=1):
            eng.set_filter_tree(tree)
            eng.upload_snapshot(ep, snap.packed)
            eng.set_filter_tree(None)
            eng.upload_models(ep, pack_models(WL.make_models(A), snap.packed))
            full = float((eng.schedule_batch_fallbacks(ep, seed, reqs[:65536], 8)[1] >= 0).mean())
            print(json.dumps({"tree": tree_name, "fallback_entries_filled_n8": round(full, 3)}), flush=True)
            for n in (1, 4, 8):
                compare({"tree": tree_name, "form": "descriptors", "n": n},
                        lambda: eng.schedule_batch_device(ep, seed, d_reqs.data_ptr(), R, d_out.data_ptr(), st),
                        lambda: eng.schedule_batch_fallbacks_device(ep, seed, d_reqs.data_ptr(), R, d_out.data_ptr(),
                                                                    n, d_rows.data_ptr(), st),
                        args.iters, args.rounds, R * (16 + 8 + 2 * n))
                compare({"tree": tree_name, "form": "model_ids", "n": n},
                        lambda: eng.schedule_models_batches_device(ep, seed, 0, [d_ids.data_ptr()], R,
                                                                   [d_out.data_ptr()], st),
                        lambda: eng.schedule_models_batch_fallbacks_device(ep, seed, 0, d_ids.data_ptr(), R,
                                                                           d_out.data_ptr(), n, d_rows.data_ptr(), st),
                        args.iters, args.rounds, R * (4 + 4 + 2 * n))
        print(json.dumps({"R": R, "P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
