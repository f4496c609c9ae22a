"""Survivor lists of a whole batch on one GPU: lig_filter_batch_device against lig_schedule_batch_device
in the same process, and the model-id form lig_filter_models_batch_device against
lig_schedule_models_batches_device.

C4 (R = 2^20, P = 4096, A = 1024), HBM-resident buffers, one stream.  The two calls of a pair
alternate, each timed with CUDA events over --iters back-to-back calls, --rounds times.  Prints the
card and its power limit first, then one JSON line per form: median time per call, and the bytes per
call the survivor-list call moves by the formula
    R x (16 B descriptor or 4 B id in + 8 B or 4 B pick out + 8 B offset) + 2 B x sum(n)
(class tables and the compact pool are not counted: they stay in L2).

Usage: python bench_filter_batch.py [--iters 20] [--rounds 15]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import pack_models  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters   # us per call


def compare(name, base, filt, iters, rounds, bytes_per_call):
    for _ in range(3):                       # warm-up
        base()
        filt()
    torch.cuda.synchronize()
    tb, tf = [], []
    for r in range(rounds):                  # alternate which call goes first
        if r % 2:
            tf.append(timed(filt, iters))
            tb.append(timed(base, iters))
        else:
            tb.append(timed(base, iters))
            tf.append(timed(filt, iters))
    mf, mb = float(np.median(tf)), float(np.median(tb))
    print(json.dumps({"form": name, "filter_us": round(mf, 2), "schedule_us": round(mb, 2),
                      "filter_over_schedule": round(mf / mb, 3), "filter_bytes_per_call": bytes_per_call,
                      "filter_gb_per_s": round(bytes_per_call / mf / 1e3, 1),
                      "filter_us_min_max": [round(min(tf), 2), round(max(tf), 2)],
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
        eng.upload_snapshot(1, snap.packed)
        eng.upload_models(1, pack_models(WL.make_models(A), snap.packed))
        reqs = WL.make_requests(R, A)
        ids = WL.make_model_requests(R, A)
        seed = 0xC0FFEE
        # sizes of the lists, from one host call of each form
        total = int(eng.filter_batch(1, seed, reqs)[1][-1])
        mtotal = int(eng.filter_models_batch(1, seed, ids)[1][-1])
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_off = torch.empty(R + 1, dtype=torch.int64, device="cuda")
        d_pods = torch.empty(max(total, mtotal, 1), dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream

        compare("descriptors",
                lambda: eng.schedule_batch_device(1, seed, d_reqs.data_ptr(), R, d_out.data_ptr(), st),
                lambda: eng.filter_batch_device(1, seed, d_reqs.data_ptr(), R, d_out.data_ptr(), d_off.data_ptr(),
                                                d_pods.data_ptr(), total, st),
                args.iters, args.rounds, R * (16 + 8 + 8) + 2 * total)
        compare("model_ids",
                lambda: eng.schedule_models_batches_device(1, seed, 0, [d_ids.data_ptr()], R, [d_out.data_ptr()], st),
                lambda: eng.filter_models_batch_device(1, seed, 0, d_ids.data_ptr(), R, d_out.data_ptr(),
                                                       d_off.data_ptr(), d_pods.data_ptr(), mtotal, st),
                args.iters, args.rounds, R * (4 + 4 + 8) + 2 * mtotal)
        print(json.dumps({"R": R, "P": P, "A": A, "survivors_descriptors": total, "survivors_model_ids": mtotal,
                          "mean_n_descriptors": round(total / R, 3), "mean_n_model_ids": round(mtotal / R, 3)}),
              flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
