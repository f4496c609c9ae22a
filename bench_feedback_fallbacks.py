"""Fallback rows under the load-feedback chain on one GPU, at C4 (P = 4096, A = 1024, built-in tree).

1. Host-buffer calls with page-locked buffers, n = 8, R in {1, 16, 256, 4096}, descriptors and model
   ids.  Four calls alternate, one of each per round, --calls rounds after a warm-up, each timed on
   the host clock around the blocking call:
     chain            lig_schedule_[models_]batch_feedback_chain, W larger than the run (no window closes)
     chain_fb         lig_schedule_[models_]batch_feedback_chain_fallbacks, the same chain
     chain_fb_close   the chain fallback call with W = R on a second context: every call closes one
                      window, and the next call rebuilds the class tables first
     resident_fb      lig_schedule_[models_]batch_fallbacks on the resident epoch
   Prints median and p99 per call.
2. The device form at R = 2^20, n = 8: lig_schedule_batch_feedback_chain_fallbacks_device with W
   larger than the run (no window closes) against lig_schedule_batch_fallbacks_device and the plain
   chain device call, CUDA events over --iters back-to-back calls, --rounds times, alternating.
   Bytes per call by the formula R x (16 B in + 8 B pick + 2 B x n); the 4-byte atomics of the window
   histogram and the class tables (L2-resident) are not counted.
Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_feedback_fallbacks.py [--calls 400] [--iters 20] [--rounds 11]"""
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
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, pack_models  # noqa: E402

NF = N.LIG_MAX_FALLBACKS
NO_CLOSE = (1 << 31) - 1


class Pinned:
    def __init__(self, lib, nbytes):
        self.lib, self.ptr = lib, lib.lig_host_alloc(max(nbytes, 16))
        assert self.ptr

    def free(self):
        self.lib.lig_host_free(self.ptr)


def host_part(calls):
    c = WL.CONFIGS["C4"]
    P, A = c["P"], c["A"]
    snap = WL.make_snapshot(P, A)
    models = pack_models(WL.make_models(A), snap.packed)
    lib = N.load()
    engines = [Engine(0, max_pods=P, max_adapters=A, max_batch=4096) for _ in range(2)]
    bufs = []
    try:
        for e in engines:
            e.upload_snapshot(1, snap.packed)
            e.upload_models(1, models)
        a, b = engines
        for R in (1, 16, 256, 4096):
            for kind in ("descriptors", "model_ids"):
                m = kind == "model_ids"
                data = WL.make_model_requests(R, A) if m else WL.make_requests(R, A)
                pin = Pinned(lib, data.nbytes)
                pout = Pinned(lib, R * (MPICK_DTYPE if m else PICK_DTYPE).itemsize)
                prows = Pinned(lib, R * NF * 2)
                bufs += [pin, pout, prows]
                np.ctypeslib.as_array((C.c_uint8 * data.nbytes).from_address(pin.ptr))[:] = \
                    np.frombuffer(data.tobytes(), np.uint8)
                first = [0]

                def fi():
                    first[0] += R
                    return first[0]
                if m:
                    fns = {"chain": lambda: a.schedule_models_batch_feedback_chain_ptr(1, 5, fi(), pin.ptr, R, pout.ptr,
                                                                                      NO_CLOSE),
                           "chain_fb": lambda: a.schedule_models_batch_feedback_chain_fallbacks_ptr(
                               1, 5, fi(), pin.ptr, R, pout.ptr, NF, prows.ptr, NO_CLOSE),
                           "chain_fb_close": lambda: b.schedule_models_batch_feedback_chain_fallbacks_ptr(
                               1, 5, fi(), pin.ptr, R, pout.ptr, NF, prows.ptr, R),
                           "resident_fb": lambda: a.schedule_models_batch_fallbacks_ptr(1, 5, fi(), pin.ptr, R,
                                                                                         pout.ptr, NF, prows.ptr)}
                else:
                    fns = {"chain": lambda: a.schedule_batch_feedback_chain_ptr(1, 5, pin.ptr, R, pout.ptr, NO_CLOSE),
                           "chain_fb": lambda: a.schedule_batch_feedback_chain_fallbacks_ptr(
                               1, 5, pin.ptr, R, pout.ptr, NF, prows.ptr, NO_CLOSE),
                           "chain_fb_close": lambda: b.schedule_batch_feedback_chain_fallbacks_ptr(
                               1, 5, pin.ptr, R, pout.ptr, NF, prows.ptr, R),
                           "resident_fb": lambda: a.schedule_batch_fallbacks_ptr(1, 5, pin.ptr, R, pout.ptr, NF,
                                                                                  prows.ptr)}
                for e in engines:
                    e.feedback_chain_reset()
                for _ in range(20):                        # warm-up (and the chains' starts)
                    for fn in fns.values():
                        fn()
                times = {k: [] for k in fns}
                for r in range(calls):
                    order = list(fns) if r % 2 == 0 else list(fns)[::-1]
                    for k in order:
                        t0 = time.perf_counter()
                        fns[k]()
                        times[k].append((time.perf_counter() - t0) * 1e6)
                row = {"part": "host", "kind": kind, "R": R, "n": NF, "calls": calls}
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
    c = WL.CONFIGS["C4"]
    R, P, A = c["R"], c["P"], c["A"]
    snap = WL.make_snapshot(P, A)
    eng = Engine(0, max_pods=P, max_adapters=A, max_batch=4096)
    try:
        eng.upload_snapshot(1, snap.packed)
        reqs = WL.make_requests(R, A)
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.empty(R * NF, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        fns = {
            "resident_fb": lambda: eng.schedule_batch_fallbacks_device(1, 7, d_reqs.data_ptr(), R, d_out.data_ptr(),
                                                                       NF, d_rows.data_ptr(), st),
            "chain_fb": lambda: eng.schedule_batch_feedback_chain_fallbacks_device(
                1, 7, d_reqs.data_ptr(), R, d_out.data_ptr(), NF, d_rows.data_ptr(), NO_CLOSE, 0, st),
            "chain": lambda: eng.schedule_batch_feedback_chain_device(1, 7, d_reqs.data_ptr(), R, d_out.data_ptr(),
                                                                      NO_CLOSE, 0, st),
        }
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
        row = {"part": "device", "R": R, "P": P, "A": A, "n": NF, "iters": iters, "rounds": rounds,
               "bytes_per_call": R * (16 + 8 + 2 * NF)}
        for k, v in times.items():
            row[k + "_median_us"] = round(float(np.median(v)), 2)
            row[k + "_us_min_max"] = [round(min(v), 2), round(max(v), 2)]
            if k != "chain":
                row[k + "_gb_per_s"] = round(R * (16 + 8 + 2 * NF) / float(np.median(v)) / 1e3, 1)
        print(json.dumps(row), flush=True)
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=11)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    host_part(args.calls)
    device_part(args.iters, args.rounds)


if __name__ == "__main__":
    main()
