"""Session affinity on one GPU: the affinity calls against the fallback and plain calls they sit beside.

C4 (R = 2^20, P = 4096, A = 1024, built-in tree: at most 4 survivors per class), HBM-resident buffers,
one stream.  Each group's calls are timed with CUDA events over --iters back-to-back calls, interleaved
over --rounds rounds (the first call of a round rotates), and reported as the median per call with the
spread:
    descriptors  lig_schedule_batch_affinity_device n = 0 and 8, lig_schedule_batch_fallbacks_device n = 8,
                 lig_schedule_batch_device
    model ids    lig_schedule_models_batch_affinity_device n = 0 and 8,
                 lig_schedule_models_batch_fallbacks_device n = 8, lig_schedule_models_batches_device (one batch)
Then the host-buffer forms (page-locked buffers, the call blocks) at R = 1, 64 and 4096 against
lig_schedule_batch_fallbacks, and the long-list shape: P = 32768 under a caller tree of one predicate
node that keeps every pod, R = 4096, where every request is served by a whole warp.  Prints the card
and its power limit first, then one JSON line per group.

Usage: python bench_affinity.py [--iters 20] [--rounds 15]"""
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
from llm_instance_gateway_b200 import scheduling as S  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.engine import Engine  # noqa: E402
from llm_instance_gateway_b200.packer import pack_columns, pack_models  # noqa: E402

KEEP_ALL = [N.LigFilterNode(N.LIG_F_LOW_QUEUEING, -1, -1, -1, 1 << 62, 0.0)]


def group(label, calls, iters, rounds):
    """calls: {name: fn}; interleaved CUDA-event medians in us per call."""
    names = list(calls)
    for _ in range(3):
        for n in names:
            calls[n]()
    torch.cuda.synchronize()
    t = {n: [] for n in names}
    for r in range(rounds):
        order = names[r % len(names):] + names[:r % len(names)]
        for n in order:
            t[n].append(timed(calls[n], iters))
    out = {**label}
    for n in names:
        out[n + "_us"] = round(float(np.median(t[n])), 2)
        out[n + "_us_min_max"] = [round(min(t[n]), 2), round(max(t[n]), 2)]
    print(json.dumps(out), flush=True)
    return out


def pinned(lib, nbytes):
    ptr = lib.lig_host_alloc(max(nbytes, 16))
    assert ptr
    return ptr


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
    lib = eng._lib
    ptrs = []
    try:
        reqs = WL.make_requests(R, A)
        ids = WL.make_model_requests(R, A)
        keys = np.random.default_rng(1).integers(0, 1 << 64, size=R, dtype=np.uint64)
        reqs["rand_key"] = keys
        seed = 0xC0FFEE
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        d_keys = torch.from_numpy(keys.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.empty(R * N.LIG_MAX_FALLBACKS, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        eng.upload_snapshot(1, snap.packed)
        eng.upload_pod_keys(1, np.array([S.pod_key(p) for p in snap.packed.pods], dtype=np.uint64))
        eng.upload_models(1, pack_models(WL.make_models(A), snap.packed))
        o, rw = d_out.data_ptr(), d_rows.data_ptr()
        dr, di, dk = d_reqs.data_ptr(), d_ids.data_ptr(), d_keys.data_ptr()
        group({"shape": "C4", "form": "descriptors", "R": R}, {
            "affinity_n0": lambda: eng.schedule_batch_affinity_device(1, dr, R, o, 0, 0, st),
            "affinity_n8": lambda: eng.schedule_batch_affinity_device(1, dr, R, o, 8, rw, st),
            "fallbacks_n8": lambda: eng.schedule_batch_fallbacks_device(1, seed, dr, R, o, 8, rw, st),
            "schedule": lambda: eng.schedule_batch_device(1, seed, dr, R, o, st)}, args.iters, args.rounds)
        group({"shape": "C4", "form": "model_ids", "R": R}, {
            "affinity_n0": lambda: eng.schedule_models_batch_affinity_device(1, di, dk, R, o, 0, 0, st),
            "affinity_n8": lambda: eng.schedule_models_batch_affinity_device(1, di, dk, R, o, 8, rw, st),
            "fallbacks_n8": lambda: eng.schedule_models_batch_fallbacks_device(1, seed, 0, di, R, o, 8, rw, st),
            "schedule": lambda: eng.schedule_models_batches_device(1, seed, 0, [di], R, [o], st)},
            args.iters, args.rounds)
        # host-buffer forms: page-locked buffers read and written in place, the call blocks
        h_reqs, h_ids, h_keys = pinned(lib, 16 * 4096), pinned(lib, 4 * 4096), pinned(lib, 8 * 4096)
        h_out, h_rows = pinned(lib, 8 * 4096), pinned(lib, 2 * 8 * 4096)
        ptrs += [h_reqs, h_ids, h_keys, h_out, h_rows]
        import ctypes as C
        C.memmove(h_reqs, reqs[:4096].ctypes.data, 16 * 4096)
        C.memmove(h_ids, ids[:4096].ctypes.data, 4 * 4096)
        C.memmove(h_keys, keys[:4096].ctypes.data, 8 * 4096)
        for r in (1, 64, 4096):
            group({"shape": "C4", "form": "host_buffers", "R": r}, {
                "affinity_n8": lambda: eng.schedule_batch_affinity_ptr(1, h_reqs, r, h_out, 8, h_rows),
                "fallbacks_n8": lambda: eng.schedule_batch_fallbacks_ptr(1, seed, h_reqs, r, h_out, 8, h_rows),
                "models_affinity_n8": lambda: eng.schedule_models_batch_affinity_ptr(1, h_ids, h_keys, r, h_out, 8,
                                                                                     h_rows),
                "models_fallbacks_n8": lambda: eng.schedule_models_batch_fallbacks_ptr(1, seed, 0, h_ids, r, h_out,
                                                                                       8, h_rows)},
                max(1, args.iters // 2), args.rounds)
    finally:
        for p in ptrs:
            lib.lig_host_free(p)
        eng.close()
    # long lists: every request's survivor list is all P = 32768 pods
    P, R = 32768, 4096
    eng = Engine(0, max_pods=P, max_adapters=1, max_batch=R)
    try:
        eng.set_filter_tree(KEEP_ALL)
        eng.upload_snapshot(1, pack_columns(np.full(P, 0.1), np.zeros(P, np.int64), np.zeros(P, np.int64),
                                            np.zeros(P, np.int64), np.zeros((1, P // 32), np.uint32)))
        eng.set_filter_tree(None)
        eng.upload_pod_keys(1, np.arange(P, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        reqs = np.zeros(R, dtype=WL.make_requests(1, 1).dtype)
        reqs["rand_key"] = np.random.default_rng(2).integers(0, 1 << 64, size=R, dtype=np.uint64)
        d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).cuda()
        d_out = torch.empty(R * 8, dtype=torch.uint8, device="cuda")
        d_rows = torch.empty(R * N.LIG_MAX_FALLBACKS, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        dr, o, rw = d_reqs.data_ptr(), d_out.data_ptr(), d_rows.data_ptr()
        group({"shape": "P32768_keep_all", "form": "descriptors", "R": R}, {
            "affinity_n0": lambda: eng.schedule_batch_affinity_device(1, dr, R, o, 0, 0, st),
            "affinity_n8": lambda: eng.schedule_batch_affinity_device(1, dr, R, o, 8, rw, st),
            "fallbacks_n8": lambda: eng.schedule_batch_fallbacks_device(1, 7, dr, R, o, 8, rw, st)},
            args.iters, args.rounds)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
