"""Round-trip latency of the doorbell stream (include/lig.h, lig_stream_submit and
lig_stream_submit_models) on one GPU.  Prints the card and its power limit first, then JSON lines:

* round_trip: at C4 (P = 4096, A = 1024, WL.make_models), micro-batches of 1, 16, 256 and 4096
  requests; descriptor submits and model-id submits alternate one by one.  Median and p99 wall time
  per submit over --reps submits of each kind, timed on the host around the blocking call (the
  call returns when the picks are back in host memory).
* descriptors_ab (with --baseline-lib PATH): the descriptor round trip of this build and of another
  build of liblig.so (e.g. the parent commit's), each in a fresh process, the two alternated over
  --rounds rounds.  Per build and size: the median of every round, so the run-to-run spread shows.

The library is driven through ctypes directly (descriptor submits only need entry points every ABI
version has), so --baseline-lib may be an older build.

Usage: python bench_doorbell_models.py [--reps 400] [--baseline-lib PATH --rounds 6]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from llm_instance_gateway_b200 import _native as N  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, _ptr, pack_models  # noqa: E402

SIZES = (1, 16, 256, 4096)
WARMUP = 50


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable ({e})"
    return out


def stats_us(ts):
    a = np.array(ts) * 1e6
    return {"p50_us": round(float(np.median(a)), 2), "p99_us": round(float(np.percentile(a, 99)), 2), "n": len(a)}


def open_stream(lib_path, with_models):
    """(lib, ctx) with the C4 snapshot (and model table) of epoch 1 resident and the stream open."""
    lib = C.CDLL(lib_path)
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    lib.lig_create.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    lib.lig_upload_snapshot.argtypes = [vp, u64, i32, i32, vp, vp, vp, vp, vp]
    lib.lig_stream_open.argtypes = [vp]
    lib.lig_stream_close.argtypes = [vp]
    lib.lig_stream_submit.argtypes = [vp, u64, u64, vp, i32, vp]
    lib.lig_destroy.argtypes = [vp]
    lib.lig_destroy.restype = None
    lib.lig_last_error.restype = C.c_char_p

    def check(rc):
        if rc != 0:
            raise RuntimeError(f"lig error {rc}: {lib.lig_last_error().decode()}")

    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"]).packed
    ctx = C.c_void_p()
    check(lib.lig_create(C.byref(ctx), 0, c["P"], c["A"], max(SIZES)))
    check(lib.lig_upload_snapshot(ctx, 1, snap.P, snap.A, _ptr(snap.kv), _ptr(snap.q), _ptr(snap.n_active),
                                  _ptr(snap.max_active), _ptr(snap.bitmap)))
    if with_models:
        pm = pack_models(WL.make_models(c["A"]), snap)
        lib.lig_upload_models.argtypes = [vp, u64, i32, vp, vp, vp, vp, vp, vp]
        lib.lig_stream_submit_models.argtypes = [vp, u64, u64, u64, vp, i32, vp]
        check(lib.lig_upload_models(ctx, 1, pm.n_models, _ptr(pm.target_offsets), _ptr(pm.target_adapter_ids),
                                    _ptr(pm.target_weights), _ptr(pm.critical), _ptr(pm.self_adapter_ids),
                                    _ptr(pm.present)))
    check(lib.lig_stream_open(ctx))
    return lib, ctx, check


def close_stream(lib, ctx):
    lib.lig_stream_close(ctx)
    lib.lig_destroy(ctx)


def time_round_trips(lib_path, reps, with_models):
    """{n: {"descriptors": stats, "models": stats}}; the two kinds alternate submit by submit."""
    lib, ctx, check = open_stream(lib_path, with_models)
    A = WL.CONFIGS["C4"]["A"]
    reqs = WL.make_requests(max(SIZES), A, seed=7)
    ids = WL.make_model_requests(max(SIZES), A, seed=8)
    picks = np.empty(max(SIZES), dtype=PICK_DTYPE)
    mpicks = np.empty(max(SIZES), dtype=MPICK_DTYPE)
    out = {}
    try:
        for n in SIZES:
            r = np.ascontiguousarray(reqs[:n])
            m = np.ascontiguousarray(ids[:n])
            td, tm = [], []
            for k in range(WARMUP + reps):
                t0 = time.perf_counter()
                check(lib.lig_stream_submit(ctx, 1, k, _ptr(r), n, _ptr(picks)))
                t1 = time.perf_counter()
                if with_models:
                    check(lib.lig_stream_submit_models(ctx, 1, k, 0, _ptr(m), n, _ptr(mpicks)))
                t2 = time.perf_counter()
                if k >= WARMUP:
                    td.append(t1 - t0)
                    tm.append(t2 - t1)
            out[n] = {"descriptors": stats_us(td)}
            if with_models:
                out[n]["models"] = stats_us(tm)
    finally:
        close_stream(lib, ctx)
    return out


def child(lib_path, reps):
    res = time_round_trips(lib_path, reps, with_models=False)
    print(json.dumps({str(n): v["descriptors"]["p50_us"] for n, v in res.items()}))


def descriptors_ab(baseline, reps, rounds):
    libs = {"this": N.LIB_PATH, "baseline": os.path.abspath(baseline)}
    med = {k: {str(n): [] for n in SIZES} for k in libs}
    for r in range(rounds):
        order = ["this", "baseline"] if r % 2 == 0 else ["baseline", "this"]
        for k in order:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", libs[k], "--reps", str(reps)],
                                 capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
            for n, v in json.loads(out).items():
                med[k][n].append(v)
    return {"part": "descriptors_ab", "rounds": rounds, "reps": reps, "p50_us_per_round": med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=400)
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.reps)
        return
    N.load()                       # this build must be complete (no fallback)
    print(json.dumps({"card": card()}), flush=True)
    res = time_round_trips(N.LIB_PATH, a.reps, with_models=True)
    print(json.dumps({"part": "round_trip", "config": "C4", "reps": a.reps,
                      "results": {str(n): v for n, v in res.items()}}), flush=True)
    if a.baseline_lib:
        print(json.dumps(descriptors_ab(a.baseline_lib, a.reps, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
