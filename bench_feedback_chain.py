"""Cost and effect of the load-feedback chain (include/lig.h, lig_schedule_batch_feedback_chain) on
one GPU, in one process.  Prints the card and its power limit first, then one JSON line per part:

* latency: host-buffer calls at C4 (P = 4096, A = 1024) with page-locked buffers, for micro-batches
  of 1, 16, 256 and 4096 requests: lig_schedule_batch, chain calls that close no window (W = 2^30)
  and chain calls that close one window each (W = the micro-batch: a pick, a window apply and one
  class build per call).  Median and p99 wall time per call over --reps calls;
* models: the same for model-id requests at C4 with WL.make_models: lig_schedule_models_batch and
  lig_schedule_models_batch_feedback_chain with no window closing and with one window per call;
* herd: 5000 C4-distributed requests in micro-batches of 8 against one epoch: the most picks one
  pod received and the number of pods used, without feedback and with W in {1, 8, 64, 512};
* stream: the C5 stream (100 K req/s Poisson) through the C++ runtime, p50 / p99 service latency
  without feedback and with one window.

Usage: python bench_feedback_chain.py [--reps 400] [--seconds 2] [--stream-window 64]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import time

import numpy as np
import torch

from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import host as H
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable ({e})"
    return out or torch.cuda.get_device_name(0)


def pinned(lib, n, dtype):
    dtype = np.dtype(dtype)
    nbytes = max(n, 1) * dtype.itemsize
    ptr = lib.lig_host_alloc(nbytes)
    return ptr, np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr)).view(dtype)[:n]


def stats_us(ts):
    a = np.array(ts) * 1e6
    return {"p50_us": round(float(np.median(a)), 2), "p99_us": round(float(np.percentile(a, 99)), 2)}


def latency(reps):
    lib = N.load()
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    out = {}
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=4096) as e:
        e.upload_snapshot(1, snap.packed)
        for m in (1, 16, 256, 4096):
            rp, ra = pinned(lib, m, REQ_DTYPE)
            op, _ = pinned(lib, m, PICK_DTYPE)
            ra[:] = WL.make_requests(m, c["A"], seed=m)
            row = {}
            for name, call in (
                    ("schedule_batch", lambda s: e.schedule_batch_ptr(1, s, rp, m, op)),
                    ("chain_no_window", lambda s: e.schedule_batch_feedback_chain_ptr(1, s, rp, m, op, 1 << 30)),
                    ("chain_one_window", lambda s: e.schedule_batch_feedback_chain_ptr(1, s, rp, m, op, m))):
                e.feedback_chain_reset()
                for s in range(20):                          # warm-up
                    call(s)
                ts = []
                for s in range(reps):
                    t0 = time.perf_counter()
                    call(s)
                    ts.append(time.perf_counter() - t0)
                row[name] = stats_us(ts)
            out[f"R={m}"] = row
            lib.lig_host_free(rp)
            lib.lig_host_free(op)
    return {"part": "latency", "config": "C4 host-buffer calls, page-locked buffers", **out}


def models(reps):
    lib = N.load()
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    out = {}
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=4096) as e:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, pack_models(WL.make_models(c["A"]), snap.packed))
        for m in (1, 16, 256, 4096):
            ip, ia = pinned(lib, m, np.uint32)
            op, _ = pinned(lib, m, MPICK_DTYPE)
            ia[:] = WL.make_model_requests(m, c["A"], seed=m)
            row = {}
            for name, call in (
                    ("schedule_models_batch", lambda s: e.schedule_models_batch_ptr(1, s, s * m, ip, m, op)),
                    ("chain_no_window",
                     lambda s: e.schedule_models_batch_feedback_chain_ptr(1, s, s * m, ip, m, op, 1 << 30)),
                    ("chain_one_window",
                     lambda s: e.schedule_models_batch_feedback_chain_ptr(1, s, s * m, ip, m, op, m))):
                e.feedback_chain_reset()
                for s in range(20):                          # warm-up
                    call(s)
                ts = []
                for s in range(reps):
                    t0 = time.perf_counter()
                    call(s)
                    ts.append(time.perf_counter() - t0)
                row[name] = stats_us(ts)
            out[f"R={m}"] = row
            lib.lig_host_free(ip)
            lib.lig_host_free(op)
    return {"part": "models", "config": "C4 model-id host-buffer calls, page-locked buffers", **out}


def herd():
    c = WL.CONFIGS["C4"]
    snap = WL.make_snapshot(c["P"], c["A"])
    reqs = WL.make_requests(5000, c["A"], seed=7)
    out = {}
    with Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=4096) as e:
        e.upload_snapshot(1, snap.packed)
        for W in (0, 1, 8, 64, 512):
            e.feedback_chain_reset()
            picks = []
            for lo in range(0, len(reqs), 8):
                b = np.ascontiguousarray(reqs[lo:lo + 8])
                picks.append(e.schedule_batch(1, 11, b) if W == 0 else e.schedule_batch_feedback_chain(1, 11, b, W))
            pods = np.concatenate(picks)["pod_idx"]
            n = np.bincount(pods[pods >= 0], minlength=c["P"])
            out["off" if W == 0 else f"W={W}"] = {"max_picks_one_pod": int(n.max()), "pods_used": int((n > 0).sum()),
                                                  "picked": int(n.sum())}
    return {"part": "herd", "config": "5000 C4 requests in micro-batches of 8, one epoch", **out}


def stream(seconds, window):
    c = WL.CONFIGS["C5"]
    snap = WL.make_snapshot(c["P"], c["A"])
    p = snap.packed
    pods = [PodMetrics(Pod(f"pod-{i}", f"address-{i}"),
                       Metrics(WaitingQueueSize=int(snap.q64[i]), KVCacheUsagePercent=float(p.kv[i]),
                               MaxActiveModels=int(snap.max_active64[i]),
                               ActiveModels={WL.adapter_name(a): 1 for a in snap.active[i]}))
            for i in range(p.P)]
    models = [WL.adapter_name(a) for a in range(c["A"])] + [WL.UNKNOWN_MODEL]
    models = models + models
    critical = [False] * (c["A"] + 1) + [True] * (c["A"] + 1)
    threads = max(2, min(16, (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 4) // 2))
    out = {}
    for W in (0, window):
        prov = H.HostProvider(pods)
        sched = H.HostScheduler(prov, max_pods=c["P"], max_adapters=c["A"], max_batch=1 << 14, flush_size=4096,
                                batch_window_us=20, refresh_interval_ms=50, busy_poll=True, caller_spin_us=100,
                                load_feedback_window=W)
        try:
            sched.stream_bench(100_000, seconds, threads, models, critical, seed=5)
            svc = sched.last_service_latency_us
            st = sched.stats()
        finally:
            sched.close()
            prov.close()
        out["off" if W == 0 else f"W={W}"] = {
            "service_p50_us": round(float(np.percentile(svc, 50)), 2),
            "service_p99_us": round(float(np.percentile(svc, 99)), 2), "requests": int(len(svc)),
            "flushes": st["batches"], "feedback_windows": st["feedback_windows"],
            "feedback_restarts": st["feedback_restarts"]}
    return {"part": "stream", "config": f"C5 100K req/s Poisson for {seconds} s, {threads} caller threads", **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=400)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--stream-window", type=int, default=64)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps(latency(a.reps)), flush=True)
    print(json.dumps(models(a.reps)), flush=True)
    print(json.dumps(herd()), flush=True)
    print(json.dumps(stream(a.seconds, a.stream_window)), flush=True)


if __name__ == "__main__":
    main()
