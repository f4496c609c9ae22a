"""Model requests through the C++ runtime (lig::scheduling::Scheduler) on one GPU: the resolve step
on the caller's thread (ScheduleModel(datastore, ...): FetchModelData + RandomWeightedDraw on the
host, then a descriptor through the batcher) against the resolve step on the device
(ScheduleModel(model, ...): the name goes through the batcher and lig_schedule_models_batch,
lig_stream_submit_models or lig_schedule_models_batch_feedback_chain resolves and picks).

C4 pool (P = 4096, A = 1024) with WL.make_models and the model mix of WL.make_model_requests.
Prints the card and its power limit first, then JSON lines:
* one_caller: one calling thread, per flush path (plain launch, doorbell, load_feedback_window = 64):
  median and p99 wall time per call of each form over --calls calls (the forms alternate in blocks).
* threads: 8 and 16 calling threads: calls per second of each form, --per-thread calls each.

Usage: python bench_scheduler_models.py [--calls 3000] [--per-thread 2000]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from llm_instance_gateway_b200 import host as H  # noqa: E402
from llm_instance_gateway_b200 import workload as WL  # noqa: E402
from llm_instance_gateway_b200.backend import Metrics, Pod, PodMetrics  # noqa: E402

P, A = WL.CONFIGS["C4"]["P"], WL.CONFIGS["C4"]["A"]
PATHS = {"launch": {}, "doorbell": {"use_doorbell": True}, "feedback_w64": {"load_feedback_window": 64}}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def pod_metrics():
    snap = WL.make_snapshot(P, A, seed=WL.SNAPSHOT_SEED)
    p = snap.packed
    return [PodMetrics(Pod(f"pod-{i}", f"address-{i}"),
                       Metrics(WaitingQueueSize=int(snap.q64[i]), KVCacheUsagePercent=float(p.kv[i]),
                               MaxActiveModels=int(snap.max_active64[i]),
                               ActiveModels={WL.adapter_name(a): 1 for a in snap.active[i]}))
            for i in range(P)]


def request_names(models, n, seed):
    names = [m.Spec.ModelName for m in models]
    return [names[i] if i < len(names) else "no-such-model" for i in WL.make_model_requests(n, A, seed=seed)]


def us(ts):
    a = np.asarray(ts) * 1e6
    return {"median_us": round(float(np.median(a)), 2), "p99_us": round(float(np.percentile(a, 99)), 2)}


def one_caller(s, ds, names, block=250):
    """Per-call wall times of both forms, alternating in blocks so both see the same machine state."""
    host, dev = [], []
    for lo in range(0, len(names), block):
        part = names[lo:lo + block]
        for form, sink in (("host", host), ("device", dev)):
            for n in part:
                t0 = time.perf_counter()
                if form == "host":
                    s.ScheduleModel(ds, n)
                else:
                    s.ScheduleModelOnDevice(n)
                sink.append(time.perf_counter() - t0)
    return host, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3000)
    ap.add_argument("--per-thread", type=int, default=2000)
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    models = WL.make_models(A)
    prov = H.HostProvider(pod_metrics())
    ds = H.HostDataStore(models)
    names = request_names(models, args.calls, seed=7)
    warm = request_names(models, 200, seed=8)
    try:
        for path, kw in PATHS.items():
            s = H.HostScheduler(prov, max_pods=P, max_adapters=A, max_batch=1 << 14, seed=11, batch_window_us=20,
                                **kw)
            try:
                s.set_inference_models(ds)
                one_caller(s, ds, warm)
                host, dev = one_caller(s, ds, names)
                print(json.dumps({"bench": "one_caller", "path": path, "calls": len(names),
                                  "datastore_form": us(host), "device_form": us(dev)}), flush=True)
                if path != "launch":
                    continue
                for threads in (8, 16):
                    row = {"bench": "threads", "path": path, "threads": threads, "calls": threads * args.per_thread}
                    st0 = s.stats()
                    for form, d in (("datastore_form", ds), ("device_form", None)):
                        s.schedule_models_concurrent(threads, 100, names, datastore=d)       # warm-up
                        t0 = time.perf_counter()
                        codes, _, _ = s.schedule_models_concurrent(threads, args.per_thread, names, datastore=d)
                        dt = time.perf_counter() - t0
                        row[form] = {"calls_per_s": round(len(codes) / dt), "ok": int((codes == 0).sum())}
                    st = s.stats()
                    row["device_form_mean_batch"] = round((st["model_scheduled"] - st0["model_scheduled"]) /
                                                          max(st["model_batches"] - st0["model_batches"], 1), 1)
                    print(json.dumps(row), flush=True)
            finally:
                s.close()
    finally:
        ds.close()
        prov.close()


if __name__ == "__main__":
    main()
