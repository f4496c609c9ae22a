"""Cost of caller filter trees on one GPU, in one process: the class-table build with the built-in
tree, with DEFAULT_FILTER as a caller tree and with a 16-node caller tree, at C4 (P = 4096, A = 1024,
2050 classes) and at a large shape (P = 32768: pod columns read from global memory, A = 4096,
8194 classes), and the C4 queue of K = 20 batches of 2^20 requests against built-in and
caller-DEFAULT_FILTER tables (alternated).  Prints the card and its power limit first; CUDA-event
medians over --reps repetitions.  Usage: python bench_filter_tree.py [--reps 50]"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys

import numpy as np
import torch

from llm_instance_gateway_b200 import _native as N
from llm_instance_gateway_b200 import scheduling as S
from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine


def node(kind, s=-1, f=-1, sf=-1, q=0, kv=0.0):
    return N.LigFilterNode(kind, s, f, sf, q, kv)


# 16 nodes, every kind, shared subtrees and both successor styles
TREE16 = [
    node(N.LIG_F_CRITICAL_REQUEST, 1, 8),
    node(N.LIG_F_LOW_QUEUEING, 2, 5, q=50),
    node(N.LIG_F_LORA_AFFINITY, 4, 3),
    node(N.LIG_F_CAN_ACCEPT_NEW_LORA, sf=4),
    node(N.LIG_F_LEAST_QUEUING, sf=7),
    node(N.LIG_F_LEAST_QUEUING, sf=6),
    node(N.LIG_F_LOW_LORA_COST, sf=7),
    node(N.LIG_F_LEAST_KV_CACHE, sf=14),
    node(N.LIG_F_NO_QUEUE_AND_LOW_KV, 10, 9, q=5, kv=0.8),
    node(N.LIG_F_NO_QUEUE_AND_LOW_KV, 13, 15, q=20, kv=0.9),
    node(N.LIG_F_LORA_AFFINITY, 12, 11),
    node(N.LIG_F_LOW_LORA_COST, sf=12),
    node(N.LIG_F_LEAST_KV_CACHE, sf=13),
    node(N.LIG_F_LEAST_QUEUING),
    node(N.LIG_F_LEAST_QUEUING),
    node(N.LIG_F_DROP),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable ({e})"
    return out or torch.cuda.get_device_name(0)


def time_builds(eng, d_blob, P, A, reps, stream, ep0):
    """Median ms of lig_upload_snapshot_device (blob copy in HBM + class build) on `stream`."""
    ts = []
    for i in range(reps + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        eng.upload_snapshot_device(ep0 + i, P, A, d_blob, stream.cuda_stream)
        b.record(stream)
        b.synchronize()
        if i >= 3:
            ts.append(a.elapsed_time(b))
    return float(np.median(ts)), ep0 + reps + 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    c = WL.CONFIGS["C4"]
    P, A, R, K = c["P"], c["A"], c["R"], 20
    snap = WL.make_snapshot(P, A)
    stream = torch.cuda.Stream()
    res = {"card": card()}
    for tag, (bP, bA) in (("C4", (P, A)), ("P32768_A4096", (32768, 4096))):
        bsnap = snap if tag == "C4" else WL.make_snapshot(bP, bA, seed=3)
        b_blob = torch.from_numpy(bsnap.packed.blob()).cuda()
        torch.cuda.synchronize()
        eng = Engine(0, max_pods=bP, max_adapters=bA, max_batch=1 << 16)
        ep = 1
        for name, tree in (("builtin", None), ("caller_default_filter", S.DEFAULT_FILTER), ("caller_16_nodes", TREE16)):
            eng.set_filter_tree(tree)
            res[f"build_ms_{tag}_{name}"], ep = time_builds(eng, b_blob.data_ptr(), bP, bA, args.reps, stream, ep)
        eng.close()
        del b_blob
    # K = 20 queue against the two tables, alternated
    builtin = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 16)
    caller = Engine(0, max_pods=P, max_adapters=A, max_batch=1 << 16)
    caller.set_filter_tree(S.DEFAULT_FILTER)
    reqs = WL.make_requests(R, A)
    d_reqs = torch.from_numpy(reqs.view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    d_out = [torch.empty(R * 8, dtype=torch.uint8, device="cuda") for _ in range(K)]
    ptrs_in, ptrs_out = [d_reqs.data_ptr()] * K, [t.data_ptr() for t in d_out]
    for e in (builtin, caller):
        e.upload_snapshot(1, snap.packed)
    same = True
    ts = {"builtin": [], "caller_default_filter": []}
    for i in range(args.reps + 2):
        for name, e in (("builtin", builtin), ("caller_default_filter", caller)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            e.schedule_batches_device(1, 42, ptrs_in, R, ptrs_out, stream.cuda_stream)
            b.record(stream)
            b.synchronize()
            if i >= 2:
                ts[name].append(a.elapsed_time(b))
            if i == 0 and e is builtin:
                want = [t.clone() for t in d_out]
            elif i == 0:
                same = all(torch.equal(x, y) for x, y in zip(want, d_out))
    for name, v in ts.items():
        res[f"queue_K20_ms_{name}"] = float(np.median(v))
        res[f"queue_K20_decisions_per_s_{name}"] = K * R / (float(np.median(v)) * 1e-3)
    res["queue_picks_identical"] = bool(same)
    res["pick_kernel_caller"] = caller.pick_kernel_info(1)
    builtin.close()
    caller.close()
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
