"""Model-id retries on one GPU: each lig_schedule_models_batch[_feedback_chain]_excluding[_fallbacks] form
against its descriptor counterpart on the same requests, at C4 (P = 4096, A = 1024) with the built-in
tree and 9 excluded pods per request (the first call's pick and its 8 fallbacks).  The model retry takes
the targets the first model call drew; the descriptor retry takes the descriptors those targets resolve to
(built here on the host from the packed model table), so both walk the same pools.

1. Device forms at R = 2^20: CUDA events over --iters back-to-back calls, the model form and its
   descriptor counterpart alternating over --rounds rounds.  The chain forms use a window no call fills.
   The picks of each pair must agree (pod and status) on every request that resolves.
2. Blocking host calls with page-locked buffers at R = 1, 16, 256, 4096, alternating call by call with the
   descriptor counterpart.  Median and p99 wall time over --calls calls each.

Prints the card and its power limit first, then one JSON line per measurement.

Usage: python bench_models_retry.py [--calls 400] [--iters 5] [--rounds 7]"""
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
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, REQ_DTYPE, pack_models  # noqa: E402

NO_CLOSE = 1 << 30
N_FB = 8
FORMS = ("resident", "resident_rows", "chain", "chain_rows")


def descriptors(pm, ids, targets, first_index=0):
    """The descriptors the fixed targets resolve to (absent models and bad targets: adapter A, which
    is a miss, as LIG_NO_MODEL requests are not walked by the model form)."""
    R = len(ids)
    reqs = np.zeros(R, dtype=REQ_DTYPE)
    reqs["rand_key"] = (np.uint64(first_index) + np.arange(R, dtype=np.uint64))
    m = np.minimum(ids, pm.n_models - 1).astype(np.int64)
    nt = (pm.target_offsets[m + 1] - pm.target_offsets[m]).astype(np.int64)
    t = targets.astype(np.int64)
    ok = (ids < pm.n_models) & (pm.present[m] == 1) & np.where(nt == 0, t == 255, t < nt)
    tgt = pm.target_adapter_ids[np.clip(pm.target_offsets[m] + np.where(t == 255, 0, t), 0,
                                        max(len(pm.target_adapter_ids) - 1, 0))] if len(pm.target_adapter_ids) else 0
    reqs["adapter_id"] = np.where(ok, np.where(t == 255, pm.self_adapter_ids[m], tgt), 1 << 20)
    reqs["flags"] = np.where(ok, pm.critical[m], 0)
    return reqs, ok


def device_pairs(eng, ep, seed, d, R, k):
    """(model call, descriptor call) per form on the device buffers in d."""
    p = {n: t.data_ptr() for n, t in d.items()}
    st = torch.cuda.current_stream().cuda_stream
    return {
        "resident": (lambda: eng.schedule_models_batch_excluding_device(ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k,
                                                                        p["mout"], st),
                     lambda: eng.schedule_batch_excluding_device(ep, seed, p["reqs"], R, p["rows"], k, p["out"], st)),
        "resident_rows": (lambda: eng.schedule_models_batch_excluding_fallbacks_device(
                              ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], N_FB, p["mfb"], st),
                          lambda: eng.schedule_batch_excluding_fallbacks_device(ep, seed, p["reqs"], R, p["rows"], k,
                                                                                p["out"], N_FB, p["fb"], st)),
        "chain": (lambda: eng.schedule_models_batch_feedback_chain_excluding_device(
                      ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], NO_CLOSE, 0, st),
                  lambda: eng.schedule_batch_feedback_chain_excluding_device(ep, seed, p["reqs"], R, p["rows"], k,
                                                                             p["out"], NO_CLOSE, 0, st)),
        "chain_rows": (lambda: eng.schedule_models_batch_feedback_chain_excluding_fallbacks_device(
                           ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], N_FB, p["mfb"], NO_CLOSE, 0, st),
                       lambda: eng.schedule_batch_feedback_chain_excluding_fallbacks_device(
                           ep, seed, p["reqs"], R, p["rows"], k, p["out"], N_FB, p["fb"], NO_CLOSE, 0, st)),
    }


def agree(d, ok, R):
    m = d["mout"].cpu().numpy().view(MPICK_DTYPE)[:R]
    x = d["out"].cpu().numpy().view(PICK_DTYPE)[:R]
    return bool(np.array_equal(m["pod_idx"][ok], x["pod_idx"][ok]) and np.array_equal(m["status"][ok], x["status"][ok]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    c = WL.CONFIGS["C4"]
    P, A, R_dev = c["P"], c["A"], 1 << 20
    snap = WL.make_snapshot(P, A)
    pm = pack_models(WL.make_models(A), snap.packed)
    lib = N.load()
    eng = Engine(0, max_pods=P, max_adapters=A, max_batch=4096)
    try:
        ep, seed = 1, 0xC0FFEE
        eng.upload_snapshot(ep, snap.packed)
        eng.upload_models(ep, pm)
        ids = WL.make_model_requests(R_dev, A)
        d_ids = torch.from_numpy(ids.view(np.uint8).copy()).cuda()
        d_first = torch.empty(R_dev * 4, dtype=torch.uint8, device="cuda")
        eng.schedule_models_batches_device(ep, seed, 0, [d_ids.data_ptr()], R_dev, [d_first.data_ptr()], 0)
        torch.cuda.synchronize()
        first = d_first.cpu().numpy().view(MPICK_DTYPE)
        targets = np.ascontiguousarray(first["target_idx"])
        picks, fb = eng.schedule_models_batch_fallbacks(ep, seed, ids[:4096], N_FB)
        rows9 = np.concatenate([np.where(picks["status"] == N.LIG_OK, picks["pod_idx"], -1)[:, None].astype(np.int16),
                                fb], axis=1)
        rows9 = np.ascontiguousarray(np.tile(rows9, (R_dev // 4096, 1)))
        k = rows9.shape[1]
        reqs, ok = descriptors(pm, ids, targets)
        d = {"ids": d_ids, "tg": torch.from_numpy(targets.copy()).cuda(),
             "reqs": torch.from_numpy(reqs.view(np.uint8).copy()).cuda(),
             "rows": torch.from_numpy(rows9.reshape(-1).copy()).cuda(),
             "mout": torch.empty(R_dev * 4, dtype=torch.uint8, device="cuda"),
             "out": torch.empty(R_dev * 8, dtype=torch.uint8, device="cuda"),
             "mfb": torch.empty(R_dev * N_FB, dtype=torch.int16, device="cuda"),
             "fb": torch.empty(R_dev * N_FB, dtype=torch.int16, device="cuda")}
        pairs = device_pairs(eng, ep, seed, d, R_dev, k)
        for form in FORMS:
            model, desc = pairs[form]
            eng.feedback_chain_reset()
            for _ in range(2):
                model()
                desc()
            torch.cuda.synchronize()
            same = agree(d, ok, R_dev)
            tm, td = [], []
            for r in range(args.rounds):
                for fn, acc in (((model, tm), (desc, td)) if r % 2 == 0 else ((desc, td), (model, tm))):
                    acc.append(timed(fn, args.iters))
            mm, md = float(np.median(tm)), float(np.median(td))
            print(json.dumps({"form": form, "where": "device", "R": R_dev, "excluded": int(k),
                              "n_fallbacks": N_FB if form.endswith("rows") else 0, "picks_agree": same,
                              "model_us": round(mm, 1), "descriptor_us": round(md, 1),
                              "model_us_min_max": [round(min(tm), 1), round(max(tm), 1)],
                              "descriptor_us_min_max": [round(min(td), 1), round(max(td), 1)],
                              "model_over_descriptor": round(mm / md, 3)}), flush=True)
        for R in (1, 16, 256, 4096):
            bufs = {"ids": Pinned(lib, np.ascontiguousarray(ids[:R])),
                    "tg": Pinned(lib, np.ascontiguousarray(targets[:R])),
                    "reqs": Pinned(lib, np.ascontiguousarray(reqs[:R])),
                    "rows": Pinned(lib, np.ascontiguousarray(rows9[:R])),
                    "mout": Pinned(lib, np.zeros(R, MPICK_DTYPE)), "out": Pinned(lib, np.zeros(R, PICK_DTYPE)),
                    "mfb": Pinned(lib, np.zeros((R, N_FB), np.int16)), "fb": Pinned(lib, np.zeros((R, N_FB), np.int16))}
            p = {n: b.ptr for n, b in bufs.items()}
            host = {
                "resident": (lambda: eng.schedule_models_batch_excluding_ptr(ep, seed, 0, p["ids"], p["tg"], R,
                                                                             p["rows"], k, p["mout"]),
                             lambda: eng.schedule_batch_excluding_ptr(ep, seed, p["reqs"], R, p["rows"], k, p["out"])),
                "resident_rows": (lambda: eng.schedule_models_batch_excluding_fallbacks_ptr(
                                      ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], N_FB, p["mfb"]),
                                  lambda: eng.schedule_batch_excluding_fallbacks_ptr(ep, seed, p["reqs"], R, p["rows"],
                                                                                     k, p["out"], N_FB, p["fb"])),
                "chain": (lambda: eng.schedule_models_batch_feedback_chain_excluding_ptr(
                              ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], NO_CLOSE),
                          lambda: eng.schedule_batch_feedback_chain_excluding_ptr(ep, seed, p["reqs"], R, p["rows"], k,
                                                                                  p["out"], NO_CLOSE)),
                "chain_rows": (lambda: eng.schedule_models_batch_feedback_chain_excluding_fallbacks_ptr(
                                   ep, seed, 0, p["ids"], p["tg"], R, p["rows"], k, p["mout"], N_FB, p["mfb"], NO_CLOSE),
                               lambda: eng.schedule_batch_feedback_chain_excluding_fallbacks_ptr(
                                   ep, seed, p["reqs"], R, p["rows"], k, p["out"], N_FB, p["fb"], NO_CLOSE)),
            }
            try:
                for form in FORMS:
                    model, desc = host[form]
                    eng.feedback_chain_reset()
                    for _ in range(20):
                        model()
                        desc()
                    tm, td = [], []
                    for i in range(args.calls):
                        for fn, acc in (((model, tm), (desc, td)) if i % 2 == 0 else ((desc, td), (model, tm))):
                            t0 = time.perf_counter()
                            fn()
                            acc.append((time.perf_counter() - t0) * 1e6)
                    print(json.dumps({"form": form, "where": "host_pinned", "R": R, "excluded": int(k),
                                      "model_us_median": round(float(np.median(tm)), 2),
                                      "model_us_p99": round(float(np.percentile(tm, 99)), 2),
                                      "descriptor_us_median": round(float(np.median(td)), 2),
                                      "descriptor_us_p99": round(float(np.percentile(td, 99)), 2)}), flush=True)
            finally:
                for b in bufs.values():
                    b.free()
        print(json.dumps({"P": P, "A": A}), flush=True)
    finally:
        eng.close()


if __name__ == "__main__":
    main()
