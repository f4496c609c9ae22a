"""The persistent kernels (pick and model-request) hand out tiles from claim counters, one per
launch in flight, taken from a ring of 16 in the ctx.  A launch that reuses a counter must wait, on
the device, for the counter's previous launch even when that one is still pending on another
stream: the counter's base on the host already counts the earlier launch's claims."""
import numpy as np
import pytest

from llm_instance_gateway_b200 import workload as WL
from llm_instance_gateway_b200.engine import Engine
from llm_instance_gateway_b200.packer import MPICK_DTYPE, PICK_DTYPE, pack_models

pytestmark = pytest.mark.gpu

CLAIM_SLOTS = 16          # lig_ctx::kClaimSlots


def test_more_persistent_launches_in_flight_than_claim_counters():
    import torch
    c = WL.CONFIGS["C3"]
    snap = WL.make_snapshot(c["P"], c["A"], seed=61)
    R, nb = 150_000, 2
    host = [WL.make_requests(R, c["A"], seed=62 + b) for b in range(nb)]
    mhost = [WL.make_model_requests(R, c["A"], seed=64 + b) for b in range(nb)]
    e = Engine(0, max_pods=c["P"], max_adapters=c["A"], max_batch=R)
    try:
        e.upload_snapshot(1, snap.packed)
        e.upload_models(1, pack_models(WL.make_models(c["A"]), snap.packed))
        d_reqs = [torch.from_numpy(h.view(np.uint8).reshape(-1)).cuda() for h in host]
        d_ids = [torch.from_numpy(h.view(np.uint8)).cuda() for h in mhost]
        # Three laps of the counter ring.  Lap 0 queues on one stream held by a spin kernel; laps 1
        # and 2 go to 16 other streams, one launch each per lap, so launch CLAIM_SLOTS + k shares a
        # counter with launch k while launch k is still pending, and nothing else orders the two.
        held = torch.cuda.Stream()
        others = [torch.cuda.Stream() for _ in range(CLAIM_SLOTS)]
        plan, outs = [], []
        for i in range(3 * CLAIM_SLOTS):
            models = i % 3 == 2
            Rq = 1000 if i % 4 == 3 else R            # two tiles on two CTAs: a claim-ahead leaves one idle
            st = held if i < CLAIM_SLOTS else others[i % CLAIM_SLOTS]
            outs.append([torch.zeros(Rq * (4 if models else 8), dtype=torch.uint8, device="cuda") for _ in range(nb)])
            plan.append((models, Rq, 100 * i, st))
        torch.cuda.synchronize()                      # the fills / copies ran on torch's default stream
        with torch.cuda.stream(held):
            torch.cuda._sleep(100_000_000)            # ~50 ms: every launch below is enqueued meanwhile
        for i, (models, Rq, seed, st) in enumerate(plan):
            if models:
                e.schedule_models_batches_device(1, seed, 7, [t.data_ptr() for t in d_ids], Rq,
                                                 [t.data_ptr() for t in outs[i]], st.cuda_stream)
            else:
                e.schedule_batches_device(1, seed, [t.data_ptr() for t in d_reqs], Rq,
                                          [t.data_ptr() for t in outs[i]], st.cuda_stream)
        assert not held.query()                       # lap 0 was still pending when lap 1 was enqueued
        torch.cuda.synchronize()
        for i, (models, Rq, seed, _) in enumerate(plan):
            for b in range(nb):
                if models:
                    got = outs[i][b].cpu().numpy().view(MPICK_DTYPE)
                    want = e.schedule_models_batch(1, seed + b, np.ascontiguousarray(mhost[b][:Rq]), first_index=7)
                else:
                    got = outs[i][b].cpu().numpy().view(PICK_DTYPE)
                    want = e.schedule_batch(1, seed + b, np.ascontiguousarray(host[b][:Rq]))
                assert np.array_equal(got, want), (i, models, Rq, b)
    finally:
        e.close()
