"""Host-side mirror of the reference's ``scheduling`` package interface, backed by the GPU.

Same names, argument meaning and error behaviour as the reference so that it drops in behind
``handlers.Scheduler`` (pkg/ext-proc/handlers/server.go:37-39):

    scheduler = NewScheduler(pod_metrics_provider)       # scheduling/scheduler.go:93-99
    pod = scheduler.Schedule(LLMRequest(...))            # scheduling/scheduler.go:113-122

``Schedule`` returns a ``backend.Pod`` or raises ``StatusError``; its ``.code`` is
``"ResourceExhausted"`` when the tree shed the request (scheduler.go:83-89), which the ext-proc
server turns into HTTP 429 (handlers/server.go:97-109).  ``NewScheduler(pmp, filter=...)`` runs a
caller-built flow chart of the reference's filter nodes (``Filter``, filter.go:17-73) instead of
``defaultFilter``; ``DEFAULT_FILTER`` restates defaultFilter node for node.  ``ScheduleBatch`` is the micro-batched
form the Go adapter uses under load (one C-ABI call per batch); ``NewScheduler(pmp, load_feedback_window=W)``
carries load feedback across those calls until the next refresh (off by default).  ``SetInferenceModels`` plus
``ScheduleModel`` / ``ScheduleModelBatch`` take the request's model name instead of a resolved request: the
resolve step of HandleRequestBody (handlers/request.go:42-56) runs on the device against a model table that
every snapshot epoch carries.  ``FilterBatch`` / ``FilterModelBatch`` return the survivor slices of a whole
batch (Filter.Filter, filter.go:12-15) in one device call, for any filter tree.  ``ScheduleBatchWithFallbacks`` /
``ScheduleWithFallbacks`` / ``ScheduleModelBatchWithFallbacks`` return the pick followed by up to n more distinct
survivors in retry order (include/lig.h, fallback endpoints); under load_feedback_window they need
``feedback_fallbacks=True`` and then rank the feedback chain's own tables.  ``ScheduleRetry`` / ``ScheduleBatchRetry``
schedule a request again without the pods it already tried, as Schedule would once those pods left the provider
(lig_schedule_batch_excluding); under load_feedback_window they need ``feedback_retries=True`` and then run as
feedback-chain calls.  ``ScheduleRetryWithFallbacks`` / ``ScheduleBatchRetryWithFallbacks`` return the retry's
pick followed by up to n more distinct survivors of the reduced pool (lig_schedule_batch_excluding_fallbacks), so
one call serves several attempts; under load_feedback_window they need both ``feedback_retries=True`` and
``feedback_fallbacks=True`` and then run as feedback-chain calls whose rows rank the chain's reduced pool.  ``NewScheduler(pmp, affinity=True)`` adds
``ScheduleAffinity`` and its relatives: requests that share a key go to the same surviving pod, by rendezvous hashing
over the survivors on the device (lig_schedule_batch_affinity); under load_feedback_window they need
``feedback_affinity=True`` and then rank the feedback chain's load-adjusted survivors.  There is
no CPU path here: without liblig.so or without a CUDA device construction fails.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Protocol, Sequence, Tuple

import numpy as np

from . import _native as N
from .backend import InferenceModel, Pod, PodMetrics
from .engine import Engine
from .packer import REQ_DTYPE, PackedModels, PackedSnapshot, pack_models, pack_pod_metrics


@dataclass
class LLMRequest:                            # scheduling/types.go:4-11
    Model: str = ""
    TargetModels: Dict[str, int] = field(default_factory=dict)
    ResolvedTargetModel: str = ""
    Critical: bool = False


class PodMetricsProvider(Protocol):          # scheduling/scheduler.go:108-110
    def AllPodMetrics(self) -> Sequence[PodMetrics]: ...


class StatusError(Exception):
    """A Go error carrying a gRPC status code (google.golang.org/grpc/status)."""

    def __init__(self, code: str, message: str):
        super().__init__(message)
        self.code = code


_DROP_DESC = "dropping request due to limited backend resources"          # scheduler.go:87
_ERR_PREFIX = "failed to apply filter, resulted 0 pods, this should never happen: "   # scheduler.go:117

# ---- caller filter trees (lig_set_filter_tree) --------------------------------------------------
# Node kinds: the filter functions of filter.go / scheduler.go.
CRITICAL_REQUEST = N.LIG_F_CRITICAL_REQUEST        # criticalRequestPredicate            filter.go:179-181
LOW_QUEUEING = N.LIG_F_LOW_QUEUEING                # q < queue_threshold                 filter.go:124-126
LORA_AFFINITY = N.LIG_F_LORA_AFFINITY              # loRAAffinityPredicate               filter.go:169-172
CAN_ACCEPT_NEW_LORA = N.LIG_F_CAN_ACCEPT_NEW_LORA  # canAcceptNewLoraPredicate           filter.go:175-177
LOW_LORA_COST = N.LIG_F_LOW_LORA_COST              # lowLoRACostPredicate                filter.go:163-166
NO_QUEUE_AND_LOW_KV = N.LIG_F_NO_QUEUE_AND_LOW_KV  # q <= queue_threshold && kv <= kv_threshold  filter.go:183-187
LEAST_QUEUING = N.LIG_F_LEAST_QUEUING              # leastQueuingFilterFunc              filter.go:102-122
LEAST_KV_CACHE = N.LIG_F_LEAST_KV_CACHE            # leastKVCacheFilterFunc              filter.go:134-154
DROP = N.LIG_F_DROP                                # the "drop request" func             scheduler.go:83-89


class Filter:
    """One node of a flow chart, as the reference's ``filter`` struct (filter.go:20-35).  Successors
    are other ``Filter`` objects (or None); a node may be the successor of several parents."""

    def __init__(self, name: str, kind: int, next_on_success: "Optional[Filter]" = None,
                 next_on_failure: "Optional[Filter]" = None,
                 next_on_success_or_failure: "Optional[Filter]" = None,
                 queue_threshold: int = 0, kv_threshold: float = 0.0):
        self.name, self.kind = name, kind
        self.next_on_success, self.next_on_failure = next_on_success, next_on_failure
        self.next_on_success_or_failure = next_on_success_or_failure
        self.queue_threshold, self.kv_threshold = queue_threshold, kv_threshold

    def Name(self) -> str:                                                    # filter.go:37-42
        return self.name

    def _successors(self):
        return (self.next_on_success, self.next_on_failure, self.next_on_success_or_failure)

    def flatten(self) -> List[N.LigFilterNode]:
        """The chart as lig_set_filter_tree's table: this node first, every edge pointing forward
        (a topological order), each node object once, so shared subtrees stay shared.  ValueError
        for a cyclic chart or one of more than LIG_MAX_FILTER_NODES nodes."""
        post: List[Filter] = []
        state: Dict[int, int] = {}            # id -> 1 on the DFS path, 2 finished
        stack = [(self, iter(self._successors()))]
        state[id(self)] = 1
        while stack:
            node, it = stack[-1]
            nxt = next(it, StopIteration)
            if nxt is StopIteration:
                state[id(node)] = 2
                post.append(node)
                stack.pop()
            elif nxt is not None:
                st = state.get(id(nxt))
                if st == 1:
                    raise ValueError(f"filter chart has a cycle through {nxt.name!r}")
                if st is None:
                    state[id(nxt)] = 1
                    stack.append((nxt, iter(nxt._successors())))
        order = post[::-1]                    # reverse post-order: parents before children
        if len(order) > N.LIG_MAX_FILTER_NODES:
            raise ValueError(f"filter chart has {len(order)} nodes (at most {N.LIG_MAX_FILTER_NODES})")
        index = {id(n): i for i, n in enumerate(order)}
        ix = lambda n: -1 if n is None else index[id(n)]
        return [N.LigFilterNode(n.kind, ix(n.next_on_success), ix(n.next_on_failure),
                                ix(n.next_on_success_or_failure), int(n.queue_threshold), float(n.kv_threshold))
                for n in order]


# defaultFilter, node for node                                                scheduler.go:26-91
kvCacheThreshold, queueThresholdCritical, queueingThresholdLoRA = 0.8, 5, 50   # scheduler.go:15-24
queueLoRAAndKVCacheFilter = Filter(
    "least queuing", LEAST_QUEUING,
    next_on_success_or_failure=Filter("low cost LoRA", LOW_LORA_COST,
                                      next_on_success_or_failure=Filter("least KV cache percent", LEAST_KV_CACHE)))
queueAndKVCacheFilter = Filter(
    "least queuing", LEAST_QUEUING,
    next_on_success_or_failure=Filter("least KV cache percent", LEAST_KV_CACHE))
lowLatencyFilter = Filter(
    "low queueing filter", LOW_QUEUEING, queue_threshold=queueingThresholdLoRA,
    next_on_success=Filter("affinity LoRA", LORA_AFFINITY, next_on_success=queueAndKVCacheFilter,
                           next_on_failure=Filter("can accept LoRA Adapter", CAN_ACCEPT_NEW_LORA,
                                                  next_on_success_or_failure=queueAndKVCacheFilter)),
    next_on_failure=queueLoRAAndKVCacheFilter)
sheddableRequestFilter = Filter(
    "has capacity for sheddable requests", NO_QUEUE_AND_LOW_KV,
    queue_threshold=queueThresholdCritical, kv_threshold=kvCacheThreshold,
    next_on_success=queueLoRAAndKVCacheFilter,
    next_on_failure=Filter("drop request", DROP))
DEFAULT_FILTER = Filter("critical request", CRITICAL_REQUEST,
                        next_on_success=lowLatencyFilter, next_on_failure=sheddableRequestFilter)


def _schedule_error(status: int) -> StatusError:
    # fmt.Errorf("failed to apply filter, resulted %v pods, this should never happen: %w", len(pods), err)
    #                                                                       scheduler.go:117
    if status == N.LIG_DROP:
        inner = f"rpc error: code = ResourceExhausted desc = {_DROP_DESC}"
        return StatusError("ResourceExhausted", _ERR_PREFIX + inner)
    if status == N.LIG_NO_PODS_LEFT:       # a caller tree ended on a predicate that kept no pod
        return StatusError("Unknown", _ERR_PREFIX + "no pods left")           # filter.go:88-90
    # tree returned ([], nil): Go prints a nil error under %w as %!w(<nil>); status.Code(err) of a
    # plain fmt error is Unknown.
    return StatusError("Unknown", _ERR_PREFIX + "%!w(<nil>)")


_POD_PREFIX = "failed to find target pod: "                                  # request.go:73-75


def _no_model_entry(model_id: int, name: str) -> str:
    """LIG_NO_MODEL from the device, which absent models never reach: an Internal status error as
    the Go adapter wraps it (request.go:73-75)."""
    return f"{_POD_PREFIX}rpc error: code = Internal desc = model id {model_id} ({name}) has no model entry on the device"


# What a call under load_feedback_window is refused with when the scheduler was not built for its form,
# by (retry, fallback rows).
_FEEDBACK_REFUSALS = {
    (False, True): "fallback endpoints are not defined under load_feedback_window: the picks come from the "
                   "feedback chain's copy of the snapshot, the fallbacks would not",
    (True, False): "retries are not defined under load_feedback_window: the picks come from the feedback "
                   "chain's load-adjusted copy of the snapshot, a retry would not",
    (True, True): "retries with fallbacks are not defined under load_feedback_window without "
                  "feedback_retries and feedback_fallbacks: the picks come from the feedback chain's "
                  "load-adjusted copy of the snapshot, these would not",
}


def _rows_array(rows: Sequence[Sequence[int]]) -> np.ndarray:
    """Excluded rows as the excluding calls take them: -1 padded to the widest row (at least 1)."""
    out = np.full((len(rows), max([1] + [len(r) for r in rows])), -1, dtype=np.int16)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return out


def _picks(results: list) -> list:
    """Results of a batch body with the pick alone in place of the pod list (None on error)."""
    return [(pods[0] if pods else None, *rest) for pods, *rest in results]


_M64 = (1 << 64) - 1


def pod_key(pod: Pod) -> int:
    """A pod's affinity identity: FNV-1a 64 over Name, a zero byte, then Address (the provider's own
    identity of a pod, so the key does not depend on where the pod is listed)."""
    h = 0xCBF29CE484222325
    for b in pod.Name.encode() + b"\0" + pod.Address.encode():
        h = ((h ^ b) * 0x100000001B3) & _M64
    return h


def _check_models(models: Sequence[InferenceModel]) -> None:
    """What lig_upload_models refuses with LIG_ERR_RANGE, named by model.  A model whose weights sum
    to <= 0 is not refused: pack_models packs it as absent."""
    for m in models:
        tms = m.Spec.TargetModels
        total = sum(int(t.Weight) for t in tms)
        if not tms or total <= 0:
            continue
        if len(tms) > 255:
            raise ValueError(f"model {m.Spec.ModelName} has {len(tms)} target models (at most 255)")
        if any(t.Weight < 0 for t in tms):
            raise ValueError(f"model {m.Spec.ModelName} has a negative weight")
        if total > (1 << 31) - 1:
            raise ValueError(f"the weights of model {m.Spec.ModelName} sum to {total} (at most 2^31-1)")


class Scheduler:
    def __init__(self, podMetricsProvider: PodMetricsProvider, device: int = 0,
                 max_pods: int = 4096, max_adapters: int = 1024, max_batch: int = 1 << 16,
                 seed: Optional[int] = None, filter: Optional[Filter] = None, load_feedback_window: int = 0,
                 feedback_fallbacks: bool = False, feedback_retries: bool = False, affinity: bool = False,
                 feedback_affinity: bool = False):
        if load_feedback_window < 0:
            raise ValueError(f"load_feedback_window must be >= 0, got {load_feedback_window}")
        self.podMetricsProvider = podMetricsProvider
        self._window = load_feedback_window  # 0: the reference's behaviour (no load feedback)
        # fallback rows under load_feedback_window come from the chain's tables; opt-in because the
        # *WithFallbacks calls refuse under feedback without it (documented behaviour kept as is)
        self._feedback_fallbacks = bool(feedback_fallbacks)
        # retries under load_feedback_window run on the chain's copy and load it; opt-in for the same reason
        self._feedback_retries = bool(feedback_retries)
        # every published epoch carries the pods' keys (lig_upload_pod_keys) only with affinity on
        self._affinity = bool(affinity)
        # affinity under load_feedback_window ranks the chain's tables and loads it; opt-in for the same reason
        self._feedback_affinity = bool(feedback_affinity)
        self._pod_keys: Optional[np.ndarray] = None
        self._engine = Engine(device, max_pods, max_adapters, max_batch)
        self._filter = filter                # None: the built-in defaultFilter
        if filter is not None:
            self._engine.set_filter_tree(filter)
        self._epoch = 0                      # the published epoch
        self._uploaded = 0                   # the last epoch number used (never reused)
        self._snap: Optional[PackedSnapshot] = None
        self._models: Optional[List[InferenceModel]] = None          # SetInferenceModels' list
        self._packed_models: Optional[PackedModels] = None           # that list packed for self._epoch
        self._model_index = 0                # first_index of the next model-id call
        self._ejected: List[Pod] = []        # EjectPods' set
        self._ejected_idx: List[int] = []    # its pods in the published epoch
        self._rng = random.Random(seed)      # the Go global source is auto-seeded (scheduler.go:120)
        self._seed = self._rng.getrandbits(64)

    def close(self) -> None:
        self._engine.close()

    # The reference re-reads the provider on every Schedule call; here the snapshot is re-packed
    # once per refresh tick (refreshMetricsInterval, main.go:39).  A provider that exposes
    # ``Version()`` is re-packed only when the version changes; otherwise every call re-packs,
    # which is exactly the reference's per-call semantics.
    def Refresh(self) -> PackedSnapshot:
        return self._refresh(self._models)

    def _refresh(self, models: Optional[List[InferenceModel]]) -> PackedSnapshot:
        # With a model list, the epoch is published only together with its model table, interned
        # against the epoch's own adapter ids.
        snap = pack_pod_metrics(list(self.podMetricsProvider.AllPodMetrics()))
        self._uploaded += 1
        self._engine.upload_snapshot(self._uploaded, snap)
        if self._affinity:
            self._pod_keys = np.array([pod_key(p) for p in snap.pods], dtype=np.uint64)
            self._engine.upload_pod_keys(self._uploaded, self._pod_keys)
        packed = pack_models(models, snap) if models is not None else None
        self._epoch, self._snap, self._packed_models, self._ejected_idx = self._uploaded, snap, packed, []
        idx = self._ejected_indices()
        if idx:                              # a full upload has every pod: derive once more
            self._derive(idx)
        elif packed is not None:
            self._engine.upload_models(self._uploaded, packed)
        self._version = self._provider_version()
        return snap

    def _ejected_indices(self) -> List[int]:
        gone = set(self._ejected)
        return [p for p, pod in enumerate(self._snap.pods) if pod in gone] if gone else []

    def _derive(self, idx: List[int]) -> None:
        """Publish an epoch derived from the published one (the newest resident epoch) without `idx`,
        with the model table when a list is set."""
        self._uploaded += 1
        self._engine.eject_pods(self._uploaded, self._epoch, idx)
        if self._affinity:                   # same pods in the same order: the same keys
            self._engine.upload_pod_keys(self._uploaded, self._pod_keys)
        if self._packed_models is not None:
            self._engine.upload_models(self._uploaded, self._packed_models)
        self._epoch, self._ejected_idx = self._uploaded, idx

    def EjectPods(self, pods: Sequence[Pod]) -> None:
        """Schedule as if `pods` had left the provider (lig_eject_pods), until a later call lets them
        back.  `pods` is the complete ejected set (empty: every pod back), matched by value against the
        snapshot; pods it does not hold are ignored.  Before the return a derived epoch is published
        (with the model table when a list is set), so every later call avoids them; every Refresh
        derives again from its new snapshot.  Publishing an epoch restarts the load-feedback chain."""
        self._ejected = list(pods)
        before = self._epoch
        self._current()                      # a refresh here already applies the new set
        if self._epoch == before:
            idx = self._ejected_indices()
            if idx != self._ejected_idx:
                self._derive(idx)

    def SetInferenceModels(self, models: Sequence[InferenceModel]) -> None:
        """The InferenceModels ScheduleModel resolves against (of two with one ModelName the later
        wins).  Publishes a new epoch, which restarts the load-feedback chain.  ValueError, naming the
        model, for a list the device cannot take; the previous list then stays in force."""
        by_name: Dict[str, int] = {}
        unique: List[InferenceModel] = []
        for m in models:                     # the reference's datastore is a map: the later one wins
            if m.Spec.ModelName in by_name:
                unique[by_name[m.Spec.ModelName]] = m
            else:
                by_name[m.Spec.ModelName] = len(unique)
                unique.append(m)
        _check_models(unique)
        self._refresh(unique)
        self._models = unique

    def ResolvesModels(self) -> bool:
        """Whether ScheduleModel has a list to resolve against (SetInferenceModels was called)."""
        return self._models is not None

    def _provider_version(self):
        v = getattr(self.podMetricsProvider, "Version", None)
        return v() if callable(v) else None

    def _current(self) -> PackedSnapshot:
        ver = self._provider_version()
        if self._snap is None or ver is None or ver != self._version:
            return self.Refresh()
        return self._snap

    # ---- the two batch bodies: descriptor requests and model names, each plain, with fallback rows, as a
    # retry without the pods already tried, or both ----
    def _check_form(self, n: Optional[int], tried_lists: Optional[Sequence[Sequence[Pod]]] = None,
                    mismatch: Optional[str] = None, affinity: bool = False) -> None:
        """The refusals of a call with fallback rows (n), a retry (tried_lists) or an affinity call, in
        this order.  `mismatch` is the message for argument lists of different lengths, if they differ."""
        retry, rows = tried_lists is not None, n is not None
        if affinity and not self._affinity:
            raise ValueError("affinity calls need a scheduler built with affinity=True (it uploads the pods' keys)")
        if affinity and self._window and not self._feedback_affinity:
            raise ValueError("affinity is not defined under load_feedback_window: affinity picks would bypass the "
                             "feedback chain's per-pod counts")
        if self._window and not affinity and ((retry and not self._feedback_retries) or (rows and not self._feedback_fallbacks)):
            raise ValueError(_FEEDBACK_REFUSALS[retry, rows])
        if rows and not 1 <= n <= N.LIG_MAX_FALLBACKS:
            raise ValueError(f"n must be in [1, {N.LIG_MAX_FALLBACKS}], got {n}")
        if mismatch:
            raise ValueError(mismatch)
        for tried in tried_lists or ():
            if len(tried) > N.LIG_MAX_EXCLUDED:
                raise ValueError(f"{len(tried)} tried pods (at most {N.LIG_MAX_EXCLUDED})")

    @staticmethod
    def _tried_rows(snap: PackedSnapshot, tried_lists: Sequence[Sequence[Pod]]) -> List[List[int]]:
        """Each list's tried pods as indices into the snapshot, matched by value; pods no longer in it
        are ignored."""
        where: Dict[Pod, List[int]] = {}
        for p, pod in enumerate(snap.pods):
            where.setdefault(pod, []).append(p)
        return [[p for pod in tried for p in where.get(pod, ())] for tried in tried_lists]

    def _call(self, kind: str, arr: np.ndarray, excluded: tuple, n: Optional[int],
              keys: Optional[np.ndarray] = None, **kw):
        """The Engine call of a batch: ``schedule_<kind>`` (kind "batch" or "models_batch"), as a chain
        call under load_feedback_window, an excluding call for a retry (`excluded` holds the retry's
        arrays), a fallback call for n rows, an affinity call with `keys` (the descriptors carry theirs
        as rand_key, model ids take them beside).  Returns (picks, rows); without n every row is empty."""
        if keys is not None:
            extra = (keys,) if kind == "models_batch" else ()
            chain = ("_feedback_chain", (self._window,)) if self._window else ("", ())
            out, rows = getattr(self._engine, "schedule_" + kind + chain[0] + "_affinity")(self._epoch, arr, *extra,
                                                                                         n or 0, *chain[1])
            return (out, rows) if n is not None else (out, [()] * len(out))
        name = ("schedule_" + kind + ("_feedback_chain" if self._window else "") + ("_excluding" if excluded else "")
                + ("_fallbacks" if n is not None else ""))
        args = (self._epoch, self._seed, arr, *excluded) + ((n,) if n is not None else ()) + \
            ((self._window,) if self._window else ())
        out = getattr(self._engine, name)(*args, **kw)
        return out if n is not None else (out, [()] * len(out))

    def _batch(self, reqs: Sequence[LLMRequest], tried_lists: Optional[Sequence[Sequence[Pod]]] = None,
               n: Optional[int] = None, keys: Optional[Sequence[int]] = None
               ) -> List[Tuple[List[Pod], Optional[StatusError]]]:
        """(pods, error) per request: pods the pick and then its fallback row, [] on error.  One rand_key
        per request, in order, from ScheduleBatch's sequence; an affinity call (keys) takes none."""
        affinity = keys is not None
        if affinity:
            self._check_form(n, None, None if len(keys) == len(reqs) else f"{len(reqs)} requests but {len(keys)} keys",
                             True)
        else:
            self._check_form(n, tried_lists, None if tried_lists is None or len(tried_lists) == len(reqs)
                             else f"{len(reqs)} requests but {len(tried_lists)} tried lists")
        snap = self._current()
        excluded: tuple = ()
        if tried_lists is not None:
            rows = self._tried_rows(snap, tried_lists)
            width = max([1] + [len(r) for r in rows])
            if width > N.LIG_MAX_EXCLUDED:
                raise ValueError(f"the tried pods match {width} pods of the snapshot (at most {N.LIG_MAX_EXCLUDED})")
            excluded = (_rows_array(rows),)
        arr = np.zeros(len(reqs), dtype=REQ_DTYPE)
        for i, r in enumerate(reqs):
            arr[i] = (snap.adapter_id(r.ResolvedTargetModel), N.LIG_REQ_CRITICAL if r.Critical else 0,
                      int(keys[i]) & _M64 if affinity else self._rng.getrandbits(64))
        # under load_feedback_window each window of `_window` requests, across calls, adds its picks to
        # the pods' WaitingQueueSize until the next refresh uploads a new epoch
        picks, rows = self._call("batch", arr, excluded, n, keys=arr["rand_key"] if affinity else None)
        return [([snap.pods[int(pk["pod_idx"])]] + [snap.pods[int(p)] for p in row if p >= 0], None)
                if pk["status"] == N.LIG_OK else ([], _schedule_error(int(pk["status"])))
                for pk, row in zip(picks, rows)]

    def _map_models(self, names: Sequence[str], resolved: Optional[Sequence[str]] = None,
                    rows: Optional[List[List[int]]] = None):
        """(errors, model ids, target indices, slots): the names the device is sent, in order, as model
        ids at positions `slots`, and for a retry (resolved) each resolved target as the first
        TargetModels entry of that name (255 for a model without TargetModels whose own name it is).
        A name the list alone answers gets its error instead."""
        pm = self._packed_models
        errors: List[Optional[StatusError]] = [None] * len(names)
        ids, targets, slots = [], [], []
        for i, name in enumerate(names):
            m = pm.model_ids.get(name) if pm is not None else None
            if m is None:                                                       # request.go:42-45
                errors[i] = StatusError("Unknown", f"error finding a model object in InferenceModel for input {name}")
                continue
            if not pm.present[m]:                                               # request.go:48-51
                errors[i] = StatusError("Unknown", f"error getting target model name for model {name}")
                continue
            if resolved is not None:
                res, tgt = resolved[i], pm.target_names[m]
                t = (255 if res == name else None) if not tgt else next((j for j, x in enumerate(tgt) if x == res), None)
                if t is None:
                    errors[i] = StatusError("InvalidArgument", f"{res} is not a target model of {name}")
                    continue
                if len(rows[i]) > N.LIG_MAX_EXCLUDED:
                    raise ValueError(f"the tried pods match {len(rows[i])} pods of the snapshot (at most "
                                     f"{N.LIG_MAX_EXCLUDED})")
                targets.append(t)
            ids.append(m)
            slots.append(i)
        return errors, ids, targets, slots

    def _model_batch(self, names: Sequence[str], resolved: Optional[Sequence[str]] = None,
                     tried_lists: Optional[Sequence[Sequence[Pod]]] = None, n: Optional[int] = None,
                     keys: Optional[Sequence[int]] = None) -> List[Tuple[List[Pod], str, Optional[StatusError]]]:
        """(pods, resolved target model, error) per name: pods the pick and then its fallback row, [] on
        error.  A retry (resolved, tried_lists) keeps the target the first attempt drew.  Names the host
        answers take no rand_key; request k sent to the device has rand_key = _model_index + k.  An
        affinity call (keys) draws on its keys and leaves the sequence alone."""
        retry, affinity = tried_lists is not None, keys is not None
        if affinity:
            self._check_form(n, None, None if len(keys) == len(names) else f"{len(names)} names but {len(keys)} keys",
                             True)
        else:
            self._check_form(n, tried_lists, None if not retry or len(names) == len(resolved) == len(tried_lists)
                             else f"{len(names)} names, {len(resolved)} resolved targets, {len(tried_lists)} tried "
                                  "lists")
        snap = self._current()
        rows = self._tried_rows(snap, tried_lists) if retry else None
        errors, ids, targets, slots = self._map_models(names, resolved if retry else None, rows)
        out = [([], resolved[i] if retry else "", err) for i, err in enumerate(errors)]
        if not ids:
            return out
        excluded = (np.array(targets, dtype=np.uint8), _rows_array([rows[i] for i in slots])) if retry else ()
        if affinity:
            picks, fbs = self._call("models_batch", np.array(ids, dtype=np.uint32), (), n,
                                    keys=np.array([int(keys[i]) & _M64 for i in slots], dtype=np.uint64))
        else:
            picks, fbs = self._call("models_batch", np.array(ids, dtype=np.uint32), excluded, n,
                                    first_index=self._model_index)
            self._model_index += len(ids)
        pm = self._packed_models
        for i, m, pk, row in zip(slots, ids, picks, fbs):
            t, st = int(pk["target_idx"]), int(pk["status"])
            res = resolved[i] if retry else names[i] if t == 255 else pm.target_names[m][t]   # 255: request.go:47
            if st == N.LIG_OK:
                out[i] = ([snap.pods[int(pk["pod_idx"])]] + [snap.pods[int(p)] for p in row if p >= 0], res, None)
            elif st == N.LIG_NO_MODEL:       # absent models and targets never reach the device
                out[i] = ([], res, StatusError("Internal", _no_model_entry(m, names[i])))
            else:
                err = _schedule_error(st)
                out[i] = ([], res, StatusError(err.code, _POD_PREFIX + str(err)))
        return out

    def ScheduleBatch(self, reqs: Sequence[LLMRequest]) -> List[Tuple[Optional[Pod], Optional[StatusError]]]:
        return _picks(self._batch(reqs))

    def ScheduleModelBatch(self, names: Sequence[str]) -> List[Tuple[Optional[Pod], str, Optional[StatusError]]]:
        """The resolve step and the pick on the device, one call per batch: (pod, resolved target
        model, error) per name.  Names the host answers from the list alone (unknown, or weights
        summing to <= 0) take no rand_key; request k sent to the device has rand_key = k."""
        return _picks(self._model_batch(names))

    def ScheduleModel(self, name: str) -> Tuple[str, Pod]:
        """HandleRequestBody's resolve step and Schedule for one request: (resolved target model,
        pod), or raises StatusError."""
        pod, resolved, err = self.ScheduleModelBatch([name])[0]
        if err is not None:
            raise err
        return resolved, pod

    def Schedule(self, req: LLMRequest) -> Pod:                     # scheduler.go:113-122
        pod, err = self.ScheduleBatch([req])[0]
        if err is not None:
            raise err
        return pod

    # ---- fallback endpoints: the pick, then up to n more distinct survivors in retry order ----
    def ScheduleBatchWithFallbacks(self, reqs: Sequence[LLMRequest], n: int
                                   ) -> List[Tuple[List[Pod], Optional[StatusError]]]:
        """ScheduleBatch plus up to n fallback pods per request (lig_schedule_batch_fallbacks):
        (pods, error) per request, pods[0] the pod ScheduleBatch would have returned, then distinct
        survivors in the order a proxy should retry them.  One rand_key per request from the same
        sequence as ScheduleBatch.  Under load_feedback_window the call is a feedback-chain call
        (lig_schedule_batch_feedback_chain_fallbacks) when the scheduler was built with
        feedback_fallbacks=True, and raises ValueError otherwise."""
        return self._batch(reqs, n=n)

    def ScheduleWithFallbacks(self, req: LLMRequest, n: int) -> List[Pod]:
        """Schedule plus up to n fallback pods: [pick, fallback 1, ...]; raises like Schedule."""
        pods, err = self.ScheduleBatchWithFallbacks([req], n)[0]
        if err is not None:
            raise err
        return pods

    def ScheduleModelBatchWithFallbacks(self, names: Sequence[str], n: int
                                        ) -> List[Tuple[List[Pod], str, Optional[StatusError]]]:
        """ScheduleModelBatch plus up to n fallback pods per request: (pods, resolved target model,
        error) per name, pods[0] the pod ScheduleModelBatch would have returned.  Host-answered errors
        and the rand_key sequence (_model_index) as ScheduleModelBatch.  Under load_feedback_window
        as ScheduleBatchWithFallbacks: a chain call with feedback_fallbacks=True, else ValueError."""
        return self._model_batch(names, n=n)

    # ---- retry scheduling: Schedule again over the pool without the pods already tried ----
    def ScheduleBatchRetry(self, reqs: Sequence[LLMRequest], tried_lists: Sequence[Sequence[Pod]]
                           ) -> List[Tuple[Optional[Pod], Optional[StatusError]]]:
        """ScheduleBatch with request i scheduled over the current snapshot's pods without the pods of
        tried_lists[i] (lig_schedule_batch_excluding): what Schedule returns once those pods have left
        the provider.  Tried pods are matched by value against the snapshot current when the call
        runs; those no longer in it are ignored.  One rand_key per request from ScheduleBatch's
        sequence; errors as ScheduleBatch.  ValueError for more than LIG_MAX_EXCLUDED tried pods.  Under
        load_feedback_window the call is a feedback-chain call (lig_schedule_batch_feedback_chain_excluding:
        the pool is the chain's load-adjusted copy, and each pick counts toward the chain's windows)
        when the scheduler was built with feedback_retries=True, and raises ValueError otherwise."""
        return _picks(self._batch(reqs, tried_lists))

    def ScheduleRetry(self, req: LLMRequest, tried: Sequence[Pod]) -> Pod:
        """Schedule over the pool without the pods in `tried`; raises like Schedule."""
        pod, err = self.ScheduleBatchRetry([req], [tried])[0]
        if err is not None:
            raise err
        return pod

    def ScheduleBatchRetryWithFallbacks(self, reqs: Sequence[LLMRequest], tried_lists: Sequence[Sequence[Pod]],
                                        n: int) -> List[Tuple[List[Pod], Optional[StatusError]]]:
        """ScheduleBatchRetry plus up to n fallback pods per request (lig_schedule_batch_excluding_fallbacks):
        (pods, error) per request, pods[0] the pod ScheduleBatchRetry would have returned, then distinct
        survivors of the same reduced pool in the order a proxy should try them, none of them tried.
        Tried pods, the rand_key sequence and errors as ScheduleBatchRetry.  ValueError for n outside
        [1, LIG_MAX_FALLBACKS] and more than LIG_MAX_EXCLUDED tried pods.  Under load_feedback_window the
        call is a feedback-chain call (lig_schedule_batch_feedback_chain_excluding_fallbacks: the picks and
        loads are ScheduleBatchRetry's chain call's, the rows rank the reduced pool of the chain's
        load-adjusted copy) when the scheduler was built with both feedback_retries=True and
        feedback_fallbacks=True, and raises ValueError otherwise."""
        return self._batch(reqs, tried_lists, n)

    def ScheduleRetryWithFallbacks(self, req: LLMRequest, tried: Sequence[Pod], n: int) -> List[Pod]:
        """ScheduleRetry plus up to n fallback pods: [pick, fallback 1, ...]; raises like Schedule."""
        pods, err = self.ScheduleBatchRetryWithFallbacks([req], [tried], n)[0]
        if err is not None:
            raise err
        return pods

    # ---- model-id retries: the retry of a model request at the target its first attempt drew ----
    def ScheduleModelBatchRetry(self, names: Sequence[str], resolved: Sequence[str],
                                tried_lists: Sequence[Sequence[Pod]]
                                ) -> List[Tuple[Optional[Pod], str, Optional[StatusError]]]:
        """The retry of ScheduleModelBatch requests without the pods they tried, keeping the targets they
        drew (resolved[i], the name ScheduleModelBatch returned): (pod, resolved target model, error) per
        name, as lig_schedule_models_batch_excluding returns it; no second draw.  Names the host answers
        from the list alone take no rand_key: unknown models and models whose weights sum to <= 0 with
        ScheduleModelBatch's errors, a resolved name that is not a target of the model with
        InvalidArgument.  Requests sent to the device take rand_keys from ScheduleModelBatch's sequence.
        Tried pods are matched by value as in ScheduleBatchRetry.  Under load_feedback_window the call is
        a chain call (lig_schedule_models_batch_feedback_chain_excluding) when the scheduler was built
        with feedback_retries=True, and raises ValueError otherwise."""
        return _picks(self._model_batch(names, resolved, tried_lists))

    def ScheduleModelRetry(self, name: str, resolved: str, tried: Sequence[Pod]) -> Pod:
        """The retry of one ScheduleModel request at its resolved target; raises like ScheduleModel."""
        pod, _, err = self.ScheduleModelBatchRetry([name], [resolved], [tried])[0]
        if err is not None:
            raise err
        return pod

    def ScheduleModelBatchRetryWithFallbacks(self, names: Sequence[str], resolved: Sequence[str],
                                             tried_lists: Sequence[Sequence[Pod]], n: int
                                             ) -> List[Tuple[List[Pod], str, Optional[StatusError]]]:
        """ScheduleModelBatchRetry plus up to n fallback pods of the same reduced pool per request
        (lig_schedule_models_batch_excluding_fallbacks): (pods, resolved target model, error), pods[0] the
        pod ScheduleModelBatchRetry would have returned.  ValueError for n outside [1, LIG_MAX_FALLBACKS];
        under load_feedback_window it needs both feedback_retries=True and feedback_fallbacks=True."""
        return self._model_batch(names, resolved, tried_lists, n)

    def ScheduleModelRetryWithFallbacks(self, name: str, resolved: str, tried: Sequence[Pod], n: int) -> List[Pod]:
        """ScheduleModelRetry plus up to n fallback pods: [pick, fallback 1, ...]; raises like ScheduleModel."""
        pods, _, err = self.ScheduleModelBatchRetryWithFallbacks([name], [resolved], [tried], n)[0]
        if err is not None:
            raise err
        return pods

    # ---- session affinity: requests that share a key go to the same surviving pod ----
    def ScheduleBatchAffinity(self, reqs: Sequence[LLMRequest], keys: Sequence[int], n: Optional[int] = None):
        """ScheduleBatch with request i placed by its affinity key keys[i] (lig_schedule_batch_affinity):
        the survivor with the highest rendezvous score mix(key ^ mix(pod_key(pod))), so a key keeps its
        pod while that pod survives, whatever order the provider lists pods in.  (pod, error) per
        request, or with n (1..LIG_MAX_FALLBACKS) (pods, error): the pick, then up to n more survivors in
        descending score.  Takes no rand_key.  Errors as ScheduleBatch.  ValueError unless the scheduler
        was built with affinity=True, and under load_feedback_window unless it was built with
        feedback_affinity=True: then the call is a chain call (lig_schedule_batch_feedback_chain_affinity)
        that ranks the chain's load-adjusted survivors and loads the chain with its picks."""
        results = self._batch(reqs, n=n, keys=keys)
        return results if n is not None else _picks(results)

    def ScheduleAffinity(self, req: LLMRequest, key: int) -> Pod:
        """Schedule placed by the affinity key `key`; raises like Schedule."""
        pod, err = self.ScheduleBatchAffinity([req], [key])[0]
        if err is not None:
            raise err
        return pod

    def ScheduleAffinityWithFallbacks(self, req: LLMRequest, key: int, n: int) -> List[Pod]:
        """ScheduleAffinity plus up to n fallback pods in descending score; raises like Schedule."""
        pods, err = self.ScheduleBatchAffinity([req], [key], n)[0]
        if err is not None:
            raise err
        return pods

    def ScheduleModelBatchAffinity(self, names: Sequence[str], keys: Sequence[int], n: Optional[int] = None):
        """ScheduleModelBatch with name i placed by keys[i] (lig_schedule_models_batch_affinity): the target
        is drawn on the key (so a session keeps its target while the model's targets and weights stay),
        then the pick is ScheduleBatchAffinity's.  (pod, resolved target model, error) per name, or with n
        (pods, resolved, error).  Names the host answers as ScheduleModelBatch; takes no rand_key."""
        results = self._model_batch(names, n=n, keys=keys)
        return results if n is not None else _picks(results)

    def ScheduleModelAffinity(self, name: str, key: int) -> Tuple[str, Pod]:
        """ScheduleModel placed by the affinity key `key`: (resolved target model, pod); raises like
        ScheduleModel."""
        pod, resolved, err = self.ScheduleModelBatchAffinity([name], [key])[0]
        if err is not None:
            raise err
        return resolved, pod

    def ScheduleModelAffinityWithFallbacks(self, name: str, key: int, n: int) -> Tuple[str, List[Pod]]:
        """ScheduleModelAffinity plus up to n fallback pods: (resolved target model, [pick, ...])."""
        pods, resolved, err = self.ScheduleModelBatchAffinity([name], [key], n)[0]
        if err is not None:
            raise err
        return resolved, pods

    # Filter-level view (the GPU analogue of Filter.Filter, filter.go:12-15): survivor slice.
    def Filter(self, req: LLMRequest) -> Tuple[List[Pod], Optional[StatusError]]:
        """The survivors of `req` against the scraped snapshot.  With load_feedback_window set this
        is still the scraped epoch: the queue sizes the feedback chain has added are not in it."""
        snap = self._current()
        # the class table holds the caller tree's survivor set, and the pool's: the direct scan walks
        # the built-in tree over every pod
        if self._filter is not None or self._ejected_idx:
            st, _, lst = self._engine.read_class(self._epoch, req.Critical, snap.adapter_id(req.ResolvedTargetModel),
                                                 snap.P)
            if st == N.LIG_DROP:
                return [], StatusError("ResourceExhausted", _DROP_DESC)
            if st == N.LIG_NO_PODS_LEFT:
                return [], StatusError("Unknown", "no pods left")
            return [snap.pods[int(p)] for p in lst], None
        arr = np.zeros(1, dtype=REQ_DTYPE)
        arr[0] = (snap.adapter_id(req.ResolvedTargetModel), N.LIG_REQ_CRITICAL if req.Critical else 0, 0)
        picks, masks = self._engine.schedule_scan(self._epoch, self._seed, arr, True, snap.W)
        st = int(picks[0]["status"])
        survivors = [snap.pods[p] for p in range(snap.P) if (int(masks[0, p >> 5]) >> (p & 31)) & 1]
        if st == N.LIG_DROP:
            return [], StatusError("ResourceExhausted", _DROP_DESC)
        return survivors, None

    def _survivors(self, snap: PackedSnapshot, status: int, pods: np.ndarray) -> Tuple[List[Pod], Optional[StatusError]]:
        if status == N.LIG_DROP:
            return [], StatusError("ResourceExhausted", _DROP_DESC)
        if status == N.LIG_NO_PODS_LEFT:
            return [], StatusError("Unknown", "no pods left")
        return [snap.pods[int(p)] for p in pods], None

    def FilterBatch(self, reqs: Sequence[LLMRequest]) -> List[Tuple[List[Pod], Optional[StatusError]]]:
        """Filter for a whole batch in one device call (lig_filter_batch): (survivors, error) per
        request, as Filter returns them, for the built-in tree and for a caller tree alike.  The
        scraped epoch, like Filter; the requests take no rand_key."""
        snap = self._current()
        arr = np.zeros(len(reqs), dtype=REQ_DTYPE)
        for i, r in enumerate(reqs):
            arr[i] = (snap.adapter_id(r.ResolvedTargetModel), N.LIG_REQ_CRITICAL if r.Critical else 0, 0)
        picks, offsets, pods = self._engine.filter_batch(self._epoch, self._seed, arr)
        return [self._survivors(snap, int(pk["status"]), pods[offsets[i]:offsets[i + 1]])
                for i, pk in enumerate(picks)]

    def FilterModelBatch(self, names: Sequence[str]) -> List[Tuple[List[Pod], Optional[StatusError]]]:
        """The survivors of model requests (lig_filter_models_batch): the resolve step of
        ScheduleModelBatch, then Filter on the resolved request.  (survivors, error) per name; names
        the host answers from the list alone get ScheduleModelBatch's errors.  The draws use
        ScheduleModelBatch's rand_key sequence without advancing it."""
        snap = self._current()
        errors, ids, _, slots = self._map_models(names)
        out = [([], err) for err in errors]
        if not ids:
            return out
        picks, offsets, pods = self._engine.filter_models_batch(self._epoch, self._seed, np.array(ids, dtype=np.uint32),
                                                                first_index=self._model_index)
        for k, (i, m, pk) in enumerate(zip(slots, ids, picks)):
            st = int(pk["status"])
            if st == N.LIG_NO_MODEL:         # absent models never reach the device
                out[i] = ([], StatusError("Internal", _no_model_entry(m, names[i])))
            else:
                out[i] = self._survivors(snap, st, pods[offsets[k]:offsets[k + 1]])
        return out


def NewScheduler(pmp: PodMetricsProvider, filter: Optional[Filter] = None, load_feedback_window: int = 0,
                 feedback_fallbacks: bool = False, feedback_retries: bool = False, affinity: bool = False,
                 feedback_affinity: bool = False, **kw) -> Scheduler:  # scheduler.go:93-99
    """filter: a caller flow chart (None = defaultFilter, the reference's only tree).
    load_feedback_window > 0: ScheduleBatch goes through the load-feedback chain (include/lig.h,
    lig_schedule_batch_feedback_chain): every window of that many requests, counted across calls,
    adds its picks to the pods' WaitingQueueSize until the next refresh.  0 = off.
    feedback_fallbacks: under load_feedback_window, let the *WithFallbacks calls run as chain calls
    whose rows rank the chain's load-adjusted survivors (lig_schedule_batch_feedback_chain_fallbacks);
    without it they raise ValueError there, as they always have.  The picks and the chain's loads do
    not depend on it.
    feedback_retries: under load_feedback_window, let ScheduleRetry / ScheduleBatchRetry run as chain calls
    (lig_schedule_batch_feedback_chain_excluding): each retry is scheduled on the chain's load-adjusted copy
    without the pods it tried, and its pick loads the chain like any other; without it they raise
    ValueError there, as they always have.
    With both feedback_fallbacks and feedback_retries, ScheduleRetryWithFallbacks /
    ScheduleBatchRetryWithFallbacks run as chain calls too
    (lig_schedule_batch_feedback_chain_excluding_fallbacks); with either one alone they raise ValueError
    under load_feedback_window.
    affinity: upload the pods' keys (pod_key) with every published epoch, so that ScheduleAffinity and its
    relatives can place requests by a caller key (lig_schedule_batch_affinity); without it they raise
    ValueError and nothing else changes.
    feedback_affinity: with affinity, under load_feedback_window, let the affinity calls run as chain calls
    (lig_schedule_batch_feedback_chain_affinity): each request takes the top-scoring pod of the chain's
    load-adjusted survivors, and its pick loads the chain like any other, so a hot key moves off a pod
    the chain has loaded out of the survivor set; without it they raise ValueError there, as they
    always have.  Without load_feedback_window it has no effect."""
    return Scheduler(pmp, filter=filter, load_feedback_window=load_feedback_window,
                     feedback_fallbacks=feedback_fallbacks, feedback_retries=feedback_retries, affinity=affinity,
                     feedback_affinity=feedback_affinity, **kw)
