"""ctypes view of the native C++ host runtime (csrc/host/lig_host.hpp -> liblig_host.so).

The C++ ``lig::scheduling::Scheduler`` is the compiled-language counterpart of the Go adapter
(INTEGRATION.md): concurrent blocking ``Schedule`` calls folded into one C-ABI call per flush,
snapshot re-packed per refresh tick.  This module only drives it from Python for the tests and the
streaming benchmark.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .backend import Pod, PodMetrics

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblig_host.so")

GRPC_OK, GRPC_UNKNOWN, GRPC_RESOURCE_EXHAUSTED, GRPC_INTERNAL = 0, 2, 8, 13

EXPORTED_SYMBOLS = (
    "ligh_provider_new", "ligh_provider_free", "ligh_provider_set_pods", "ligh_scheduler_new",
    "ligh_scheduler_new2",
    "ligh_scheduler_free", "ligh_schedule", "ligh_refresh", "ligh_stats",
    "ligh_schedule_concurrent", "ligh_stream_bench", "ligh_refresh_timing", "ligh_flush_timing",
    "ligh_scheduler_new_devices", "ligh_datastore_new", "ligh_datastore_free", "ligh_datastore_set_model",
    "ligh_schedule_model", "ligh_scheduler_new_tree", "ligh_scheduler_new_feedback", "ligh_feedback_stats",
    "ligh_scheduler_set_models", "ligh_schedule_model_device", "ligh_model_stats", "ligh_schedule_models_concurrent",
    "ligh_filter", "ligh_schedule_with_fallbacks", "ligh_fallback_scheduled", "ligh_schedule_model_with_fallbacks",
    "ligh_schedule_retry", "ligh_retry_scheduled", "ligh_schedule_retry_with_fallbacks",
    "ligh_schedule_model_retry", "ligh_schedule_model_retry_with_fallbacks",
    "ligh_eject_pods", "ligh_eject_stats",
    "ligh_scheduler_new_affinity", "ligh_schedule_affinity", "ligh_schedule_model_affinity", "ligh_affinity_scheduled",
    "ligh_pod_key", "ligh_scheduler_new_feedback_affinity",
)

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} not found: run `make -C llm_instance_gateway_b200/csrc`")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    cpp = C.POINTER(C.c_char_p)
    lib.ligh_provider_new.restype = vp
    lib.ligh_provider_free.argtypes = [vp]
    lib.ligh_provider_free.restype = None
    lib.ligh_provider_set_pods.argtypes = [vp, i32, cpp, cpp, vp, vp, vp, cpp, vp]
    lib.ligh_scheduler_new.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, u64, C.c_char_p, i32]
    lib.ligh_scheduler_new.restype = vp
    lib.ligh_scheduler_new2.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, u64, i32, i32, i32, C.c_char_p, i32]
    lib.ligh_scheduler_new2.restype = vp
    lib.ligh_scheduler_new_devices.argtypes = [vp, C.POINTER(i32), i32, i32, i32, i32, i32, i32, i32, u64, C.c_char_p, i32]
    lib.ligh_scheduler_new_devices.restype = vp
    lib.ligh_scheduler_new_tree.argtypes = [vp, i32, C.POINTER(i32), i32, i32, i32, i32, i32, i32, i32, u64, i32, i32,
                                            i32, vp, i32, C.c_char_p, i32]
    lib.ligh_scheduler_new_tree.restype = vp
    lib.ligh_scheduler_new_feedback.argtypes = [vp, i32, C.POINTER(i32), i32, i32, i32, i32, i32, i32, i32, u64, i32,
                                                i32, i32, vp, i32, i32, i32, i32, C.c_char_p, i32]
    lib.ligh_scheduler_new_feedback.restype = vp
    lib.ligh_scheduler_new_affinity.argtypes = [vp, i32, C.POINTER(i32), i32, i32, i32, i32, i32, i32, i32, u64, i32,
                                                i32, i32, vp, i32, i32, i32, i32, i32, C.c_char_p, i32]
    lib.ligh_scheduler_new_affinity.restype = vp
    lib.ligh_scheduler_new_feedback_affinity.argtypes = [vp, i32, C.POINTER(i32), i32, i32, i32, i32, i32, i32, i32,
                                                         u64, i32, i32, i32, vp, i32, i32, i32, i32, i32, i32,
                                                         C.c_char_p, i32]
    lib.ligh_scheduler_new_feedback_affinity.restype = vp
    lib.ligh_schedule_affinity.argtypes = [vp, C.c_char_p, i32, u64, i32, C.c_char_p, i32, C.POINTER(i32),
                                           C.c_char_p, i32]
    lib.ligh_schedule_model_affinity.argtypes = [vp, C.c_char_p, u64, i32, C.c_char_p, i32, C.c_char_p, i32,
                                                 C.POINTER(i32), C.c_char_p, i32]
    lib.ligh_affinity_scheduled.argtypes = [vp]
    lib.ligh_affinity_scheduled.restype = u64
    lib.ligh_pod_key.argtypes = [C.c_char_p, C.c_char_p]
    lib.ligh_pod_key.restype = u64
    lib.ligh_feedback_stats.argtypes = [vp, vp]
    lib.ligh_feedback_stats.restype = None
    lib.ligh_datastore_new.restype = vp
    lib.ligh_datastore_free.argtypes = [vp]
    lib.ligh_datastore_free.restype = None
    lib.ligh_datastore_set_model.argtypes = [vp, C.c_char_p, i32, i32, cpp, vp]
    lib.ligh_schedule_model.argtypes = [vp, vp, C.c_char_p, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32]
    lib.ligh_scheduler_set_models.argtypes = [vp, vp, C.c_char_p, i32]
    lib.ligh_schedule_model_device.argtypes = [vp, C.c_char_p, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32,
                                               C.c_char_p, i32]
    lib.ligh_model_stats.argtypes = [vp, vp]
    lib.ligh_model_stats.restype = None
    lib.ligh_schedule_models_concurrent.argtypes = [vp, vp, i32, i32, cpp, i32, vp, vp, vp]
    lib.ligh_scheduler_free.argtypes = [vp]
    lib.ligh_scheduler_free.restype = None
    lib.ligh_schedule.argtypes = [vp, C.c_char_p, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32,
                                  C.c_char_p, i32]
    lib.ligh_refresh.argtypes = [vp, C.c_char_p, i32]
    lib.ligh_filter.argtypes = [vp, C.c_char_p, i32, C.c_char_p, i32, C.POINTER(i32), C.c_char_p, i32]
    lib.ligh_schedule_with_fallbacks.argtypes = [vp, C.c_char_p, i32, i32, C.c_char_p, i32, C.POINTER(i32),
                                                 C.c_char_p, i32]
    lib.ligh_schedule_model_with_fallbacks.argtypes = [vp, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32,
                                                       C.POINTER(i32), C.c_char_p, i32]
    lib.ligh_fallback_scheduled.argtypes = [vp]
    lib.ligh_schedule_retry.argtypes = [vp, C.c_char_p, i32, cpp, cpp, i32, C.c_char_p, i32, C.c_char_p, i32,
                                        C.c_char_p, i32]
    lib.ligh_schedule_retry_with_fallbacks.argtypes = [vp, C.c_char_p, i32, cpp, cpp, i32, i32, C.c_char_p, i32,
                                                       C.POINTER(i32), C.c_char_p, i32]
    lib.ligh_retry_scheduled.argtypes = [vp]
    lib.ligh_schedule_model_retry.argtypes = [vp, C.c_char_p, C.c_char_p, cpp, cpp, i32, C.c_char_p, i32, C.c_char_p,
                                              i32, C.c_char_p, i32]
    lib.ligh_schedule_model_retry_with_fallbacks.argtypes = [vp, C.c_char_p, C.c_char_p, cpp, cpp, i32, i32,
                                                             C.c_char_p, i32, C.POINTER(i32), C.c_char_p, i32]
    lib.ligh_eject_pods.argtypes = [vp, cpp, cpp, i32, C.c_char_p, i32]
    lib.ligh_eject_stats.argtypes = [vp, vp]
    lib.ligh_eject_stats.restype = None
    lib.ligh_retry_scheduled.restype = u64
    lib.ligh_fallback_scheduled.restype = u64
    lib.ligh_stats.argtypes = [vp, vp]
    lib.ligh_stats.restype = None
    lib.ligh_refresh_timing.argtypes = [vp, vp]
    lib.ligh_refresh_timing.restype = None
    lib.ligh_flush_timing.argtypes = [vp, vp]
    lib.ligh_flush_timing.restype = None
    lib.ligh_schedule_concurrent.argtypes = [vp, i32, i32, cpp, vp, i32, vp, vp]
    lib.ligh_stream_bench.argtypes = [vp, C.c_double, C.c_double, i32, cpp, vp, i32, u64, vp, vp, i32,
                                      C.POINTER(i32), C.POINTER(i32)]
    for name in EXPORTED_SYMBOLS:
        getattr(lib, name)
    _lib = lib
    return lib


def _strs(items: Sequence[str]):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode()
    return arr


class HostSchedulerError(RuntimeError):
    pass


class HostProvider:
    """A mutable fake PodMetricsProvider living on the C++ side."""

    def __init__(self, pods: Sequence[PodMetrics] = ()):
        self._lib = load()
        self._p = self._lib.ligh_provider_new()
        self.set_pods(pods)

    def set_pods(self, pods: Sequence[PodMetrics]) -> None:
        self.pods = list(pods)
        n = len(self.pods)
        q = np.array([p.Metrics.WaitingQueueSize for p in self.pods], dtype=np.int64)
        kv = np.array([p.Metrics.KVCacheUsagePercent for p in self.pods], dtype=np.float64)
        ma = np.array([p.Metrics.MaxActiveModels for p in self.pods], dtype=np.int64)
        flat: List[str] = []
        off = [0]
        for p in self.pods:
            flat.extend(p.Metrics.ActiveModels.keys())
            off.append(len(flat))
        off = np.array(off, dtype=np.int32)
        rc = self._lib.ligh_provider_set_pods(
            self._p, n, _strs([p.Pod.Name for p in self.pods]), _strs([p.Pod.Address for p in self.pods]),
            q.ctypes.data, kv.ctypes.data, ma.ctypes.data, _strs(flat), off.ctypes.data)
        assert rc == 0

    def close(self):
        if self._p:
            self._lib.ligh_provider_free(self._p)
            self._p = None


class HostScheduler:
    def __init__(self, provider: HostProvider, device: int = 0, max_pods: int = 4096,
                 max_adapters: int = 1024, max_batch: int = 1 << 16, flush_size: int = 4096,
                 batch_window_us: int = 50, refresh_interval_ms: int = 0, seed: int = 1,
                 busy_poll: bool = False, caller_spin_us: int = 0, use_doorbell: bool = False,
                 devices: Optional[Sequence[int]] = None, filter=None, load_feedback_window: int = 0,
                 feedback_fallbacks: bool = False, feedback_retries: bool = False, affinity: bool = False,
                 feedback_affinity: bool = False):
        self._lib = load()
        self.provider = provider
        err = C.create_string_buffer(512)
        if (filter is not None or load_feedback_window or feedback_fallbacks or feedback_retries or affinity
                or feedback_affinity):
            # Options::filter (a scheduling.Filter chart or a node table),
            # Options::load_feedback_window (load feedback carried across flushes, 0 = off) and
            # Options::feedback_fallbacks / feedback_retries (the *WithFallbacks calls and ScheduleRetry
            # under that feedback; with both, ScheduleRetryWithFallbacks too) and Options::affinity (the pods'
            # keys with every published epoch, for ScheduleAffinity and its relatives; with
            # Options::feedback_affinity those run as chain calls under load_feedback_window)
            from .engine import _node_table
            nodes, n = _node_table(filter)
            devs = list(devices) if devices is not None else []
            arr = (C.c_int * max(len(devs), 1))(*devs)
            self._s = self._lib.ligh_scheduler_new_feedback_affinity(
                provider._p, device, arr, len(devs), max_pods, max_adapters, max_batch, flush_size, batch_window_us,
                refresh_interval_ms, seed, int(busy_poll), caller_spin_us, int(use_doorbell), C.cast(nodes, C.c_void_p),
                n, load_feedback_window, int(feedback_fallbacks), int(feedback_retries), int(affinity),
                int(feedback_affinity), err, 512)
        elif devices is not None and len(devices) > 1:
            arr = (C.c_int * len(devices))(*devices)
            self._s = self._lib.ligh_scheduler_new_devices(provider._p, arr, len(devices), max_pods, max_adapters,
                                                           max_batch, flush_size, batch_window_us, refresh_interval_ms,
                                                           seed, err, 512)
        else:
            self._s = self._lib.ligh_scheduler_new2(provider._p, device, max_pods, max_adapters, max_batch,
                                                    flush_size, batch_window_us, refresh_interval_ms, seed,
                                                    int(busy_poll), caller_spin_us, int(use_doorbell), err, 512)
        if not self._s:
            raise HostSchedulerError(err.value.decode("utf-8", "replace"))

    def close(self):
        if getattr(self, "_s", None):
            self._lib.ligh_scheduler_free(self._s)
            self._s = None

    def Schedule(self, model: str, resolved: str, critical: bool) -> Tuple[int, Optional[Pod], str]:  # noqa: N802
        name, addr = C.create_string_buffer(256), C.create_string_buffer(256)
        err = C.create_string_buffer(512)
        code = self._lib.ligh_schedule(self._s, model.encode(), resolved.encode(), int(critical),
                                       name, 256, addr, 256, err, 512)
        if code == GRPC_OK:
            return code, Pod(name.value.decode(), addr.value.decode()), ""
        return code, None, err.value.decode("utf-8", "replace")

    def Filter(self, resolved: str, critical: bool) -> Tuple[int, List[str], str]:  # noqa: N802
        """Scheduler::Filter: (gRPC code, survivor pod names in slice order, error message)."""
        cap = 4 << 20
        names, err, n = C.create_string_buffer(cap), C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_filter(self._s, resolved.encode(), int(critical), names, cap, C.byref(n), err, 512)
        pods = names.value.decode().split("\n") if n.value else []
        return code, pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleWithFallbacks(self, resolved: str, critical: bool, n: int) -> Tuple[int, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleWithFallbacks: (gRPC code, pod names [pick, fallbacks in retry order], error)."""
        cap = 64 * 1024
        names, err, k = C.create_string_buffer(cap), C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_with_fallbacks(self._s, resolved.encode(), int(critical), n, names, cap,
                                                      C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleRetry(self, resolved: str, critical: bool, tried: Sequence[Pod]
                      ) -> Tuple[int, Optional[Pod], str]:  # noqa: N802
        """Scheduler::ScheduleRetry: Schedule without the pods in `tried` (matched by value):
        (gRPC code, pod, error)."""
        name, addr = C.create_string_buffer(256), C.create_string_buffer(256)
        err = C.create_string_buffer(512)
        code = self._lib.ligh_schedule_retry(self._s, resolved.encode(), int(critical), _strs([p.Name for p in tried]),
                                             _strs([p.Address for p in tried]), len(tried), name, 256, addr, 256,
                                             err, 512)
        if code == GRPC_OK:
            return code, Pod(name.value.decode(), addr.value.decode()), ""
        return code, None, err.value.decode("utf-8", "replace")

    def ScheduleRetryWithFallbacks(self, resolved: str, critical: bool, tried: Sequence[Pod], n: int
                                   ) -> Tuple[int, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleRetryWithFallbacks: ScheduleRetry plus up to n fallback pods of the same reduced
        pool: (gRPC code, pod names [pick, fallbacks in retry order], error).  Under load_feedback_window it
        needs both feedback_retries and feedback_fallbacks, and then runs on the feedback chain."""
        cap = 64 * 1024
        names, err, k = C.create_string_buffer(cap), C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_retry_with_fallbacks(self._s, resolved.encode(), int(critical),
                                                            _strs([p.Name for p in tried]),
                                                            _strs([p.Address for p in tried]), len(tried), n, names,
                                                            cap, C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleModelRetry(self, model: str, resolved: str, tried: Sequence[Pod]
                           ) -> Tuple[int, Optional[Pod], str]:  # noqa: N802
        """Scheduler::ScheduleModelRetry: the retry of a model request at the target it drew (`resolved`, the
        name ScheduleModel returned), without the pods in `tried`: (gRPC code, pod, error)."""
        name, addr = C.create_string_buffer(256), C.create_string_buffer(256)
        err = C.create_string_buffer(512)
        code = self._lib.ligh_schedule_model_retry(self._s, model.encode(), resolved.encode(),
                                                   _strs([p.Name for p in tried]), _strs([p.Address for p in tried]),
                                                   len(tried), name, 256, addr, 256, err, 512)
        if code == GRPC_OK:
            return code, Pod(name.value.decode(), addr.value.decode()), ""
        return code, None, err.value.decode("utf-8", "replace")

    def ScheduleModelRetryWithFallbacks(self, model: str, resolved: str, tried: Sequence[Pod], n: int
                                        ) -> Tuple[int, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleModelRetryWithFallbacks: ScheduleModelRetry plus up to n fallback pods of the
        same reduced pool: (gRPC code, pod names [pick, fallbacks in retry order], error)."""
        cap = 64 * 1024
        names, err, k = C.create_string_buffer(cap), C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_model_retry_with_fallbacks(self._s, model.encode(), resolved.encode(),
                                                                  _strs([p.Name for p in tried]),
                                                                  _strs([p.Address for p in tried]), len(tried), n,
                                                                  names, cap, C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleModelWithFallbacks(self, model: str, n: int) -> Tuple[int, str, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleModelWithFallbacks: (gRPC code, resolved target model, pod names [pick,
        fallbacks in retry order], error)."""
        cap = 64 * 1024
        resolved, names = C.create_string_buffer(256), C.create_string_buffer(cap)
        err, k = C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_model_with_fallbacks(self._s, model.encode(), n, resolved, 256, names, cap,
                                                            C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, resolved.value.decode(), pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleAffinity(self, resolved: str, critical: bool, key: int, n: int = 0
                         ) -> Tuple[int, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleAffinity (n = 0) or ScheduleAffinityWithFallbacks (n fallbacks): (gRPC code, pod
        names [pick, then the row in descending score], error)."""
        cap = 64 * 1024
        names, err, k = C.create_string_buffer(cap), C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_affinity(self._s, resolved.encode(), int(critical), key & ((1 << 64) - 1), n,
                                                names, cap, C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def ScheduleModelAffinity(self, model: str, key: int, n: int = 0
                              ) -> Tuple[int, str, List[str], str]:  # noqa: N802
        """Scheduler::ScheduleModelAffinity[WithFallbacks]: (gRPC code, resolved target model, pod names, error)."""
        cap = 64 * 1024
        resolved, names = C.create_string_buffer(256), C.create_string_buffer(cap)
        err, k = C.create_string_buffer(512), C.c_int(0)
        code = self._lib.ligh_schedule_model_affinity(self._s, model.encode(), key & ((1 << 64) - 1), n, resolved, 256,
                                                      names, cap, C.byref(k), err, 512)
        pods = names.value.decode().split("\n") if k.value else []
        return code, resolved.value.decode(), pods, err.value.decode("utf-8", "replace") if code != GRPC_OK else ""

    def EjectPods(self, pods: Sequence[Pod]) -> None:  # noqa: N802
        """Scheduler::EjectPods: schedule as if `pods` (the complete set, matched by value; empty = every
        pod back) had left the provider, from the return on and across refreshes."""
        err = C.create_string_buffer(512)
        code = self._lib.ligh_eject_pods(self._s, _strs([p.Name for p in pods]), _strs([p.Address for p in pods]),
                                         len(pods), err, 512)
        if code != GRPC_OK:
            raise HostSchedulerError(err.value.decode("utf-8", "replace"))

    def Refresh(self) -> None:  # noqa: N802
        err = C.create_string_buffer(512)
        if self._lib.ligh_refresh(self._s, err, 512) != 0:
            raise HostSchedulerError(err.value.decode())

    def stats(self) -> dict:
        out = (C.c_uint64 * 9)()
        self._lib.ligh_stats(self._s, out)
        fb = (C.c_uint64 * 2)()
        self._lib.ligh_feedback_stats(self._s, fb)
        ms = (C.c_uint64 * 2)()
        self._lib.ligh_model_stats(self._s, ms)
        ej = (C.c_uint64 * 2)()
        self._lib.ligh_eject_stats(self._s, ej)
        return dict(zip(("scheduled", "batches", "max_batch", "refreshes", "stale_retries", "failed_refreshes",
                         "excluded_pods", "delta_refreshes", "last_dirty_pods", "feedback_windows",
                         "feedback_restarts", "model_scheduled", "model_batches", "fallback_scheduled",
                         "retry_scheduled", "ejected_pods", "eject_publishes", "affinity_scheduled"),
                        map(int, list(out) + list(fb) + list(ms) + [self._lib.ligh_fallback_scheduled(self._s),
                                                                    self._lib.ligh_retry_scheduled(self._s)] +
                            list(ej) + [self._lib.ligh_affinity_scheduled(self._s)])))

    def ScheduleModel(self, datastore: "HostDataStore", model: str):  # noqa: N802
        """resolve (FetchModelData + RandomWeightedDraw + IsCritical) + Schedule: (code, resolved, pod, err)."""
        resolved, name, addr = C.create_string_buffer(256), C.create_string_buffer(256), C.create_string_buffer(256)
        err = C.create_string_buffer(512)
        code = self._lib.ligh_schedule_model(self._s, datastore._d, model.encode(), resolved, 256, name, 256, addr, 256, err, 512)
        pod = Pod(name.value.decode(), addr.value.decode()) if code == GRPC_OK else None
        return code, resolved.value.decode(), pod, err.value.decode("utf-8", "replace")

    def set_inference_models(self, datastore: "HostDataStore") -> None:
        """Scheduler::SetInferenceModels with the datastore's current models: ScheduleModelOnDevice
        resolves against them from the epoch this call publishes.  HostSchedulerError on refusal."""
        err = C.create_string_buffer(512)
        if self._lib.ligh_scheduler_set_models(self._s, datastore._d, err, 512) != GRPC_OK:
            raise HostSchedulerError(err.value.decode("utf-8", "replace"))

    def ScheduleModelOnDevice(self, model: str):  # noqa: N802
        """The resolve step on the device + the pick: (code, resolved, pod, err), as ScheduleModel."""
        resolved, name, addr = C.create_string_buffer(256), C.create_string_buffer(256), C.create_string_buffer(256)
        err = C.create_string_buffer(512)
        code = self._lib.ligh_schedule_model_device(self._s, model.encode(), resolved, 256, name, 256, addr, 256,
                                                    err, 512)
        pod = Pod(name.value.decode(), addr.value.decode()) if code == GRPC_OK else None
        return code, resolved.value.decode(), pod, err.value.decode("utf-8", "replace")

    def schedule_models_concurrent(self, n_threads: int, per_thread: int, models: Sequence[str],
                                   datastore: Optional["HostDataStore"] = None):
        """n_threads callers of ScheduleModelOnDevice (or of ScheduleModel with `datastore`), caller i
        sending models[i % len(models)]: (codes, pod index in the provider's slice or -1, index of the
        resolved target or 255/-1)."""
        n = n_threads * per_thread
        codes, pods, targets = (np.zeros(n, dtype=np.int32) for _ in range(3))
        rc = self._lib.ligh_schedule_models_concurrent(self._s, datastore._d if datastore else None, n_threads,
                                                       per_thread, _strs(models), len(models), codes.ctypes.data,
                                                       pods.ctypes.data, targets.ctypes.data)
        assert rc == 0
        return codes, pods, targets

    def refresh_timing(self) -> dict:
        out = (C.c_double * 2)()
        self._lib.ligh_refresh_timing(self._s, out)
        return {"pack_us": float(out[0]), "upload_us": float(out[1])}

    def flush_timing(self) -> dict:
        """Slowest single device call and slowest Flush (resolve + call + wake) since creation, us."""
        out = (C.c_double * 4)()
        self._lib.ligh_flush_timing(self._s, out)
        return {"max_device_call_us": float(out[0]), "max_flush_us": float(out[1]), "slowest_call_batch": int(out[2]),
                "slowest_call_cpu_us": float(out[3])}

    def schedule_concurrent(self, n_threads: int, per_thread: int, models: Sequence[str],
                            critical: Sequence[bool]):
        n = n_threads * per_thread
        codes = np.zeros(n, dtype=np.int32)
        pods = np.zeros(n, dtype=np.int32)
        crit = np.array([int(c) for c in critical], dtype=np.int32)
        rc = self._lib.ligh_schedule_concurrent(self._s, n_threads, per_thread, _strs(models),
                                                crit.ctypes.data, len(models), codes.ctypes.data,
                                                pods.ctypes.data)
        assert rc == 0
        return codes, pods

    def stream_bench(self, rate: float, seconds: float, n_threads: int, models: Sequence[str],
                     critical: Sequence[bool], seed: int = 1):
        cap = int(rate * seconds * 1.2) + 1024
        lat = np.zeros(cap, dtype=np.float32)
        svc = np.zeros(cap, dtype=np.float32)
        crit = np.array([int(c) for c in critical], dtype=np.int32)
        n_done, n_err = C.c_int(), C.c_int()
        rc = self._lib.ligh_stream_bench(self._s, rate, seconds, n_threads, _strs(models),
                                         crit.ctypes.data, len(models), seed, lat.ctypes.data, svc.ctypes.data, cap,
                                         C.byref(n_done), C.byref(n_err))
        assert rc == 0
        self.last_service_latency_us = svc[: n_done.value].copy()
        return lat[: n_done.value].copy(), n_err.value


class HostDataStore:
    """backend.FakeDataStore on the C++ side: model name -> InferenceModel."""

    def __init__(self, models=()):
        self._lib = load()
        self._d = self._lib.ligh_datastore_new()
        for m in models:
            self.set_model(m)

    def set_model(self, m) -> None:
        tms = m.Spec.TargetModels
        w = np.array([t.Weight for t in tms], dtype=np.int32)
        rc = self._lib.ligh_datastore_set_model(self._d, m.Spec.ModelName.encode(), int(m.Spec.Criticality == "Critical"),
                                                len(tms), _strs([t.Name for t in tms]), w.ctypes.data if len(tms) else None)
        assert rc == 0

    def close(self):
        if self._d:
            self._lib.ligh_datastore_free(self._d)
            self._d = None
