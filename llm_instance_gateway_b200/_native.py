"""ctypes binding of the C ABI in include/lig.h (liblig.so, built in-tree for sm_90a).

There is no fallback: if the library is missing, import fails loudly with the build command; if
there is no CUDA device, ``lig_create`` returns LIG_ERR_CUDA and ``LigError`` is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblig.so")

LIG_OK, LIG_DROP, LIG_EMPTY, LIG_NO_MODEL, LIG_NO_PODS_LEFT = 0, 1, 2, 3, 4
LIG_DRAW_DOMAIN = 0xA0761D6478BD642F
LIG_ERR_INVALID, LIG_ERR_CUDA, LIG_ERR_STALE_EPOCH, LIG_ERR_NO_SNAPSHOT, LIG_ERR_RANGE = -1, -2, -3, -4, -5
LIG_ERR_BUSY, LIG_ERR_NCCL = -6, -7
LIG_MAX_TICKETS, LIG_COMM_ID_BYTES = 256, 128
LIG_ABI_VERSION = 7
# filter node kinds of a caller filter tree (lig_set_filter_tree)
(LIG_F_CRITICAL_REQUEST, LIG_F_LOW_QUEUEING, LIG_F_LORA_AFFINITY, LIG_F_CAN_ACCEPT_NEW_LORA, LIG_F_LOW_LORA_COST,
 LIG_F_NO_QUEUE_AND_LOW_KV, LIG_F_LEAST_QUEUING, LIG_F_LEAST_KV_CACHE, LIG_F_DROP) = range(9)
LIG_MAX_FILTER_NODES = 32
LIG_REQ_CRITICAL = 1
LIG_MAX_PODS, LIG_MAX_ADAPTERS = 32768, 65534
LIG_MAX_FALLBACKS = 8
LIG_MAX_EXCLUDED = 32
(LIG_KERNEL_NONE, LIG_KERNEL_PERSISTENT, LIG_KERNEL_LOOP, LIG_KERNEL_PLAIN, LIG_KERNEL_QUEUE, LIG_KERNEL_MODELS,
 LIG_KERNEL_MODELS_PLAIN) = range(7)

# Every symbol include/lig.h declares (tests check the library exports all of them).
EXPORTED_SYMBOLS = (
    "lig_create", "lig_destroy", "lig_set_thresholds", "lig_get_thresholds", "lig_snapshot_bytes",
    "lig_pack_pods", "lig_pack_snapshot", "lig_upload_snapshot", "lig_upload_snapshot_device",
    "lig_schedule_batch", "lig_schedule_batch_device", "lig_schedule_batches_device", "lig_schedule_scan_device",
    "lig_schedule_scan", "lig_read_class", "lig_last_error", "lig_version", "lig_abi_version",
    "lig_device_count", "lig_kernel_launches", "lig_sm_count", "lig_host_alloc", "lig_host_free",
    "lig_stream_capacity", "lig_stream_open", "lig_stream_submit", "lig_stream_close",
    "lig_schedule_batch_async", "lig_schedule_wait",
    "lig_group_create", "lig_group_destroy", "lig_group_size", "lig_group_ctx", "lig_group_set_thresholds",
    "lig_group_upload_snapshot", "lig_group_schedule_batch",
    "lig_comm_unique_id", "lig_comm_init_rank", "lig_comm_upload_snapshot_device", "lig_comm_upload_snapshot",
    "lig_comm_allreduce_i32",
    "lig_upload_models", "lig_schedule_models_batch", "lig_schedule_models_batches_device", "lig_resolve_models",
    "lig_pick_kernel_info", "lig_schedule_batch_feedback_device", "lig_update_snapshot",
    "lig_upload_snapshot_async", "lig_upload_models_async", "lig_set_filter_tree", "lig_group_set_filter_tree",
    "lig_schedule_batch_feedback_chain", "lig_schedule_batch_feedback_chain_device", "lig_feedback_chain_reset",
    "lig_schedule_models_batch_feedback_chain", "lig_schedule_models_batch_feedback_chain_device",
    "lig_stream_submit_models",
    "lig_filter_batch", "lig_filter_batch_device", "lig_filter_models_batch", "lig_filter_models_batch_device",
    "lig_last_pick_launch",
    "lig_schedule_batch_fallbacks", "lig_schedule_batch_fallbacks_device", "lig_schedule_models_batch_fallbacks",
    "lig_schedule_models_batch_fallbacks_device",
    "lig_schedule_batch_feedback_chain_fallbacks", "lig_schedule_batch_feedback_chain_fallbacks_device",
    "lig_schedule_models_batch_feedback_chain_fallbacks", "lig_schedule_models_batch_feedback_chain_fallbacks_device",
    "lig_schedule_batch_excluding", "lig_schedule_batch_excluding_device",
    "lig_schedule_batch_feedback_chain_excluding", "lig_schedule_batch_feedback_chain_excluding_device",
    "lig_schedule_batch_excluding_fallbacks", "lig_schedule_batch_excluding_fallbacks_device",
    "lig_schedule_batch_feedback_chain_excluding_fallbacks",
    "lig_schedule_batch_feedback_chain_excluding_fallbacks_device",
    "lig_eject_pods",
    "lig_schedule_models_batch_excluding", "lig_schedule_models_batch_excluding_device",
    "lig_schedule_models_batch_excluding_fallbacks", "lig_schedule_models_batch_excluding_fallbacks_device",
    "lig_schedule_models_batch_feedback_chain_excluding", "lig_schedule_models_batch_feedback_chain_excluding_device",
    "lig_schedule_models_batch_feedback_chain_excluding_fallbacks",
    "lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device",
    "lig_upload_pod_keys", "lig_schedule_batch_affinity", "lig_schedule_batch_affinity_device",
    "lig_schedule_models_batch_affinity", "lig_schedule_models_batch_affinity_device",
    "lig_schedule_batch_feedback_chain_affinity", "lig_schedule_batch_feedback_chain_affinity_device",
    "lig_schedule_models_batch_feedback_chain_affinity", "lig_schedule_models_batch_feedback_chain_affinity_device",
)


class LigReq(C.Structure):
    _fields_ = [("adapter_id", C.c_int32), ("flags", C.c_uint32), ("rand_key", C.c_uint64)]


class LigPick(C.Structure):
    _fields_ = [("pod_idx", C.c_int32), ("status", C.c_uint16), ("n_survivors", C.c_uint16)]


class LigThresholds(C.Structure):
    _fields_ = [("kv_cache_threshold", C.c_double), ("queue_threshold_critical", C.c_int64),
                ("queueing_threshold_lora", C.c_int64)]


class LigFilterNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("next_on_success", C.c_int32), ("next_on_failure", C.c_int32),
                ("next_on_success_or_failure", C.c_int32), ("queue_threshold", C.c_int64),
                ("kv_threshold", C.c_double)]


class LigLaunchInfo(C.Structure):
    _fields_ = [("kernel", C.c_int32), ("groups", C.c_int32), ("stages", C.c_int32), ("bulk_store", C.c_int32),
                ("tables_in_smem", C.c_int32), ("per_thread", C.c_int32)]


class LigError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"lig error {code}: {message}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    """Load liblig.so (once).  Raises if it has not been built — no silent fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
            f"g.build()'` or `make -C llm_instance_gateway_b200/csrc` (needs nvcc, sm_90a). "
            "There is no CPU fallback for the scheduling path.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    lib.lig_create.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    lib.lig_destroy.argtypes = [vp]
    lib.lig_destroy.restype = None
    lib.lig_set_thresholds.argtypes = [vp, C.POINTER(LigThresholds)]
    lib.lig_get_thresholds.argtypes = [vp, C.POINTER(LigThresholds)]
    lib.lig_set_filter_tree.argtypes = [vp, C.POINTER(LigFilterNode), i32]
    lib.lig_group_set_filter_tree.argtypes = [vp, C.POINTER(LigFilterNode), i32]
    lib.lig_snapshot_bytes.argtypes = [i32, i32]
    lib.lig_snapshot_bytes.restype = C.c_size_t
    lib.lig_pack_pods.argtypes = [i32, vp, vp, vp, vp, vp, vp]
    lib.lig_pack_snapshot.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp]
    lib.lig_upload_snapshot.argtypes = [vp, u64, i32, i32, vp, vp, vp, vp, vp]
    lib.lig_upload_snapshot_async.argtypes = [vp, u64, i32, i32, vp, vp, vp, vp, vp]
    lib.lig_upload_snapshot_device.argtypes = [vp, u64, i32, i32, vp, vp]
    lib.lig_schedule_batch.argtypes = [vp, u64, u64, vp, i32, vp]
    lib.lig_schedule_batch_device.argtypes = [vp, u64, u64, vp, i32, vp, vp]
    lib.lig_schedule_batches_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_scan_device.argtypes = [vp, u64, u64, vp, i32, vp, vp, vp]
    lib.lig_schedule_scan.argtypes = [vp, u64, u64, vp, i32, vp, vp]
    lib.lig_read_class.argtypes = [vp, u64, i32, i32, C.POINTER(i32), C.POINTER(i32), vp]
    lib.lig_last_error.restype = C.c_char_p
    lib.lig_version.restype = C.c_char_p
    lib.lig_kernel_launches.argtypes = [vp]
    lib.lig_kernel_launches.restype = u64
    lib.lig_sm_count.argtypes = [vp]
    lib.lig_host_alloc.argtypes = [C.c_size_t]
    lib.lig_host_alloc.restype = vp
    lib.lig_host_free.argtypes = [vp]
    lib.lig_host_free.restype = None
    lib.lig_stream_open.argtypes = [vp]
    lib.lig_stream_submit.argtypes = [vp, u64, u64, vp, i32, vp]
    lib.lig_stream_submit_models.argtypes = [vp, u64, u64, u64, vp, i32, vp]
    lib.lig_stream_close.argtypes = [vp]
    lib.lig_schedule_batch_async.argtypes = [vp, u64, u64, vp, i32, vp, C.POINTER(i32)]
    lib.lig_schedule_wait.argtypes = [vp, i32]
    lib.lig_group_create.argtypes = [C.POINTER(vp), C.POINTER(i32), i32, i32, i32, i32]
    lib.lig_group_destroy.argtypes = [vp]
    lib.lig_group_destroy.restype = None
    lib.lig_group_size.argtypes = [vp]
    lib.lig_group_ctx.argtypes = [vp, i32]
    lib.lig_group_ctx.restype = vp
    lib.lig_group_set_thresholds.argtypes = [vp, C.POINTER(LigThresholds)]
    lib.lig_group_upload_snapshot.argtypes = [vp, u64, i32, i32, vp, vp, vp, vp, vp]
    lib.lig_group_schedule_batch.argtypes = [vp, u64, u64, vp, i32, vp]
    lib.lig_comm_unique_id.argtypes = [vp]
    lib.lig_comm_init_rank.argtypes = [vp, i32, i32, vp]
    lib.lig_comm_upload_snapshot_device.argtypes = [vp, u64, i32, i32, vp, i32, vp]
    lib.lig_comm_upload_snapshot.argtypes = [vp, u64, i32, i32, vp, vp, vp, vp, vp, i32]
    lib.lig_comm_allreduce_i32.argtypes = [vp, vp, i32, vp]
    lib.lig_upload_models.argtypes = [vp, u64, i32, vp, vp, vp, vp, vp, vp]
    lib.lig_upload_models_async.argtypes = [vp, u64, i32, vp, vp, vp, vp, vp, vp]
    lib.lig_schedule_models_batch.argtypes = [vp, u64, u64, u64, vp, i32, vp]
    lib.lig_schedule_models_batches_device.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_resolve_models.argtypes = [vp, u64, u64, u64, vp, i32, vp, vp]
    lib.lig_schedule_batch_feedback_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, i32, vp, vp]
    lib.lig_schedule_batch_feedback_chain.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_feedback_chain_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_feedback_chain.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_feedback_chain_device.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_feedback_chain_reset.argtypes = [vp]
    i64 = C.c_int64
    lib.lig_filter_batch.argtypes = [vp, u64, u64, vp, i32, vp, vp, vp, i64]
    lib.lig_filter_batch_device.argtypes = [vp, u64, u64, vp, i32, vp, vp, vp, i64, vp]
    lib.lig_filter_models_batch.argtypes = [vp, u64, u64, u64, vp, i32, vp, vp, vp, i64]
    lib.lig_filter_models_batch_device.argtypes = [vp, u64, u64, u64, vp, i32, vp, vp, vp, i64, vp]
    lib.lig_schedule_batch_fallbacks.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_fallbacks_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_fallbacks.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_fallbacks_device.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_batch_feedback_chain_fallbacks.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_feedback_chain_fallbacks_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp,
                                                                       vp]
    lib.lig_schedule_models_batch_feedback_chain_fallbacks.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32, vp, i32,
                                                                       vp]
    lib.lig_schedule_models_batch_feedback_chain_fallbacks_device.argtypes = [vp, u64, u64, u64, vp, i32, vp, i32,
                                                                              vp, i32, vp, vp]
    lib.lig_schedule_batch_excluding.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_excluding_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_batch_excluding_fallbacks.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_excluding_fallbacks_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_batch_feedback_chain_excluding.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_feedback_chain_excluding_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32, vp,
                                                                       vp]
    lib.lig_schedule_batch_feedback_chain_excluding_fallbacks.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp, i32,
                                                                          vp, i32, vp]
    lib.lig_schedule_batch_feedback_chain_excluding_fallbacks_device.argtypes = [vp, u64, u64, vp, i32, vp, i32, vp,
                                                                                 i32, vp, i32, vp, vp]
    # model-id retries: the descriptor counterpart's arguments with first_index, model_ids, targets
    lib.lig_schedule_models_batch_excluding.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_excluding_device.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_excluding_fallbacks.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp, i32, vp, i32,
                                                                  vp]
    lib.lig_schedule_models_batch_excluding_fallbacks_device.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp, i32, vp,
                                                                         i32, vp, vp]
    lib.lig_schedule_models_batch_feedback_chain_excluding.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp, i32, vp,
                                                                       i32, vp]
    lib.lig_schedule_models_batch_feedback_chain_excluding_device.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp,
                                                                              i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks.argtypes = [vp, u64, u64, u64, vp, vp, i32, vp,
                                                                                 i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_feedback_chain_excluding_fallbacks_device.argtypes = [
        vp, u64, u64, u64, vp, vp, i32, vp, i32, vp, i32, vp, i32, vp, vp]
    # session affinity: no seed, no first_index; the model forms take one key per request
    lib.lig_upload_pod_keys.argtypes = [vp, u64, i32, vp]
    lib.lig_schedule_batch_affinity.argtypes = [vp, u64, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_affinity_device.argtypes = [vp, u64, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_affinity.argtypes = [vp, u64, vp, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_affinity_device.argtypes = [vp, u64, vp, vp, i32, vp, i32, vp, vp]
    # ... and under the feedback chain: the chain fallback calls' arguments without seed or first_index
    lib.lig_schedule_batch_feedback_chain_affinity.argtypes = [vp, u64, vp, i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_batch_feedback_chain_affinity_device.argtypes = [vp, u64, vp, i32, vp, i32, vp, i32, vp, vp]
    lib.lig_schedule_models_batch_feedback_chain_affinity.argtypes = [vp, u64, vp, vp, i32, vp, i32, vp, i32, vp]
    lib.lig_schedule_models_batch_feedback_chain_affinity_device.argtypes = [vp, u64, vp, vp, i32, vp, i32, vp, i32,
                                                                             vp, vp]
    lib.lig_update_snapshot.argtypes = [vp, u64, u64, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.lig_eject_pods.argtypes = [vp, u64, u64, vp, i32]
    lib.lig_pick_kernel_info.argtypes = [vp, u64, C.c_char_p, i32, C.POINTER(i32), C.POINTER(i32),
                                         C.POINTER(i32), C.POINTER(i32)]
    lib.lig_last_pick_launch.argtypes = [vp, C.POINTER(LigLaunchInfo)]
    for name in EXPORTED_SYMBOLS:
        getattr(lib, name)  # AttributeError if the library does not export it
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise LigError(rc, load().lig_last_error().decode("utf-8", "replace"))
