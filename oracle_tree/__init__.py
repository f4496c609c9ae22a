"""ctypes binding of the CPU oracle for caller filter trees (lig_oracle_tree.c): the oracle's port of
the reference, walking a table of filter nodes instead of defaultFilter.  Test infrastructure: only
tests/ and bench scripts load it.  Status numbers are include/lig.h's (0 OK, 1 DROP, 2 EMPTY,
4 NO_PODS_LEFT)."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblig_oracle_tree.so")

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} not found: build it with `make -C oracle_tree` (or __graft_entry__.build())")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl, u64 = C.c_void_p, C.c_int, C.c_int64, C.c_double, C.c_uint64
    cpp = C.POINTER(C.c_char_p)
    lib.lig_oracle_pool_new.argtypes = [i32]
    lib.lig_oracle_pool_new.restype = vp
    lib.lig_oracle_pool_free.argtypes = [vp]
    lib.lig_oracle_pool_free.restype = None
    lib.lig_oracle_pool_set_pod.argtypes = [vp, i32, C.c_char_p, C.c_char_p, i64, dbl, i64, cpp, i32]
    lib.lig_oracle_set_filter_tree.argtypes = [vp, i32]
    lib.lig_oracle_tree_filter.argtypes = [vp, C.c_char_p, i32, vp, C.POINTER(i32)]
    lib.lig_oracle_tree_schedule_batch.argtypes = [vp, cpp, i32, C.c_char_p, vp, i32, u64, vp]
    _lib = lib
    return lib


def _names(items: Sequence[str]):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, s in enumerate(items):
        arr[i] = s.encode()
    return arr


def set_filter_tree(nodes) -> None:
    """nodes: a sequence of rows with include/lig.h's lig_filter_node layout (LigFilterNode), or
    None for defaultFilter.  Process-wide, like lig_oracle_set_thresholds."""
    if nodes is None:
        assert load().lig_oracle_set_filter_tree(None, 0) == 0
        return
    from llm_instance_gateway_b200 import _native as N
    rows = [n if isinstance(n, N.LigFilterNode) else N.LigFilterNode(*n) for n in nodes]
    arr = (N.LigFilterNode * max(len(rows), 1))(*rows)
    if load().lig_oracle_set_filter_tree(C.cast(arr, C.c_void_p), len(rows)) != 0:
        raise ValueError("invalid filter tree")


class Pool:
    """A fake PodMetricsProvider (oracle records: name, address, waiting_queue_size,
    kv_cache_usage_percent, max_active_models, active_models)."""

    def __init__(self, pods: Sequence[dict]):
        self._lib = load()
        self.n = len(pods)
        self._p = self._lib.lig_oracle_pool_new(self.n)
        for i, p in enumerate(pods):
            act = list(p.get("active_models", []))
            rc = self._lib.lig_oracle_pool_set_pod(
                self._p, i, p.get("name", "").encode(), p.get("address", "").encode(),
                int(p.get("waiting_queue_size", 0)), float(p.get("kv_cache_usage_percent", 0.0)),
                int(p.get("max_active_models", 0)), _names(act), len(act))
            assert rc == 0

    def __del__(self):
        try:
            self._lib.lig_oracle_pool_free(self._p)
        except Exception:
            pass

    def filter(self, model: str, critical: bool) -> Tuple[int, List[int]]:
        out = np.zeros(max(self.n, 1), dtype=np.int32)
        n = C.c_int()
        rc = self._lib.lig_oracle_tree_filter(self._p, model.encode(), int(critical), out.ctypes.data, C.byref(n))
        assert rc >= 0
        return rc, out[: n.value].tolist()

    def schedule_batch(self, adapter_names: Sequence[str], unknown_name: str, reqs: np.ndarray,
                       seed: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        from llm_instance_gateway_b200.packer import PICK_DTYPE, REQ_DTYPE
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        R = int(reqs.shape[0])
        if out is None:
            out = np.zeros(R, dtype=PICK_DTYPE)
        rc = self._lib.lig_oracle_tree_schedule_batch(self._p, _names(adapter_names), len(adapter_names),
                                                      unknown_name.encode(), reqs.ctypes.data if R else None, R,
                                                      seed, out.ctypes.data if R else None)
        assert rc == 0
        return out
