"""The survivor-list entry points without a GPU: declared in include/lig.h, exported by liblig.so,
listed in _native.EXPORTED_SYMBOLS, and bound by ctypes with the header's parameter list."""
import ctypes as C
import os
import re

from llm_instance_gateway_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("lig_filter_batch", "lig_filter_batch_device", "lig_filter_models_batch", "lig_filter_models_batch_device")

# C parameter type -> the ctypes type _native binds it with
CTYPE = {"lig_ctx*": C.c_void_p, "uint64_t": C.c_uint64, "int": C.c_int, "int64_t": C.c_int64, "void*": C.c_void_p}


def prototypes():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lig.h")).read(), flags=re.S)
    out = {}
    for name in NAMES:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
        assert m, f"{name} is not declared"
        params = []
        for p in m.group(1).split(","):
            p = " ".join(p.replace("*", " * ").split())
            p = re.sub(r"\bconst\b\s*", "", p).strip()
            typ = " ".join(p.split()[:-1]).replace(" *", "*")
            params.append(typ)
        out[name] = params
    return out


def test_declared_exported_and_listed():
    lib = N.load()
    for name in NAMES:
        assert hasattr(lib, name)
        assert name in N.EXPORTED_SYMBOLS
    assert lib.lig_abi_version() == N.LIG_ABI_VERSION == 7


def test_ctypes_signatures_match_the_header():
    lib = N.load()
    for name, params in prototypes().items():
        got = getattr(lib, name).argtypes
        assert len(got) == len(params), (name, params)
        for typ, ct in zip(params, got):
            want = CTYPE.get(typ, C.c_void_p if typ.endswith("*") else None)
            assert want is ct, (name, typ, ct)
        assert getattr(lib, name).restype in (C.c_int, None)


def test_null_context_is_refused_without_a_device():
    lib = N.load()
    assert lib.lig_filter_batch(None, 1, 0, None, 0, None, None, None, 0) == N.LIG_ERR_INVALID
    assert lib.lig_filter_models_batch_device(None, 1, 0, 0, None, 0, None, None, None, 0, None) == N.LIG_ERR_INVALID
