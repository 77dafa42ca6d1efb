"""The asynchronous paced-presentation entry points: declared in include/espflix_b200.h, exported by the library, and bound
in capi.py with argtypes that match the declared parameters."""
import ctypes
import os
import re

import espflix_b200
from espflix_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("ef_present_picture_async", "ef_present_idle_async", "ef_present_wait")
C_TYPES = {"int": ctypes.c_int, "uint64_t": ctypes.c_uint64, "int*": ctypes.POINTER(ctypes.c_int)}


def _params(name):
    h = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "espflix_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, h)
    assert m, name
    out = []
    for p in m.group(1).split(","):
        t = re.sub(r"\s+", " ", p.strip()).rsplit(" ", 1)[0].replace("const ", "")
        t = t.replace(" *", "*")
        out.append(t + "*" if p.strip().split()[-1].startswith("*") else t)
    return out


def test_header_declares_the_async_present_calls():
    assert _params("ef_present_picture_async") == ["ef_ctx*", "int", "uint8_t*", "uint16_t*", "uint64_t", "ef_present_info*", "void*"]
    assert _params("ef_present_idle_async") == ["ef_ctx*", "uint32_t*", "uint16_t*", "uint64_t", "ef_present_info*", "void*"]
    assert _params("ef_present_wait") == ["ef_ctx*", "int*"]


def test_capi_binds_them_with_matching_argtypes():
    lib = ctypes.CDLL(espflix_b200.lib_path())
    for name in NAMES:
        assert hasattr(lib, name), name
        res, args = capi._SIGNATURES[name]
        assert res is ctypes.c_int
        params = _params(name)
        assert len(args) == len(params), name
        for a, p in zip(args, params):
            want = C_TYPES.get(p, ctypes.c_void_p if p.endswith("*") else None)
            assert want is not None, (name, p)
            assert a == want or (a is ctypes.c_void_p and want is ctypes.c_void_p), (name, p, a)
    # the synchronous calls take the same arguments in the same order
    assert capi._SIGNATURES["ef_present_picture_async"] == capi._SIGNATURES["ef_present_picture"]
    assert capi._SIGNATURES["ef_present_idle_async"] == capi._SIGNATURES["ef_present_idle"]


def test_context_methods_exist():
    for m in ("present_picture_async", "present_idle_async", "present_wait", "present_info"):
        assert callable(getattr(espflix_b200.Context, m)), m
