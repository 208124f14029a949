"""Every function include/prophet_b200.h exports has a ctypes prototype in _lib.load() of the same arity, argument kinds
and return kind (no GPU needed: the library is only opened)."""
import ctypes as C
import os
import re

import pytest

from time_series_spark_b200 import _lib as L

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "prophet_b200.h")
DECL = re.compile(r"PB200_API\s+([^;{]*?)\b(pb200_\w+)\s*\(([^)]*)\)\s*;", re.S)
C_KINDS = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "uint64_t": "uint64", "double": "double",
           "void": "void"}
CTYPES_KINDS = {C.c_int32: "int32", C.c_int64: "int64", C.c_uint64: "uint64", C.c_double: "double"}


def _c_kind(decl: str) -> str:
    """``int64_t n_series`` -> int64, any pointer -> pointer (a parameter or a return type)."""
    if "*" in decl:
        return "pointer"
    words = [w for w in decl.split() if w not in ("const", "struct")]
    return C_KINDS[words[0]]


def _ctypes_kind(t) -> str:
    if t is None:
        return "void"
    if t in (C.c_void_p, C.c_char_p) or hasattr(t, "contents"):
        return "pointer"
    return CTYPES_KINDS[t]


def _declarations():
    with open(HEADER) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    out = {}
    for ret, name, params in DECL.findall(text):
        params = " ".join(params.split())
        out[name] = (_c_kind(ret), [] if params in ("", "void") else [_c_kind(p) for p in params.split(",")])
    return out


DECLARATIONS = _declarations()


def test_header_declarations_are_found():
    assert len(DECLARATIONS) == 54
    assert sorted(DECLARATIONS) == sorted(L.EXPORTS)


@pytest.mark.parametrize("name", sorted(DECLARATIONS))
def test_prototype_matches_header(name):
    ret, params = DECLARATIONS[name]
    f = getattr(L.load(), name)
    assert f.argtypes is not None, f"{name} has no ctypes prototype"
    assert [_ctypes_kind(t) for t in f.argtypes] == params
    assert _ctypes_kind(f.restype) == ret
