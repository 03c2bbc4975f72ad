"""ORACLE — ctypes binding of the strict inflater (inflate.hpp), test infrastructure only. The library is built from the header with
the host C++ compiler into oracle/liboracle_inflate.so (by __graft_entry__.build(), or on first use)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "inflate.hpp")
_SO = os.path.join(_HERE, "liboracle_inflate.so")
INFLATE_RAW, INFLATE_ZLIB, INFLATE_GZIP = 0, 1, 2
_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-DORC_INFLATE_EXPORT", "-x", "c++", _SRC, "-o", _SO])
    return _SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_inflate.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_char_p, C.c_uint64]
        L.orc_inflate.restype = C.c_int64
        _lib = L
    return _lib


def inflate(data: bytes, container: int, chunk: int = 0):
    """(text, None, info) or (None, broken rule, None). container INFLATE_RAW / _ZLIB / _GZIP; chunk > 0 also checks the engine's
    container layout. info = {"stored", "fixed", "dynamic", "markers"}: block counts by type, "max_len": the longest literal/length
    code of a dynamic block."""
    err = C.create_string_buffer(200); info = (C.c_uint64 * 5)()
    n = lib().orc_inflate(data, len(data), container, chunk, None, 0, info, err, len(err))
    if n < 0:
        return None, err.value.decode(), None
    dst = C.create_string_buffer(max(1, n))
    lib().orc_inflate(data, len(data), container, chunk, dst, n, info, err, len(err))
    return dst.raw[:n], None, {"stored": info[0], "fixed": info[1], "dynamic": info[2], "markers": info[3], "max_len": info[4]}
