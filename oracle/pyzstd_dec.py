"""ORACLE — ctypes binding of the strict zstd decoder (zstd_dec.hpp), test infrastructure only. The library is built from the header
with the host C++ compiler into oracle/liboracle_zstd.so (by __graft_entry__.build(), or on first use)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "zstd_dec.hpp")
_SO = os.path.join(_HERE, "liboracle_zstd.so")
_lib = None
INFO_KEYS = ("raw", "rle", "compressed", "huf_literals", "fse_weights", "fse_tables", "predefined_tables", "rle_tables")


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-DORC_ZSTD_EXPORT", "-x", "c++", _SRC, "-o", _SO])
    return _SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_zstd_decode.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_char_p, C.c_uint64]
        L.orc_zstd_decode.restype = C.c_int64
        _lib = L
    return _lib


def decode(data: bytes, chunk: int = 0):
    """(content, None, info) or (None, broken rule, None). chunk > 0 also checks the engine's frame layout (TF_WIRE_F_ZSTD).
    info: block counts by type, Huffman-coded literal sections, FSE-compressed Huffman weights, sequence tables by mode."""
    err = C.create_string_buffer(200); info = (C.c_uint64 * 8)()
    n = lib().orc_zstd_decode(data, len(data), chunk, None, 0, info, err, len(err))
    if n < 0:
        return None, err.value.decode(), None
    dst = C.create_string_buffer(max(1, n))
    lib().orc_zstd_decode(data, len(data), chunk, dst, n, info, err, len(err))
    return dst.raw[:n], None, dict(zip(INFO_KEYS, info))
