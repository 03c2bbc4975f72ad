"""ORACLE — test infrastructure only (tests/, __graft_entry__.smoke(), bench.py cpu_baseline /
--impl reference).  Never imported by the product package.

Python front of the CPU oracle:
  * loads oracle/liboracle.so (C++ restatement of the per-row hot path, oracle.cpp);
  * restates the filter-expression grammar used by `filter_rows`
        library/go/yandex/cloud/filter/grammar/grammar.go:256-313 (lexer regexp + participle grammar)
        library/go/yandex/cloud/filter/filters.go:237-313      (opFromG / validateTerm / Parse)
    config-level logic runs once per plan, so pure Python is adequate here;
  * restates plan building for the transformers on the path
        pkg/transformer/transformation.go:46-85 (Suitable -> ResultSchema chain)
        filter_rows.go:445-519, hmac_hasher.go:76-89, mask.go:20-67, to_string.go:99-113.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import re
import subprocess
import sys
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(_HERE))
from transferia_b200 import abi  # noqa: E402  (memory layout only)

# ----------------------------------------------------------------------------- library


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cpp", ".h", ".hpp"))] + [os.path.join(_HERE, "..", "include", "tfgpu.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"], stdout=subprocess.DEVNULL)
    return so


class OrcVal(C.Structure):
    _fields_ = [("kind", C.c_int32), ("nsec", C.c_uint32), ("i", C.c_int64), ("u", C.c_uint64),
                ("f", C.c_double), ("s", C.c_char_p), ("slen", C.c_uint64)]


class OrcTerm(C.Structure):
    _fields_ = [("col", C.c_int32), ("op", C.c_int32), ("vtype", C.c_int32), ("nlist", C.c_int32),
                ("i", C.c_int64), ("f", C.c_double), ("s", C.c_char_p), ("slen", C.c_uint64),
                ("ilist", C.c_void_p), ("flist", C.c_void_p), ("soffs", C.c_void_p), ("sheap", C.c_void_p)]


class OrcColSchema(C.Structure):
    _fields_ = [("name", C.c_char_p), ("type", C.c_int32), ("required", C.c_int32), ("original_type", C.c_char_p)]


class OrcStep(C.Structure):
    _fields_ = [("kind", C.c_int32), ("terms", C.POINTER(OrcTerm)), ("expr_off", C.c_void_p), ("nexpr", C.c_int32),
                ("cols", C.c_void_p), ("ncols", C.c_int32), ("salt", C.c_char_p), ("salt_len", C.c_uint64),
                ("convert_to_bytes", C.c_int32), ("pass_all", C.c_int32), ("kind_mask", C.c_int32)]


class OrcRegions(C.Structure):
    _fields_ = [("values", C.c_uint64), ("validity", C.c_uint64), ("aux", C.c_uint64), ("offsets", C.c_uint64), ("heap", C.c_uint64), ("heap_len", C.c_uint64)]


class OrcCsvOpts(C.Structure):
    _fields_ = [("delimiter", C.c_uint8), ("quote", C.c_uint8), ("escape", C.c_uint8), ("double_quote", C.c_uint8), ("strings_can_be_null", C.c_uint8),
                ("quoted_strings_can_be_null", C.c_uint8), ("include_missing", C.c_uint8), ("pad", C.c_uint8),
                ("null_values", C.c_char_p), ("true_values", C.c_char_p), ("false_values", C.c_char_p), ("skip_lines", C.c_uint64)]


class OrcJsonOpts(C.Structure):
    _fields_ = [("add_rest", C.c_uint8), ("add_dedupe_keys", C.c_uint8), ("null_keys_allowed", C.c_uint8), ("use_numbers_in_any", C.c_uint8),
                ("unpack_bytes_base64", C.c_uint8), ("pad", C.c_uint8 * 3), ("partition", C.c_char_p)]


class OrcJsonMsg(C.Structure):
    _fields_ = [("end", C.c_uint64), ("offset", C.c_uint64), ("write_sec", C.c_int64), ("write_nsec", C.c_uint32), ("pad", C.c_uint32)]


class OrcBuf(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_uint8)), ("len", C.c_uint64)]


(OG_NIL, OG_INT8, OG_INT16, OG_INT32, OG_INT64, OG_UINT8, OG_UINT16, OG_UINT32, OG_UINT64, OG_FLOAT32, OG_FLOAT64,
 OG_BOOL, OG_STRING, OG_BYTES, OG_TIME, OG_DURATION, OG_JSON, OG_INT, OG_UINT) = range(19)
OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_IN, OP_NOTIN, OP_MATCH, OP_NOTMATCH = range(10)
LV_INT, LV_FLOAT, LV_BOOL, LV_STRING, LV_TIME, LV_NULL, LV_LIST = 1, 2, 3, 4, 5, 6, 16
STEP_FILTER_ROWS, STEP_MASK, STEP_TO_STRING, STEP_SKIP_EVENTS, STEP_SELECT_COLS, STEP_TO_DATETIME, STEP_NUMBER_TO_FLOAT = 1, 2, 3, 4, 5, 6, 7
STEP_SHARDER = 8

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_fmt_float64.argtypes = [C.c_double, C.c_int, C.c_char_p, C.c_int]
        L.orc_fmt_float32.argtypes = [C.c_float, C.c_int, C.c_char_p, C.c_int]
        L.orc_fmt_duration.argtypes = [C.c_int64, C.c_char_p, C.c_int]
        L.orc_fmt_rfc3339nano.argtypes = [C.c_int64, C.c_uint32, C.c_char_p, C.c_int]
        L.orc_serialize_to_string.argtypes = [C.POINTER(OrcVal), C.c_int32, C.c_char_p, C.c_int]
        L.orc_hmac_sha256_hex.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_char_p]
        L.orc_hmac_sha256_hex.restype = None
        L.orc_sha256.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p]
        L.orc_sha256.restype = None
        L.orc_cityhash128.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.orc_cityhash128.restype = None
        L.orc_lz4_bound.argtypes = [C.c_uint64]; L.orc_lz4_bound.restype = C.c_uint64
        L.orc_lz4_compress.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]; L.orc_lz4_compress.restype = C.c_uint64
        L.orc_lz4_decompress.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]; L.orc_lz4_decompress.restype = C.c_int64
        L.orc_match_value.argtypes = [C.POINTER(OrcVal), C.POINTER(OrcTerm), C.POINTER(C.c_int)]
        L.orc_ch_type.argtypes = [C.POINTER(OrcColSchema), C.c_char_p, C.c_int]
        L.orc_push_encode.argtypes = [C.POINTER(abi.TfBatch), C.POINTER(OrcColSchema), C.POINTER(OrcStep), C.c_int,
                                      C.c_int, C.c_uint64, C.POINTER(OrcBuf), C.POINTER(OrcBuf),
                                      C.POINTER(C.c_uint64), C.POINTER(abi.TfRowErr), C.POINTER(C.c_uint64)]
        L.orc_push_columns.argtypes = [C.POINTER(abi.TfBatch), C.POINTER(OrcColSchema), C.POINTER(OrcStep), C.c_int, C.POINTER(OrcBuf),
                                       C.POINTER(OrcRegions), C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(abi.TfRowErr), C.POINTER(C.c_uint64)]
        L.orc_csv_parse.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(OrcCsvOpts), C.POINTER(OrcBuf), C.POINTER(OrcRegions),
                                    C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(abi.TfRowErr), C.c_uint64, C.POINTER(C.c_uint64)]
        L.orc_json_parse.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(OrcJsonMsg), C.c_uint64, C.POINTER(C.c_char_p), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.POINTER(OrcJsonOpts), C.POINTER(OrcBuf), C.POINTER(OrcRegions), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                     C.POINTER(abi.TfRowErr), C.c_uint64, C.POINTER(C.c_uint64)]
        L.orc_queue_json_batches.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]
        L.orc_measure.argtypes = [C.POINTER(abi.TfBatch), C.c_void_p, C.POINTER(C.c_uint64)]
        L.orc_ch_decode_frames.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(OrcBuf), C.POINTER(C.c_uint64)]
        L.orc_free.argtypes = [C.POINTER(OrcBuf)]; L.orc_free.restype = None
        _lib = L
    return _lib


# ----------------------------------------------------------------------------- scalar helpers

def fmt_float64(v: float, fmt: int = 0) -> str:
    b = C.create_string_buffer(400); n = lib().orc_fmt_float64(v, fmt, b, 400); return b.raw[:n].decode()


def fmt_float32(v, fmt: int = 0) -> str:
    b = C.create_string_buffer(400); n = lib().orc_fmt_float32(float(np.float32(v)), fmt, b, 400); return b.raw[:n].decode()


def fmt_duration(ns: int) -> str:
    b = C.create_string_buffer(64); n = lib().orc_fmt_duration(ns, b, 64); return b.raw[:n].decode()


def fmt_rfc3339nano(sec: int, nsec: int = 0) -> str:
    b = C.create_string_buffer(64); n = lib().orc_fmt_rfc3339nano(sec, nsec, b, 64); return b.raw[:n].decode()


def make_val(kind: int, *, i: int = 0, u: int = 0, f: float = 0.0, s: bytes = b"", nsec: int = 0) -> OrcVal:
    v = OrcVal(); v.kind = kind; v.i = i; v.u = u; v.f = f; v.nsec = nsec
    v._s = s; v.s = s; v.slen = len(s)
    return v


def serialize_to_string(v: OrcVal, yt_type: int) -> bytes:
    b = C.create_string_buffer(1 << 16); n = lib().orc_serialize_to_string(C.byref(v), yt_type, b, 1 << 16); return b.raw[:n]


def hmac_hex(salt: bytes, msg: bytes) -> str:
    out = C.create_string_buffer(65); lib().orc_hmac_sha256_hex(salt, len(salt), msg, len(msg), out); return out.value.decode()


def cityhash128(data: bytes) -> Tuple[int, int]:
    lo, hi = C.c_uint64(), C.c_uint64()
    buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    lib().orc_cityhash128(buf, len(data), C.byref(lo), C.byref(hi)); return lo.value, hi.value


def lz4_compress(data: bytes) -> bytes:
    n = len(data); cap = lib().orc_lz4_bound(n)
    src = (C.c_uint8 * max(1, n)).from_buffer_copy(data or b"\0"); dst = (C.c_uint8 * cap)()
    c = lib().orc_lz4_compress(src, n, dst); return bytes(dst[:c])


def lz4_decompress(data: bytes, raw_len: int) -> Optional[bytes]:
    """The block of exactly raw_len bytes, or None when it is malformed or breaks an LZ4 end-of-block rule (lz4_block.hpp)."""
    src = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0"); dst = (C.c_uint8 * max(1, raw_len))()
    r = lib().orc_lz4_decompress(src, len(data), dst, raw_len)
    return None if r < 0 else bytes(dst[:r])


def ch_decode_frames(wire: bytes) -> Tuple[Optional[bytes], int]:
    src = (C.c_uint8 * max(1, len(wire))).from_buffer_copy(wire or b"\0")
    raw = OrcBuf(); nf = C.c_uint64()
    rc = lib().orc_ch_decode_frames(src, len(wire), C.byref(raw), C.byref(nf))
    if rc != 0:
        return None, 0
    out = C.string_at(raw.data, raw.len); lib().orc_free(C.byref(raw)); return out, nf.value


# ----------------------------------------------------------------------------- filter grammar
# grammar.go:256-266 — the lexer is literally this regexp, tried at every position, first alternative wins.
_LEX = re.compile(
    r"(?P<Operator>!=|<=|>=|!~|[=<>~])"
    r"|(?P<String>'((\\'|[^']))*'|\"(\\\"|[^\"])*\")"
    r"|(?P<DateTime>\d{4}-\d{2}-\d{2}(T\d{2}:\d{2}(:\d{2}(\.\d+)?)?(Z|[+-]\d+(:\d+)?)?)?)"
    r"|(?P<Ident>[a-zA-Z][a-zA-Z0-9_.]*)"
    r"|(?P<Float>[-+]?\d+\.\d+)"
    r"|(?P<Int>[-+]?\d+)"
    r"|(?P<Punctuation>[(),])"
    r"|(?P<WS>\s+)")


class FilterSyntaxError(ValueError):
    pass


def _unquote(tok: str) -> str:
    """participle.Unquote("String"): strconv.UnquoteChar over the body with the token's own quote."""
    q, body, out, i = tok[0], tok[1:-1], [], 0
    raw = body.encode("utf-8", "surrogateescape")
    res = bytearray()
    while i < len(raw):
        c = raw[i]
        if c != 0x5C:
            res.append(c); i += 1; continue
        i += 1
        if i >= len(raw):
            raise FilterSyntaxError("invalid syntax")
        e = chr(raw[i]); i += 1
        simple = {"a": 7, "b": 8, "f": 12, "n": 10, "r": 13, "t": 9, "v": 11, "\\": 0x5C}
        if e in simple:
            res.append(simple[e])
        elif e in ("'", '"'):
            if e != q:
                raise FilterSyntaxError("invalid syntax")
            res.append(ord(e))
        elif e == "x":
            res.append(int(raw[i:i + 2], 16)); i += 2
        elif e in "uU":
            n = 4 if e == "u" else 8
            res += chr(int(raw[i:i + n], 16)).encode(); i += n
        elif e in "01234567":
            res.append(int(raw[i - 1:i + 2], 8)); i += 2
        else:
            raise FilterSyntaxError("invalid syntax")
    return bytes(res)


_DAYS = [0, 31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]


def _days_from_civil(y, m, d):
    y -= m <= 2
    era = (y if y >= 0 else y - 399) // 400
    yoe = y - era * 400
    doy = (153 * (m - 3 if m > 2 else m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def parse_filter_time(value: str) -> int:
    """DateTime.delayedParse grammar.go:176-188 with findTimeLayout :120-149; returns UnixMicro."""
    m = re.fullmatch(r"(\d{4})-(\d{2})-(\d{2})(?:T(\d{2}):(\d{2})(?::(\d{2})(?:\.(\d+))?)?(Z|[+-]\d+(?::\d+)?)?)?", value)
    if not m:
        raise FilterSyntaxError("bad time " + value)
    y, mo, d = int(m[1]), int(m[2]), int(m[3])
    leap = (y % 4 == 0 and y % 100 != 0) or y % 400 == 0
    if not (1 <= mo <= 12) or not (1 <= d <= _DAYS[mo] + (1 if mo == 2 and leap else 0)):
        raise FilterSyntaxError("day out of range")
    hh = int(m[4] or 0); mi = int(m[5] or 0); ss = int(m[6] or 0)
    if hh > 23 or mi > 59 or ss > 59:
        raise FilterSyntaxError("time out of range")
    frac = (m[7] or "")
    nsec = int((frac + "000000000")[:9]) if frac else 0
    off = 0
    tz = m[8]
    if tz and tz != "Z":
        sign = -1 if tz[0] == "-" else 1
        if ":" in tz:
            h, mm = tz[1:].split(":")
            if len(h) != 2 or len(mm) != 2:
                raise FilterSyntaxError("bad zone")
            off = sign * (int(h) * 3600 + int(mm) * 60)
        else:
            if len(tz) != 3:
                raise FilterSyntaxError("bad zone")
            off = sign * int(tz[1:]) * 3600
    sec = _days_from_civil(y, mo, d) * 86400 + hh * 3600 + mi * 60 + ss - off
    return sec * 1_000_000 + nsec // 1000


@dataclass
class Term:
    attribute: str
    op: int
    vtype: int            # LV_* | LV_LIST
    value: Any            # python value / list


_OPS = {"=": OP_EQ, "!=": OP_NE, "<": OP_LT, "<=": OP_LE, ">": OP_GT, ">=": OP_GE, "~": OP_MATCH, "!~": OP_NOTMATCH}


def parse_filter(src: str) -> List[Term]:
    """filter.Parse (filters.go:293-313) over grammar.Parse (grammar.go:275-313)."""
    if src == "":
        return []
    toks: List[Tuple[str, str]] = []
    pos = 0
    while pos < len(src):
        m = _LEX.match(src, pos)
        if not m or m.end() == pos:
            raise FilterSyntaxError(f"invalid token at {pos}")
        kind = next(k for k in ("Operator", "String", "DateTime", "Ident", "Float", "Int", "Punctuation", "WS") if m.group(k) is not None)
        toks.append((kind, m.group(0))); pos = m.end()
    p = 0

    def peek(k=0):
        return toks[p + k] if p + k < len(toks) else ("EOF", "")

    def skip_ws():
        nonlocal p
        while peek()[0] == "WS":
            p += 1

    def is_kw(tok, *names):
        return tok[0] == "Ident" and tok[1].upper() in names

    def parse_value() -> Tuple[int, Any]:
        nonlocal p
        kind, text = peek()
        if kind == "String":
            p += 1; return LV_STRING, _unquote(text)
        if kind == "DateTime":
            p += 1; return LV_TIME, parse_filter_time(text)
        if is_kw((kind, text), "TRUE", "FALSE"):
            p += 1; return LV_BOOL, text.upper() == "TRUE"
        if kind == "Float":
            p += 1
            v = float(text)
            if math.isinf(v):                                   # strconv.ParseFloat: ErrRange beyond the float64 range
                raise FilterSyntaxError("value out of range")
            return LV_FLOAT, v
        if kind == "Int":
            p += 1
            v = int(text)
            if not (-(1 << 63) <= v < (1 << 63)):
                raise FilterSyntaxError("value out of range")
            return LV_INT, v
        if is_kw((kind, text), "NULL", "NIL"):
            p += 1; return LV_NULL, None
        if kind == "Punctuation" and text == "(":
            p += 1; skip_ws()
            items = [parse_value()]; skip_ws()
            while True:
                skip_ws()
                if peek() == ("Punctuation", ","):
                    p += 1; skip_ws(); items.append(parse_value()); skip_ws(); continue
                break
            if peek() != ("Punctuation", ")"):
                raise FilterSyntaxError(f"unexpected token {peek()[1]!r}")
            p += 1
            head = items[0][0]
            for i, it in enumerate(items):                      # validateTerm filters.go:255-270
                if it[0] != head:
                    raise FilterSyntaxError("list items should have same type")
                if it[0] & LV_LIST:
                    raise FilterSyntaxError("nested list are not supported")
            return head | LV_LIST, [it[1] for it in items]
        raise FilterSyntaxError(f"unexpected token {text!r}")

    def parse_term() -> Term:
        nonlocal p
        kind, text = peek()
        if kind != "Ident":
            raise FilterSyntaxError(f"unexpected token {text!r}")
        attr = text; p += 1; skip_ws()
        kind, text = peek()
        if kind == "Operator":
            op = _OPS[text]; p += 1
        elif is_kw((kind, text), "IN"):
            op = OP_IN; p += 1
        elif is_kw((kind, text), "NOT"):
            p += 1; skip_ws()
            if not is_kw(peek(), "IN"):
                raise FilterSyntaxError(f"unexpected token {peek()[1]!r}")
            op = OP_NOTIN; p += 1
        else:
            raise FilterSyntaxError(f"unexpected token {text!r}")
        skip_ws()
        vt, val = parse_value(); skip_ws()
        is_list = bool(vt & LV_LIST)
        if is_list and op not in (OP_IN, OP_NOTIN):
            raise FilterSyntaxError("list values require [ NOT ] IN operator")
        if not is_list and op in (OP_IN, OP_NOTIN):
            raise FilterSyntaxError("operator expect list value")
        if vt == LV_NULL and op not in (OP_EQ, OP_NE):
            raise FilterSyntaxError('NULL expects "=" or "!=" operator')
        return Term(attr, op, vt, val)

    terms: List[Term] = []
    skip_ws()
    if peek()[0] != "EOF":
        terms.append(parse_term())
        while True:
            skip_ws()
            if peek()[0] == "EOF":
                break
            if not is_kw(peek(), "AND"):
                raise FilterSyntaxError(f"unexpected token {peek()[1]!r}")
            p += 1; skip_ws()
            terms.append(parse_term())
    return terms


# ----------------------------------------------------------------------------- plan (Suitable / ResultSchema)

def _fqtn_variants(ns: str, name: str) -> List[str]:
    """transformer_common.go:9-23 + table_id.go:14-30."""
    full = name if ns == "" else f"{ns}.{name}"
    q = lambda s: '"' + s.replace('"', '""') + '"'
    parts = ([q(ns)] if ns else []) + ([name] if name == "*" else [q(name)])
    return [full, ".".join(parts)]


def _filter_match(include: List[str], exclude: List[str], value: str) -> bool:
    """filter.Filter.Match filter.go:27-44 (Go regexp ~ Python re for the anchored/simple patterns used in configs)."""
    for ex in exclude or []:
        if re.search(ex, value):
            return False
    if not include:
        return True
    return any(re.search(inc, value) for inc in include)


def _tables_match(tables_cfg: Optional[dict], ns: str, name: str) -> bool:
    inc = (tables_cfg or {}).get("includeTables") or (tables_cfg or {}).get("include_tables") or []
    exc = (tables_cfg or {}).get("excludeTables") or (tables_cfg or {}).get("exclude_tables") or []
    if not inc and not exc:
        return True
    return any(_filter_match(inc, exc, v) for v in _fqtn_variants(ns, name))


_NUMERIC = {"int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float", "double"}


def _column_suitable(term: Term, yt: str) -> bool:
    """checkColumnSuitable filter_rows.go:489-519."""
    base, is_list = term.vtype & 15, bool(term.vtype & LV_LIST)
    if is_list and base in (LV_INT, LV_FLOAT, LV_STRING, LV_TIME):
        return True
    if is_list:
        return False
    if base == LV_BOOL:
        return yt == "boolean"
    if base in (LV_FLOAT, LV_INT):
        return yt in _NUMERIC
    if base == LV_STRING:
        return yt in ("utf8", "string", "any")
    if base == LV_TIME:
        return yt in ("timestamp", "date", "datetime")
    if base == LV_NULL:
        return True
    return False


@dataclass
class Plan:
    schema: List[dict]                 # input ColSchema dicts
    result_schema: List[dict]
    steps: List[dict]                  # {"kind":..., "index": position among the kept transformers, ...}
    out_cols: List[int] = None         # input index of every surviving column
    result_table: Tuple[str, str] = None


def build_plan(ns: str, name: str, schema: List[dict], transformers: List[dict]) -> Plan:
    """transformation.AddTablePlan transformation.go:46-85. Suitable() is asked with the ORIGINAL table id for every
    transformer (:54); transformers that re-check item.TableID() inside Apply (filter_rows.go:109) see renames."""
    cur = [dict(c, _in=i) for i, c in enumerate(schema)]
    cur_ns, cur_name = ns, name
    steps: List[dict] = []
    idx = 0
    for tr in transformers:
        (ttype, cfg), = [(k, v) for k, v in tr.items() if k != "transformerId"]
        cfg = cfg or {}
        names = [c["name"] for c in cur]
        if ttype == "filter_rows":
            if cfg.get("filter") and cfg.get("filters"):
                raise ValueError("Settings 'filters' and 'filter' cannot be enabled at the same time")
            filters = cfg.get("filters") or [cfg.get("filter", "")]
            exprs = [parse_filter(f) for f in filters]
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            ok = True
            for terms in exprs:                                  # Suitable filter_rows.go:445-476
                for t in terms:
                    if t.attribute not in names or not _column_suitable(t, cur[names.index(t.attribute)]["type"]):
                        ok = False
            if not ok:
                continue
            steps.append({"kind": "filter_rows", "index": idx, "pass_all": not _tables_match(cfg.get("tables"), cur_ns, cur_name),
                          "exprs": [[(cur[names.index(t.attribute)]["_in"], t) for t in terms] for terms in exprs]}); idx += 1
        elif ttype == "skip_events":
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            mask = 0
            for ev in cfg.get("events") or []:
                mask |= {"insert": 1, "update": 2, "delete": 4}.get(ev, 0)
            steps.append({"kind": "skip_events", "index": idx, "kind_mask": mask}); idx += 1
        elif ttype == "filter_columns":
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            ccfg = cfg.get("columns") or {}
            inc = ccfg.get("includeColumns") or ccfg.get("include_columns") or []
            exc = ccfg.get("excludeColumns") or ccfg.get("exclude_columns") or []
            if any((not _filter_match(inc, exc, c["name"])) and c.get("key") for c in cur):   # validSchema :219-226
                continue
            cur = [c for c in cur if _filter_match(inc, exc, c["name"])]
            steps.append({"kind": "filter_columns", "index": idx, "keep": [c["_in"] for c in cur]}); idx += 1
        elif ttype == "replace_primary_key":                       # replace_primary_key.go:84-117 (Suitable :84-86, ResultSchema :88-117)
            keys = list(cfg.get("keys") or [])
            if len(set(keys)) != len(keys):
                raise ValueError("replace_primary_key: Can't use same keys column names twice")      # :133-137
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            if sum(1 for n_ in names if n_ in keys) != len(keys):
                continue
            if len(keys) == 1:
                cur = [dict(c, key=(c["name"] == keys[0])) for c in cur]
                steps.append({"kind": "replace_primary_key", "index": idx, "keep": None}); idx += 1
            else:
                by = {c["name"]: c for c in cur}
                cur = [dict(by[k], key=True) for k in keys] + [dict(c, key=False) for c in cur if c["name"] not in keys]
                steps.append({"kind": "replace_primary_key", "index": idx, "keep": [c["_in"] for c in cur]}); idx += 1
        elif ttype == "rename_tables":
            hit = None
            for r in cfg.get("renameTables") or []:
                o, nw = r.get("originalName") or {}, r.get("newName") or {}
                if o.get("nameSpace", "") == ns and o.get("name", "") == name:
                    hit = (nw.get("nameSpace", ""), nw.get("name", ""))
            if hit is None:
                continue
            nxt = None                                        # Apply: AltNames[current id] (rename.go:50-54), the last entry for an id wins
            for r in cfg.get("renameTables") or []:
                o, nw = r.get("originalName") or {}, r.get("newName") or {}
                if (o.get("nameSpace", ""), o.get("name", "")) == (cur_ns, cur_name):
                    nxt = (nw.get("nameSpace", ""), nw.get("name", ""))
            if nxt is not None:
                cur_ns, cur_name = nxt
            steps.append({"kind": "rename_tables", "index": idx}); idx += 1
        elif ttype == "mask_field":
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            cols = cfg.get("columns") or []
            if cols and not any(c in names for c in cols):       # hmac_hasher.go:76-89
                continue
            salt = ((cfg.get("maskFunctionHash") or {}).get("userDefinedSalt", ""))
            pos = [i for i, n_ in enumerate(names) if n_ in cols]
            steps.append({"kind": "mask_field", "index": idx, "cols": [cur[i]["_in"] for i in pos], "salt": salt.encode()}); idx += 1
            for i in pos:                                        # hmac_hasher.go:35-47
                cur[i] = dict(cur[i]); cur[i]["type"] = "utf8"; cur[i]["original_type"] = ""
        elif ttype == "convert_to_datetime":                     # to_datetime.go:56-135
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            ccfg = cfg.get("columns") or {}
            inc = ccfg.get("includeColumns") or []; exc = ccfg.get("excludeColumns") or []
            if not inc and not exc:
                continue
            pos = [i for i, c in enumerate(cur) if _filter_match(inc, exc, c["name"]) and c["type"] in ("int32", "uint32")]
            if not pos:
                continue
            steps.append({"kind": "convert_to_datetime", "index": idx, "cols": [cur[i]["_in"] for i in pos]}); idx += 1
            for i in pos:
                cur[i] = dict(cur[i]); cur[i]["type"] = "datetime"
        elif ttype == "number_to_float_transformer":             # number_to_float.go:54-125
            if not _tables_match(cfg.get("tables"), ns, name):
                continue                                             # Suitable :123-125 (original id)
            if not _tables_match(cfg.get("tables"), cur_ns, cur_name):
                idx += 1; continue                                   # Apply re-checks item.TableID() :62-66: a renamed table no longer matches
            pos = [i for i, c in enumerate(cur) if c["type"] == "any"]
            steps.append({"kind": "number_to_float", "index": idx, "cols": [cur[i]["_in"] for i in pos]}); idx += 1
        elif ttype == "sharder_transformer":                      # sharder.go:83-145
            if cfg.get("is_random"):
                raise NotImplementedError("sharder is_random: PartID is uuid + rand.Intn, host only")
            ccfg = cfg.get("columns") or {}
            inc = ccfg.get("includeColumns") or []; exc = ccfg.get("excludeColumns") or []
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            pos = [i for i, n_ in enumerate(names) if _filter_match(inc, exc, n_)]
            if (inc or exc) and not pos:
                continue                                             # Suitable :93-105
            shards = int(cfg.get("shardsCount"))
            if shards & 0xffffffff == 0:
                raise ValueError("sharder: shardsCount is zero modulo 2^32 (the reference divides by zero)")
            steps.append({"kind": "sharder", "index": idx, "cols": [cur[i]["_in"] for i in pos], "shards": shards & 0xffffffff}); idx += 1
        elif ttype == "convert_to_string":
            if not _tables_match(cfg.get("tables"), ns, name):
                continue
            ccfg = cfg.get("columns") or {}
            inc = ccfg.get("includeColumns") or []; exc = ccfg.get("excludeColumns") or []
            pos = [i for i, n_ in enumerate(names) if _filter_match(inc, exc, n_)]
            if (inc or exc) and not pos:
                continue
            to_bytes = bool(cfg.get("convert_to_bytes"))
            steps.append({"kind": "convert_to_string", "index": idx, "cols": [cur[i]["_in"] for i in pos], "to_bytes": to_bytes}); idx += 1
            for i in pos:
                cur[i] = dict(cur[i]); cur[i]["type"] = "string" if to_bytes else "utf8"
        else:
            raise NotImplementedError(ttype)
    return Plan(schema, [{k: v for k, v in c.items() if k != "_in"} for c in cur], steps, [c["_in"] for c in cur], (cur_ns, cur_name))


# ----------------------------------------------------------------------------- marshaling to liboracle

class _Keep:
    def __init__(self):
        self.refs = []

    def add(self, x):
        self.refs.append(x); return x


def term_to_c(col: int, t: Term, keep: _Keep) -> OrcTerm:
    ct = OrcTerm(); ct.col = col; ct.op = t.op; ct.vtype = t.vtype; ct.nlist = 0
    base, is_list = t.vtype & 15, bool(t.vtype & LV_LIST)
    if not is_list:
        if base == LV_INT or base == LV_TIME:
            ct.i = t.value
        elif base == LV_BOOL:
            ct.i = 1 if t.value else 0
        elif base == LV_FLOAT:
            ct.f = t.value
        elif base == LV_STRING:
            b = keep.add(bytes(t.value)); ct.s = b; ct.slen = len(b)
    else:
        ct.nlist = len(t.value)
        if base in (LV_INT, LV_TIME):
            a = keep.add(np.asarray(t.value, dtype=np.int64)); ct.ilist = a.ctypes.data
        elif base == LV_FLOAT:
            a = keep.add(np.asarray(t.value, dtype=np.float64)); ct.flist = a.ctypes.data
        elif base == LV_STRING:
            offs = keep.add(np.zeros(len(t.value) + 1, dtype=np.uint32)); np.cumsum([len(x) for x in t.value], out=offs[1:])
            heap = keep.add(np.frombuffer(b"".join(t.value) or b"\0", dtype=np.uint8).copy())
            ct.soffs = offs.ctypes.data; ct.sheap = heap.ctypes.data
    return ct


def match_value(v: OrcVal, t: Term) -> Tuple[int, bool]:
    keep = _Keep(); ct = term_to_c(0, t, keep); m = C.c_int(0)
    rc = lib().orc_match_value(C.byref(v), C.byref(ct), C.byref(m)); return rc, bool(m.value)


def _schema_to_c(schema: List[dict], keep: _Keep):
    arr = (OrcColSchema * len(schema))()
    for i, c in enumerate(schema):
        arr[i].name = keep.add(c["name"].encode())
        arr[i].type = abi.YT_NAME_TO_TF[c["type"]]
        arr[i].required = 1 if c.get("required") else 0
        arr[i].original_type = keep.add((c.get("original_type") or "").encode())
    return arr


def ch_type(col: dict) -> str:
    keep = _Keep(); arr = _schema_to_c([col], keep); b = C.create_string_buffer(128)
    n = lib().orc_ch_type(arr, b, 128); return b.raw[:n].decode()


@dataclass
class PushResult:
    rows_out: int
    raw: bytes
    wire: bytes
    errors: List[Tuple[int, int, int]]
    raw_len: int = 0
    wire_len: int = 0


def _marshal(plan: Plan):
    keep = _Keep()
    cschema = _schema_to_c(plan.schema, keep)
    csteps = (OrcStep * max(1, len(plan.steps)))()
    for si, st in enumerate(plan.steps):
        s = csteps[si]
        if st["kind"] == "filter_rows":
            flat = [(c, t) for terms in st["exprs"] for (c, t) in terms]
            tarr = keep.add((OrcTerm * max(1, len(flat)))())
            for k, (c, t) in enumerate(flat):
                tarr[k] = term_to_c(c, t, keep)
            off = keep.add(np.zeros(len(st["exprs"]) + 1, dtype=np.uint32)); np.cumsum([len(x) for x in st["exprs"]], out=off[1:])
            s.kind = STEP_FILTER_ROWS; s.terms = C.cast(tarr, C.POINTER(OrcTerm)); s.expr_off = off.ctypes.data; s.nexpr = len(st["exprs"])
            s.pass_all = 1 if st.get("pass_all") else 0; s.convert_to_bytes = st["index"]     # (reused as the step's transformer index in error rows)
        elif st["kind"] == "convert_to_datetime":
            cols = keep.add(np.asarray(st["cols"], dtype=np.int32))
            s.kind = STEP_TO_DATETIME; s.cols = cols.ctypes.data; s.ncols = len(st["cols"])
        elif st["kind"] == "number_to_float":
            cols = keep.add(np.asarray(st["cols"], dtype=np.int32))
            s.kind = STEP_NUMBER_TO_FLOAT; s.cols = cols.ctypes.data; s.ncols = len(st["cols"])
        elif st["kind"] == "sharder":
            cols = keep.add(np.asarray(st["cols"], dtype=np.int32))
            s.kind = STEP_SHARDER; s.cols = cols.ctypes.data; s.ncols = len(st["cols"]); s.kind_mask = C.c_int32(st["shards"] & 0xffffffff).value
        elif st["kind"] == "skip_events":
            s.kind = STEP_SKIP_EVENTS; s.kind_mask = st["kind_mask"]
        elif st["kind"] == "filter_columns":
            cols = keep.add(np.asarray(st["keep"], dtype=np.int32))
            s.kind = STEP_SELECT_COLS; s.cols = cols.ctypes.data; s.ncols = len(st["keep"])
        elif st["kind"] == "replace_primary_key":
            if st["keep"] is None:
                s.kind = 0
            else:                                                        # the reordered schema: the same column selection step filter_columns uses
                cols = keep.add(np.asarray(st["keep"], dtype=np.int32))
                s.kind = STEP_SELECT_COLS; s.cols = cols.ctypes.data; s.ncols = len(st["keep"])
        elif st["kind"] == "rename_tables":
            s.kind = 0
        elif st["kind"] == "mask_field":
            cols = keep.add(np.asarray(st["cols"], dtype=np.int32))
            s.kind = STEP_MASK; s.cols = cols.ctypes.data; s.ncols = len(st["cols"]); s.salt = keep.add(st["salt"]); s.salt_len = len(st["salt"])
        elif st["kind"] == "convert_to_string":
            cols = keep.add(np.asarray(st["cols"], dtype=np.int32))
            s.kind = STEP_TO_STRING; s.cols = cols.ctypes.data; s.ncols = len(st["cols"]); s.convert_to_bytes = 1 if st["to_bytes"] else 0
    return keep, cschema, csteps


def push_encode(batch: abi.Batch, plan: Plan, wire_fmt: int, frame_bytes: int = 32768, want_bytes: bool = True) -> PushResult:
    """Row-at-a-time reference path over one batch: transformers -> Restore -> native block -> LZ4 frames."""
    keep, cschema, csteps = _marshal(plan)
    tb = batch.as_struct()
    raw, wire = OrcBuf(), OrcBuf()
    rows = C.c_uint64(); nerr = C.c_uint64()
    errs = (abi.TfRowErr * max(1, batch.nrows))()
    rc = lib().orc_push_encode(C.byref(tb), cschema, csteps, len(plan.steps), wire_fmt, frame_bytes,
                               C.byref(raw), C.byref(wire), C.byref(rows), errs, C.byref(nerr))
    if rc != 0:
        raise RuntimeError(f"oracle push_encode rc={rc}")
    res = PushResult(rows.value,
                     C.string_at(raw.data, raw.len) if (want_bytes and raw.len) else b"",
                     C.string_at(wire.data, wire.len) if (want_bytes and wire.len) else b"",
                     [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)])
    res.raw_len = raw.len; res.wire_len = wire.len
    lib().orc_free(C.byref(raw)); lib().orc_free(C.byref(wire))
    return res


def shard_ids(batch: abi.Batch, plan: Plan):
    """ChangeItem.PartID (as the integer the sharder prints) of every row the chain keeps; 0xFFFFFFFF without a sharder."""
    keep, cschema, csteps = _marshal(plan)
    tb = batch.as_struct()
    out = np.zeros(max(1, batch.nrows), dtype=np.uint32); rows = C.c_uint64()
    L = lib()
    L.orc_shard_ids.argtypes = [C.POINTER(abi.TfBatch), C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_uint64)]
    rc = L.orc_shard_ids(C.byref(tb), C.cast(cschema, C.c_void_p), C.cast(csteps, C.c_void_p), len(plan.steps), out.ctypes.data, C.byref(rows))
    if rc != 0:
        raise RuntimeError(f"oracle shard_ids rc={rc}")
    return out[:rows.value].copy()


def crc32_ieee(data: bytes) -> int:
    L = lib(); L.orc_crc32_ieee.argtypes = [C.c_char_p, C.c_uint64]; L.orc_crc32_ieee.restype = C.c_uint32
    return int(L.orc_crc32_ieee(data, len(data)))


def push_columns(batch: abi.Batch, plan: Plan):
    """TransformerResult of the chain: (Batch of Transformed rows, errors)."""
    keep, cschema, csteps = _marshal(plan)
    tb = batch.as_struct()
    no = len(plan.out_cols)
    out = OrcBuf(); regs = (OrcRegions * max(1, no))(); types = (C.c_int32 * max(1, no))()
    rows = C.c_uint64(); nerr = C.c_uint64()
    errs = (abi.TfRowErr * max(1, batch.nrows))()
    rc = lib().orc_push_columns(C.byref(tb), cschema, csteps, len(plan.steps), C.byref(out), regs, types, C.byref(rows), errs, C.byref(nerr))
    if rc != 0:
        raise RuntimeError(f"oracle push_columns rc={rc}")
    buf = C.string_at(out.data, out.len) if out.len else b""
    lib().orc_free(C.byref(out))
    n = rows.value
    NONE = 2 ** 64 - 1
    cols = []
    for k in range(no):
        g, t = regs[k], types[k]
        def arr(off, nbytes, dtype):
            if off == NONE:
                return None
            return np.frombuffer(buf[off:off + nbytes], dtype=dtype).copy()
        if t in abi.VAR_TYPES:
            cols.append(abi.Column(t, offsets=arr(g.offsets, 4 * (n + 1), np.uint32), heap=arr(g.heap, g.heap_len, np.uint8),
                                   validity=arr(g.validity, (n + 7) // 8, np.uint8), aux=arr(g.aux, n, np.uint8)))
        else:
            dt = abi.FIXED_DTYPE[t]
            cols.append(abi.Column(t, values=arr(g.values, n * np.dtype(dt).itemsize, dt), validity=arr(g.validity, (n + 7) // 8, np.uint8),
                                   aux=arr(g.aux, 4 * n, np.uint32)))
    return abi.Batch(n, cols), [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)]


def _regions_to_batch(buf: bytes, regs, types, n: int) -> abi.Batch:
    NONE = 2 ** 64 - 1
    cols = []
    for k, t in enumerate(types):
        g = regs[k]
        def arr(off, nbytes, dtype):
            if off == NONE:
                return None
            return np.frombuffer(buf[off:off + nbytes], dtype=dtype).copy()
        if t in abi.VAR_TYPES:
            cols.append(abi.Column(t, offsets=arr(g.offsets, 4 * (n + 1), np.uint32), heap=arr(g.heap, g.heap_len, np.uint8),
                                   validity=arr(g.validity, (n + 7) // 8, np.uint8), aux=arr(g.aux, n, np.uint8)))
        else:
            dt = abi.FIXED_DTYPE[t]
            cols.append(abi.Column(t, values=arr(g.values, n * np.dtype(dt).itemsize, dt), validity=arr(g.validity, (n + 7) // 8, np.uint8),
                                   aux=arr(g.aux, 4 * n, np.uint32)))
    return abi.Batch(n, cols)


def csv_options(opts: Optional[dict], keep: "_Keep") -> OrcCsvOpts:
    opts = opts or {}
    o = OrcCsvOpts()
    q = opts.get("quote", '"'); e = opts.get("escape", "\\")
    o.delimiter = ord(opts.get("delimiter", ",")); o.quote = ord(q) if q else 0
    o.escape = ord(e) if e else 0
    o.double_quote = 1 if opts.get("double_quote", True) else 0
    o.strings_can_be_null = 1 if opts.get("strings_can_be_null") else 0
    o.quoted_strings_can_be_null = 1 if opts.get("quoted_strings_can_be_null") else 0
    o.include_missing = 1 if opts.get("include_missing_columns") else 0
    for k in ("null_values", "true_values", "false_values"):
        v = opts.get(k)
        setattr(o, k, keep.add("\n".join(v).encode()) if v else None)
    o.skip_lines = int(opts.get("skip_lines", 0))
    return o


def csv_parse(data: bytes, schema: List[dict], opts: Optional[dict] = None):
    """Reference CSV path over one chunk of bytes -> (Batch, errors[(data line, code, 0)], lines, consumed)."""
    keep = _Keep()
    o = csv_options(opts, keep)
    types = keep.add(np.asarray([abi.YT_NAME_TO_TF[c["type"]] for c in schema], dtype=np.int32))
    paths = keep.add(np.asarray([int(c.get("path", i)) if str(c.get("path", "")) != "" else i for i, c in enumerate(schema)], dtype=np.int32))
    src = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    out = OrcBuf(); regs = (OrcRegions * max(1, len(schema)))()
    rows, lines, consumed, nerr = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    cap = data.count(b"\n") + 1
    errs = (abi.TfRowErr * cap)()
    rc = lib().orc_csv_parse(src, len(data), types.ctypes.data, paths.ctypes.data, len(schema), C.byref(o), C.byref(out), regs,
                             C.byref(rows), C.byref(lines), C.byref(consumed), errs, cap, C.byref(nerr))
    assert rc == 0
    buf = C.string_at(out.data, out.len) if out.len else b""
    lib().orc_free(C.byref(out))
    return (_regions_to_batch(buf, regs, list(types), rows.value), [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)],
            lines.value, consumed.value)


# ----------------------------------------------------------------------------- generic JSON parser
JSON_FIELD_TYPES = ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "double", "boolean", "utf8", "string", "any", "datetime")


def json_result_schema(fields: List[dict], opts: Optional[dict] = None) -> List[dict]:
    """addAuxFields (generic_parser.go:115-164): the parser's result schema for declared `fields`."""
    opts = opts or {}
    out = [dict(f) for f in fields]
    for f in out:
        if f["type"] not in JSON_FIELD_TYPES:
            raise ValueError(f"json parser: field type {f['type']} is not handled")
        if f.get("path"):
            raise ValueError("json parser: nested paths are not handled")
        if f.get("key"):
            f["required"] = True
    def dedup(name):
        while any(c["name"] == name for c in out):
            name = "_delivery_" + name
        return name
    if opts.get("add_rest"):
        out.append({"name": dedup("_rest"), "type": "any"})
    if opts.get("add_dedupe_keys"):
        sys_key = not (opts.get("mark_dedupe_keys_as_system") and any(f.get("key") for f in fields))
        for n, t in (("_timestamp", "timestamp"), ("_partition", "string"), ("_offset", "uint64"), ("_idx", "uint32")):
            out.append({"name": dedup(n), "type": t, "key": sys_key, "required": sys_key})
    return out


def json_parse(data: bytes, fields: List[dict], opts: Optional[dict] = None, msgs: Optional[list] = None):
    """Reference generic JSON parser over concatenated messages -> (Batch of the result schema, errors[(line, code, col)], lines).
    msgs: [(end, offset, write_sec, write_nsec)], default = one message covering `data` with offset 0 / time 0."""
    opts = opts or {}
    schema = json_result_schema(fields, opts)
    msgs = msgs if msgs is not None else [(len(data), 0, 0, 0)]
    keep = _Keep()
    o = OrcJsonOpts()
    o.add_rest = 1 if opts.get("add_rest") else 0; o.add_dedupe_keys = 1 if opts.get("add_dedupe_keys") else 0
    o.null_keys_allowed = 1 if opts.get("null_keys_allowed") else 0; o.use_numbers_in_any = 1 if opts.get("use_numbers_in_any") else 0
    o.unpack_bytes_base64 = 1 if opts.get("unpack_bytes_base64") else 0
    o.partition = keep.add(opts.get("partition", "").encode())
    nc = len(schema)
    names = (C.c_char_p * nc)(*[c["name"].encode() for c in schema])
    types = keep.add(np.asarray([abi.YT_NAME_TO_TF[c["type"]] for c in schema], dtype=np.int32))
    keys = keep.add(np.asarray([1 if c.get("key") else 0 for c in schema], dtype=np.uint8))
    req = keep.add(np.asarray([1 if c.get("required") else 0 for c in schema], dtype=np.uint8))
    ms = (OrcJsonMsg * max(1, len(msgs)))()
    for k, (end, off, ws, wn) in enumerate(msgs):
        ms[k].end, ms[k].offset, ms[k].write_sec, ms[k].write_nsec = end, off, ws, wn
    src = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    out = OrcBuf(); regs = (OrcRegions * nc)()
    rows, lines, nerr = C.c_uint64(), C.c_uint64(), C.c_uint64()
    cap = data.count(b"\n") + len(msgs) + 1
    errs = (abi.TfRowErr * cap)()
    rc = lib().orc_json_parse(src, len(data), ms, len(msgs), names, types.ctypes.data, keys.ctypes.data, req.ctypes.data, nc, C.byref(o),
                              C.byref(out), regs, C.byref(rows), C.byref(lines), errs, cap, C.byref(nerr))
    assert rc == 0
    buf = C.string_at(out.data, out.len) if out.len else b""
    lib().orc_free(C.byref(out))
    return (_regions_to_batch(buf, regs, list(types), rows.value), [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)], lines.value)


def measure(batch: abi.Batch):
    """Measurer middleware: (per-row Size.Values, total)."""
    tb = batch.as_struct(); per = np.zeros(batch.nrows, dtype=np.uint64); tot = C.c_uint64()
    assert lib().orc_measure(C.byref(tb), per.ctypes.data, C.byref(tot)) == 0
    return per, tot.value


def queue_json_batches(lens, max_message_size=0, max_change_items=0):
    """BatchJSON: start row of every message (+ n at the end)."""
    a = np.asarray(lens, dtype=np.uint64); st = np.zeros(len(a) + 1, dtype=np.uint64); k = C.c_uint64()
    assert lib().orc_queue_json_batches(a.ctypes.data, len(a), max_message_size, max_change_items, st.ctypes.data, C.byref(k)) == 0
    return [int(x) for x in st[:k.value + 1]]


def queue_debezium_merge(values, max_message_size):
    """MergeWithMaxMessageSize (pkg/serializer/queue/debezium_multithreading.go:67-106) over the values of one TablePartID, restated
    literally: the merged message values."""
    out = []
    for v in values:
        if not out or len(out[-1]) + 1 + len(v) > max_message_size:      # expandArrIfNeeded :76-86
            out.append(b"")
        out[-1] += v
    return out


# ----------------------------------------------------------------------------- debezium
class OrcDbzField(C.Structure):
    _fields_ = [("name", C.c_char_p), ("recv", C.c_int32), ("scale", C.c_int32), ("key", C.c_int32)]


class OrcDbzOpts(C.Structure):
    _fields_ = [("schema_text", C.c_char_p), ("schema_len", C.c_uint64), ("use_sr", C.c_uint8), ("check_table", C.c_uint8), ("pad", C.c_uint8 * 2),
                ("schema_id", C.c_uint32), ("table_schema", C.c_char_p), ("table_name", C.c_char_p)]


(R_INT8, R_INT16, R_INT32, R_INT64, R_BOOL, R_STRING, R_F64, R_BYTES, R_DECIMAL, R_POINT, R_VSD) = range(1, 12)
_RECV_YT = {R_INT8: "int8", R_INT16: "int16", R_INT32: "int32", R_INT64: "int64", R_BOOL: "boolean", R_STRING: "utf8", R_F64: "double", R_BYTES: "string",
            R_DECIMAL: "utf8", R_POINT: "utf8", R_VSD: "double"}


def debezium_fields(schema_text: str, which: str = "after"):
    """receiveTableSchema / receiveFieldColSchema (pkg/debezium/receiver.go:46-62, receiver_engine.go:104-141) with the DEFAULT
    receivers (common/field_receiver_default.go:15-30): [(name, receiver, scale, key)], and the yt schema of the result."""
    import json as _json
    sch = _json.loads(schema_text)
    node = next((f for f in sch.get("fields", []) if f.get("field") == which), None)
    if node is None:
        raise ValueError(f"schema has no '{which}' struct")
    out = []
    for f in node.get("fields", []):
        if (f.get("__dt_original_type_info") or {}).get("original_type"):
            raise ValueError("database specific receivers are not handled")
        kt, nm = f.get("type"), f.get("name", "")
        scale = 0
        if kt in ("int8", "int16", "int32", "int64"): recv = {"int8": R_INT8, "int16": R_INT16, "int32": R_INT32, "int64": R_INT64}[kt]
        elif kt == "boolean": recv = R_BOOL
        elif kt == "string": recv = R_STRING
        elif kt in ("float", "double"): recv = R_F64
        elif kt == "bytes":
            if nm == "org.apache.kafka.connect.data.Decimal":
                recv = R_DECIMAL; sc = (f.get("parameters") or {}).get("scale", "")
                scale = int(sc) if sc != "" else 0
            else: recv = R_BYTES
        elif kt == "struct" and nm == "io.debezium.data.geometry.Point": recv = R_POINT
        elif kt == "struct" and nm == "io.debezium.data.VariableScaleDecimal": recv = R_VSD
        else: raise ValueError(f"kafka type {kt} / {nm} has no default receiver handled here")
        out.append((f["field"], recv, scale, not f.get("optional", False)))
    schema = [{"name": n, "type": _RECV_YT[r], "key": k} for n, r, _, k in out]
    return out, schema


def debezium_parse(data: bytes, msg_ends, schema_text: str, use_sr: bool = False, schema_id: int = 0, table=None):
    """Reference debezium parser over concatenated messages -> (Batch, kinds, tx_ids, lsns, commit_times, row_msg, errors)."""
    fields, schema = debezium_fields(schema_text)
    if debezium_fields(schema_text, "before")[0] != fields:
        raise ValueError("before / after structs differ")
    nf = len(fields); nm = len(msg_ends)
    fa = (OrcDbzField * max(1, nf))()
    keep = _Keep()
    for k, (n, r, sc, key) in enumerate(fields):
        fa[k].name = keep.add(n.encode()); fa[k].recv = r; fa[k].scale = sc; fa[k].key = 1 if key else 0
    o = OrcDbzOpts(); st = keep.add(schema_text.encode()); o.schema_text = st; o.schema_len = len(st); o.use_sr = 1 if use_sr else 0; o.schema_id = schema_id
    if table: o.check_table = 1; o.table_schema = keep.add(table[0].encode()); o.table_name = keep.add(table[1].encode())
    ends = keep.add(np.asarray(msg_ends, dtype=np.uint64))
    src = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    out = OrcBuf(); regs = (OrcRegions * max(1, nf))(); types = np.zeros(max(1, nf), dtype=np.int32)
    kinds = np.zeros(nm, dtype=np.uint8); tx = np.zeros(nm, dtype=np.uint32); lsn = np.zeros(nm, dtype=np.uint64); ct = np.zeros(nm, dtype=np.uint64); rm = np.zeros(nm, dtype=np.uint32)
    rows, nerr = C.c_uint64(), C.c_uint64(); errs = (abi.TfRowErr * max(1, nm))()
    L = lib()
    L.orc_debezium_parse.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(OrcDbzField), C.c_int, C.POINTER(OrcDbzOpts), C.POINTER(OrcBuf), C.POINTER(OrcRegions),
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(abi.TfRowErr), C.POINTER(C.c_uint64)]
    rc = L.orc_debezium_parse(src, len(data), ends.ctypes.data, nm, fa, nf, C.byref(o), C.byref(out), regs, types.ctypes.data, kinds.ctypes.data, tx.ctypes.data, lsn.ctypes.data,
                              ct.ctypes.data, rm.ctypes.data, C.byref(rows), errs, C.byref(nerr))
    assert rc == 0
    buf = C.string_at(out.data, out.len) if out.len else b""
    L.orc_free(C.byref(out))
    n = rows.value
    return (_regions_to_batch(buf, regs, [int(t) for t in types[:nf]], n), kinds[:n].copy(), tx[:n].copy(), lsn[:n].copy(), ct[:n].copy(), rm[:n].copy(),
            [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)], schema)


def base64_to_numeric(b64: str, scale: int) -> str:
    L = lib(); L.orc_base64_to_numeric.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
    b = C.create_string_buffer(4096); n = L.orc_base64_to_numeric(b64.encode(), scale, b, 4096)
    if n < 0: raise ValueError(f"base64_to_numeric rc {n}")
    return b.raw[:n].decode()


# ----------------------------------------------------------------------------- Debezium emitter

class OrcDbzEmitOpts(C.Structure):
    _fields_ = [("version", C.c_char_p), ("name", C.c_char_p), ("database", C.c_char_p), ("schema", C.c_char_p), ("table", C.c_char_p),
                ("source_type", C.c_int32), ("snapshot", C.c_uint8), ("drop_keys", C.c_uint8), ("pad", C.c_uint8 * 2),
                ("key_schema", C.c_char_p), ("val_schema", C.c_char_p), ("key_schema_id", C.c_int64), ("val_schema_id", C.c_int64)]


_DBZ_SOURCE = {"": 0, None: 0, "pg": 1, "mysql": 2}


_PG_STRING_TYPES = {"pg:text", "pg:uuid", "pg:cidr", "pg:macaddr", "pg:citext", "pg:int4range", "pg:int8range", "pg:character", "pg:character varying"}


def debezium_pg_form(col: dict) -> int:
    """The AddPg branch (pkg/debezium/pg/emitter.go:265-629) the emitter takes for a result column: 0 = addCommon (no original type, or
    a pg type whose branch stores the typed value unchanged); -1 = a type or (type, column type) pair left to the Go emitter."""
    import re
    ot, yt = col.get("original_type") or "", col["type"]
    if not ot.startswith(("pg:", "mysql:", "ydb:")):
        return 0
    same = {"pg:boolean": "boolean", "pg:smallint": "int16", "pg:integer": "int32", "pg:bigint": "int64", "pg:bytea": "string"}
    if ot in same:
        return 0 if yt == same[ot] else -1
    if ot == "pg:real":
        return 2 if yt in ("double", "float") else -1
    if ot == "pg:double precision":
        return 3 if yt == "double" else -1
    if ot in _PG_STRING_TYPES or re.fullmatch(r"pg:character( varying)?\(\d+\)", ot):
        return 4 if yt in ("utf8", "any") else -1
    if ot in ("pg:json", "pg:jsonb"):
        return 6 if yt == "any" else -1
    if ot == "pg:inet":
        return 11 if yt in ("utf8", "any") else -1
    if ot == "pg:date":
        return 7 if yt == "date" else -1
    m = re.fullmatch(r"pg:timestamp(?:\((\d)\))? without time zone", ot)
    if m:
        if yt != "timestamp":
            return -1
        return 9 if (m.group(1) and 1 <= int(m.group(1)) <= 3) else 8          # GetTimeDivider typeutil/helpers.go:104-120
    if re.fullmatch(r"pg:timestamp(?:\([0-6]\))? with time zone", ot):
        return 10 if yt == "timestamp" else -1
    return -1


def debezium_emit(batch: abi.Batch, plan: Plan, opts: dict, meta: Optional[dict] = None, old: Optional[abi.Batch] = None, old_present=None, old_row_has=None, want_msg_sizes: bool = False):
    """Emitter.EmitKV over the rows of `batch` after the plan's chain (emitter_value_converter.go:626-690), every row kind; OldKeys as a
    second batch. Returns (messages bytes, key_sizes, row_sizes, errors[, msg_sizes (rows x 7)])."""
    L = lib()
    keep, cschema, csteps = _marshal(plan)
    tb = batch.as_struct()
    key_by_name = {c["name"]: bool(c.get("key")) for c in plan.result_schema}
    is_key = np.zeros(len(plan.schema), dtype=np.uint8)
    forms = np.zeros(len(plan.schema), dtype=np.uint8)
    for k, ci in enumerate(plan.out_cols):
        is_key[ci] = 1 if key_by_name.get(plan.result_schema[k]["name"]) else 0
        f = debezium_pg_form(plan.result_schema[k])
        if f < 0:
            raise NotImplementedError(f"column {plan.result_schema[k]['name']}: original type {plan.result_schema[k].get('original_type')} is emitted by the Go emitter")
        forms[ci] = f
    meta = meta or {}
    m, mkeep = abi.make_row_meta(meta.get("id"), meta.get("lsn"), meta.get("commit_time"), meta.get("txid_offsets"), meta.get("txid_heap"))
    o = OrcDbzEmitOpts()
    enc = lambda v: None if v is None else keep.add(str(v).encode())
    o.version = enc(opts.get("version", "")); o.name = enc(opts.get("topic_prefix", "")); o.database = enc(opts.get("database", ""))
    o.schema = enc(plan.result_table[0]); o.table = enc(plan.result_table[1])
    o.source_type = _DBZ_SOURCE[opts.get("source_type", "")]; o.snapshot = 1 if opts.get("snapshot") else 0; o.drop_keys = 1 if opts.get("drop_keys") else 0
    o.key_schema = enc(opts.get("key_schema")); o.val_schema = enc(opts.get("val_schema"))
    o.key_schema_id = opts["key_schema_id"] if opts.get("key_schema_id") is not None else -1
    o.val_schema_id = opts["val_schema_id"] if opts.get("val_schema_id") is not None else -1
    n = batch.nrows
    ks = np.zeros(max(1, n), dtype=np.uint32); rs = np.zeros(max(1, n), dtype=np.uint32)
    out = OrcBuf(); rows = C.c_uint64(); nerr = C.c_uint64()
    errs = (abi.TfRowErr * max(1, 2 * n))()
    ms = np.zeros((max(1, n), 7), dtype=np.uint32)
    ok, okeep = (abi.make_old_keys(old, old_present or [], old_row_has) if old is not None else (None, None))
    tomb = 0 if opts.get("tombstones_on_delete") is False else 1
    L.orc_debezium_emit_crud.argtypes = [C.POINTER(abi.TfBatch), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(abi.TfRowMeta), C.POINTER(OrcDbzEmitOpts),
                                         C.POINTER(OrcBuf), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]
    rc = L.orc_debezium_emit_crud(C.byref(tb), C.cast(C.pointer(ok), C.c_void_p) if ok is not None else None, tomb, C.cast(cschema, C.c_void_p), is_key.ctypes.data, forms.ctypes.data,
                                  C.cast(csteps, C.c_void_p), len(plan.steps), C.byref(m), C.byref(o),
                                  C.byref(out), ks.ctypes.data, rs.ctypes.data, ms.ctypes.data, C.byref(rows), C.cast(errs, C.c_void_p), C.byref(nerr))
    if rc != 0:
        raise RuntimeError(f"oracle debezium_emit rc={rc}")
    data = C.string_at(out.data, out.len) if out.len else b""
    L.orc_free(C.byref(out))
    k = rows.value
    res = (data, ks[:k].copy(), rs[:k].copy(), [(errs[i].row, errs[i].code, errs[i].term) for i in range(nerr.value)])
    return res + (ms[:k].copy(),) if want_msg_sizes else res


def debezium_messages(data: bytes, msg_sizes):
    """[[(key bytes, value bytes | None), ...] per row] of a CRUD emission."""
    out = []; at = 0
    for row in msg_sizes:
        msgs = []
        for m in range(int(row[0])):
            k, v = int(row[1 + 2 * m]), int(row[2 + 2 * m])
            key = data[at:at + k]; at += k
            if v == 0xffffffff: msgs.append((key, None))
            else: msgs.append((key, data[at:at + v])); at += v
        out.append(msgs)
    return out


def debezium_split(data: bytes, key_sizes, row_sizes):
    """[(key bytes, value bytes)] of a debezium_emit / tfgpu_emit_debezium result."""
    out = []; at = 0
    for k, r in zip(key_sizes, row_sizes):
        out.append((data[at:at + int(k)], data[at + int(k):at + int(r)])); at += int(r)
    return out


# ---------------------------------------------------------------- typesystem casts over boxed Go values (cast_oracle.hpp)
def _goval_call(fn, go: str, v, third):
    L = lib()
    raw = bytes.fromhex(v) if go == "[]byte" else (v.encode("utf-8") if isinstance(v, str) else bytes(v))
    og = C.create_string_buffer(32); ov = C.create_string_buffer(max(4096, 4 * len(raw) + 64)); on = C.c_uint64()
    f = getattr(L, fn); f.restype = C.c_int
    f.argtypes = [C.c_char_p, C.c_char_p, C.c_uint64, (C.c_int32 if fn == "orc_strictify_value" else C.c_char_p), C.c_char_p, C.c_int, C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64)]
    rc = f(go.encode(), raw, len(raw), third, og, 32, ov, len(ov), C.byref(on))
    g = og.value.decode(); val = ov.raw[:on.value]
    return rc, {"go": g, "v": val.hex() if g == "[]byte" else val.decode("utf-8")}


def strictify_value(go: str, v, tf: int):
    """strictify.strictifyValue over one boxed Go value: (rc, {"go", "v"}); rc 0 ok, 1 cast error, 2 range error."""
    return _goval_call("orc_strictify_value", go, v, tf)


def restore_value(go: str, v, data_type: str):
    """abstract.Restore over one boxed Go value."""
    return _goval_call("orc_restore_value", go, v, data_type.encode())


def csv_split_rows(data: bytes):
    """csv.Splitter.ConsumeRow until io.EOF: (rows, remainder written by the call that returned io.EOF)."""
    L = lib(); L.orc_csv_split_rows.restype = C.c_uint64
    L.orc_csv_split_rows.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64]
    ends = (C.c_uint64 * (len(data) + 1))()
    n = L.orc_csv_split_rows(data, len(data), ends, len(data) + 1)
    rows, pos = [], 0
    for k in range(n):
        rows.append(data[pos:ends[k]]); pos = ends[k]
    return rows, data[pos:]
