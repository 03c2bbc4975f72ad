"""ctypes view of include/tfgpu.h and include/tfgpu_sink.h: the structs that cross the C-ABI and the prototype of every function.

This module only describes memory; it computes nothing.  The engine binding
(transferia_b200.engine) uses it, and so do the tests' CPU checker and the workload generator,
because they all speak the same `tf_batch` struct.
"""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass, field
from typing import Any, List, Optional, Sequence

import numpy as np

# tf_type — YT type strings of pkg/abstract/typesystem/schema.go:48-68
TF_INT8, TF_INT16, TF_INT32, TF_INT64 = 1, 2, 3, 4
TF_UINT8, TF_UINT16, TF_UINT32, TF_UINT64 = 5, 6, 7, 8
TF_FLOAT, TF_DOUBLE, TF_BOOLEAN = 9, 10, 11
TF_BYTES, TF_UTF8, TF_ANY = 12, 13, 14
TF_DATE, TF_DATETIME, TF_TIMESTAMP, TF_INTERVAL = 15, 16, 17, 18

YT_NAME_TO_TF = {
    "int8": TF_INT8, "int16": TF_INT16, "int32": TF_INT32, "int64": TF_INT64,
    "uint8": TF_UINT8, "uint16": TF_UINT16, "uint32": TF_UINT32, "uint64": TF_UINT64,
    "float": TF_FLOAT, "double": TF_DOUBLE, "boolean": TF_BOOLEAN,
    "string": TF_BYTES, "utf8": TF_UTF8, "any": TF_ANY,
    "date": TF_DATE, "datetime": TF_DATETIME, "timestamp": TF_TIMESTAMP, "interval": TF_INTERVAL,
}
TF_TO_YT_NAME = {v: k for k, v in YT_NAME_TO_TF.items()}

FIXED_DTYPE = {
    TF_INT8: np.int8, TF_INT16: np.int16, TF_INT32: np.int32, TF_INT64: np.int64,
    TF_UINT8: np.uint8, TF_UINT16: np.uint16, TF_UINT32: np.uint32, TF_UINT64: np.uint64,
    TF_FLOAT: np.float32, TF_DOUBLE: np.float64, TF_BOOLEAN: np.uint8,
    TF_DATE: np.int64, TF_DATETIME: np.int64, TF_TIMESTAMP: np.int64, TF_INTERVAL: np.int64,
}
VAR_TYPES = (TF_BYTES, TF_UTF8, TF_ANY)
TIME_TYPES = (TF_DATE, TF_DATETIME, TF_TIMESTAMP)

TF_MEM_HOST, TF_MEM_DEVICE = 0, 1
TF_KIND_INSERT, TF_KIND_UPDATE, TF_KIND_DELETE = 0, 1, 2

TF_WIRE_CH_NATIVE, TF_WIRE_CH_NATIVE_LZ4, TF_WIRE_CH_JSONEACHROW = 1, 2, 3

TF_ROWERR_FILTER_KIND, TF_ROWERR_FILTER_OVERFLOW, TF_ROWERR_FILTER_TYPEPAIR = 1, 2, 3


class TfCol(C.Structure):
    _fields_ = [
        ("type", C.c_int32), ("flags", C.c_int32),
        ("values", C.c_void_p), ("validity", C.c_void_p), ("offsets", C.c_void_p),
        ("heap", C.c_void_p), ("aux", C.c_void_p), ("heap_len", C.c_uint64),
    ]


class TfBatch(C.Structure):
    _fields_ = [
        ("nrows", C.c_uint64), ("ncols", C.c_uint32), ("mem", C.c_uint32),
        ("cols", C.POINTER(TfCol)), ("kinds", C.c_void_p),
    ]


class TfRowErr(C.Structure):
    _fields_ = [("row", C.c_uint32), ("code", C.c_uint16), ("term", C.c_uint16)]


class TfMsg(C.Structure):
    """tf_msg: one queue message of a tfgpu_parse_json call (parsers.Message, pkg/parsers/abstract.go:13-27)."""
    _fields_ = [("end", C.c_uint64), ("offset", C.c_uint64), ("write_sec", C.c_int64), ("write_nsec", C.c_uint32), ("pad", C.c_uint32)]


class TfRowMeta(C.Structure):
    """tf_row_meta: the ChangeItem fields Debezium's `source` block carries (change_item.go:27-40)."""
    _fields_ = [("id", C.c_void_p), ("lsn", C.c_void_p), ("commit_time", C.c_void_p), ("txid_offsets", C.c_void_p), ("txid_heap", C.c_void_p)]


class TfOldKeys(C.Structure):
    """tf_old_keys: ChangeItem.OldKeys of a batch as a second set of typed columns (old_keys.go:3-7)."""
    _fields_ = [("values", C.c_void_p), ("present_cols", C.c_void_p), ("row_has", C.c_void_p)]


def schema_json(schema) -> str:
    """A table schema as the ColSchema JSON array the calls take: JSON text as it is, or ColSchema dicts without their "_" keys."""
    return schema if isinstance(schema, str) else json.dumps([{k: v for k, v in c.items() if not k.startswith("_")} for c in schema])


def make_old_keys(old_batch, present_cols, row_has=None):
    """(struct, keepalive): `old_batch` an abi.Batch with the plan's input schema, present_cols the column indexes listed in OldKeys.KeyNames."""
    tb = old_batch.as_struct()
    pres = np.zeros(len(old_batch.columns), dtype=np.uint8); pres[list(present_cols)] = 1
    ok = TfOldKeys(C.cast(C.pointer(tb), C.c_void_p), pres.ctypes.data, _ptr(row_has))
    return ok, (tb, pres, row_has, old_batch)


def make_row_meta(id=None, lsn=None, commit_time=None, txid_offsets=None, txid_heap=None):
    """(struct, keepalive) from numpy arrays / torch tensors; None stays NULL."""
    m = TfRowMeta(_ptr(id), _ptr(lsn), _ptr(commit_time), _ptr(txid_offsets), _ptr(txid_heap))
    return m, (id, lsn, commit_time, txid_offsets, txid_heap)


TF_COL_LENS8, TF_COL_LENS16 = 1, 2
TF_WIRE_SER_JSON, TF_WIRE_SER_CSV = 4, 5
TF_WIRE_F_CLOSING_NEWLINE, TF_WIRE_F_ANY_AS_STRING = 0x100, 0x200
TF_WIRE_F_GZIP, TF_WIRE_F_ZLIB = 0x400, 0x800     # the row text as one gzip member / zlib stream (include/tfgpu.h)
TF_WIRE_F_ZSTD = 0x1000                            # the JSONEachRow text as one zstd frame (include/tfgpu.h)
TF_WIRE_DEBEZIUM = 6
TF_ROWERR_CSV_BAD_FLOAT, TF_ROWERR_CSV_UNSUPPORTED, TF_ROWERR_CSV_DQ_DISABLED, TF_ROWERR_CSV_QUOTING_DISABLED = 22, 23, 24, 25
TF_ROWERR_N2F_HOST = 52
TF_ROWERR_DBZ_EMIT_HOST = 53
TF_ROWERR_SINK_KIND_HOST = 54
TF_ROWERR_DBZ_UNPARSED, TF_ROWERR_DBZ_HOST, TF_ROWERR_DBZ_OTHER_SCHEMA, TF_ROWERR_DBZ_OTHER_TABLE = 48, 49, 50, 51
TF_ROWERR_JSON_PARSE, TF_ROWERR_JSON_SKIP, TF_ROWERR_JSON_NIL_REQUIRED, TF_ROWERR_JSON_PARSEVAL, TF_ROWERR_JSON_HOST = 32, 33, 34, 35, 36


def _ptr(a) -> Optional[int]:
    """Address of a numpy array or torch tensor (None stays NULL)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data if a.size else None
    # torch tensor (host pinned or device)
    return a.data_ptr() if a.numel() else None


@dataclass
class Column:
    """One column in the physical layout documented in include/tfgpu.h."""
    type: int
    values: Any = None      # fixed-width / time seconds
    validity: Any = None    # uint8 bitmap, bit=1 non-null
    offsets: Any = None     # uint32[nrows+1]
    heap: Any = None        # uint8[]
    aux: Any = None         # time: uint32 nanos; any: uint8 tags
    lens_width: int = 0     # 0: `offsets` holds uint32 offsets; 1 / 2: it holds uint8 / uint16 per-row LENGTHS (TF_COL_LENS8 / 16)

    def heap_len(self) -> int:
        if self.heap is None:
            return 0
        return int(self.heap.size if isinstance(self.heap, np.ndarray) else self.heap.numel())


@dataclass
class Batch:
    """A single-table batch of ChangeItems, transposed (pkg/abstract/changeitem/change_item.go:27-78)."""
    nrows: int
    columns: List[Column]
    kinds: Any = None
    mem: int = TF_MEM_HOST
    _keep: list = field(default_factory=list, repr=False)

    def as_struct(self) -> TfBatch:
        arr = (TfCol * len(self.columns))()
        for i, c in enumerate(self.columns):
            arr[i].type = c.type
            arr[i].flags = {0: 0, 1: TF_COL_LENS8, 2: TF_COL_LENS16}[getattr(c, "lens_width", 0)]
            arr[i].values = _ptr(c.values)
            arr[i].validity = _ptr(c.validity)
            arr[i].offsets = _ptr(c.offsets)
            arr[i].heap = _ptr(c.heap)
            arr[i].aux = _ptr(c.aux)
            arr[i].heap_len = c.heap_len()
        b = TfBatch()
        b.nrows = self.nrows
        b.ncols = len(self.columns)
        b.mem = self.mem
        b.cols = C.cast(arr, C.POINTER(TfCol))
        b.kinds = _ptr(self.kinds)
        self._keep = [arr]
        return b

    def narrow(self) -> "Batch":
        """The same host batch with per-row LENGTHS (uint8 where every cell of the column is shorter than 256 bytes, else uint16) in place
        of the uint32 offsets of its var-width columns: what a shim sends to save PCIe bytes (tf_col.flags TF_COL_LENS8 / 16)."""
        cols = []
        for c in self.columns:
            if c.offsets is None or c.type not in VAR_TYPES or getattr(c, "lens_width", 0):
                cols.append(c); continue
            off = np.asarray(c.offsets).view(np.uint32) if isinstance(c.offsets, np.ndarray) else None
            if off is None:
                cols.append(c); continue
            ln = np.diff(off.astype(np.int64))
            mx = int(ln.max()) if len(ln) else 0
            if mx < 256: cols.append(Column(c.type, c.values, c.validity, ln.astype(np.uint8), c.heap, c.aux, 1))
            elif mx < 65536: cols.append(Column(c.type, c.values, c.validity, ln.astype(np.uint16), c.heap, c.aux, 2))
            else: cols.append(c)
        return Batch(self.nrows, cols, self.kinds, self.mem)

    def input_bytes(self) -> int:
        """Columnar input bytes (SURVEY §8d `I`): values + offsets + heap (+validity/aux when present)."""
        tot = 0
        for c in self.columns:
            for a in (c.values, c.validity, c.offsets, c.heap, c.aux):
                if a is None:
                    continue
                tot += int(a.nbytes if isinstance(a, np.ndarray) else a.numel() * a.element_size())
        if self.kinds is not None:
            a = self.kinds
            tot += int(a.nbytes if isinstance(a, np.ndarray) else a.numel() * a.element_size())
        return tot

    def slice(self, lo: int, hi: int) -> "Batch":
        """Host-only row slice [lo, hi) — used to deal sub-batches to pipelines / ranks."""
        assert self.mem == TF_MEM_HOST
        cols = []
        for c in self.columns:
            if c.type in VAR_TYPES:
                off = c.offsets[lo:hi + 1]
                base = int(off[0]) if len(off) else 0
                end = int(off[-1]) if len(off) else 0
                cols.append(Column(c.type, offsets=(off - np.uint32(base)).astype(np.uint32),
                                   heap=np.ascontiguousarray(c.heap[base:end]),
                                   validity=_slice_bits(c.validity, lo, hi),
                                   aux=None if c.aux is None else np.ascontiguousarray(c.aux[lo:hi])))
            else:
                cols.append(Column(c.type, values=np.ascontiguousarray(c.values[lo:hi]),
                                   validity=_slice_bits(c.validity, lo, hi),
                                   aux=None if c.aux is None else np.ascontiguousarray(c.aux[lo:hi])))
        kinds = None if self.kinds is None else np.ascontiguousarray(self.kinds[lo:hi])
        return Batch(hi - lo, cols, kinds)

    def pin_arena(self) -> "Batch":
        """Same batch in ONE page-locked arena laid out like the engine's device staging (each non-empty buffer at the next multiple of 256
        past the previous one's end + 16; values / validity / offsets / heap / aux per column, then kinds): tfgpu_push_* then needs a single
        DMA for the whole batch (the pooled buffers of a shim's transposer are laid out this way)."""
        import torch
        bufs = []
        for c in self.columns:
            for a in (c.values, c.validity, c.offsets, c.heap, c.aux):
                bufs.append(None if a is None else np.ascontiguousarray(a).reshape(-1).view(np.uint8))
        bufs.append(None if self.kinds is None else np.ascontiguousarray(self.kinds).reshape(-1).view(np.uint8))
        stride = lambda nb: (nb + 16 + 255) // 256 * 256
        total = sum(stride(b.size) for b in bufs if b is not None and b.size) + 256
        arena = torch.empty(total, dtype=torch.uint8).pin_memory()
        base = (-arena.data_ptr()) % 256                       # the device staging is 256-byte aligned: keep the same phase
        views, at = [], base
        for b in bufs:
            if b is None or not b.size:
                views.append(None if b is None else arena[at:at]); continue
            v = arena[at:at + b.size]; v.copy_(torch.from_numpy(b)); views.append(v); at += stride(b.size)
        cols = []
        for i, c in enumerate(self.columns):
            v = views[5 * i:5 * i + 5]
            cols.append(Column(c.type, v[0], v[1], v[2], v[3], v[4], getattr(c, "lens_width", 0)))
        out = Batch(self.nrows, cols, views[-1], TF_MEM_HOST); out._keep = [arena]
        return out

    def pin(self) -> "Batch":
        """Same batch with every buffer in page-locked host memory (what the cgo shim hands over)."""
        import torch
        def pn(a):
            if a is None:
                return None
            return torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).pin_memory()
        cols = [Column(c.type, pn(c.values), pn(c.validity), pn(c.offsets), pn(c.heap), pn(c.aux), getattr(c, "lens_width", 0)) for c in self.columns]
        return Batch(self.nrows, cols, pn(self.kinds), TF_MEM_HOST)

    def to_device(self, device="cuda:0", pinned_first: bool = False) -> "Batch":
        """Copy every buffer to HBM with torch (plumbing only)."""
        import torch
        def mv(a):
            if a is None:
                return None
            t = torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8))
            if pinned_first:
                t = t.pin_memory()
            return t.to(device, non_blocking=pinned_first)
        cols = [Column(c.type, mv(c.values), mv(c.validity), mv(c.offsets), mv(c.heap), mv(c.aux), getattr(c, "lens_width", 0)) for c in self.columns]
        return Batch(self.nrows, cols, mv(self.kinds), TF_MEM_DEVICE)


def _slice_bits(bm, lo, hi):
    if bm is None:
        return None
    bits = np.unpackbits(bm, bitorder="little")[lo:hi]
    return np.packbits(bits, bitorder="little")


def pack_validity(mask: np.ndarray) -> np.ndarray:
    """bool[nrows] (True = non-null) -> LSB-first bitmap."""
    return np.packbits(mask.astype(np.uint8), bitorder="little")


def strings_to_column(tf_type: int, values: Sequence[Optional[bytes]], tags=None) -> Column:
    """Build a var-width column from python bytes (None = nil)."""
    n = len(values)
    lens = np.fromiter((0 if v is None else len(v) for v in values), dtype=np.int64, count=n)
    offs = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(lens, out=offs[1:])
    heap = np.frombuffer(b"".join(v for v in values if v is not None), dtype=np.uint8).copy()
    validity = None
    if any(v is None for v in values):
        validity = pack_validity(np.array([v is not None for v in values]))
    aux = None if tags is None else np.asarray(tags, dtype=np.uint8)
    return Column(tf_type, offsets=offs, heap=heap, validity=validity, aux=aux)


def fixed_to_column(tf_type: int, values: Sequence, nulls: Optional[Sequence[bool]] = None, nanos=None) -> Column:
    arr = np.asarray(values, dtype=FIXED_DTYPE[tf_type])
    validity = None
    if nulls is not None and any(nulls):
        validity = pack_validity(~np.asarray(nulls, dtype=bool))
    aux = None if nanos is None else np.asarray(nanos, dtype=np.uint32)
    return Column(tf_type, values=arr, validity=validity, aux=aux)


# ------------------------------------------------------------------ include/tfgpu_sink.h
class TfTable(C.Structure):
    _fields_ = [("schema", C.c_char_p), ("table", C.c_char_p), ("schema_json", C.c_char_p)]


class TfItem(C.Structure):
    _fields_ = [("lsn", C.c_uint64), ("commit_time", C.c_uint64), ("size_read", C.c_uint64), ("size_values", C.c_uint64), ("values_off", C.c_uint64), ("old_keys_off", C.c_uint64),
                ("id", C.c_uint32), ("table", C.c_uint32), ("n_values", C.c_uint32), ("txid_off", C.c_uint32), ("txid_len", C.c_uint32),
                ("part_off", C.c_uint32), ("part_len", C.c_uint32), ("counter", C.c_int32), ("kind", C.c_uint8), ("flags", C.c_uint8), ("pad", C.c_uint8 * 2)]


class TfRows(C.Structure):
    _fields_ = [("n_items", C.c_uint64), ("items", C.POINTER(TfItem)), ("n_tables", C.c_uint32), ("pad", C.c_uint32), ("tables", C.POINTER(TfTable)),
                ("values", C.c_void_p), ("values_len", C.c_uint64), ("strings", C.c_void_p), ("strings_len", C.c_uint64)]


class TfSinkEvent(C.Structure):
    _fields_ = [("type", C.c_int32), ("table", C.c_uint32), ("out_schema", C.c_char_p), ("out_table", C.c_char_p), ("n_items", C.c_uint64),
                ("item_idx", C.POINTER(C.c_uint64)), ("errors", C.c_void_p), ("batch", C.c_void_p), ("wire", C.c_void_p),
                ("wire_len", C.c_uint64), ("raw_len", C.c_uint64), ("n_frames", C.c_uint64), ("msg_sizes", C.POINTER(C.c_uint32)), ("plan_id", C.c_int32), ("pad", C.c_int32)]


class TfSinkStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("pushes", "downstream_pushes", "change_items_pushed", "row_events_pushed", "inflight_bytes", "filter_dropped",
                                          "transform_dropped", "transform_errors", "max_commit_time", "min_commit_time", "without_commit_time", "wire_bytes",
                                          "metering_input_rows", "metering_output_rows")]


TF_SINK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(TfSinkEvent))      # tf_sink_fn


# ------------------------------------------------------------------ every function of both headers
# name -> (restype, argtypes), one table per header; engine.load_library() applies PROTOTYPES (both) once. Handles are void*, char buffers char*, byte and integer arrays
# void* (numpy addresses, bytes and string buffers pass as they are); structs go by their class, and scalars, scalar out-parameters and
# returned arrays at the header's width.
_v, _s, _i, _u32, _u64, _P = C.c_void_p, C.c_char_p, C.c_int, C.c_uint32, C.c_uint64, C.POINTER
TFGPU_H_PROTOTYPES = {
    "tfgpu_engine_create": (_i, [_s, _P(_i), _i, _P(_v)]),
    "tfgpu_engine_destroy": (_i, [_v]),
    "tfgpu_last_error": (_s, [_v]),
    "tfgpu_engine_set_stream": (_i, [_v, _v]),
    "tfgpu_plan": (_i, [_v, _s, _s, _s, _s, _s, _P(_i)]),
    "tfgpu_plan_validate": (_i, [_s, _s, _s, _s, _s, _s, _u64, _s, _u64]),
    "tfgpu_plan_describe": (_s, [_v, _i]),
    "tfgpu_push_columns": (_i, [_v, _i, _P(TfBatch), _P(_v)]),
    "tfgpu_push_encode": (_i, [_v, _i, _i, _P(TfBatch), _P(_v)]),
    "tfgpu_push_encode_selective": (_i, [_v, _i, _i, _P(TfBatch), _i, _P(_v)]),
    "tfgpu_engine_h2d_bytes": (_u64, [_v]),
    "tfgpu_emit_debezium": (_i, [_v, _i, _s, _P(TfBatch), _P(TfRowMeta), _P(_v)]),
    "tfgpu_emit_debezium_crud": (_i, [_v, _i, _s, _P(TfBatch), _P(TfOldKeys), _P(TfRowMeta), _P(_v)]),
    "tfgpu_result_dbz_msg_sizes": (_P(_u32), [_v]),
    "tfgpu_emit_debezium_validate": (_i, [_s, _s, _s, _s, _s, _s, _u64, _s, _u64]),
    "tfgpu_measure": (_i, [_v, _P(TfBatch), _v, _P(_u64)]),
    "tfgpu_parse_csv": (_i, [_v, _i, _s, _v, _u64, _i, _i, _P(_v)]),
    "tfgpu_result_consumed": (_u64, [_v]),
    "tfgpu_push_encode_resident": (_i, [_v, _i, _i, _P(TfBatch)]),
    "tfgpu_resident_stats": (_i, [_v, _P(_u64), _P(_u64), _P(_u64), _P(_u64)]),
    "tfgpu_resident_fetch": (_i, [_v, _i, _v, _u64]),
    "tfgpu_result_rows_in": (_u64, [_v]),
    "tfgpu_parse_json": (_i, [_v, _i, _s, _v, _u64, _i, _P(TfMsg), _u32, _i, _P(_v)]),
    "tfgpu_parse_debezium": (_i, [_v, _i, _s, _v, _u64, _i, _v, _u32, _i, _P(_v)]),
    "tfgpu_debezium_schema_validate": (_i, [_s, _s, _u64, _s, _u64]),
    "tfgpu_debug_lz4_phases": (_i, [_v, _i, _P(_u64)]),
    "tfgpu_result_selection": (_P(_u32), [_v]),
    "tfgpu_result_meta_kinds": (_P(C.c_uint8), [_v]),
    "tfgpu_result_meta_tx_id": (_P(_u32), [_v]),
    "tfgpu_result_meta_lsn": (_P(_u64), [_v]),
    "tfgpu_result_meta_commit_time": (_P(_u64), [_v]),
    "tfgpu_result_rows_out": (_u64, [_v]),
    "tfgpu_result_n_errors": (_u64, [_v]),
    "tfgpu_result_errors": (_P(TfRowErr), [_v]),
    "tfgpu_result_batch": (_P(TfBatch), [_v]),
    "tfgpu_result_bytes": (_v, [_v]),
    "tfgpu_result_bytes_len": (_u64, [_v]),
    "tfgpu_result_raw_len": (_u64, [_v]),
    "tfgpu_result_n_frames": (_u64, [_v]),
    "tfgpu_result_row_sizes": (_P(_u32), [_v]),
    "tfgpu_result_part_ids": (_P(_u32), [_v]),
    "tfgpu_result_key_sizes": (_P(_u32), [_v]),
    "tfgpu_queue_json_batches": (_i, [_v, _u64, _u64, _u64, _v, _u64, _P(_u64)]),
    "tfgpu_queue_debezium_batches": (_i, [_v, _u64, _u64, _v, _u64, _P(_u64)]),
    "tfgpu_result_release": (None, [_v]),
    "tfgpu_deflate_stream_open": (_i, [_i, _P(_v)]),
    "tfgpu_deflate_stream_append": (_i, [_v, _v, _u64, _u64, _v, _u64, _P(_u64)]),
    "tfgpu_deflate_stream_close": (_i, [_v, _v, _u64, _P(_u64)]),
    "tfgpu_deflate_stream_free": (None, [_v]),
    "tfgpu_zstd_prefix": (_i, [_v, _u64, _v, _u64, _v, _u64, _P(_u64)]),
    "tfgpu_engine_launch_count": (_u64, [_v]),
    "tfgpu_profile_enable": (_i, [_v, _i]),
    "tfgpu_profile_read": (_s, [_v]),
    "tfgpu_version": (_s, []),
}
TFGPU_SINK_H_PROTOTYPES = {
    "tfgpu_ch_open": (_i, [_i, _s, _P(_v)]),
    "tfgpu_ch_close": (_i, [_v]),
    "tfgpu_ch_last_error": (_s, [_v]),
    "tfgpu_ch_server_info": (_s, [_v]),
    "tfgpu_ch_exception_code": (_i, [_v]),
    "tfgpu_ch_insert_begin": (_i, [_v, _s, _s, _s]),
    "tfgpu_ch_insert_columns": (_s, [_v]),
    "tfgpu_ch_insert_data": (_i, [_v, _v, _u64]),
    "tfgpu_ch_insert_end": (_i, [_v, _P(_u64), _P(_u64)]),
    "tfgpu_ch_stats": (_i, [_v, _P(_u64), _P(_u64), _P(_u64)]),
    "tfgpu_ch_insert_query": (C.c_int64, [_s, _s, _s, _i, _s, _u64]),
    "tfgpu_columnar_create": (_i, [_P(_v)]),
    "tfgpu_columnar_destroy": (_i, [_v]),
    "tfgpu_columnar_last_error": (_s, [_v]),
    "tfgpu_rows_to_batch": (_i, [_v, _P(TfRows), _u32, _v, _u64, _i, _P(_P(TfBatch)), _P(_P(TfRowMeta)), _P(_P(TfOldKeys))]),
    "tfgpu_batch_to_rows": (_i, [_P(TfBatch), _v, _u64, _v, _P(_u64)]),
    "tfgpu_batch_gather": (_i, [_v, _P(TfBatch), _v, _i, _P(_P(TfBatch)), _P(_P(_u32))]),
    "tfgpu_batch_gather_sel": (_i, [_v, _P(TfBatch), _v, _u64, _i, _P(_P(TfBatch))]),
    "tfgpu_sink_create": (_i, [_v, _s, _P(_v)]),
    "tfgpu_sink_destroy": (_i, [_v]),
    "tfgpu_sink_last_error": (_s, [_v]),
    "tfgpu_sink_set_callback": (_i, [_v, TF_SINK_FN, _v]),
    "tfgpu_sink_set_clickhouse": (_i, [_v, _v]),
    "tfgpu_sink_push": (_i, [_v, _P(TfRows)]),
    "tfgpu_sink_stats": (_i, [_v, _P(TfSinkStats)]),
    "tfgpu_dispatcher_create": (_i, [_P(_v), _i, _P(_v)]),
    "tfgpu_dispatcher_submit": (_i, [_v, _P(TfRows), _P(_u64)]),
    "tfgpu_dispatcher_wait": (_i, [_v, _u64]),
    "tfgpu_dispatcher_drain": (_i, [_v]),
    "tfgpu_dispatcher_destroy": (_i, [_v]),
    "tfgpu_host_cityhash128": (None, [_v, _u64, _P(_u64)]),
    "tfgpu_regex_replace_all": (C.c_int64, [_s, _s, _v, _u64, _v, _u64]),
}
PROTOTYPES = {**TFGPU_H_PROTOTYPES, **TFGPU_SINK_H_PROTOTYPES}
