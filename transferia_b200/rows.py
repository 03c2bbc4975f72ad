"""[]abstract.ChangeItem in row form (include/tfgpu_sink.h `tf_rows`) — the Python stand-in for what the Go shim writes while it walks a
batch (pkg/abstract/changeitem/change_item.go:27-78): one fixed header per item, one byte image of the boxed values, and the binding of
the C++ transposer (tfgpu_rows_to_batch / tfgpu_batch_to_rows).  Go's dynamic value types are spelled as (tag, value) pairs built with the
helpers below (`go.int32(5)`, `go.string("x")`, `go.time(sec, nsec)`), because Python's own types do not carry a width."""
from __future__ import annotations

import ctypes as C
import struct
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi, engine
from .abi import TfItem, TfRows, TfTable

# kinds (kind.go:5-43)
KIND_INSERT, KIND_UPDATE, KIND_DELETE = 0, 1, 2
KIND_INIT_SHARDED_TABLE_LOAD, KIND_INIT_TABLE_LOAD, KIND_DONE_TABLE_LOAD, KIND_DONE_SHARDED_TABLE_LOAD = 16, 17, 18, 19
KIND_DROP_TABLE, KIND_TRUNCATE, KIND_DDL, KIND_PG_DDL, KIND_SYNCHRONIZE, KIND_OTHER = 20, 21, 22, 23, 24, 31
KIND_NAMES = {"insert": 0, "update": 1, "delete": 2, "init_sharded_table_load": 16, "init_load_table": 17, "done_load_table": 18,
              "done_sharded_table_load": 19, "drop_table": 20, "truncate": 21, "DDL": 22, "pg:DDL": 23, "": 24}

V_NIL, V_BOOL, V_INT8, V_INT16, V_INT32, V_INT64, V_UINT8, V_UINT16, V_UINT32, V_UINT64 = range(10)
V_FLOAT32, V_FLOAT64, V_STRING, V_BYTES, V_TIME, V_DURATION, V_JSONNUM, V_JSON = range(10, 18)
_FIXED_FMT = {V_BOOL: "<B", V_INT8: "<b", V_INT16: "<h", V_INT32: "<i", V_INT64: "<q", V_UINT8: "<B", V_UINT16: "<H", V_UINT32: "<I",
              V_UINT64: "<Q", V_FLOAT32: "<f", V_FLOAT64: "<d", V_DURATION: "<q"}


class go:
    """Constructors for Go-typed values: go.int64(7) == (V_INT64, 7)."""
    nil = (V_NIL, None)
    bool = staticmethod(lambda v: (V_BOOL, 1 if v else 0))
    int8 = staticmethod(lambda v: (V_INT8, int(v))); int16 = staticmethod(lambda v: (V_INT16, int(v)))
    int32 = staticmethod(lambda v: (V_INT32, int(v))); int64 = staticmethod(lambda v: (V_INT64, int(v)))
    uint8 = staticmethod(lambda v: (V_UINT8, int(v))); uint16 = staticmethod(lambda v: (V_UINT16, int(v)))
    uint32 = staticmethod(lambda v: (V_UINT32, int(v))); uint64 = staticmethod(lambda v: (V_UINT64, int(v)))
    float32 = staticmethod(lambda v: (V_FLOAT32, float(v))); float64 = staticmethod(lambda v: (V_FLOAT64, float(v)))
    string = staticmethod(lambda v: (V_STRING, v.encode() if isinstance(v, str) else bytes(v)))
    bytes = staticmethod(lambda v: (V_BYTES, bytes(v)))
    time = staticmethod(lambda sec, nsec=0: (V_TIME, (int(sec), int(nsec))))
    duration = staticmethod(lambda ns: (V_DURATION, int(ns)))
    number = staticmethod(lambda text: (V_JSONNUM, text.encode() if isinstance(text, str) else bytes(text)))
    json = staticmethod(lambda text: (V_JSON, text.encode() if isinstance(text, str) else bytes(text)))


def encode_value(out: bytearray, v) -> None:
    tag, x = v
    out.append(tag)
    if tag == V_NIL:
        return
    if tag in _FIXED_FMT:
        out += struct.pack(_FIXED_FMT[tag], x)
    elif tag == V_TIME:
        out += struct.pack("<qI", x[0], x[1])
    else:
        out += struct.pack("<I", len(x)); out += x


@dataclass
class ChangeItem:
    """pkg/abstract/changeitem/change_item.go:27-78 (the fields this path reads)."""
    kind: int = KIND_INSERT
    table: int = 0                                   # index into the tables list (Schema, Table, TableSchema)
    values: Optional[Sequence] = None                # ColumnValues as Go-typed pairs, schema order (or {column index: value} when sparse)
    old_keys: Optional[Dict[int, Any]] = None        # OldKeys: {column index: value}
    id: int = 0; lsn: int = 0; commit_time: int = 0; counter: int = 0; size_read: int = 0; size_values: int = 0
    txid: bytes = b""; part_id: bytes = b""


NO_OLD_KEYS = (1 << 64) - 1


class RowsImage:
    """tf_rows + the buffers it points into. tables: [(namespace, name, schema list of ColSchema dicts)]."""

    def __init__(self, items: Sequence[ChangeItem], tables: Sequence[Tuple[str, str, list]]):
        self.tables = list(tables)
        vals, strs = bytearray(), bytearray()
        arr = (TfItem * max(1, len(items)))()
        for i, it in enumerate(items):
            a = arr[i]
            a.lsn, a.commit_time, a.size_read, a.size_values, a.id, a.table, a.counter, a.kind = it.lsn, it.commit_time, it.size_read, it.size_values, it.id, it.table, it.counter, it.kind
            a.txid_off, a.txid_len = len(strs), len(it.txid); strs += it.txid
            a.part_off, a.part_len = len(strs), len(it.part_id); strs += it.part_id
            a.values_off = len(vals); a.flags = 0; a.n_values = 0
            if it.values is not None:
                if isinstance(it.values, dict):
                    a.flags = 1; a.n_values = len(it.values)
                    for c, v in it.values.items():
                        vals += struct.pack("<H", c); encode_value(vals, v)
                else:
                    a.n_values = len(it.values)
                    for v in it.values:
                        encode_value(vals, v)
            a.old_keys_off = NO_OLD_KEYS
            if it.old_keys is not None:
                a.old_keys_off = len(vals); vals += struct.pack("<H", len(it.old_keys))
                for c, v in it.old_keys.items():
                    vals += struct.pack("<H", c); encode_value(vals, v)
        self._items = arr
        self._vals = np.frombuffer(bytes(vals) + b"\0", dtype=np.uint8).copy()
        self._strs = np.frombuffer(bytes(strs) + b"\0", dtype=np.uint8).copy()
        self._tabs = (TfTable * max(1, len(tables)))()
        self._keep = []
        for k, (ns, name, schema) in enumerate(tables):
            sj = None if schema is None else schema if isinstance(schema, bytes) else abi.schema_json(schema).encode()
            self._keep.append((ns.encode(), name.encode(), sj))
            self._tabs[k].schema, self._tabs[k].table, self._tabs[k].schema_json = self._keep[-1]
        r = TfRows()
        r.n_items = len(items); r.items = C.cast(arr, C.POINTER(TfItem)); r.n_tables = len(tables); r.tables = C.cast(self._tabs, C.POINTER(TfTable))
        r.values = self._vals.ctypes.data; r.values_len = len(vals); r.strings = self._strs.ctypes.data; r.strings_len = len(strs)
        self.struct = r
        self.values_len = len(vals)


def items_from_batch(batch: abi.Batch, table: int = 0) -> List[ChangeItem]:
    """Rows of a columnar batch as ChangeItems carrying the canonical Go type of every column (type_checkers.go:39-84)."""
    ctor = {abi.TF_INT8: go.int8, abi.TF_INT16: go.int16, abi.TF_INT32: go.int32, abi.TF_INT64: go.int64, abi.TF_UINT8: go.uint8, abi.TF_UINT16: go.uint16,
            abi.TF_UINT32: go.uint32, abi.TF_UINT64: go.uint64, abi.TF_FLOAT: go.float32, abi.TF_DOUBLE: go.float64, abi.TF_BOOLEAN: go.bool, abi.TF_INTERVAL: go.duration}
    n = batch.nrows
    cols = []
    for c in batch.columns:
        valid = np.ones(n, dtype=bool) if c.validity is None else np.unpackbits(np.asarray(c.validity), bitorder="little")[:n].astype(bool)
        if c.type in abi.VAR_TYPES:
            off = np.asarray(c.offsets).astype(np.int64); heap = np.asarray(c.heap).tobytes() if c.heap is not None else b""
            tags = None if c.aux is None else np.asarray(c.aux)
            cells = []
            for r in range(n):
                if not valid[r]: cells.append(go.nil); continue
                b = heap[off[r]:off[r + 1]]
                if c.type == abi.TF_UTF8: cells.append(go.string(b))
                elif c.type == abi.TF_BYTES: cells.append(go.bytes(b))
                else: cells.append(go.string(b) if tags is not None and tags[r] == 1 else go.json(b))
        elif c.type in abi.TIME_TYPES:
            sec = np.asarray(c.values); ns = np.zeros(n, dtype=np.uint32) if c.aux is None else np.asarray(c.aux)
            cells = [go.time(sec[r], ns[r]) if valid[r] else go.nil for r in range(n)]
        else:
            v = np.asarray(c.values); f = ctor[c.type]
            cells = [f(v[r]) if valid[r] else go.nil for r in range(n)]
        cols.append(cells)
    kinds = None if batch.kinds is None else np.asarray(batch.kinds)
    return [ChangeItem(kind=int(kinds[r]) if kinds is not None else KIND_INSERT, table=table, values=[col[r] for col in cols]) for r in range(n)]


def _view(ptr, nbytes, dtype=np.uint8):
    if not ptr or nbytes == 0:
        return None
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(nbytes,)).view(dtype)


def batch_from_struct(tb: abi.TfBatch) -> abi.Batch:
    """Zero-copy numpy view of a host tf_batch (valid as long as its owner keeps the buffers)."""
    n = int(tb.nrows); cols = []
    for i in range(tb.ncols):
        c = tb.cols[i]
        if c.type in abi.VAR_TYPES:
            lw = 1 if c.flags & abi.TF_COL_LENS8 else 2 if c.flags & abi.TF_COL_LENS16 else 0
            offs = _view(c.offsets, n * lw if lw else (n + 1) * 4, {0: np.uint32, 1: np.uint8, 2: np.uint16}[lw])
            cols.append(abi.Column(c.type, None, _view(c.validity, (n + 7) // 8), offs, _view(c.heap, int(c.heap_len)), _view(c.aux, n), lw))
        else:
            dt = abi.FIXED_DTYPE[c.type]
            cols.append(abi.Column(c.type, _view(c.values, n * np.dtype(dt).itemsize, dt), _view(c.validity, (n + 7) // 8), None, None,
                                   _view(c.aux, 4 * n, np.uint32) if c.type in abi.TIME_TYPES else None))
    return abi.Batch(n, cols, _view(tb.kinds, n), abi.TF_MEM_HOST)


@dataclass
class Transposed:
    batch: abi.Batch
    struct: Any                      # POINTER(TfBatch) owned by the pool
    meta: Any                        # POINTER(TfRowMeta) or None
    old: Any                         # POINTER(TfOldKeys) or None
    ids: np.ndarray = None; lsn: np.ndarray = None; commit_time: np.ndarray = None
    old_batch: Optional[abi.Batch] = None; old_present: Optional[np.ndarray] = None; old_row_has: Optional[np.ndarray] = None


class Columnar:
    """Pooled column buffers + the transposer (tfgpu_columnar)."""

    def __init__(self):
        self._L = engine.load_library(); self._h = C.c_void_p()
        rc = self._L.tfgpu_columnar_create(C.byref(self._h))
        if rc: raise engine.EngineError(rc, "tfgpu_columnar_create")

    def rows_to_batch(self, rows: RowsImage, table: int = 0, item_idx: Optional[Sequence[int]] = None, threads: int = 0) -> Transposed:
        pb, pm, po = C.POINTER(abi.TfBatch)(), C.POINTER(abi.TfRowMeta)(), C.POINTER(abi.TfOldKeys)()
        idx = None if item_idx is None else np.asarray(item_idx, dtype=np.uint64)
        rc = self._L.tfgpu_rows_to_batch(self._h, C.byref(rows.struct), table, None if idx is None else idx.ctypes.data, 0 if idx is None else len(idx),
                                         threads, C.byref(pb), C.byref(pm), C.byref(po))
        if rc: raise engine.EngineError(rc, self._L.tfgpu_columnar_last_error(self._h).decode())
        b = batch_from_struct(pb.contents); n = b.nrows
        t = Transposed(b, pb, pm if pm else None, po if po else None)
        if pm:
            m = pm.contents
            t.ids, t.lsn, t.commit_time = _view(m.id, 4 * n, np.uint32), _view(m.lsn, 8 * n, np.uint64), _view(m.commit_time, 8 * n, np.uint64)
        if po:
            o = po.contents
            t.old_batch = batch_from_struct(C.cast(o.values, C.POINTER(abi.TfBatch)).contents)
            t.old_present = _view(o.present_cols, len(b.columns)); t.old_row_has = _view(o.row_has, n)
        return t

    def gather(self, batch: abi.Batch, keep: np.ndarray, threads: int = 0) -> Tuple[abi.Batch, np.ndarray]:
        """tfgpu_batch_gather: (rows with keep != 0 as a batch in the pool's buffers, the input row of every output row)."""
        tb = batch.as_struct(); keep = np.ascontiguousarray(keep, dtype=np.uint8)
        pb, ps = C.POINTER(abi.TfBatch)(), C.POINTER(C.c_uint32)()
        rc = self._L.tfgpu_batch_gather(self._h, C.byref(tb), keep.ctypes.data, threads, C.byref(pb), C.byref(ps))
        if rc: raise engine.EngineError(rc, self._L.tfgpu_columnar_last_error(self._h).decode())
        out = batch_from_struct(pb.contents)
        return out, (np.ctypeslib.as_array(ps, shape=(out.nrows,)).copy() if out.nrows else np.zeros(0, np.uint32))

    def close(self):
        if self._h: self._L.tfgpu_columnar_destroy(self._h); self._h = None


def batch_to_rows(batch: abi.Batch) -> Tuple[bytes, np.ndarray]:
    """tfgpu_batch_to_rows: (value images back to back, nrows + 1 offsets)."""
    L = engine.load_library(); tb = batch.as_struct()
    off = np.zeros(batch.nrows + 1, dtype=np.uint64); need = C.c_uint64()
    L.tfgpu_batch_to_rows(C.byref(tb), None, 0, off.ctypes.data, C.byref(need))
    out = np.zeros(int(need.value) + 1, dtype=np.uint8)
    rc = L.tfgpu_batch_to_rows(C.byref(tb), out.ctypes.data, int(need.value), off.ctypes.data, C.byref(need))
    if rc: raise engine.EngineError(rc, "tfgpu_batch_to_rows")
    return out[:int(need.value)].tobytes(), off
