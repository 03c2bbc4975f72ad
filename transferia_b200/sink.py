"""Host side of the boundary (include/tfgpu_sink.h) bound over ctypes: the ClickHouse native client writer that ships the device's
frames (the reference's streamer, pkg/providers/clickhouse/async/streamer.go:64-265), mirrored with the reference's method names.

    ClickHouseWriter.prepare_batch()  ~ conn.PrepareBatch          streamer.go:246, sink_table.go:655 (tx.PrepareContext)
    ClickHouseWriter.append_frames()  ~ batch.Append ... Flush     streamer.go:64-118,196
    ClickHouseWriter.send()           ~ batch.Send                 streamer.go:143,212
"""
from __future__ import annotations

import ctypes as C
import json
from typing import List, Optional, Tuple

import numpy as np

from . import abi, engine
from .abi import TF_SINK_FN, TfSinkEvent, TfSinkStats  # noqa: F401  (TfSinkEvent: the struct a callback receives)

SINK_SYMBOLS = list(abi.TFGPU_SINK_H_PROTOTYPES)    # the functions of include/tfgpu_sink.h


def host_cityhash128(data: bytes) -> Tuple[int, int]:
    out = (C.c_uint64 * 2)()
    buf = C.create_string_buffer(data, len(data)) if data else None
    engine.load_library().tfgpu_host_cityhash128(C.cast(buf, C.c_void_p) if buf else None, len(data), out)
    return int(out[0]), int(out[1])


def regex_replace_all(pattern: str, rule: str, src: bytes) -> bytes:
    """regexp.MustCompile(pattern).ReplaceAll(src, rule) (regex_replace/transformer.go:127-142) as tfgpu_sink_push applies it; EngineError with
    rc TF_E_FATAL_CONFIG for an expression Go refuses too, TF_E_FATAL_UNSUPPORTED for syntax the library does not carry."""
    pat, rl = pattern.encode("utf-8", "surrogateescape"), rule.encode("utf-8", "surrogateescape")
    if b"\0" in pat or b"\0" in rl:
        raise ValueError("a NUL inside the expression does not travel as a C string (write \\x00)")
    cap = max(64, 2 * len(src) + 64)
    while True:
        out = C.create_string_buffer(cap)
        n = engine.load_library().tfgpu_regex_replace_all(pat, rl, src, len(src), out, cap)
        if n < 0:
            raise engine.EngineError(int(n), "tfgpu_regex_replace_all")
        if n <= cap:
            return out.raw[:n]
        cap = int(n)


def insert_query(database: str, table: str, columns: List[str], updateable: bool = False) -> str:
    """doOperation's statement (sink_table.go:633-660) as clickhouse-go sends it (cut at VALUES)."""
    out = C.create_string_buffer(1 << 16)
    n = engine.load_library().tfgpu_ch_insert_query(database.encode(), table.encode(), json.dumps(columns).encode(), int(updateable), out, len(out))
    if n < 0:
        raise engine.EngineError(int(n), "tfgpu_ch_insert_query")
    return out.raw[:n].decode()


class ClickHouseWriter:
    """One native-protocol connection over a connected socket (the caller dials and keeps the socket object alive)."""

    def __init__(self, sock, database="default", user="default", password="", compression=True, read_timeout_ms=300000, client_name=None):
        self._L = engine.load_library()
        self._sock = sock
        self._h = C.c_void_p()
        opts = {"database": database, "user": user, "password": password, "compression": compression, "read_timeout_ms": read_timeout_ms}
        if client_name:
            opts["client_name"] = client_name
        rc = self._L.tfgpu_ch_open(sock.fileno(), json.dumps(opts).encode(), C.byref(self._h))
        if rc != 0:
            msg = self._L.tfgpu_ch_last_error(self._h).decode(errors="replace") if self._h else "open failed"
            code = self._L.tfgpu_ch_exception_code(self._h) if self._h else 0
            if self._h:
                self._L.tfgpu_ch_close(self._h); self._h = None
            err = engine.EngineError(rc, msg); err.exception_code = code
            raise err

    def _check(self, rc):
        if rc != 0:
            err = engine.EngineError(rc, self._L.tfgpu_ch_last_error(self._h).decode(errors="replace"))
            err.exception_code = self._L.tfgpu_ch_exception_code(self._h)
            raise err

    @property
    def server_info(self) -> dict:
        return json.loads(self._L.tfgpu_ch_server_info(self._h).decode())

    def prepare_batch(self, query: str, query_id: str = "", settings: Optional[dict] = None) -> List[dict]:
        self._check(self._L.tfgpu_ch_insert_begin(self._h, query.encode(), query_id.encode(), json.dumps(settings).encode() if settings else None))
        return json.loads(self._L.tfgpu_ch_insert_columns(self._h).decode())

    def append_frames(self, wire) -> None:
        """One Data packet around the bytes tfgpu_result_bytes returned (TF_WIRE_CH_NATIVE_LZ4 frames, or the raw block without compression)."""
        if isinstance(wire, (bytes, bytearray)):
            buf = (C.c_uint8 * len(wire)).from_buffer_copy(wire) if len(wire) else None
            self._check(self._L.tfgpu_ch_insert_data(self._h, C.cast(buf, C.c_void_p) if buf is not None else None, len(wire)))
        else:                                                   # (address, length): the engine's pinned landing buffer, no copy
            self._check(self._L.tfgpu_ch_insert_data(self._h, C.c_void_p(wire[0]), wire[1]))

    def send(self) -> Tuple[int, int]:
        wr, wb = C.c_uint64(), C.c_uint64()
        self._check(self._L.tfgpu_ch_insert_end(self._h, C.byref(wr), C.byref(wb)))
        return int(wr.value), int(wb.value)

    def stats(self) -> dict:
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._L.tfgpu_ch_stats(self._h, C.byref(a), C.byref(b), C.byref(c))
        return {"bytes_out": int(a.value), "bytes_in": int(b.value), "data_packets": int(c.value)}

    def close(self):
        if self._h:
            self._L.tfgpu_ch_close(self._h); self._h = None


# ------------------------------------------------------------------ Sinker.Push as one call (tfgpu_sink_*)
EV_ROWS, EV_ITEM, EV_ERRORS = 1, 2, 3


class Sink:
    """The reference's sink pipeline below the user transformers as one object (middlewares.PlugTransformer position, Appendix A of SURVEY):
    Sink.push(rows) ~ Sinker.Push([]ChangeItem). `downstream(event dict) -> int` plays the destination Sinker for what the ClickHouse writer
    does not take."""

    def __init__(self, eng=None, transformers=None, wire_fmt=0, system_tables=(), exclude_system_tables=True, errors_output="sink",
                 database="default", downstream=None, clickhouse: Optional[ClickHouseWriter] = None, debezium: Optional[dict] = None, updateable: bool = False,
                 record: str = "full"):
        """record: "full" keeps item indexes and copies of the delivered columns per event (tests); "counts" keeps type / table / n_items
        only (timing runs: the copies would be what is measured)."""
        from . import rows as _rows
        self._L = engine.load_library()
        cfg = {"transformers": transformers or [], "wire_fmt": wire_fmt, "system_tables": list(system_tables), "exclude_system_tables": exclude_system_tables,
               "errors_output": errors_output, "database": database, "updateable": updateable}
        if debezium is not None:
            cfg["debezium"] = debezium
        self._h = C.c_void_p()
        rc = self._L.tfgpu_sink_create(eng._h if eng is not None else None, json.dumps(cfg).encode(), C.byref(self._h))
        if rc:
            raise engine.EngineError(rc, "tfgpu_sink_create")
        self.events: List[dict] = []
        self._downstream = downstream

        def _cb(_ctx, evp):
            ev = evp.contents
            if record == "counts":
                d = {"type": ev.type, "table": ev.table, "n_items": int(ev.n_items)}
                self.events.append(d)
                return int(self._downstream(d)) if self._downstream else 0
            d = {"type": ev.type, "table": ev.table, "out": ((ev.out_schema or b"").decode(), (ev.out_table or b"").decode()), "n_items": int(ev.n_items),
                 "items": [int(ev.item_idx[k]) for k in range(ev.n_items)] if ev.item_idx else None, "plan_id": ev.plan_id,
                 "raw_len": int(ev.raw_len), "n_frames": int(ev.n_frames)}
            if ev.wire:
                d["wire"] = C.string_at(ev.wire, ev.wire_len)
            if ev.msg_sizes:
                d["msg_sizes"] = np.ctypeslib.as_array(ev.msg_sizes, shape=(int(ev.n_items), 7)).copy()
            if ev.batch:
                b = _rows.batch_from_struct(C.cast(ev.batch, C.POINTER(abi.TfBatch)).contents)
                d["batch"] = b
                d["columns"] = [None if c.values is None else np.asarray(c.values).copy() for c in b.columns]
                # the batch's buffers are the pool's (the next push overwrites them): var-width columns are copied here, read with var_cells()
                d["var"] = [None if c.values is not None else tuple(None if a is None else np.asarray(a).copy() for a in (c.offsets, c.heap, c.validity)) + (c.lens_width, b.nrows)
                            for c in b.columns]
            if ev.errors:
                errs = C.cast(ev.errors, C.POINTER(abi.TfRowErr))
                d["errors"] = [(errs[k].row, errs[k].code, errs[k].term) for k in range(ev.n_items)]
            self.events.append(d)
            return int(self._downstream(d)) if self._downstream else 0
        self._cb = TF_SINK_FN(_cb)
        self._L.tfgpu_sink_set_callback(self._h, self._cb, None)
        if clickhouse is not None:
            rc = self._L.tfgpu_sink_set_clickhouse(self._h, clickhouse._h)
            if rc:
                raise engine.EngineError(rc, self._L.tfgpu_sink_last_error(self._h).decode())

    def push(self, rows_image) -> None:
        rc = self._L.tfgpu_sink_push(self._h, C.byref(rows_image.struct))
        if rc:
            raise engine.EngineError(rc, self._L.tfgpu_sink_last_error(self._h).decode(errors="replace"))

    def stats(self) -> dict:
        st = TfSinkStats(); self._L.tfgpu_sink_stats(self._h, C.byref(st))
        return {n: int(getattr(st, n)) for n, _ in TfSinkStats._fields_}

    def close(self):
        if self._h:
            self._L.tfgpu_sink_destroy(self._h); self._h = None


def var_cells(event: dict, c: int) -> list:
    """The cells of var-width column `c` of a rows event as bytes (None = null), from the copies the callback took."""
    offsets, heap, validity, lens_width, n = event["var"][c]
    raw = offsets.astype(np.int64)
    off = np.concatenate([[0], np.cumsum(raw)]) if lens_width else raw
    text = heap.tobytes() if heap is not None else b""
    valid = np.ones(n, bool) if validity is None else np.unpackbits(validity, bitorder="little")[:n].astype(bool)
    return [text[off[r]:off[r + 1]] if valid[r] else None for r in range(n)]


class Dispatcher:
    """tfgpu_dispatcher: batches dealt round-robin over N sinks (one engine per GPU behind each), every sink on a host thread of its own,
    deliveries in submission order (SURVEY §8e). submit() returns a sequence number; wait(seq) the outcome of that batch's push."""

    def __init__(self, sinks):
        self._L = engine.load_library(); vp = C.c_void_p
        self.sinks = list(sinks)
        arr = (vp * len(self.sinks))(*[s._h for s in self.sinks])
        self._h = vp(); self._keep = {}
        rc = self._L.tfgpu_dispatcher_create(arr, len(self.sinks), C.byref(self._h))
        if rc:
            raise engine.EngineError(rc, "tfgpu_dispatcher_create")

    def submit(self, rows_image) -> int:
        seq = C.c_uint64()
        rc = self._L.tfgpu_dispatcher_submit(self._h, C.byref(rows_image.struct), C.byref(seq))
        if rc:
            raise engine.EngineError(rc, "tfgpu_dispatcher_submit")
        self._keep[int(seq.value)] = rows_image                 # the image must outlive the push
        return int(seq.value)

    def wait(self, seq: int) -> None:
        rc = self._L.tfgpu_dispatcher_wait(self._h, seq)
        self._keep.pop(seq, None)
        if rc:
            s = self.sinks[seq % len(self.sinks)]
            raise engine.EngineError(rc, s._L.tfgpu_sink_last_error(s._h).decode(errors="replace"))

    def drain(self) -> int:
        return int(self._L.tfgpu_dispatcher_drain(self._h))

    def close(self):
        if self._h:
            self._L.tfgpu_dispatcher_destroy(self._h); self._h = None; self._keep.clear()
