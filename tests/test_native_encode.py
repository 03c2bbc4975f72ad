"""The ClickHouse native-block encoder at its internal limits: k_str_sizes / k_layout_scan / k_layout_finish / k_encode_fixed /
k_encode_str_plain / k_encode_str, and k_layout_columnar / k_pack_validity behind tfgpu_push_columns.

The expected block comes from a small writer in this file, built from the native format and the cast rules
(columntypes/types.go: Date = clamped seconds // 86400 as UInt16, DateTime clamped to [0, 4291747200] as UInt32, DateTime64(6) =
s * 10^6 + ns // 1000, bool as 0 / 1, zero values under nulls, LEB128 + bytes for strings) and not from either encoder. On the CPU it
is checked against the oracle's block and read back by tests/ch_block_reader.py; on the device every case must equal both.

Each case is chosen to reach one internal boundary of the kernels (a residue mod 4 of a column start, a full or partial 256-row
tile at the 16 KiB staging limit of k_encode_str, empty tiles inside a 4-tile group, a capped k_encode_fixed grid that loops, more
than 1024 tiles in k_layout_scan, more than 256 columns or String columns) and asserts, from the expected block, that it does."""
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ch_block_reader  # noqa: E402

from transferia_b200 import abi  # noqa: E402

RAW, LZ, SER_JSON = abi.TF_WIRE_CH_NATIVE, abi.TF_WIRE_CH_NATIVE_LZ4, abi.TF_WIRE_SER_JSON
STRICT_RANGE, SER_VALUE = 58, 40
TILE, GROUP, STAGE, FIX_TILE_WORDS = 256, 4, 16384, 2048       # TF_STR_TILE, TF_STR_GROUP, TF_STR_STAGE, TF_FIX_TILE_WORDS
CH_MAX = 4291747200                                              # 2106-01-01T00:00:00Z
KEEP = [{"filter_rows": {"filter": "keep > 0"}}]
CH_TYPE = {abi.TF_INT8: "Int8", abi.TF_INT16: "Int16", abi.TF_INT32: "Int32", abi.TF_INT64: "Int64", abi.TF_UINT8: "UInt8",
           abi.TF_UINT16: "UInt16", abi.TF_UINT32: "UInt32", abi.TF_UINT64: "UInt64", abi.TF_FLOAT: "Float32", abi.TF_DOUBLE: "Float64",
           abi.TF_BOOLEAN: "UInt8", abi.TF_DATE: "Date", abi.TF_DATETIME: "DateTime", abi.TF_TIMESTAMP: "DateTime64(6)",
           abi.TF_INTERVAL: "Int64", abi.TF_BYTES: "String", abi.TF_UTF8: "String"}
OUT_DTYPE = {"Int8": "<i1", "Int16": "<i2", "Int32": "<i4", "Int64": "<i8", "UInt8": "<u1", "UInt16": "<u2", "UInt32": "<u4",
             "UInt64": "<u8", "Float32": "<f4", "Float64": "<f8", "Date": "<u2", "DateTime": "<u4", "DateTime64(6)": "<i8"}


# ----------------------------------------------------------------------------- the writer
def uvarint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7f) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def varint_len(lens: np.ndarray) -> np.ndarray:
    return 1 + (lens >= 1 << 7) + (lens >= 1 << 14) + (lens >= 1 << 21) + (lens >= 1 << 28)


def valid_mask(col: abi.Column, n: int) -> np.ndarray:
    if col.validity is None:
        return np.ones(n, bool)
    return np.unpackbits(np.asarray(col.validity), bitorder="little")[:n].astype(bool)


class Encoded:
    """One column of the expected block: where its parts start, what it holds (values with the casts applied, None under nulls of
    Nullable columns) and, for String columns, the encoded length of every kept row."""
    def __init__(self, name, typ, nullable):
        self.name, self.type, self.nullable = name, typ, nullable
        self.hdr_off = self.null_off = self.data_off = self.end = 0
        self.width, self.enc = 0, None          # fixed width, or per-row LEB128 + payload lengths
        self.payload = None                     # String payload length per kept row
        self.values, self.valid = None, None

    def tile_totals(self):
        """Encoded bytes of every 256-row tile of kept rows (the k_str_sizes tile sums)."""
        if not len(self.enc):
            return np.zeros(0, np.int64)
        return np.add.reduceat(self.enc, np.arange(0, len(self.enc), TILE))


def cast_fixed(col: abi.Column, tf: int, rows: np.ndarray, todt: bool) -> np.ndarray:
    v = np.asarray(col.values)[rows]
    ns = np.asarray(col.aux).astype(np.int64)[rows] if col.aux is not None else np.zeros(len(rows), np.int64)
    if todt:                                        # to_datetime.go:137-151 seconds, then the DateTime clamp
        return np.clip(v.astype(np.int64), 0, CH_MAX).astype("<u4")
    if tf in (abi.TF_DATE, abi.TF_DATETIME):
        s = v.astype(np.int64)
        s = np.where((s > CH_MAX) | ((s == CH_MAX) & (ns > 0)), CH_MAX, np.maximum(s, 0))
        return (s // 86400).astype("<u2") if tf == abi.TF_DATE else s.astype("<u4")
    if tf == abi.TF_TIMESTAMP:
        with np.errstate(over="ignore"):
            return (v.astype(np.int64) * 10 ** 6 + ns // 1000).astype("<i8")
    if tf == abi.TF_BOOLEAN:
        return (v != 0).astype("<u1")
    return v.astype(v.dtype.newbyteorder("<"))


def write_block(batch: abi.Batch, schema, keep: np.ndarray, tostr=(), todt=()):
    """-> (block bytes, [Encoded]) for the kept input rows `keep` (in order); tostr / todt: names of utf8 columns under
    convert_to_string (the text of a string is itself) and int32 / uint32 columns under convert_to_datetime."""
    keep = np.asarray(keep, dtype=np.int64); n = len(keep)
    out = [b"\x01\x00\x02\xff\xff\xff\xff\x00", uvarint(len(schema)), uvarint(n)]
    pos = sum(map(len, out)); cols = []
    for sc, col in zip(schema, batch.columns):
        tf = abi.YT_NAME_TO_TF[sc["type"]]
        typ = "DateTime" if sc["name"] in todt else CH_TYPE[tf]
        nullable = not sc.get("required", False)
        e = Encoded(sc["name"], f"Nullable({typ})" if nullable else typ, nullable)
        name = sc["name"].encode()
        hdr = uvarint(len(name)) + name + uvarint(len(e.type)) + e.type.encode() + b"\x00"
        v = src_valid = valid_mask(col, batch.nrows)[keep]
        if sc["name"] in tostr:
            assert tf == abi.TF_UTF8 and not nullable
        if sc["name"] in todt:
            v = np.ones(n, bool)                    # nil -> time.Unix(0, 0): a value, never NULL
        e.valid = v
        nullmap = (~v).astype(np.uint8).tobytes() if nullable and n else b""
        if typ == "String":
            off = np.asarray(col.offsets).astype(np.int64); heap = np.asarray(col.heap).view(np.uint8) if col.heap is not None else np.zeros(0, np.uint8)
            starts, lens = off[keep], np.where(v, off[keep + 1] - off[keep], 0)
            vl = varint_len(lens); enc = vl + lens
            data = np.zeros(int(enc.sum()), np.uint8)
            at = np.concatenate([[0], np.cumsum(enc)[:-1]]).astype(np.int64) if n else np.zeros(0, np.int64)
            for k in range(5):                      # LEB128 of the payload length
                m = vl > k
                data[at[m] + k] = ((lens[m] >> (7 * k)) & 0x7f) | np.where(vl[m] > k + 1, 0x80, 0)
            P = int(lens.sum())
            if P:
                before = np.concatenate([[0], np.cumsum(lens)[:-1]])
                step = np.arange(P) - np.repeat(before, lens)
                data[np.repeat(at + vl, lens) + step] = heap[np.repeat(starts, lens) + step]
            body = data.tobytes()
            e.enc, e.payload = enc, lens
            e.values = [heap[s:s + L].tobytes() if ok else (None if nullable else b"") for s, L, ok in zip(starts, lens, v)]
        else:
            vals = cast_fixed(col, tf, keep, sc["name"] in todt)
            raw = vals.view(f"<u{vals.itemsize}").copy(); raw[~src_valid] = 0
            body = raw.tobytes(); e.width = vals.itemsize
            e.values = raw.view(vals.dtype)
        e.hdr_off = pos; e.null_off = pos + len(hdr); e.data_off = e.null_off + len(nullmap); e.end = e.data_off + len(body)
        out += [hdr, nullmap, body]; pos = e.end; cols.append(e)
    return b"".join(out), cols


def locate(got: bytes, want: bytes, cols) -> str:
    """Where two blocks first differ: the column, the part, the kept row j, its tile and the byte offset inside the column's data."""
    a, b = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
    m = min(len(a), len(b))
    d = np.flatnonzero(a[:m] != b[:m])
    d = int(d[0]) if len(d) else m
    where = f"block of {len(got)} B vs {len(want)} B, first difference at byte {d}"
    for e in cols:
        if e.hdr_off <= d < max(e.end, e.hdr_off + 1) or e is cols[-1]:
            if d < e.null_off:
                return f"{where}: header of column {e.name!r}"
            if d < e.data_off:
                j = d - e.null_off
                return f"{where}: null map of column {e.name!r}, kept row j={j}, tile {j // TILE}"
            x = d - e.data_off
            j = x // e.width if e.width else int(np.searchsorted(np.cumsum(e.enc), x, side="right"))
            return f"{where}: data of column {e.name!r} ({e.type}), kept row j={j}, tile {j // TILE}, byte {x} of the column"
    return f"{where}: in the block header"


def columnar_mismatch(got: abi.Batch, ref: abi.Batch, names) -> str:
    """The first difference between two push_columns batches, by column, field, kept row and tile ('' when equal)."""
    if got.nrows != ref.nrows:
        return f"rows {got.nrows} vs {ref.nrows}"
    n = got.nrows
    for k, (x, y) in enumerate(zip(got.columns, ref.columns)):
        for f in ("values", "validity", "offsets", "heap", "aux"):
            u, w = getattr(x, f), getattr(y, f)
            if not n and f in ("validity", "aux") and (u is None or not len(u)) and (w is None or not len(w)):
                continue                            # without rows an absent bitmap / aux array and an empty one are the same column
            if (u is None) != (w is None):
                return f"column {names[k]!r}: {f} present on one side only"
            if u is None:
                continue
            if f == "validity":
                u, w = np.unpackbits(u, bitorder="little")[:n], np.unpackbits(w, bitorder="little")[:n]
            u, w = np.asarray(u), np.asarray(w)
            if u.shape == w.shape and np.array_equal(u.view(np.uint8), w.view(np.uint8)):
                continue
            m = min(len(u), len(w))
            d = np.flatnonzero(u[:m].view(np.uint8)[:m * u.itemsize] != w[:m].view(np.uint8)[:m * u.itemsize]) if m else []
            i = int(d[0]) // u.itemsize if len(d) else m
            j = int(np.searchsorted(np.asarray(y.offsets), i, side="right")) - 1 if f == "heap" else i
            return f"column {names[k]!r}: {f} differs at element {i} (kept row j={j}, tile {j // TILE})"
    return ""


# ----------------------------------------------------------------------------- cases
class Case:
    def __init__(self, batch, schema, trs, keep, tostr=(), todt=(), reach=None, lz=False, narrow=False, selective=False):
        self.batch, self.schema, self.trs, self.keep = batch, schema, trs, np.asarray(keep, dtype=np.int64)
        self.tostr, self.todt, self.reach = tuple(tostr), tuple(todt), reach
        self.lz, self.narrow, self.selective = lz, narrow, selective
        all_trs = list(trs)
        if tostr:
            all_trs.append({"convert_to_string": {"columns": {"includeColumns": [f"^{c}$" for c in tostr]}}})
        if todt:
            all_trs.append({"convert_to_datetime": {"columns": {"includeColumns": [f"^{c}$" for c in todt]}}})
        self.all_trs = all_trs

    @functools.cached_property
    def expected(self):
        return write_block(self.batch, self.schema, self.keep, self.tostr, self.todt)


def rand_strings(rng, n, lo, hi, alphabet=b"abcdefghijklmnopqrstuvwxyz0123456789"):
    lens = rng.integers(lo, hi + 1, n)
    pool = np.frombuffer(alphabet, np.uint8)
    flat = pool[rng.integers(0, len(pool), int(lens.sum()))].tobytes()
    at = np.concatenate([[0], np.cumsum(lens)])
    return [flat[at[i]:at[i + 1]] for i in range(n)]


def build(cols, keepcol=None, trs=KEEP, **kw):
    """cols: [(name, yt type, required, Column)]; keepcol: the int8 `keep` values (None: no filter, every row kept)."""
    schema, columns = [], []
    if keepcol is not None:
        keepcol = np.asarray(keepcol, dtype=np.int8)
        schema.append({"name": "keep", "type": "int8", "required": True}); columns.append(abi.fixed_to_column(abi.TF_INT8, keepcol))
    for name, typ, req, col in cols:
        schema.append({"name": name, "type": typ, "required": req}); columns.append(col)
    n = len(columns[0].values) if columns[0].values is not None else len(columns[0].offsets) - 1
    keep = np.flatnonzero(keepcol > 0) if keepcol is not None else np.arange(n)
    return Case(abi.Batch(n, columns), schema, trs if keepcol is not None else [], keep, **kw)


def base_cols(rng, n, nulls=0.1):
    """A mixed table: nullable utf8 of 0..40 bytes, bytes of 0..300 (1- and 2-byte lengths), nullable int32, timestamp with nanos."""
    null = lambda: rng.random(n) < nulls
    s = rand_strings(rng, n, 0, 40); ns = null()
    return [("s", "utf8", False, abi.strings_to_column(abi.TF_UTF8, [None if z else x for x, z in zip(s, ns)])),
            ("b", "string", True, abi.strings_to_column(abi.TF_BYTES, rand_strings(rng, n, 0, 300))),
            ("i", "int32", False, abi.fixed_to_column(abi.TF_INT32, rng.integers(-2 ** 31, 2 ** 31, n), null())),
            ("t", "timestamp", True, abi.fixed_to_column(abi.TF_TIMESTAMP, rng.integers(-2 * 10 ** 9, 9 * 10 ** 9, n), nanos=rng.integers(0, 10 ** 9, n)))]


def keep_exactly(rng, n_in, n_kept):
    k = np.zeros(n_in, np.int8); k[rng.choice(n_in, n_kept, replace=False)] = 1
    k[k == 0] = rng.choice(np.array([0, -1, -128], np.int8), int((k == 0).sum()))
    return k


def case_kept(n_kept):
    rng = np.random.default_rng(n_kept)
    n_in = 2 * n_kept + 300
    def reach(c, cols):
        assert len(c.keep) == n_kept and len(cols[1].tile_totals()) == -(-n_kept // TILE)
    return build(base_cols(rng, n_in), keep_exactly(rng, n_in, n_kept), reach=reach, lz=n_kept in (1, 257, 4097), narrow=n_kept in (255, 1025))


def case_all_kept(n):
    rng = np.random.default_rng(1000 + n)
    def reach(c, cols):
        assert len(c.keep) == n and not c.trs
    return build(base_cols(rng, n), None, reach=reach, lz=n in (0, 4097))


def case_tile_end(which):
    """Only the first (or only the last) input row of every 256-row block is kept: one kept row per k_filter block."""
    rng = np.random.default_rng(7 if which == "first" else 8)
    n_in = 256 * 40
    k = np.zeros(n_in, np.int8); k[(0 if which == "first" else 255)::256] = 1
    def reach(c, cols):
        assert np.array_equal(np.bincount(c.keep // 256, minlength=40), np.ones(40, np.int64))
    return build(base_cols(rng, n_in), k, reach=reach)


def case_string_groups(which):
    """Kept rows whose strings leave empty tiles: a 4-tile group with only its last tile non-empty, or a whole empty group (tiles 4..7)
    between two non-empty ones. Empty strings cost one LEB128 byte in the block and nothing in the columnar heap."""
    rng = np.random.default_rng(11 if which == "last_tile" else 12)
    n_kept = 1024 if which == "last_tile" else 3 * 1024
    n_in = n_kept + n_kept // 2
    k = keep_exactly(rng, n_in, n_kept); kept = np.flatnonzero(k > 0)
    empty_tiles = [0, 1, 2] if which == "last_tile" else [4, 5, 6, 7]
    s = rand_strings(rng, n_in, 1, 50)
    for j in range(n_kept):
        if j // TILE in empty_tiles: s[kept[j]] = b""
    nulls = (rng.random(n_in) < 0.2) & ~np.isin(np.arange(n_in), kept[np.isin(np.arange(n_kept) // TILE, empty_tiles)])
    cols = [("s", "utf8", True, abi.strings_to_column(abi.TF_UTF8, s)),
            ("ns", "string", False, abi.strings_to_column(abi.TF_BYTES, [None if z or (j in kept[np.isin(np.arange(n_kept) // TILE, empty_tiles)]) else x for j, (x, z) in enumerate(zip(s, nulls))]))]
    def reach(c, cols):
        per_tile = np.add.reduceat(cols[1].payload, np.arange(0, n_kept, TILE))
        assert [t for t in range(len(per_tile)) if per_tile[t] == 0] == empty_tiles and (per_tile[[t for t in range(len(per_tile)) if t not in empty_tiles]] > 0).all()
        assert all(cols[1].tile_totals()[t] == TILE for t in empty_tiles)
    return build(cols, k, reach=reach, lz=True)


def case_keep_rate(rate):
    rng = np.random.default_rng(int(rate * 1000))
    n_in = 20000
    k = (rng.random(n_in) < rate).astype(np.int8)
    def reach(c, cols):
        assert abs(len(c.keep) / n_in - rate) < 0.01 + rate * 0.1
    return build(base_cols(rng, n_in, nulls=0.3), k, reach=reach, selective=True, narrow=True)


# every stream kind of k_encode_fixed: (name stem, yt type, values, nanos, to_datetime)
def fixed_kinds(rng, n):
    def edge(vals, dtype):
        return np.resize(np.asarray(vals, dtype=dtype), n)[rng.permutation(n)]
    i64 = edge([-2 ** 63, 2 ** 63 - 1, 0, -1, 1], np.int64)
    f32 = np.resize(np.array([0x80000000, 0x7fc00001, 0xff800001, 0x7f800000, 0x3f800000], np.uint32), n).view(np.float32)
    f64 = np.resize(np.array([0x8000000000000000, 0x7ff8000000000123, 0xfff0000000000001, 0x7ff0000000000000, 1], np.uint64), n).view(np.float64)
    secs = edge([-1, 0, 4291747199, CH_MAX, CH_MAX, CH_MAX + 1, 86399, 86400], np.int64)
    nanos = edge([0, 1, 0, 0, 1, 0, 999999999, 0], np.int64)
    return [("i8", "int8", edge([-128, 127, 0, -1], np.int8), None, False), ("u8", "uint8", edge([0, 255, 1], np.uint8), None, False),
            ("i16", "int16", edge([-32768, 32767, 0], np.int16), None, False), ("u16", "uint16", edge([65535, 0, 1], np.uint16), None, False),
            ("i32", "int32", edge([-2 ** 31, 2 ** 31 - 1, 0], np.int32), None, False), ("f32", "float", f32, None, False),
            ("u32", "uint32", edge([2 ** 32 - 1, 0], np.uint32), None, False), ("i64", "int64", i64, None, False), ("f64", "double", f64, None, False),
            ("u64", "uint64", edge([2 ** 64 - 1, 0, 2 ** 63], np.uint64), None, False), ("iv", "interval", i64, None, False),
            ("bool", "boolean", edge([0, 1, 2, 255], np.uint8), None, False), ("date", "date", secs, nanos, False),
            ("dt", "datetime", secs, nanos, False), ("ts", "timestamp", secs, nanos, False), ("tsn", "timestamp", secs, None, False),
            ("todt", "int32", edge([-1, 0, 2 ** 31 - 1, -2 ** 31, 86400], np.int32), None, True),
            ("todtu", "uint32", edge([2 ** 32 - 1, CH_MAX - 1, CH_MAX, 0], np.uint32), None, True)]


def stream_kind(e, todt):
    t = e.type[9:-1] if e.nullable else e.type
    return "todt" if todt else t if t in ("Date", "DateTime", "DateTime64(6)") else f"w{e.width}"


def case_alignment(filtered):
    """Every fixed stream kind (copy at widths 1 / 2 / 4 / 8, bool, Date, DateTime, DateTime64 with and without nanos,
    convert_to_datetime) and the null map start at each residue mod 4 of the block: each column's name length is picked from what
    the columns before it take."""
    rng = np.random.default_rng(21 if filtered else 22)
    n_in = 3001
    k = (rng.random(n_in) < 0.55).astype(np.int8) if filtered else None
    n = int((k > 0).sum()) if filtered else n_in
    pos = 8 + len(uvarint(0)) + len(uvarint(n))            # (the column count stays below 128: one byte)
    if filtered:
        pos += len(b"\x04keep\x04Int8\x00") + n
    cols, todt = [], []
    for stem, typ, vals, nanos, dt in fixed_kinds(rng, n_in):
        tf = abi.YT_NAME_TO_TF[typ]
        chtyp = "DateTime" if dt else CH_TYPE[tf]
        w = np.dtype(OUT_DTYPE[chtyp]).itemsize
        for nullable in (False, True):
            for r in range(4):
                full = f"Nullable({chtyp})" if nullable else chtyp
                for pad in range(4):
                    name = f"{stem}_{int(nullable)}{r}" + "_" * pad
                    hdr = 1 + len(name) + 1 + len(full) + 1
                    if (pos + hdr) % 4 == r:                             # null map start (nullable) or data start

                        break
                nulls = rng.random(n_in) < 0.3 if nullable else None
                cols.append((name, typ, not nullable, abi.fixed_to_column(tf, vals, nulls, nanos)))
                if dt: todt.append(name)
                pos += hdr + (n if nullable else 0) + w * n
    def reach(c, enc):
        got = {}
        for e in enc:
            if e.name == "keep": continue
            kind = stream_kind(e, e.name in c.todt)
            got.setdefault(kind, set()).add(e.data_off % 4)
            if e.nullable: got.setdefault("nullmap", set()).add(e.null_off % 4)
        assert set(got) == {"w1", "w2", "w4", "w8", "Date", "DateTime", "DateTime64(6)", "todt", "nullmap"}
        assert all(v == {0, 1, 2, 3} for v in got.values()), got
        ts = [e for e in enc if e.name.startswith("ts") and not e.nullable]
        assert {e.name[:3] for e in ts} == {"ts_", "tsn"}                   # with and without nanos
    return build(cols, k, todt=todt, reach=reach, lz=filtered, narrow=True)


def case_leb128():
    """Payload lengths where the LEB128 length grows a byte, next to short strings, across tile edges."""
    rng = np.random.default_rng(31)
    L = [0, 1, 127, 128, 16383, 16384, 2097151, 2097152]
    n = 1200
    s = rand_strings(rng, n, 0, 20)
    at = [0, 1, 255, 256, 257, 511, 512, 1023]
    for p, ln in zip(at, L):
        s[p] = bytes(rng.integers(0, 256, ln, dtype=np.uint8))
    def reach(c, enc):
        e = enc[0]
        assert sorted(set(varint_len(np.array(L)).tolist())) == [1, 2, 3, 4] and set(L) <= set(e.payload.tolist())
    return build([("s", "string", True, abi.strings_to_column(abi.TF_BYTES, s))], None, reach=reach, lz=True)


def case_big_row():
    """One tile that holds a single 5 MB row and 255 empty strings, then tiles of empty strings only."""
    n = 4 * TILE + 10
    s = [b""] * n; s[3] = bytes(np.random.default_rng(32).integers(0, 256, 5 << 20, dtype=np.uint8))
    def reach(c, enc):
        t = enc[0].tile_totals()
        assert t[0] == (5 << 20) + 4 + 255 and (t[1:] == [TILE, TILE, TILE, 10]).all()
    return build([("s", "utf8", True, abi.strings_to_column(abi.TF_UTF8, s)), ("x", "int16", True, abi.fixed_to_column(abi.TF_INT16, np.arange(n)))], None, reach=reach, lz=True)


def case_nulls_at_tile_edges():
    rng = np.random.default_rng(33)
    n_in = 5000
    k = keep_exactly(rng, n_in, 2100); kept = np.flatnonzero(k > 0)
    edges = [0, 255, 256, 511, 512, 1023, 1024, 1025, 2047, 2048, 2099]
    nulls = np.zeros(n_in, bool); nulls[kept[edges]] = True
    s = rand_strings(rng, n_in, 0, 30)
    cols = [("ns", "utf8", False, abi.strings_to_column(abi.TF_UTF8, [None if z else x for x, z in zip(s, nulls)])),
            ("nb", "string", False, abi.strings_to_column(abi.TF_BYTES, [None if z else x for x, z in zip(s[::-1], nulls)]))]
    def reach(c, enc):
        assert set(np.flatnonzero(~enc[1].valid).tolist()) == set(edges)
    return build(cols, k, reach=reach, narrow=True)


def case_staging(L, n_kept):
    """convert_to_string over a utf8 column of L-byte cells: a full tile is 256 * (L + 1) bytes, 16384 for L = 63 (staged in shared
    memory) and 16640 for L = 64 (written directly); partial last tiles just under and over the limit."""
    rng = np.random.default_rng(40 + L + n_kept)
    n_in = n_kept + 700
    k = keep_exactly(rng, n_in, n_kept)
    cols = [("txt", "utf8", True, abi.strings_to_column(abi.TF_UTF8, rand_strings(rng, n_in, L, L))),
            ("plain", "utf8", True, abi.strings_to_column(abi.TF_UTF8, rand_strings(rng, n_in, L, L)))]
    def reach(c, enc):
        t = enc[1].tile_totals().tolist()
        full, part = n_kept // TILE, n_kept % TILE
        assert t[:full] == [TILE * (L + 1)] * full and (not part or t[-1] == part * (L + 1))
        assert {x <= STAGE for x in t} == {L + 1 <= STAGE // TILE} | ({part * (L + 1) <= STAGE} if part else set())
    return build(cols, k, tostr=["txt"], reach=reach, lz=n_kept % TILE == 0)


def case_scale():
    """About 300 k kept rows: more than 1024 tiles, so k_layout_scan's 1024-thread CTA loops over its tiles."""
    rng = np.random.default_rng(50)
    n_in = 320_000
    k = (rng.random(n_in) < 0.95).astype(np.int8)
    cols = [("s", "utf8", False, abi.strings_to_column(abi.TF_UTF8, [None if z else x for x, z in zip(rand_strings(rng, n_in, 0, 12), rng.random(n_in) < 0.1)])),
            ("v", "int64", True, abi.fixed_to_column(abi.TF_INT64, rng.integers(-2 ** 63, 2 ** 63 - 1, n_in)))]
    def reach(c, enc):
        assert len(enc[1].tile_totals()) > 1024
    return build(cols, k, reach=reach, lz=True, selective=True)


FIXED_GRID_COLS, FIXED_GRID_ROWS = 128, 72_000


def case_fixed_grid():
    """Enough fixed-width slots that k_encode_fixed's grid is capped (grid_cap) below the tiles of its 8-byte streams, so the CTAs
    loop over them (asserted on the device from the SM count)."""
    rng = np.random.default_rng(60)
    n_in = FIXED_GRID_ROWS
    k = (rng.random(n_in) < 0.9).astype(np.int8)
    cols = [(f"v{i:03d}", "int64", i % 8 != 0, abi.fixed_to_column(abi.TF_INT64, rng.integers(-2 ** 40, 2 ** 40, n_in), rng.random(n_in) < 0.1 if i % 8 == 0 else None))
            for i in range(FIXED_GRID_COLS)]
    return build(cols, k, reach=lambda c, enc: fixed_loops(c, 132) >= 2 or pytest.fail("no second pass at 132 SMs"))


def fixed_slots(case):
    return sum(1 + (not sc.get("required", False)) for sc in case.schema if abi.YT_NAME_TO_TF[sc["type"]] not in abi.VAR_TYPES)


def fixed_loops(case, sm_count):
    """CTA passes of k_encode_fixed over its widest stream (grid_cap in tfgpu.cu: 6 resident CTAs per SM, 6 waves, at least 8)."""
    slots, n_in, n = fixed_slots(case), case.batch.nrows, len(case.keep)
    want = -(-(sm_count * 36) // slots)
    gx = max(1, min(-(-(2 * n_in + 2) // FIX_TILE_WORDS), max(want, 8)))
    words = -(-(3 + 8 * n) // 4)
    return -(-(-(-words // FIX_TILE_WORDS)) // gx)


def wide_table(n_str, loose=True, seed=70):
    """320 columns: keep (0), doubles at 255 and 300 (NaN in some rows), an int32 column at 280 (loose: its values arrive as int64 and
    some are out of range), a few other fixed columns, and n_str utf8 / bytes columns, a third of them nullable. Names run up to 130
    bytes. -> (Case over the strict batch with the failing rows dropped, loose batch, rows that fail Strictify)."""
    rng = np.random.default_rng(seed)
    n_in, ncols = 700, 320
    keepv = (rng.random(n_in) < 0.75).astype(np.int8)
    fixed_at = {255: "double", 280: "int32", 300: "double"}
    others = [i for i in range(1, ncols) if i not in fixed_at]
    for i in others[: ncols - 1 - len(fixed_at) - n_str]:
        fixed_at[i] = ("int16", "uint64", "date", "float", "boolean")[i % 5]
    nan255 = np.zeros(n_in, bool); nan255[rng.choice(n_in, 30, replace=False)] = True
    nan300 = np.zeros(n_in, bool); nan300[rng.choice(np.flatnonzero(~nan255), 30, replace=False)] = True
    v280 = rng.integers(-2 ** 31, 2 ** 31, n_in)
    bad = rng.choice(np.flatnonzero(~nan255 & ~nan300), 25, replace=False)
    v280[bad] = rng.choice(np.array([2 ** 31, -2 ** 31 - 1, 2 ** 40, -2 ** 62]), len(bad))
    cols = []
    for i in range(1, ncols):
        name = f"c{i}_" + "w" * max(0, (i * 37) % 131 - len(f"c{i}_"))
        if i in fixed_at:
            typ = fixed_at[i]; tf = abi.YT_NAME_TO_TF[typ]
            if i in (255, 300):
                v = rng.standard_normal(n_in); v[nan255 if i == 255 else nan300] = np.nan
                col = abi.fixed_to_column(tf, v)
            elif i == 280:
                col = abi.fixed_to_column(abi.TF_INT32, np.where(np.isin(np.arange(n_in), bad), 0, v280))
            else:
                col = abi.fixed_to_column(tf, rng.integers(0, 2 ** 15, n_in), rng.random(n_in) < 0.2)
            cols.append((name, typ, i in (255, 280, 300), col))
        else:
            typ = "utf8" if i % 2 else "string"
            s = rand_strings(rng, n_in, 0, 20)
            nullable = i % 3 == 0
            if nullable:
                s = [None if z else x for x, z in zip(s, rng.random(n_in) < 0.2)]
            cols.append((name, typ, not nullable, abi.strings_to_column(abi.YT_NAME_TO_TF[typ], s)))
    strict_keep = keepv.copy(); strict_keep[bad] = 0
    def reach(c, enc):
        assert len(enc) == ncols and sum(e.type.endswith("String") or e.type.endswith("String)") for e in enc) == n_str
        assert max(len(e.name) for e in enc) == 130 and len([e for e in enc if len(e.name) >= 128]) > 0
    case = build(cols, strict_keep, reach=reach)
    loose_cols = list(case.batch.columns)
    loose_cols[280] = abi.fixed_to_column(abi.TF_INT64, v280)
    return case, abi.Batch(n_in, loose_cols), np.sort(bad)


CASES = {}
for _n in (0, 1, 255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097):
    CASES[f"kept_{_n}"] = functools.partial(case_kept, _n)
for _n in (0, 1, 256, 257, 4097):
    CASES[f"all_kept_{_n}"] = functools.partial(case_all_kept, _n)
CASES.update({"tile_first_row": functools.partial(case_tile_end, "first"), "tile_last_row": functools.partial(case_tile_end, "last"),
              "group_last_tile_only": functools.partial(case_string_groups, "last_tile"), "empty_group_between": functools.partial(case_string_groups, "middle_group"),
              "keep_1pct": functools.partial(case_keep_rate, 0.01), "keep_50pct": functools.partial(case_keep_rate, 0.5), "keep_99pct": functools.partial(case_keep_rate, 0.99),
              "align_filtered": functools.partial(case_alignment, True), "align_all_kept": functools.partial(case_alignment, False),
              "leb128_lengths": case_leb128, "big_row_tile": case_big_row, "nulls_at_tile_edges": case_nulls_at_tile_edges,
              "stage_63_full": functools.partial(case_staging, 63, 4 * TILE), "stage_63_partial": functools.partial(case_staging, 63, 3 * TILE + 200),
              "stage_64_full": functools.partial(case_staging, 64, 4 * TILE), "stage_64_partial_under": functools.partial(case_staging, 64, 3 * TILE + 252),
              "stage_64_partial_over": functools.partial(case_staging, 64, 3 * TILE + 253),
              "scale_300k": case_scale, "fixed_grid_loops": case_fixed_grid,
              "wide_308_strings": lambda: wide_table(308)[0], "wide_250_strings": lambda: wide_table(250)[0]})


@functools.lru_cache(maxsize=None)
def get_case(name) -> Case:
    return CASES[name]()


# ----------------------------------------------------------------------------- CPU: the writer against the oracle and the reader
@pytest.mark.parametrize("name", list(CASES))
def test_writer_matches_oracle(po, name):
    c = get_case(name)
    block, enc = c.expected
    if c.reach:
        c.reach(c, enc)
    ref = po.push_encode(c.batch, po.build_plan("db", "t", c.schema, c.all_trs), RAW)
    assert ref.rows_out == len(c.keep) and ref.errors == []
    assert block == ref.raw, locate(block, ref.raw, enc)


@pytest.mark.parametrize("name", list(CASES))
def test_reader_reads_writer_back(name):
    """The block parsed by tests/ch_block_reader.py gives back the names, types and kept input values after the casts."""
    c = get_case(name)
    block, enc = c.expected
    cols, nrows, data = ch_block_reader.read_block(block)
    assert nrows == len(c.keep) and cols == [(e.name, e.type) for e in enc]
    for e, sc, col in zip(enc, c.schema, c.batch.columns):
        got = data[e.name]
        if isinstance(e.values, list):
            assert got == e.values, e.name
            if sc["name"] not in c.tostr:           # the kept input cells themselves
                off = np.asarray(col.offsets).astype(np.int64); heap = np.asarray(col.heap).tobytes() if col.heap is not None else b""
                assert all(g == (heap[off[r]:off[r + 1]] if ok else (None if e.nullable else b"")) for g, r, ok in zip(got, c.keep, e.valid)), e.name
            continue
        nulls = np.array([g is None for g in got], bool)
        assert np.array_equal(nulls, ~e.valid if e.nullable else np.zeros(nrows, bool)), e.name
        have = np.array([0 if g is None else g for g in got], dtype=OUT_DTYPE[e.type[9:-1] if e.nullable else e.type])
        assert have.tobytes() == e.values.tobytes(), e.name
        if abi.YT_NAME_TO_TF[sc["type"]] in (abi.TF_INT64, abi.TF_DOUBLE, abi.TF_INT32, abi.TF_UINT8) and sc["name"] not in c.todt:
            src = np.asarray(col.values)[c.keep]
            assert have[e.valid].tobytes() == src[e.valid].tobytes(), e.name       # bit patterns (NaN payloads, -0.0) kept


# ----------------------------------------------------------------------------- on the device
def _device_checks(eng, po, c, batch=None, errors=()):
    batch = batch if batch is not None else c.batch
    block, enc = c.expected
    pid = eng.plan("db", "t", c.schema, c.all_trs, {"type": "clickhouse"})
    got = eng.push_encode(pid, batch, RAW)
    assert got.rows_out == len(c.keep) and sorted(got.errors) == sorted(errors)
    assert got.wire == block, locate(got.wire, block, enc)
    return pid


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_block(eng, po, name):
    """The device block equals the writer's and the oracle's; push_columns equals the oracle's Transformed batch; a subset also
    through LZ4 frames, the two-phase selective push and narrowed (per-row length) string columns."""
    from test_gpu_parity import assert_batches_equal
    c = get_case(name)
    block, enc = c.expected
    plan = po.build_plan("db", "t", c.schema, c.all_trs)
    assert po.push_encode(c.batch, plan, RAW).raw == block
    pid = _device_checks(eng, po, c)
    names = [e.name for e in enc]
    got, gerr = eng.push_columns(pid, c.batch)
    ref, rerr = po.push_columns(c.batch, plan)
    assert gerr == rerr == []
    assert not columnar_mismatch(got, ref, names), columnar_mismatch(got, ref, names)
    if got.nrows:
        assert_batches_equal(got, ref)
    if c.lz:
        z = eng.push_encode(pid, c.batch, LZ)
        raw, nf = po.ch_decode_frames(z.wire)
        assert raw == block and nf == z.n_frames == max(1, -(-len(block) // eng.frame_bytes)), locate(raw or b"", block, enc)
    if c.selective:
        s = eng.push_encode(pid, c.batch, RAW, selective=2)
        assert s.wire == block, locate(s.wire, block, enc)
    if c.narrow:
        nb = c.batch.narrow()
        assert any(col.lens_width for col in nb.columns if col.type in abi.VAR_TYPES) or all(col.type not in abi.VAR_TYPES for col in nb.columns)
        w = eng.push_encode(pid, nb, RAW).wire
        assert w == block, locate(w, block, enc)
        g2, _ = eng.push_columns(pid, nb)
        assert not columnar_mismatch(g2, ref, names), columnar_mismatch(g2, ref, names)


@pytest.mark.gpu
def test_device_fixed_grid_loops(eng, po):
    """The case's 8-byte streams take at least two passes of k_encode_fixed's capped grid on this device."""
    import torch
    c = get_case("fixed_grid_loops")
    assert fixed_slots(c) == FIXED_GRID_COLS + FIXED_GRID_COLS // 8 + 1
    assert fixed_loops(c, torch.cuda.get_device_properties(0).multi_processor_count) >= 2
    _device_checks(eng, po, c)


def misaligned_device_batch(batch, shifts):
    """The batch in HBM with every String heap a view at byte offset shifts[k % len] into a larger tensor (values, validity and
    offsets keep their natural alignment)."""
    import torch
    d = batch.to_device("cuda:0")
    cols, keep, used = [], [], []
    for k, c in enumerate(d.columns):
        if c.type in abi.VAR_TYPES and c.heap is not None and c.heap.numel():
            s = shifts[len(used) % len(shifts)]
            big = torch.zeros(c.heap.numel() + 16, dtype=torch.uint8, device="cuda:0")
            view = big[s:s + c.heap.numel()]; view.copy_(c.heap)
            assert view.data_ptr() % 4 == s
            c = abi.Column(c.type, c.values, c.validity, c.offsets, view, c.aux); keep.append(big); used.append(s)
        cols.append(c)
    torch.cuda.synchronize()
    out = abi.Batch(d.nrows, cols, d.kinds, abi.TF_MEM_DEVICE); out._keep = keep
    return out, used


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kept_1025", "keep_50pct", "leb128_lengths", "big_row_tile", "group_last_tile_only", "stage_64_full", "wide_308_strings"])
def test_device_misaligned_heaps(eng, po, name):
    """TF_MEM_DEVICE input whose heaps start 1, 2 or 3 bytes past a 4-byte boundary: push_encode and push_encode_resident."""
    c = get_case(name)
    block, enc = c.expected
    db, used = misaligned_device_batch(c.batch, [1, 2, 3])
    assert {1, 2, 3} <= set(used) or (len(used) >= 1 and set(used) <= {1, 2, 3})
    _device_checks(eng, po, c, db)
    pid = eng.plan("db", "t", c.schema, c.all_trs, {"type": "clickhouse"})
    eng.push_encode_resident(pid, db, RAW)
    st = eng.resident_stats()
    assert st["rows_out"] == len(c.keep) and st["n_errors"] == 0
    raw = eng.resident_fetch(0, st["raw_bytes"])
    assert raw == block, locate(raw, block, enc)


@pytest.mark.gpu
@pytest.mark.parametrize("n_str", [250, 308])
def test_device_wide_table_terms(eng, po, n_str):
    """320 columns, two passes of k_layout_finish / k_layout_columnar: a loose int64 value out of int32 range at input column 280 is
    TF_ROWERR_STRICT_RANGE with term 280, and a NaN double at output column 255 or 300 of TF_WIRE_SER_JSON is TF_ROWERR_SER_VALUE with
    that column as its term (the row-error terms are 16 bits wide)."""
    c, loose, bad = wide_table(n_str)
    want = [(int(r), STRICT_RANGE, 280) for r in bad]
    pid = _device_checks(eng, po, c, loose, want)
    got, gerr = eng.push_columns(pid, loose)
    assert sorted(gerr) == want
    ref, _ = po.push_columns(c.batch, po.build_plan("db", "t", c.schema, c.all_trs))
    assert not columnar_mismatch(got, ref, [s["name"] for s in c.schema]), columnar_mismatch(got, ref, [s["name"] for s in c.schema])
    # the batch serializer: the first column (in name order) that cannot be written is the row's term
    plan = po.build_plan("db", "t", c.schema, [])
    spid = eng.plan("db", "t", c.schema, [])
    ref = po.push_encode(c.batch, plan, SER_JSON)
    js = eng.push_encode(spid, c.batch, SER_JSON)
    assert {t for _, code, t in ref.errors if code == SER_VALUE} == {255, 300}
    assert sorted(js.errors) == sorted(ref.errors)
    assert js.wire == ref.raw
