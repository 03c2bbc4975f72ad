"""Pins the CPU oracle against the reference's own golden vectors (SURVEY §8c) and against independent
implementations available in this image (hashlib, CPython repr, numpy Dragon4, liblz4, pyarrow)."""
import ctypes as C
import datetime as dt
import hashlib
import hmac
import math
import random
import struct

import numpy as np
import pytest

from transferia_b200 import abi


def _val(po, go, v):
    if go == "string":
        return po.make_val(po.OG_STRING, s=v.encode())
    if go == "bytes":
        return po.make_val(po.OG_BYTES, s=v.encode())
    if go in ("int64", "int32", "int16", "int8", "int"):
        return po.make_val({"int64": po.OG_INT64, "int32": po.OG_INT32, "int16": po.OG_INT16, "int8": po.OG_INT8, "int": po.OG_INT}[go], i=v)
    if go in ("uint64", "uint32", "uint16", "uint8"):
        return po.make_val({"uint64": po.OG_UINT64, "uint32": po.OG_UINT32, "uint16": po.OG_UINT16, "uint8": po.OG_UINT8}[go], u=v)
    if go == "bool":
        return po.make_val(po.OG_BOOL, i=1 if v else 0)
    if go == "float64":
        return po.make_val(po.OG_FLOAT64, f=v)
    if go == "float32":
        return po.make_val(po.OG_FLOAT32, f=float(np.float32(v)))
    if go == "duration":
        return po.make_val(po.OG_DURATION, i=v)
    if go == "time":
        t = dt.datetime.fromisoformat(v.replace("Z", "+00:00"))
        us = (t - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(microseconds=1)
        return po.make_val(po.OG_TIME, i=us // 1_000_000, nsec=(us % 1_000_000) * 1000)
    if go == "nil":
        return po.make_val(po.OG_NIL)
    raise KeyError(go)


def test_mask_golden_digests(po, goldens):
    """pkg/transformer/registry/mask/gotest/canondata/result.json: all 11 digests."""
    salt = goldens["mask"]["salt"].encode()
    assert len(goldens["mask"]["cases"]) == 11
    for c in goldens["mask"]["cases"]:
        text = po.serialize_to_string(_val(po, c["go"], c["value"]), abi.YT_NAME_TO_TF[c["type"]])
        assert po.hmac_hex(salt, text) == c["digest"], (c, text)
        assert hmac.new(salt, text, hashlib.sha256).hexdigest() == c["digest"]


def test_to_string_forms(po):
    """to_string.go:145-171 text forms (mask golden inputs + to_string_test.go:16-194 style cases)."""
    s = lambda go, v, t: po.serialize_to_string(_val(po, go, v), abi.YT_NAME_TO_TF[t]).decode()
    assert s("float64", 123.123, "double") == "123.123"
    assert s("float32", 312.321, "float") == "312.321"
    assert s("duration", 60_000_000_000, "date") == "1m0s"
    assert s("time", "1703-01-02T00:00:00Z", "date") == "1703-01-02"
    assert s("time", "2022-02-03T04:05:06.123456Z", "timestamp") == "2022-02-03T04:05:06.123456Z"
    assert s("time", "2022-02-03T04:05:06Z", "datetime") == "2022-02-03T04:05:06Z"
    assert s("bool", True, "boolean") == "true"
    assert s("int8", -3, "int8") == "-3"
    assert s("uint32", 12345, "uint32") == "12345"
    assert s("nil", None, "int32") == "<nil>"
    assert s("nil", None, "any") == "null"
    assert s("string", 'a"b<c', "any") == '"a\\"b\\u003cc"'
    assert s("bytes", "raw", "string") == "raw"


def test_float_shortest_matches_repr(po):
    """strconv shortest digits == CPython repr digits (both: shortest round-trip, closest)."""
    rnd = random.Random(7)
    vals = [0.1, 0.3, 1 / 3, 1e21, 1e22, 1e23, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 9007199254740993.0, 123456.7, 1234567.0, 1e-5, 1e-4]
    vals += [struct.unpack("<d", struct.pack("<Q", rnd.getrandbits(64) & 0x7FEFFFFFFFFFFFFF))[0] for _ in range(3000)]
    vals += [rnd.random() * 10 ** rnd.randint(-20, 20) for _ in range(2000)]
    for v in vals:
        if v == 0 or math.isinf(v) or math.isnan(v):
            continue
        got = po.fmt_float64(v, 1)         # 'f', -1: plain decimal
        assert float(got) == v, (v, got)
        r = repr(v)
        mant = r.split("e")[0].replace(".", "").lstrip("0").rstrip("0") or "0"
        assert got.replace(".", "").strip("0") == mant.strip("0"), (v, got, r)


def test_float32_shortest_matches_numpy(po):
    rnd = np.random.default_rng(5)
    bits = rnd.integers(1, 0x7F7FFFFF, 3000, dtype=np.uint32)
    for f in bits.view(np.float32):
        want = np.format_float_positional(f, unique=True, trim="-")
        assert po.fmt_float32(f, 1) == want, (f, po.fmt_float32(f, 1), want)


def test_float_layouts(po):
    """%v ('g' shortest, exponent when exp < -4 || exp >= 21? no: >= 6... eprec = 6), 'f', encoding/json."""
    f = po.fmt_float64
    assert f(1000000.0) == "1e+06" and f(123456.0) == "123456" and f(1234567.0) == "1.234567e+06"
    assert f(0.0001) == "0.0001" and f(0.00001) == "1e-05" and f(0.0) == "0" and f(-0.0) == "-0"
    assert f(float("inf")) == "+Inf" and f(float("-inf")) == "-Inf" and f(float("nan")) == "NaN"
    assert f(1e21, 2) == "1e+21" and f(1e20, 2) == "100000000000000000000" and f(1e-7, 2) == "1e-7" and f(0.000001, 2) == "0.000001"
    assert f(123456789.0, 1) == "123456789" and f(1e-7, 1) == "0.0000001"


def test_duration_and_time_text(po):
    assert po.fmt_duration(0) == "0s" and po.fmt_duration(1) == "1ns" and po.fmt_duration(1500) == "1.5µs"
    assert po.fmt_duration(1_000_000) == "1ms" and po.fmt_duration(3600 * 10**9 + 5 * 10**8) == "1h0m0.5s" and po.fmt_duration(-60 * 10**9) == "-1m0s"
    for y, m, d, hh in ((1703, 1, 2, 0), (1970, 1, 1, 0), (2013, 7, 14, 21), (2106, 1, 1, 0), (1, 1, 1, 0), (1969, 12, 31, 23)):
        t = dt.datetime(y, m, d, hh, 44, 35, tzinfo=dt.timezone.utc)
        sec = (t - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(seconds=1)
        assert po.fmt_rfc3339nano(sec, 0) == t.strftime("%Y-%m-%dT%H:%M:%SZ").replace(str(y) + "-", "%04d-" % y, 1)
    assert po.fmt_rfc3339nano(0, 120_000_000) == "1970-01-01T00:00:00.12Z"


def test_filter_rows_reference_tables(po, goldens):
    """filter_rows_test.go:47-560 input/expected tables through parse_filter + matchValue."""
    for case in goldens["filter_rows"]:
        terms = po.parse_filter(case["filter"])
        kept, nerr = [], 0
        for item in case["input"]:
            go, v = (item if case["go"] == "mixed" else (case["go"], item))
            val = _val(po, go, v)
            ok, err = True, False
            for t in terms:
                rc, m = po.match_value(val, t)
                if rc:
                    err = True
                    assert rc == case.get("error_code", rc)
                    break
                if not m:
                    ok = False
                    break
            if err:
                nerr += 1
            elif ok:
                kept.append(v)
        assert kept == case["expected"], (case["name"], kept)
        assert nerr == case["errors"], case["name"]


def test_filter_null_semantics(po):
    """TestNullFiltering filter_rows_test.go:336-365."""
    terms = po.parse_filter("column1 != NULL AND column2 = NULL")
    rows = [("abc", 128), ("str", None), (None, 32), (None, None)]
    keep = []
    for s, i in rows:
        v1 = _val(po, "nil", None) if s is None else _val(po, "string", s)
        v2 = _val(po, "nil", None) if i is None else _val(po, "int", i)
        r1 = po.match_value(v1, terms[0]); r2 = po.match_value(v2, terms[1])
        keep.append(r1 == (0, True) and r2 == (0, True))
    assert keep == [False, True, False, False]


def test_filter_grammar_errors_and_forms(po):
    assert [(t.attribute, t.op, t.vtype) for t in po.parse_filter("a>1 and b NOT  IN (1.5,2.5) AND c ~ 'x'")] == [("a", po.OP_GT, 1), ("b", po.OP_NOTIN, 18), ("c", po.OP_MATCH, 4)]
    assert po.parse_filter("") == []
    for bad in ('column = str"', "a IN 5", "a = (1,2)", "a > NULL", "a IN (1, 'x')", "a = ", "= 1"):
        with pytest.raises(po.FilterSyntaxError):
            po.parse_filter(bad)
    (t,) = po.parse_filter("ts >= 1990-07-22T00:00:00.001+04:00")
    want = dt.datetime(1990, 7, 21, 20, 0, 0, 1000, tzinfo=dt.timezone.utc)
    assert t.value == (want - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(microseconds=1)
    (t,) = po.parse_filter("d = 2020-02-29")
    assert t.value == 1582934400 * 10**6


def test_sha_hmac_vs_hashlib(po):
    rnd = random.Random(3)
    for n in (0, 1, 55, 56, 63, 64, 65, 119, 120, 1000):
        msg = bytes(rnd.getrandbits(8) for _ in range(n))
        for klen in (0, 5, 64, 65, 200):
            key = bytes(rnd.getrandbits(8) for _ in range(klen))
            assert po.hmac_hex(key, msg) == hmac.new(key, msg, hashlib.sha256).hexdigest()


def lz4_block(seqs, last: bytes) -> bytes:
    """An LZ4 block written by hand: (literals, offset, match length) sequences, then the literal-only last sequence.
    Offsets and lengths are written as given, legal or not."""
    def ext(x):
        out = b""
        while x >= 255:
            out += b"\xff"; x -= 255
        return out + bytes([x])
    out = b""
    for lit, off, ml in seqs:
        ll, mt = len(lit), ml - 4
        out += bytes([(min(ll, 15) << 4) | min(mt, 15)]) + (ext(ll - 15) if ll >= 15 else b"") + lit
        out += struct.pack("<H", off) + (ext(mt - 15) if mt >= 15 else b"")
    return out + bytes([min(len(last), 15) << 4]) + (ext(len(last) - 15) if len(last) >= 15 else b"") + last


def test_lz4_oracle_vs_liblz4_and_pyarrow(po):
    import pyarrow as pa
    lz = C.CDLL("liblz4.so.1")
    rnd = np.random.default_rng(11)
    samples = [b"", b"a", b"abcabcabcabcabcabcabcabc" * 50, bytes(rnd.integers(0, 256, 5000, dtype=np.uint8)), bytes(rnd.integers(0, 4, 70000, dtype=np.uint8)), b"\0" * 100000]
    # every short length (the end-of-block rules decide everything below ~40 bytes) and long runs at the length-extension steps
    noise = bytes(rnd.integers(0, 256, 600, dtype=np.uint8))
    for n in range(41):
        samples += [b"\0" * n, (b"abcab" * 9)[:n], noise[:n]]
    for n in (13, 17, 18, 19, 20, 274, 275, 529, 70000):
        samples += [b"x" * n, noise[:7] + b"y" * n + noise[7:40], noise[:300] + noise[:n % 300] + noise[:9]]
    codec = pa.Codec("lz4_raw")
    for s in samples:
        c = po.lz4_compress(s)
        assert po.lz4_decompress(c, len(s)) == s
        dst = C.create_string_buffer(max(1, len(s)))
        assert lz.LZ4_decompress_safe(c, dst, len(c), len(s)) == len(s) and dst.raw[:len(s)] == s
        if s:
            assert codec.decompress(c, decompressed_size=len(s)).to_pybytes() == s
        # and the other direction: liblz4's stream through the oracle decoder
        cap = lz.LZ4_compressBound(len(s)); buf = C.create_string_buffer(max(1, cap))
        n = lz.LZ4_compress_default(s, buf, len(s), cap)
        assert po.lz4_decompress(buf.raw[:n], len(s)) == s

    # The oracle decoder is strict: hand-built blocks of 32 raw bytes (12 for the short one), each breaking one rule.
    u = bytes(range(100, 164))                        # no byte repeats: a literal never continues a match by accident
    ok = {                                            # the limits themselves are legal
        "match at rs - 12": (lz4_block([(u[:20], 20, 4)], u[20:28]), 32),
        "match ending at rs - 5": (lz4_block([(u[:8], 8, 19)], u[8:13]), 32),
        "extended lengths": (lz4_block([(u[:15], 15, 19)], u[15:61]), 80),
        "12 literals": (lz4_block([], u[:12]), 12),
        "empty block": (b"\x00", 0),
    }
    for what, (blk, rs) in ok.items():
        got = po.lz4_decompress(blk, rs)
        assert got is not None and len(got) == rs, what
        dst = C.create_string_buffer(max(1, rs))
        assert lz.LZ4_decompress_safe(blk, dst, len(blk), rs) == rs and dst.raw[:rs] == got, what
    valid = lz4_block([(u[:8], 8, 8)], u[8:24])
    assert po.lz4_decompress(valid, 32) == u[:8] * 2 + u[8:24]
    m8 = bytes([(8 << 4) | 15]) + u[:8] + b"\x08\x00"         # a match token whose length extension is cut off
    bad = {
        "ends after a match": (lz4_block([(u[:1], 1, 31)], b"")[:-1], 32),     # (so its match also covers the last 5 bytes)
        "match starts after rs - 12": (lz4_block([(u[:21], 21, 4)], u[21:28]), 32),
        "match ends after rs - 5": (lz4_block([(u[:8], 8, 20)], u[8:12]), 32),
        "match in a block of 12 bytes": (lz4_block([(u[:1], 1, 4)], u[1:8]), 12),
        "offset 0": (lz4_block([(u[:8], 0, 8)], u[8:24]), 32),
        "offset behind the block start": (lz4_block([(u[:8], 9, 8)], u[8:24]), 32),
        "truncated literal length": (b"\xf0\xff", 270),
        "truncated match length": (m8, 32),
        "truncated offset": (bytes([8 << 4]) + u[:8] + b"\x08", 32),
        "trailing input": (valid + b"\x00", 32),
        "decodes short": (valid, 33),
        "decodes long": (valid, 31),
        "no token": (b"", 0),
    }
    for what, (blk, rs) in bad.items():
        assert po.lz4_decompress(blk, rs) is None, what
        # the same block inside a frame with valid header and checksum: the frame walk rejects it too
        body = bytes([0x82]) + struct.pack("<II", len(blk) + 9, rs) + blk
        assert po.ch_decode_frames(struct.pack("<QQ", *po.cityhash128(body)) + body) == (None, 0), what


def test_native_block_bytes_hand_computed(po):
    """ClickHouse native block, revision 54460, two columns, two rows — bytes written out by hand from the
    protocol description (block info, counts, name/type strings, custom-serialization byte, data)."""
    schema = [{"name": "id", "type": "int32", "required": True}, {"name": "s", "type": "utf8", "required": False}]
    b = abi.Batch(2, [abi.fixed_to_column(abi.TF_INT32, [7, -2]), abi.strings_to_column(abi.TF_UTF8, [b"ab", None])])
    plan = po.build_plan("db", "t", schema, [])
    r = po.push_encode(b, plan, abi.TF_WIRE_CH_NATIVE)
    want = bytes([1, 0, 2, 0xFF, 0xFF, 0xFF, 0xFF, 0, 2, 2]) \
        + b"\x02id\x05Int32\x00" + struct.pack("<ii", 7, -2) \
        + b"\x01s\x10Nullable(String)\x00" + b"\x00\x01" + b"\x02ab" + b"\x00"
    assert r.raw == want
    fr = po.push_encode(b, plan, abi.TF_WIRE_CH_NATIVE_LZ4)
    assert fr.wire[16] == 0x82 and struct.unpack_from("<II", fr.wire, 17) == (len(fr.wire) - 16, len(want))
    raw, nf = po.ch_decode_frames(fr.wire)
    assert raw == want and nf == 1
    lo, hi = po.cityhash128(fr.wire[16:])
    assert struct.unpack_from("<QQ", fr.wire, 0) == (lo, hi)


def test_ch_types(po):
    """columntypes.ToChType types.go:210-248 + Nullable(!required) sink_table.go:229-235."""
    m = {"int8": "Int8", "uint64": "UInt64", "float": "Float32", "double": "Float64", "boolean": "UInt8", "string": "String", "utf8": "String",
         "any": "String", "date": "Date", "datetime": "DateTime", "timestamp": "DateTime64(6)", "interval": "Int64"}
    for yt, ch in m.items():
        assert po.ch_type({"name": "c", "type": yt, "required": True}) == ch
        assert po.ch_type({"name": "c", "type": yt, "required": False}) == f"Nullable({ch})"


def test_date_clamp_and_units(po):
    """columntypes/types.go:15-29: date/datetime clamped to [1970-01-01, 2106-01-01], timestamp not."""
    secs = [-86400, 0, 86399, 4291747200 - 1, 4291747200, 4291747200 + 86400 * 400]
    schema = [{"name": "d", "type": "date", "required": True}, {"name": "dt", "type": "datetime", "required": True}, {"name": "ts", "type": "timestamp", "required": True}]
    b = abi.Batch(len(secs), [abi.fixed_to_column(abi.TF_DATE, secs), abi.fixed_to_column(abi.TF_DATETIME, secs), abi.fixed_to_column(abi.TF_TIMESTAMP, secs, nanos=[999] * len(secs))])
    r = po.push_encode(b, po.build_plan("db", "t", schema, []), abi.TF_WIRE_CH_NATIVE)
    tail = r.raw[r.raw.index(b"\x01d\x04Date\x00") + 8:]
    days = struct.unpack_from("<6H", tail, 0)
    assert days == (0, 0, 0, 49672, 49673, 49673)
    off = tail.index(b"\x02dt\x08DateTime\x00") + 13
    assert struct.unpack_from("<6I", tail, off) == (0, 0, 86399, 4291747199, 4291747200, 4291747200)
    off = tail.index(b"DateTime64(6)\x00") + 14
    assert struct.unpack_from("<6q", tail, off) == tuple(s * 10**6 for s in secs)


def test_to_datetime_canon(po):
    """to_datetime/gotest/canondata/result.json (TestToDateTimeTransformer, to_datetime_test.go:16-118): include column2 + column3 —
    int32 1759143061 -> 2025-09-29T10:51:01Z (int16 column3 untouched), uint32 1759143081 -> 2025-09-29T10:51:21Z (datetime column4
    untouched); the Suitable table of :67-73, through the oracle plan and the product's host plan builder."""
    from transferia_b200 import engine
    t1 = [{"name": "column1", "type": "utf8", "key": True}, {"name": "column2", "type": "int32"}, {"name": "column3", "type": "int16"}]
    t2 = [{"name": "column1", "type": "uint32"}, {"name": "column2", "type": "datetime"}, {"name": "column3", "type": "float"}]
    t3 = [{"name": "column2", "type": "int8"}, {"name": "column3", "type": "uint32"}, {"name": "column4", "type": "datetime"}]
    none = {"convert_to_datetime": {}}
    two = {"convert_to_datetime": {"columns": {"includeColumns": ["column2", "column3"]}}}
    for tr, table, schema, suitable in ((none, "table1", t1, False), (none, "table2", t2, False), (none, "a_table3", t3, False),
                                        (two, "table1", t1, True), (two, "table2", t2, False), (two, "a_table3", t3, True)):
        assert (len(po.build_plan("db", table, schema, [tr]).steps) == 1) == suitable == (len(engine.plan_validate("db", table, schema, [tr])["steps"]) == 1), (tr, table)
    b1 = abi.Batch(1, [abi.strings_to_column(abi.TF_UTF8, [b"value1"]), abi.fixed_to_column(abi.TF_INT32, [1759143061]), abi.fixed_to_column(abi.TF_INT16, [1234])])
    out, errs = po.push_columns(b1, po.build_plan("db", "table1", t1, [two]))
    assert errs == [] and [c.type for c in out.columns] == [abi.TF_UTF8, abi.TF_DATETIME, abi.TF_INT16]
    assert po.fmt_rfc3339nano(int(out.columns[1].values[0])) == "2025-09-29T10:51:01Z" and int(out.columns[2].values[0]) == 1234
    b3 = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT8, [-3]), abi.fixed_to_column(abi.TF_UINT32, [1759143081]), abi.fixed_to_column(abi.TF_DATETIME, [1759140000])])
    plan3 = po.build_plan("db", "a_table3", t3, [two])
    out, errs = po.push_columns(b3, plan3)
    assert [c["type"] for c in plan3.result_schema] == ["int8", "datetime", "datetime"]
    assert po.fmt_rfc3339nano(int(out.columns[1].values[0])) == "2025-09-29T10:51:21Z" and po.fmt_rfc3339nano(int(out.columns[2].values[0])) == "2025-09-29T10:00:00Z"
    assert int(out.columns[0].values[0]) == -3


def test_to_string_canon(po):
    """to_string/gotest/canondata/result.json (TestToStringTransformer, to_string_test.go:16-120): the three transformers (all columns /
    exclude column2 on db.table* / include column1+column3 on db.a_table3) over the three items; result types and text values as the
    canon file holds them. (item3's column4 is a `date` column holding a time.Duration in the reference; an interval column gives the
    same SerializeToString branch here.) The product's host plan builder must agree on Suitable and on the result schema."""
    from transferia_b200 import engine
    t1 = [{"name": "column1", "type": "utf8", "key": True}, {"name": "column2", "type": "int64"}, {"name": "column3", "type": "int32"}, {"name": "column4", "type": "boolean"}]
    t2 = [{"name": "column1", "type": "string"}, {"name": "column2", "type": "date"}, {"name": "column3", "type": "double"}, {"name": "column4", "type": "float"}]
    t3 = [{"name": "column2", "type": "int8"}, {"name": "column3", "type": "uint32"}, {"name": "column4", "type": "interval"}]
    b1 = abi.Batch(1, [abi.strings_to_column(abi.TF_UTF8, [b"value1"]), abi.fixed_to_column(abi.TF_INT64, [123]), abi.fixed_to_column(abi.TF_INT32, [1234]), abi.fixed_to_column(abi.TF_BOOLEAN, [1])])
    b2 = abi.Batch(1, [abi.strings_to_column(abi.TF_BYTES, [b"value1"]), abi.fixed_to_column(abi.TF_DATE, [-8425641600]), abi.fixed_to_column(abi.TF_DOUBLE, [123.123]),
                       abi.fixed_to_column(abi.TF_FLOAT, np.array([312.321], np.float32))])
    b3 = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT8, [-3]), abi.fixed_to_column(abi.TF_UINT32, [12345]), abi.fixed_to_column(abi.TF_INTERVAL, [60 * 10**9])])
    allc = {"convert_to_string": {}}
    excl = {"convert_to_string": {"tables": {"includeTables": ["db.table"]}, "columns": {"excludeColumns": ["column2"]}}}
    incl = {"convert_to_string": {"tables": {"includeTables": ["db.a_table3"]}, "columns": {"includeColumns": ["column1", "column3"]}}}

    def text(col, r=0):
        return bytes(col.heap[col.offsets[r]:col.offsets[r + 1]]).decode()

    canon = [(allc, "table1", t1, b1, ["utf8"] * 4, ["value1", "123", "1234", "true"]),
             (allc, "table2", t2, b2, ["utf8"] * 4, ["value1", "1703-01-02", "123.123", "312.321"]),
             (allc, "a_table3", t3, b3, ["utf8"] * 3, ["-3", "12345", "1m0s"]),
             (excl, "table1", t1, b1, ["utf8", "int64", "utf8", "utf8"], ["value1", 123, "1234", "true"]),
             (excl, "table2", t2, b2, ["utf8", "date", "utf8", "utf8"], ["value1", -8425641600, "123.123", "312.321"]),
             (incl, "a_table3", t3, b3, ["int8", "utf8", "interval"], [-3, "12345", 60 * 10**9])]
    for tr, table, schema, batch, types, values in canon:
        plan = po.build_plan("db", table, schema, [tr])
        assert [c["type"] for c in plan.result_schema] == types, (tr, table)
        d = engine.plan_validate("db", table, schema, [tr])
        assert len(d["steps"]) == 1 and [c["type"] for c in d["result_schema"]] == types if "result_schema" in d else len(d["steps"]) == 1
        out, errs = po.push_columns(batch, plan)
        got = [text(c) if c.type in abi.VAR_TYPES else c.values[0].item() for c in out.columns]
        assert errs == [] and got == values, (tr, table, got)
    for tr, table, schema in ((excl, "a_table3", t3), (incl, "table1", t1), (incl, "table2", t2)):      # :77-87 not Suitable
        assert po.build_plan("db", table, schema, [tr]).steps == [] and engine.plan_validate("db", table, schema, [tr])["steps"] == []


def test_measure_reference_cases(po):
    """pkg/util/sizeof_test.go:11-150 TestDeepSizeof, the cases a row of ColumnValues can hold: []interface{} = 24-byte slice header +
    16 bytes per element (interface) + payload; bool 1, int64 / uint64 8, string 16 + len ("interface slice", "string", "bool", ...)."""
    b = abi.Batch(1, [abi.strings_to_column(abi.TF_UTF8, [b"a"]), abi.strings_to_column(abi.TF_UTF8, [b"b"])])
    assert list(po.measure(b)[0]) == [24 + 2 * 16 + 2 * 16 + 2]                     # the first two elements of the test's interface slice
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_BOOLEAN, [1]), abi.fixed_to_column(abi.TF_INT64, [64]), abi.fixed_to_column(abi.TF_UINT64, [64]),
                      abi.strings_to_column(abi.TF_UTF8, [b"0123456789"])])
    per, tot = po.measure(b)
    assert list(per) == [24 + 4 * 16 + 1 + 8 + 8 + (16 + 10)] and tot == int(per[0])
    b = abi.Batch(2, [abi.strings_to_column(abi.TF_BYTES, [b"xyz", None]), abi.fixed_to_column(abi.TF_TIMESTAMP, [0, 1]), abi.fixed_to_column(abi.TF_INT16, [1, 2], [False, True])])
    assert list(po.measure(b)[0]) == [24 + 3 * 16 + (24 + 3) + 24 + 2, 24 + 3 * 16 + 0 + 24 + 0]    # []byte = slice header + len; time.Time = 3 words; nil = the interface only


def test_native_block_read_back_by_an_independent_reader(po):
    """The oracle's native block of the all-types batch (nulls, clamps, long strings) parsed by tests/ch_block_reader.py — a reader written from
    the format, not from the encoder — gives back the input values after the reference's casts (columntypes/types.go:15-115): widths, column order,
    null maps (one byte per row in front of Nullable columns), LEB128 string framing, Date as days, DateTime as seconds, DateTime64(6) as micros."""
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import ch_block_reader
    from test_gpu_parity import all_types_batch
    from transferia_b200 import abi
    batch, schema = all_types_batch(2000, seed=8)
    res = po.push_encode(batch, po.build_plan("db", "t", schema, []), abi.TF_WIRE_CH_NATIVE)
    cols, nrows, data = ch_block_reader.read_block(res.raw)
    assert nrows == 2000 and [n for n, _ in cols] == [c["name"] for c in schema]
    CH_MIN, CH_MAX = 0, 4291747200                       # 1970-01-01 .. 2106-01-01 (types.go:15-29)
    for (name, typ), col, sc in zip(cols, batch.columns, schema):
        assert typ.startswith("Nullable(") == (not sc["required"]), (name, typ)
        valid = np.ones(2000, bool) if col.validity is None else np.unpackbits(np.asarray(col.validity), bitorder="little")[:2000].astype(bool)
        got = data[name]
        if col.type in abi.VAR_TYPES:
            off = np.asarray(col.offsets).astype(np.int64); heap = np.asarray(col.heap).tobytes()
            want = [heap[off[r]:off[r + 1]] if valid[r] else (None if typ.startswith("Nullable") else b"") for r in range(2000)]
        else:
            v = np.asarray(col.values)
            if col.type == abi.TF_DATE: conv = lambda r: int(min(max(int(v[r]), CH_MIN), CH_MAX) // 86400)
            elif col.type == abi.TF_DATETIME: conv = lambda r: int(min(max(int(v[r]), CH_MIN), CH_MAX))
            elif col.type == abi.TF_TIMESTAMP: conv = lambda r: int(v[r]) * 1_000_000 + (int(np.asarray(col.aux)[r]) // 1000 if col.aux is not None else 0)
            elif col.type in (abi.TF_FLOAT, abi.TF_DOUBLE): conv = lambda r: v[r]
            else: conv = lambda r: int(v[r])
            want = [conv(r) if valid[r] else (None if typ.startswith("Nullable") else 0) for r in range(2000)]
        for r in range(2000):
            g, w = got[r], want[r]
            if w is None or g is None: assert g is None and w is None, (name, r)
            elif isinstance(w, (float, np.floating)): assert np.array(g).tobytes() == np.array(w, dtype=np.asarray(g).dtype).tobytes(), (name, r)
            else: assert int(g) == int(w) if not isinstance(w, bytes) else g == w, (name, r, g, w)


def test_to_string_all_types_reference_cases(po):
    """registry/to_string/to_string_test.go:130-168 (TestAllTypesToStringTransformer) on the C++ oracle's SerializeToString: every case of the
    reference's table incl. the `any` list / map texts, dates before year 0 and beyond 9999, nanoseconds, the interval's Duration.String()."""
    s = lambda val, t: po.serialize_to_string(val, abi.YT_NAME_TO_TF[t]).decode()
    mk = po.make_val
    secs = lambda text: int(np.datetime64(text, "s").astype(np.int64))
    cases = [(mk(po.OG_JSON, s=b'[1,"string",3,4.123,6,true]'), "any", '[1,"string",3,4.123,6,true]'),
             (mk(po.OG_JSON, s=b'{"someName":"someValue","someName2":1234}'), "any", '{"someName":"someValue","someName2":1234}'),
             (mk(po.OG_INT64, i=981274987), "int64", "981274987"), (mk(po.OG_INT32, i=-12049182), "int32", "-12049182"), (mk(po.OG_INT16, i=12313), "int16", "12313"),
             (mk(po.OG_INT8, i=-14), "int8", "-14"), (mk(po.OG_UINT64, u=1142423562), "uint64", "1142423562"), (mk(po.OG_UINT32, u=0), "uint32", "0"),
             (mk(po.OG_UINT16, u=65212), "uint16", "65212"), (mk(po.OG_UINT8, u=213), "uint8", "213"),
             (mk(po.OG_FLOAT32, f=float(np.float32(123.123))), "float", "123.123"), (mk(po.OG_FLOAT64, f=-12344.12334341), "double", "-12344.12334341"),
             (mk(po.OG_BYTES, s=b"bytes"), "string", "bytes"), (mk(po.OG_STRING, s=b"string"), "utf8", "string"), (mk(po.OG_BOOL, i=1), "boolean", "true"),
             (mk(po.OG_TIME, i=secs("-1232-02-23T00:00:00"), nsec=0), "date", "-1232-02-23"), (mk(po.OG_TIME, i=secs("14124-01-12T00:00:00"), nsec=0), "date", "14124-01-12"),
             (mk(po.OG_TIME, i=secs("2311-12-01T01:02:04"), nsec=5), "datetime", "2311-12-01T01:02:04.000000005Z"),
             (mk(po.OG_TIME, i=secs("1231-05-23T09:08:07"), nsec=6), "timestamp", "1231-05-23T09:08:07.000000006Z"),
             (mk(po.OG_DURATION, i=((12 * 3600 + 53 * 60 + 21) * 10**9 + 87_182_124)), "interval", "12h53m21.087182124s"),
             (mk(po.OG_NIL), "date", "<nil>"), (mk(po.OG_NIL), "datetime", "<nil>"), (mk(po.OG_NIL), "boolean", "<nil>"), (mk(po.OG_NIL), "utf8", "<nil>"), (mk(po.OG_NIL), "int64", "<nil>")]
    for val, typ, want in cases:
        assert s(val, typ) == want, (typ, want)
