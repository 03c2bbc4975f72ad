"""GPU parity tests proper: the CUDA path through the C-ABI vs the CPU oracle on the same seeded inputs.
Bar: bit-exact native block (integer / byte / index work); compressed frames must decode with stock liblz4
AND the oracle's decoder to exactly that block and carry valid CityHash128 checksums (LZ4 bytes themselves are
unpinned in the reference, see DESIGN.md)."""
import ctypes as C
import struct
import os, sys
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cityhash_independent

import numpy as np
import pytest

from transferia_b200 import abi, engine, workload

pytestmark = pytest.mark.gpu
LZ = abi.TF_WIRE_CH_NATIVE_LZ4
RAW = abi.TF_WIRE_CH_NATIVE


def decode_with_liblz4(wire: bytes, po):
    """Independent frame walk: header fields, CityHash128 (oracle), LZ4 block via stock liblz4."""
    lz = C.CDLL("liblz4.so.1")
    pos, out, nf = 0, bytearray(), 0
    while pos < len(wire):
        assert wire[pos + 16] == 0x82
        cs, rs = struct.unpack_from("<II", wire, pos + 17)
        lo, hi = po.cityhash128(wire[pos + 16: pos + 16 + cs])
        assert struct.unpack_from("<QQ", wire, pos) == (lo, hi), f"bad checksum in frame {nf}"
        if nf < 6:      # the device checksum also against the second, independent CityHash128 (tests/cityhash_independent.py)
            assert cityhash_independent.cityhash128(wire[pos + 16: pos + 16 + cs]) == (lo, hi), f"oracle and independent CityHash128 disagree on frame {nf}"
        dst = C.create_string_buffer(max(1, rs))
        n = lz.LZ4_decompress_safe(wire[pos + 25: pos + 16 + cs], dst, cs - 9, rs)
        assert n == rs, f"liblz4 rejected frame {nf}: {n}"
        out += dst.raw[:rs]; pos += 16 + cs; nf += 1
    return bytes(out), nf


def check(eng, po, batch, schema, trs, ns="db", name="t", lz=True):
    pid = eng.plan(ns, name, schema, trs, {"type": "clickhouse"})
    plan = po.build_plan(ns, name, schema, trs)
    ref = po.push_encode(batch, plan, RAW, eng.frame_bytes)
    got = eng.push_encode(pid, batch, RAW)
    assert got.rows_in == batch.nrows and got.rows_out == ref.rows_out
    assert got.errors == ref.errors
    assert got.raw_len == len(ref.raw)
    if got.wire != ref.raw:
        a = np.frombuffer(got.wire, dtype=np.uint8); b = np.frombuffer(ref.raw, dtype=np.uint8)
        d = np.nonzero(a[:min(len(a), len(b))] != b[:min(len(a), len(b))])[0]
        raise AssertionError(f"native block differs at byte {d[:5]} of {len(b)}")
    if lz:
        z = eng.push_encode(pid, batch, LZ)
        raw, nf = decode_with_liblz4(z.wire, po)
        assert raw == ref.raw and nf == z.n_frames == max(1, -(-len(ref.raw) // eng.frame_bytes))
        raw2, nf2 = po.ch_decode_frames(z.wire)
        assert raw2 == ref.raw and nf2 == nf
    return got, ref


def test_headline_parity_50k(eng, po):
    batch, schema = workload.make_hits_batch(50_000)
    k = workload.counterid_threshold(batch, schema)
    got, ref = check(eng, po, batch, schema, workload.headline_transformers(k), "public", "hits")
    assert 0 < got.rows_out < batch.nrows
    check(eng, po, batch, schema, [], "public", "hits")


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2049, 4097])
def test_ragged_row_counts(eng, po, n):
    batch, schema = workload.make_hits_batch(max(n, 1))
    batch = batch.slice(0, n)
    trs = workload.headline_transformers(workload.counterid_threshold(batch, schema) if n else 0)
    check(eng, po, batch, schema, trs, "public", "hits")
    check(eng, po, batch, schema, [], "public", "hits", lz=(n in (0, 1, 33, 1025)))


def all_types_batch(n=3000, seed=3):
    rng = np.random.default_rng(seed)
    nulls = lambda p: rng.random(n) < p
    schema, cols = [], []
    def add(name, typ, col, required):
        schema.append({"name": name, "type": typ, "required": required, "key": False}); cols.append(col)
    for typ in ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"):
        dt = abi.FIXED_DTYPE[abi.YT_NAME_TO_TF[typ]]; info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        v[:4] = [info.min, info.max, 0, 1]
        add("c_" + typ, typ, abi.fixed_to_column(abi.YT_NAME_TO_TF[typ], v), True)
        add("n_" + typ, typ, abi.fixed_to_column(abi.YT_NAME_TO_TF[typ], v, nulls(0.3)), False)
    f32 = rng.standard_normal(n).astype(np.float32); f32[:3] = [np.inf, -0.0, np.nan]
    add("c_float", "float", abi.fixed_to_column(abi.TF_FLOAT, f32), True)
    add("n_double", "double", abi.fixed_to_column(abi.TF_DOUBLE, rng.standard_normal(n) * 1e100, nulls(0.2)), False)
    add("n_bool", "boolean", abi.fixed_to_column(abi.TF_BOOLEAN, rng.integers(0, 2, n), nulls(0.2)), False)
    add("c_interval", "interval", abi.fixed_to_column(abi.TF_INTERVAL, rng.integers(-10**15, 10**15, n)), True)
    secs = rng.integers(-10**9, 5 * 10**9, n); secs[:6] = [-86400, 0, 86399, 4291747199, 4291747200, 4291747200 + 10**8]
    nanos = rng.integers(0, 10**9, n)
    add("c_date", "date", abi.fixed_to_column(abi.TF_DATE, secs, nanos=nanos), True)
    add("n_datetime", "datetime", abi.fixed_to_column(abi.TF_DATETIME, secs, nulls(0.1), nanos=nanos), False)
    add("n_timestamp", "timestamp", abi.fixed_to_column(abi.TF_TIMESTAMP, secs, nulls(0.1), nanos=nanos), False)
    add("c_timestamp_nonanos", "timestamp", abi.fixed_to_column(abi.TF_TIMESTAMP, secs), True)
    lens = [0, 1, 127, 128, 129, 300, 16383, 16384, 20000] + list(rng.integers(0, 60, n - 9))
    strs = [bytes(rng.integers(0, 256, int(L), dtype=np.uint8)) for L in lens]
    add("c_utf8", "utf8", abi.strings_to_column(abi.TF_UTF8, strs), True)
    ns = [None if rng.random() < 0.25 else s for s in strs]
    add("n_bytes", "string", abi.strings_to_column(abi.TF_BYTES, ns), False)
    add("n_any", "any", abi.strings_to_column(abi.TF_ANY, [None if rng.random() < 0.1 else (b'{"k":%d}' % i) for i in range(n)],
                                              tags=(rng.random(n) < 0.5).astype(np.uint8)), False)
    return abi.Batch(n, cols), schema


def test_all_types_nulls_clamps_long_strings(eng, po):
    batch, schema = all_types_batch()
    check(eng, po, batch, schema, [])
    check(eng, po, batch, schema, [{"filter_rows": {"filter": "c_int32 > 0 AND n_int16 != NULL"}}])


def typed_column(case):
    tf = abi.YT_NAME_TO_TF[case["type"]]
    vals = [v[1] if case["go"] == "mixed" else v for v in case["input"]]
    if tf in abi.VAR_TYPES:
        return abi.strings_to_column(tf, [v.encode() for v in vals])
    if tf == abi.TF_TIMESTAMP:
        import datetime as dt
        us = [(dt.datetime.fromisoformat(v) - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(microseconds=1) for v in vals]
        return abi.fixed_to_column(tf, [u // 10**6 for u in us], nanos=[(u % 10**6) * 1000 for u in us])
    if tf == abi.TF_UINT64:
        return abi.Column(tf, values=np.array(vals, dtype=np.uint64))
    return abi.fixed_to_column(tf, vals)


def test_filter_rows_reference_filters_on_device(eng, po, goldens):
    """Every filter of filter_rows_test.go on a typed column: device result == oracle (rows, errors, bytes)."""
    for case in goldens["filter_rows"]:
        col = typed_column(case)
        schema = [{"name": "column", "type": case["type"], "required": True, "key": True}]
        batch = abi.Batch(len(case["input"]), [col])
        got, ref = check(eng, po, batch, schema, [{"filter_rows": {"filter": case["filter"]}}], "db", "table", lz=False)
        assert len(got.errors) == case["errors"], case["name"]
        if case["type"] not in ("float",):      # the Go table feeds float64 values even to the float32 column
            assert got.rows_out == len(case["expected"]), case["name"]


def test_filter_rows_semantics_matrix(eng, po):
    batch, schema = all_types_batch(2000, seed=9)
    names = [c["name"] for c in schema]
    kinds = np.zeros(batch.nrows, dtype=np.uint8); kinds[5] = abi.TF_KIND_UPDATE; kinds[17] = abi.TF_KIND_DELETE
    filters = [
        "c_int8 >= -5 AND c_int8 < 100", "c_uint64 > 5",                    # uint64 > MaxInt64 rows -> errIntOverflow
        "n_int32 > -1",                                                     # nil -> cast.ToFloat64E(nil) = 0 -> matches
        "n_int32 IN (0, 1, 2)", "n_double >= 0.5", "c_float < 0.0", "c_float IN (0.0, 1.5)", "n_bool = TRUE", "n_bool != false",
        "n_bool > 0.5",                                                     # bool -> 1/0 through ToFloat64E
        "c_utf8 ~ 'a'", "c_utf8 !~ 'ab'", "n_bytes >= 'M'", "c_utf8 IN ('', 'x')", "n_any ~ 'k'", "n_bytes = NULL", "n_any != NULL",
        "n_timestamp >= 2001-09-09T01:46:40Z AND n_timestamp < 2033-05-18T03:33:20.5+00:00", "c_date NOT IN (1970-01-01, 2106-01-01)",
        "n_datetime > 1999-12-31T23:59", "c_interval = NULL", "n_int16 > 2.5 AND n_int16 <= 100.0", "c_int64 NOT IN (1, 2, 3)",
    ]
    b2 = abi.Batch(batch.nrows, batch.columns, kinds)
    for f in filters:
        check(eng, po, b2, schema, [{"filter_rows": {"filter": f}}], lz=False)
    # OR over `filters`, AND inside each (filter_rows.go:137-148)
    check(eng, po, b2, schema, [{"filter_rows": {"filters": ["c_int8 > 100", "c_utf8 ~ 'zz' AND n_bool = true", "n_int32 = NULL"]}}], lz=False)
    # two filter_rows steps in one chain
    check(eng, po, b2, schema, [{"filter_rows": {"filter": "c_int16 > 0"}}, {"filter_rows": {"filter": "c_int32 < 0"}}], lz=False)
    # type pair the reference rejects per row ("Unsupported type pair"): string literal list vs a numeric column
    got, ref = check(eng, po, batch, schema, [{"filter_rows": {"filter": "c_int32 IN ('a', 'b')"}}], lz=False)
    assert got.rows_out == 0 and len(got.errors) == batch.nrows and got.errors[0][1] == abi.TF_ROWERR_FILTER_TYPEPAIR


def test_update_delete_rows_refused_by_sink_formats(eng, po):
    """A sink / serializer wire format takes INSERT rows only on the device: update / delete rows that survive the chain come back as
    row errors (TF_ROWERR_SINK_KIND_HOST) instead of being encoded as live rows (sink_table.go:296-305, marshal.go:92-95)."""
    batch, schema = all_types_batch(700, seed=31)
    kinds = np.zeros(batch.nrows, dtype=np.uint8); kinds[::9] = abi.TF_KIND_UPDATE; kinds[4::13] = abi.TF_KIND_DELETE
    b2 = abi.Batch(batch.nrows, batch.columns, kinds)
    n_bad = int((kinds != 0).sum())
    got, ref = check(eng, po, b2, schema, [])                                  # native + LZ4, no transformer at all
    assert got.rows_out == batch.nrows - n_bad and len(got.errors) == n_bad and {c for _, c, _ in got.errors} == {abi.TF_ROWERR_SINK_KIND_HOST}
    # skip_events drops them first: no error
    got, ref = check(eng, po, b2, schema, [{"skip_events": {"events": ["update", "delete"]}}], lz=False)
    assert got.errors == [] and got.rows_out == batch.nrows - n_bad
    # JSONEachRow and the batch serializer
    pid = eng.plan("db", "t", schema, [], {"type": "clickhouse"})
    plan = po.build_plan("db", "t", schema, [])
    for fmt in (abi.TF_WIRE_CH_JSONEACHROW, abi.TF_WIRE_SER_JSON):
        g = eng.push_encode(pid, b2, fmt); r = po.push_encode(b2, plan, fmt)
        assert g.wire == r.wire and g.errors == r.errors and sum(1 for _, c, _ in g.errors if c == abi.TF_ROWERR_SINK_KIND_HOST) == n_bad


def test_skip_events_filter_columns_rename_chain(eng, po):
    """skip_events.go:52-62, filter_columns_transformer.go:228-236, rename.go:46-67 chained with filter_rows / mask_field."""
    batch, schema = all_types_batch(2500, seed=13)
    schema = [dict(c, key=(c["name"] == "c_int8")) for c in schema]
    kinds = np.zeros(batch.nrows, dtype=np.uint8); kinds[::7] = abi.TF_KIND_DELETE; kinds[3::11] = abi.TF_KIND_UPDATE
    b2 = abi.Batch(batch.nrows, batch.columns, kinds)
    chains = [
        [{"skip_events": {"events": ["delete", "update"]}}, {"filter_rows": {"filter": "c_int32 > 0"}}],        # kinds dropped before filter_rows can reject them
        [{"skip_events": {"events": ["delete"]}}, {"filter_rows": {"filter": "c_int32 > 0"}}],                  # updates still become error rows
        [{"filter_columns": {"columns": {"excludeColumns": ["^n_", "interval"]}}}],
        [{"filter_rows": {"filter": "n_int16 != NULL"}}, {"skip_events": {"events": ["insert"]}}],
        [{"rename_tables": {"renameTables": [{"originalName": {"nameSpace": "db", "name": "t"}, "newName": {"nameSpace": "x", "name": "y"}}]}},
         {"filter_rows": {"tables": {"includeTables": ["^db\\.t$"]}, "filter": "c_int32 > 0"}},            # pass_all after the rename, kinds still rejected
         {"filter_columns": {"columns": {"includeColumns": ["^c_"]}}},
         {"mask_field": {"columns": ["c_utf8", "c_int64", "n_bool"], "maskFunctionHash": {"userDefinedSalt": "salt"}}}],
    ]
    for trs in chains:
        check(eng, po, b2, schema, trs)


def test_mask_field_on_device(eng, po):
    batch, schema = all_types_batch(1500, seed=21)
    cols = ["c_int8", "n_int32", "c_uint64", "n_bool", "c_date", "n_datetime", "n_timestamp", "c_utf8", "n_bytes", "n_any", "c_int64",
            "c_float", "n_double", "c_interval"]
    trs = [{"mask_field": {"columns": cols, "maskFunctionHash": {"userDefinedSalt": "the-best-tasty-saint-petersburg-salt"}}}]
    got, ref = check(eng, po, batch, schema, trs)
    # a long key (> 64 bytes is hashed first by crypto/hmac), chained after a filter
    trs2 = [{"filter_rows": {"filter": "c_int16 > 0"}}, {"mask_field": {"columns": ["c_utf8", "c_int32"], "maskFunctionHash": {"userDefinedSalt": "k" * 100}}}]
    check(eng, po, batch, schema, trs2)


def test_mask_golden_digests_on_device(eng, po, goldens):
    """The reference's canondata digests reproduced by the device HMAC kernel (types the device formats)."""
    salt = goldens["mask"]["salt"]
    for c in goldens["mask"]["cases"]:
        tf = abi.YT_NAME_TO_TF["interval" if c["go"] == "duration" else c["type"]]
        if c["go"] == "string":
            col = abi.strings_to_column(abi.TF_UTF8 if tf == abi.TF_BYTES else tf, [c["value"].encode()]); typ = "utf8" if tf == abi.TF_BYTES else c["type"]
        elif c["go"] == "time":
            col = abi.fixed_to_column(tf, [-8425641600]); typ = c["type"]       # 1703-01-02T00:00:00Z
        elif c["go"] == "bool":
            col = abi.fixed_to_column(tf, [1]); typ = c["type"]
        elif c["go"] == "duration":
            col = abi.fixed_to_column(abi.TF_INTERVAL, [c["value"]]); typ = "interval"     # %v of time.Duration -> "1m0s"
        else:
            col = abi.fixed_to_column(tf, [c["value"]]); typ = c["type"]
        schema = [{"name": "c", "type": typ, "required": True}]
        pid = eng.plan("db", "t", schema, [{"mask_field": {"columns": ["c"], "maskFunctionHash": {"userDefinedSalt": salt}}}], {"type": "clickhouse"})
        got = eng.push_encode(pid, abi.Batch(1, [col]), RAW)
        assert got.wire.endswith(b"\x40" + c["digest"].encode()), c


def test_resident_path_equals_host_path(eng, po):
    batch, schema = workload.make_hits_batch(30_000, seed=77)
    trs = workload.headline_transformers(workload.counterid_threshold(batch, schema))
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    host = eng.push_encode(pid, batch, LZ)
    dbatch = batch.to_device("cuda:0")
    eng.push_encode_resident(pid, dbatch, LZ)
    st = eng.resident_stats()
    assert st["rows_out"] == host.rows_out and st["raw_bytes"] == host.raw_len
    plan = po.build_plan("public", "hits", schema, trs)
    ref = po.push_encode(batch, plan, RAW).raw
    assert eng.resident_fetch(0, st["raw_bytes"]) == ref
    # compressed bytes may differ between runs (hash-table insert order inside a round is a race the kernel
    # tolerates: any winner is a valid earlier position); what is invariant is what they decode to
    raw, nf = decode_with_liblz4(eng.resident_fetch(1, st["wire_bytes"]), po)
    assert raw == ref and nf == host.n_frames


def test_resident_batches_back_to_back(eng, po):
    """The checksum / gather tail of a resident LZ4 batch stays in flight while the next batch's kernels start: two different
    batches of the same shape pushed without a sync in between, then a third call in another format; every fetch must see the
    complete frames of the batch pushed last (checksums verified by the frame walk)."""
    b1, schema = workload.make_hits_batch(40_000, seed=5)
    b2, _ = workload.make_hits_batch(40_000, seed=6)
    trs = workload.headline_transformers(workload.counterid_threshold(b1, schema))
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    plan = po.build_plan("public", "hits", schema, trs)
    d1, d2 = b1.to_device("cuda:0"), b2.to_device("cuda:0")
    for _ in range(3):
        eng.push_encode_resident(pid, d1, LZ); eng.push_encode_resident(pid, d2, LZ); eng.push_encode_resident(pid, d1, LZ); eng.push_encode_resident(pid, d2, LZ)
    st = eng.resident_stats()
    ref2 = po.push_encode(b2, plan, RAW).raw
    raw, nf = decode_with_liblz4(eng.resident_fetch(1, st["wire_bytes"]), po)
    assert raw == ref2
    eng.push_encode_resident(pid, d1, LZ)
    got = eng.push_encode(pid, b2, RAW)                 # a synchronous call in another format right behind a pending tail
    assert got.wire == ref2
    eng.push_encode_resident(pid, d1, LZ)
    small = b1.slice(0, 1000)                           # another layout of the work arena: the tail is joined first
    host = eng.push_encode(pid, small, LZ)
    raw, _ = decode_with_liblz4(host.wire, po)
    assert raw == po.push_encode(small, plan, RAW).raw


@pytest.mark.parametrize("frame_bytes", [1024, 1040, 4096, 12288, 15344, 15360])
def test_other_frame_sizes(po, frame_bytes):
    e = engine.Engine(0, frame_bytes)
    try:
        batch, schema = workload.make_hits_batch(5000, seed=5)
        check(e, po, batch, schema, workload.headline_transformers(workload.counterid_threshold(batch, schema)), "public", "hits")
    finally:
        e.close()


def test_frame_size_limits():
    """frame_bytes: a multiple of 16 in [1024, 15360] (one CTA of 256 threads holds one frame in shared memory); anything else is a config error."""
    for bad in (1008, 15376, 16384, 30720, 4100):
        with pytest.raises(engine.EngineError) as ei:
            engine.Engine(0, bad)
        assert ei.value.rc == -1 and not ei.value.retriable


def test_compressible_and_incompressible_frames(eng, po):
    """LZ4 edge cases: constant column (one long run per frame), pure noise, tiny blocks, tails shorter than 13 bytes."""
    n = 70_000
    rng = np.random.default_rng(1)
    schema = [{"name": "z", "type": "int64", "required": True}, {"name": "r", "type": "int64", "required": True}, {"name": "s", "type": "utf8", "required": True}]
    cols = [abi.fixed_to_column(abi.TF_INT64, np.zeros(n, dtype=np.int64)), abi.fixed_to_column(abi.TF_INT64, rng.integers(-2**63, 2**63 - 1, n)),
            abi.strings_to_column(abi.TF_UTF8, [b"abcabcabc" * (i % 7) for i in range(n)])]
    check(eng, po, abi.Batch(n, cols), schema, [])
    for m in (1, 2, 3, 5):
        check(eng, po, abi.Batch(m, [abi.fixed_to_column(abi.TF_INT8, list(range(m)))]), [{"name": "a", "type": "int8", "required": True}], [])


def test_full_size_batch_properties(eng, po):
    """BASELINE-size step (1 M rows x 99 columns): bit-exact block vs the oracle, frames decode with liblz4,
    every frame checksum valid, the uncompressed path gives the same block (idempotence), kept rows = numpy's own count."""
    batch, schema = workload.make_hits_batch(1_000_000)
    k = workload.counterid_threshold(batch, schema)
    trs = workload.headline_transformers(k)
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    a = eng.push_encode(pid, batch, LZ)
    b = eng.push_encode(pid, batch, RAW)
    assert a.rows_out == b.rows_out and a.raw_len == len(b.wire)
    names = [c["name"] for c in schema]
    cid = batch.columns[names.index("counterid")].values
    url = batch.columns[names.index("url")]
    heap = url.heap.tobytes(); offs = url.offsets
    has = np.fromiter((heap.find(b"://", int(offs[i]), int(offs[i + 1])) >= 0 for i in range(batch.nrows)), dtype=bool, count=batch.nrows)
    assert a.rows_out == int(((cid > k) & has).sum())
    raw, nf = decode_with_liblz4(a.wire, po)
    assert nf == a.n_frames and len(raw) == a.raw_len
    ref = po.push_encode(batch, po.build_plan("public", "hits", schema, trs), RAW)
    assert raw == ref.raw and b.wire == ref.raw


def test_api_errors(eng):
    schema = [{"name": "a", "type": "int32", "required": True}]
    pid = eng.plan("db", "t", schema, [], {"type": "clickhouse"})
    unsupported, arg = -2, -3                    # TF_E_FATAL_UNSUPPORTED, TF_E_FATAL_ARG (include/tfgpu.h)
    with pytest.raises(engine.EngineError) as ei:
        eng.push_encode(pid, abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1]), abi.fixed_to_column(abi.TF_INT32, [1])]), RAW)
    assert ei.value.rc == arg
    with pytest.raises(engine.EngineError) as ei:      # a text value in an int32 column is not strictified on the device (an int64 value is: test_device_strictify_loose_value_types)
        eng.push_encode(pid, abi.Batch(1, [abi.strings_to_column(abi.TF_UTF8, [b"1"])]), RAW)
    assert ei.value.rc == arg
    with pytest.raises(engine.EngineError) as ei:
        eng.plan("db", "t", schema, [{"mask_field": {"columns": ["a"], "maskFunctionHash": {"userDefinedSalt": "s"}}}, {"filter_rows": {"filter": "a = 'x'"}}], {"type": "clickhouse"})
    assert ei.value.rc == unsupported
    with pytest.raises(engine.EngineError) as ei:
        eng.push_encode(pid, abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1])]), 99)          # unknown wire format
    assert ei.value.rc == unsupported


def assert_batches_equal(a: abi.Batch, b: abi.Batch):
    assert a.nrows == b.nrows and len(a.columns) == len(b.columns)
    n = a.nrows
    for k, (x, y) in enumerate(zip(a.columns, b.columns)):
        assert x.type == y.type, k
        for f in ("values", "offsets", "heap", "aux"):
            u, v = getattr(x, f), getattr(y, f)
            assert (u is None) == (v is None), (k, f)
            if u is not None:
                assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8)), (k, f)
        assert (x.validity is None) == (y.validity is None), k
        if x.validity is not None:
            assert np.array_equal(np.unpackbits(x.validity, bitorder="little")[:n], np.unpackbits(y.validity, bitorder="little")[:n]), k


def test_push_columns_transformed_batch(eng, po):
    """tfgpu_push_columns: TransformerResult.Transformed comes back columnar and equals the oracle's, row errors too."""
    batch, schema = all_types_batch(3000, seed=31)
    schema = [dict(c, key=(c["name"] == "c_int8")) for c in schema]
    kinds = np.zeros(batch.nrows, dtype=np.uint8); kinds[::9] = abi.TF_KIND_UPDATE
    b2 = abi.Batch(batch.nrows, batch.columns, kinds)
    chains = [
        [],
        [{"filter_rows": {"filter": "c_int32 > 0 AND n_int16 != NULL"}}],
        [{"skip_events": {"events": ["update"]}}, {"filter_columns": {"columns": {"excludeColumns": ["double", "bytes"]}}},
         {"mask_field": {"columns": ["c_utf8", "n_int32", "n_timestamp"], "maskFunctionHash": {"userDefinedSalt": "pepper"}}}],
    ]
    for trs in chains:
        pid = eng.plan("db", "t", schema, trs)
        plan = po.build_plan("db", "t", schema, trs)
        got, gerr = eng.push_columns(pid, b2)
        ref, rerr = po.push_columns(b2, plan)
        assert gerr == rerr
        assert_batches_equal(got, ref)
    # and the Transformed batch can be pushed again (it is a valid tf_batch): encode(transform(x)) == encode_with_transform(x)
    trs = [{"filter_rows": {"filter": "c_int64 > 0"}}]
    pid = eng.plan("db", "t", schema, trs, {"type": "clickhouse"}); pid0 = eng.plan("db", "t", schema, [], {"type": "clickhouse"})
    mid, _ = eng.push_columns(pid, batch)
    assert eng.push_encode(pid0, mid, RAW).wire == eng.push_encode(pid, batch, RAW).wire
    hb, hs = workload.make_hits_batch(20_000, seed=4)
    pid = eng.plan("public", "hits", hs, workload.headline_transformers(workload.counterid_threshold(hb, hs)))
    got, _ = eng.push_columns(pid, hb)
    ref, _ = po.push_columns(hb, po.build_plan("public", "hits", hs, workload.headline_transformers(workload.counterid_threshold(hb, hs))))
    assert_batches_equal(got, ref)


def float_batch(n=200_000, seed=8):
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 2**63 - 1, n, dtype=np.int64).view(np.uint64) | (rng.integers(0, 2, n).astype(np.uint64) << np.uint64(63))
    d = bits.view(np.float64).copy()
    special = [0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, 2.2250738585072014e-308, 1.7976931348623157e308, 1e21, 1e22, 1e23, 9007199254740993.0, 123456.7, 1234567.0,
               1e-5, 1e-4, 1e-7, 1e-6, 9.999999999999999e-7, 1e20, 99999.95, 0.3, 1 / 3, 100.0, 1e6, 999999.0, 123.123]
    d[:len(special)] = special
    d[len(special):n // 2] = rng.random(n // 2 - len(special)) * 10.0 ** rng.integers(-25, 25, n // 2 - len(special))
    f = rng.integers(0, 2**32 - 1, n, dtype=np.int64).astype(np.uint32).view(np.float32).copy()
    f[:len(special)] = np.array(special, dtype=np.float64).astype(np.float32)
    f[len(special):n // 2] = (rng.random(n // 2 - len(special)) * 10.0 ** rng.integers(-20, 20, n // 2 - len(special))).astype(np.float32)
    dur = rng.integers(-2**62, 2**62, n); dur[:8] = [0, 1, 999, 1000, 1_500_000, 60 * 10**9, 3600 * 10**9 + 5 * 10**8, -(2**63)]
    schema = [{"name": "d", "type": "double", "required": True}, {"name": "f", "type": "float", "required": True}, {"name": "iv", "type": "interval", "required": True}]
    return abi.Batch(n, [abi.fixed_to_column(abi.TF_DOUBLE, d), abi.fixed_to_column(abi.TF_FLOAT, f), abi.fixed_to_column(abi.TF_INTERVAL, dur)]), schema


def test_device_float_and_duration_text_forms(eng, po):
    """Go %v of float64 / float32 / time.Duration on the device (Ryu shortest digits) vs the oracle's exact big-integer
    printer, 200 k random bit patterns + the layout thresholds, through convert_to_string (to_string.go:145-171)."""
    batch, schema = float_batch()
    trs = [{"convert_to_string": {"columns": {"includeColumns": ["^d$", "^f$", "^iv$"]}}}]
    pid = eng.plan("db", "t", schema, trs)
    got, _ = eng.push_columns(pid, batch)
    ref, _ = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
    for k in range(3):
        g, r = got.columns[k], ref.columns[k]
        if not (np.array_equal(g.offsets, r.offsets) and np.array_equal(g.heap, r.heap)):
            bad = np.nonzero(np.diff(g.offsets.astype(np.int64)) != np.diff(r.offsets.astype(np.int64)))[0][:5]
            show = [(int(i), bytes(g.heap[g.offsets[i]:g.offsets[i + 1]]), bytes(r.heap[r.offsets[i]:r.offsets[i + 1]])) for i in bad]
            raise AssertionError(f"column {k}: text forms differ, e.g. {show}")
    assert_batches_equal(got, ref)


def test_convert_to_string_all_types(eng, po):
    batch, schema = all_types_batch(2000, seed=17)
    for trs in ([{"convert_to_string": {}}],                                                       # every column
                [{"convert_to_string": {"columns": {"includeColumns": ["^n_", "date"]}, "convert_to_bytes": True}}],
                [{"filter_rows": {"filter": "c_int32 > 0"}}, {"convert_to_string": {"columns": {"excludeColumns": ["utf8", "bytes"]}}}]):
        check(eng, po, batch, schema, trs)
        pid = eng.plan("db", "t", schema, trs)
        got, gerr = eng.push_columns(pid, batch)
        ref, rerr = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
        assert gerr == rerr
        assert_batches_equal(got, ref)


def test_convert_to_datetime(eng, po):
    """to_datetime.go:89-151: int32 / uint32 seconds -> time.Unix(s, 0), nil -> time.Unix(0, 0); then the ClickHouse DateTime clamp."""
    batch, schema = all_types_batch(2000, seed=23)
    trs = [{"convert_to_datetime": {"columns": {"includeColumns": ["int32", "int64"]}}}]      # int64 is not a supported type: left alone
    check(eng, po, batch, schema, trs)
    pid = eng.plan("db", "t", schema, trs)
    d = eng.describe(pid)
    assert [c["type"] for c in d["result_schema"] if "int32" in c["name"]] == ["datetime"] * 4
    got, _ = eng.push_columns(pid, batch)
    ref, _ = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
    assert_batches_equal(got, ref)
    assert eng.describe(eng.plan("db", "t", schema, [{"convert_to_datetime": {}}]))["steps"] == []          # empty column filter: not Suitable


def test_jsoneachrow_on_device(eng, po):
    """ClickHouse JSONEachRow (httpuploader/marshal.go:88-253): device rows == oracle rows, byte for byte."""
    JS = abi.TF_WIRE_CH_JSONEACHROW
    batch, schema = all_types_batch(2500, seed=41)
    chains = [[], [{"filter_rows": {"filter": "c_int32 > 0"}}],
              [{"mask_field": {"columns": ["c_utf8", "n_double"], "maskFunctionHash": {"userDefinedSalt": "s"}}}, {"convert_to_string": {"columns": {"includeColumns": ["c_float", "n_timestamp", "n_any"]}}},
               {"convert_to_datetime": {"columns": {"includeColumns": ["c_uint32"]}}}, {"filter_columns": {"columns": {"excludeColumns": ["c_interval"]}}}]]
    for trs in chains:
        pid = eng.plan("db", "t", schema, trs, {"type": "clickhouse"})
        got = eng.push_encode(pid, batch, JS)
        ref = po.push_encode(batch, po.build_plan("db", "t", schema, trs), JS)
        assert got.rows_out == ref.rows_out
        if got.wire != ref.wire:
            gl, rl = got.wire.split(b"\n"), ref.wire.split(b"\n")
            for i, (x, y) in enumerate(zip(gl, rl)):
                if x != y:
                    raise AssertionError(f"row {i}:\n got {x[:400]}\n exp {y[:400]}")
            raise AssertionError("row count differs")
    # the reference's own etalons (marshal_test.go:16-37 DateTime64 scaling; :84-110 non-UTF-8 bytes kept; null -> {})
    sch = [{"name": "t", "type": "timestamp", "required": True}, {"name": "b", "type": "string"}, {"name": "n", "type": "utf8"}]
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_TIMESTAMP, [1580637742], nanos=[123456789]), abi.strings_to_column(abi.TF_BYTES, [b'"Hello\xfe\xe4\xb8\x96']), abi.strings_to_column(abi.TF_UTF8, [None])])
    got = eng.push_encode(eng.plan("db", "t", sch, [], {"type": "clickhouse"}), b, JS)
    assert got.wire == b'{"t":1580637742123456,"b":"\\"Hello\xfe\xe4\xb8\x96"}\n'
    hb, hs = workload.make_hits_batch(30_000, seed=6)
    trs = workload.headline_transformers(workload.counterid_threshold(hb, hs))
    got = eng.push_encode(eng.plan("public", "hits", hs, trs, {"type": "clickhouse"}), hb, JS)
    assert got.wire == po.push_encode(hb, po.build_plan("public", "hits", hs, trs), JS).wire


def test_measurer_sizes(eng, po):
    """Measurer middleware (synchronizer/measurer.go:38-42): DeepSizeof(ColumnValues) per row in closed form == the oracle's walk."""
    batch, schema = all_types_batch(5000, seed=21)
    per, tot = eng.measure(batch); rper, rtot = po.measure(batch)
    assert tot == rtot and np.array_equal(per, rper) and tot == int(per.sum())
    hb, hs = workload.make_hits_batch(50_000, seed=6)
    per, tot = eng.measure(hb); rper, rtot = po.measure(hb)
    assert tot == rtot and np.array_equal(per, rper)
    # closed form by hand: one int32 + one nil utf8 + one 3-byte utf8 row
    b = abi.Batch(2, [abi.fixed_to_column(abi.TF_INT32, [1, 2]), abi.strings_to_column(abi.TF_UTF8, [None, b"abc"])])
    assert list(po.measure(b)[0]) == [24 + 16 + 4 + 16, 24 + 16 + 4 + 16 + 16 + 3]


def test_number_to_float(eng, po):
    """number_to_float_transformer (number_to_float.go:75-123) as a rewrite of the `any` JSON text, alone and before mask / to_string / sinks."""
    vals = [b'{"a":1,"b":[1.50,2e3,-0,1e21,1e-7,0.000001,123456789012345678901234567890],"s":"12 \\" 3e4","n":null}', b"17", b"1e400", b"-1.0E+2", b'"just a string 5"', b"true",
            b"[]", b'{"deep":{"x":[{"y":0.1000}]},"big":18446744073709551616,"i":9007199254740993}', None, b"3.14159265358979323846264338327950288", b'{"k":"\\\\","v":1.0}', b"0.30000000000000004"]
    tags = [0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0]
    n = len(vals)
    kinds = np.zeros(n, dtype=np.uint8); kinds[1] = abi.TF_KIND_DELETE; kinds[3] = abi.TF_KIND_UPDATE
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "a", "type": "any"}, {"name": "b", "type": "any"}]
    b = abi.Batch(n, [abi.fixed_to_column(abi.TF_INT32, list(range(n))), abi.strings_to_column(abi.TF_ANY, vals, tags=tags), abi.strings_to_column(abi.TF_ANY, vals[::-1], tags=tags[::-1])], kinds)
    chains = [[{"number_to_float_transformer": {}}],
              [{"number_to_float_transformer": {"tables": {"includeTables": ["^db.t$"]}}}, {"mask_field": {"columns": ["a"], "maskFunctionHash": {"userDefinedSalt": "s"}}}],
              [{"mask_field": {"columns": ["a"], "maskFunctionHash": {"userDefinedSalt": "s"}}}, {"number_to_float_transformer": {}}, {"convert_to_string": {"columns": {"includeColumns": ["b"]}}}],
              [{"rename_tables": {"renameTables": [{"originalName": {"nameSpace": "db", "name": "t"}, "newName": {"nameSpace": "db", "name": "u"}}]}}, {"number_to_float_transformer": {"tables": {"includeTables": ["^db.t$"]}}}],
              [{"number_to_float_transformer": {"tables": {"includeTables": ["^other$"]}}}]]
    for trs in chains:
        pid = eng.plan("db", "t", schema, trs, {"type": "clickhouse"}); plan = po.build_plan("db", "t", schema, trs)
        got, gerr = eng.push_columns(pid, b); ref, rerr = po.push_columns(b, plan)
        assert gerr == rerr, (trs, gerr, rerr)
        assert_batches_equal(got, ref)
        for fmt in (RAW, abi.TF_WIRE_CH_JSONEACHROW):
            if any("skip" in t for t in trs): continue
            bi = abi.Batch(n, b.columns, np.zeros(n, dtype=np.uint8))       # sinks take insert rows
            assert eng.push_encode(pid, bi, fmt).wire == po.push_encode(bi, plan, fmt).raw, (trs, fmt)
    # spot values
    ref, _ = po.push_columns(b, po.build_plan("db", "t", schema, chains[0]))
    a = ref.columns[1]; cell = lambda r: bytes(a.heap[a.offsets[r]:a.offsets[r + 1]])
    assert cell(0) == b'{"a":1,"b":[1.5,2000,-0,1e+21,1e-7,0.000001,1.2345678901234568e+29],"s":"12 \\" 3e4","n":null}'
    assert cell(1) == b"17" and cell(2) == b"1e400" and cell(3) == b"-100" and cell(4) == b'"just a string 5"' and cell(9) == b"3.141592653589793"


def test_device_strictify_loose_value_types(eng, po):
    """Strictify (strictify.go:18-181) as a pre-pass of the chain: values that arrive in another fixed-width type than the column's
    schema type are cast like spf13/cast does and range-checked; a row that fails is a row error on its FIRST failing column
    (TF_ROWERR_STRICT_RANGE / _CAST), the rest comes out in the schema's types. Oracle: the restatement pinned by strictify_test.go."""
    rng = np.random.default_rng(77); n = 600
    def pick(lo, hi, extra): return np.concatenate([rng.integers(lo, hi, n - len(extra)), np.array(extra, dtype=np.int64)]).astype(np.int64)
    spec = [   # (column, schema type, physical type the values arrive in, values)
        ("i8", "int8", abi.TF_INT64, pick(-128, 128, [127, 128, -128, -129, 1 << 40])),
        ("u8", "uint8", abi.TF_INT64, pick(0, 256, [255, 256, -1, 0])),
        ("i16", "int16", abi.TF_DOUBLE, np.concatenate([rng.uniform(-32768, 32767, n - 6), [32767.9, 32768.0, -32768.5, -32769.0, 1e300, float("nan")]])),
        ("u16", "uint16", abi.TF_UINT64, np.array(list(rng.integers(0, 65536, n - 3)) + [65535, 65536, 1 << 63], dtype=np.uint64)),
        ("i32", "int32", abi.TF_INT64, pick(-(1 << 31), 1 << 31, [(1 << 31) - 1, 1 << 31, -(1 << 31) - 1])),
        ("u32", "uint32", abi.TF_FLOAT, np.concatenate([rng.uniform(0, 4e9, n - 4), [4294967040.0, 4294967296.0, -0.5, -1.0]]).astype(np.float32)),
        ("i64", "int64", abi.TF_UINT64, np.array(list(rng.integers(0, 1 << 62, n - 2)) + [(1 << 64) - 1, 1 << 63], dtype=np.uint64)),
        ("u64", "uint64", abi.TF_INT64, pick(0, 1 << 62, [-1, -(1 << 63), (1 << 63) - 1])),
        ("f32", "float", abi.TF_INT64, pick(-(1 << 62), 1 << 62, [16777217, (1 << 53) + 1, -16777219])),
        ("f64", "double", abi.TF_INT64, pick(-(1 << 62), 1 << 62, [(1 << 53) + 1, -(1 << 60) - 1])),
        ("b", "boolean", abi.TF_INT32, rng.integers(-1, 2, n).astype(np.int64)),
        ("ts", "timestamp", abi.TF_INT64, pick(0, 1 << 31, [0, -5])),
        ("same", "int32", abi.TF_INT32, rng.integers(-1000, 1000, n)),
    ]
    spec = [(c, t, ptf, np.asarray(vals)[rng.permutation(n)]) for c, t, ptf, vals in spec]      # the edge values of different columns land in different rows
    go = {abi.TF_INT64: "int64", abi.TF_UINT64: "uint64", abi.TF_DOUBLE: "float64", abi.TF_FLOAT: "float32", abi.TF_INT32: "int32"}
    schema = [{"name": c, "type": t} for c, t, _, _ in spec]
    nulls = rng.random(n) < 0.1
    cols = [abi.fixed_to_column(ptf, vals, nulls if c == "i8" else None) for c, t, ptf, vals in spec]
    batch = abi.Batch(n, cols)
    pid = eng.plan("db", "t", schema, [])
    got, gerr = eng.push_columns(pid, batch)
    # the oracle, cell by cell
    want_err, keep, outv = [], [], [[] for _ in spec]
    for r in range(n):
        row, bad = [], None
        for k, (c, t, ptf, vals) in enumerate(spec):
            if c == "i8" and nulls[r]: row.append(0); continue
            v = cols[k].values[r]
            txt = repr(float(v)) if ptf in (abi.TF_DOUBLE, abi.TF_FLOAT) else str(int(v))
            rc, out = po.strictify_value(go[ptf], txt, abi.YT_NAME_TO_TF[t])
            assert rc in (0, 1, 2), (c, txt, rc)
            if rc and bad is None: bad = (r, 57 if rc == 1 else 58, k)
            if out["go"] == "time.Time": row.append(int(out["v"].split(".")[0]))
            elif out["go"] == "json.Number": row.append(float(out["v"]))
            elif out["go"] == "bool": row.append(1 if out["v"] == "true" else 0)
            elif out["go"] in ("float32",): row.append(float(out["v"]))
            else: row.append(int(out["v"]) if rc == 0 else 0)
        if bad: want_err.append(bad)
        else:
            keep.append(r)
            for k in range(len(spec)): outv[k].append(row[k])
    assert gerr == want_err, ([e for e in gerr if e not in want_err][:5], [e for e in want_err if e not in gerr][:5])
    assert 15 < len(want_err) < n // 4 and {c for _, c, _ in want_err} == {57, 58}
    assert got.nrows == len(keep)
    for k, (c, t, _, _) in enumerate(spec):
        tf = abi.YT_NAME_TO_TF[t]
        assert got.columns[k].type == tf, c
        want = np.asarray(outv[k], dtype=abi.FIXED_DTYPE[tf])
        have = np.asarray(got.columns[k].values)[:len(keep)]
        if c == "i8":      # nil rows keep an unspecified slot
            m = ~nulls[keep]; assert np.array_equal(have[m], want[m]), c
        else:
            bad = np.nonzero(have != want)[0] if have.dtype.kind != "f" else np.nonzero(have.view(np.uint32 if have.itemsize == 4 else np.uint64) != want.view(np.uint32 if want.itemsize == 4 else np.uint64))[0]
            assert len(bad) == 0, (c, bad[:5], have[bad[:5]], want[bad[:5]], [cols[k].values[keep[i]] for i in bad[:5]])
    # a pair the device does not strictify is refused up front, not converted approximately
    bad_schema = [{"name": "x", "type": "double"}]
    with pytest.raises(engine.EngineError):
        eng.push_columns(eng.plan("db", "t2", bad_schema, []), abi.Batch(2, [abi.fixed_to_column(abi.TF_FLOAT, [0.1, 0.2])]))


def test_round_robin_dispatcher_over_real_engines(po):
    """SURVEY §8e: one host process, one engine per GPU (two engines on the same GPU when the box has one), whole batches dealt
    round-robin by `dispatch.RoundRobinDispatcher`; results come back in submission order and every one decodes to the oracle's block."""
    import torch
    from transferia_b200 import dispatch
    ndev = torch.cuda.device_count()
    devs = list(range(ndev)) if ndev > 1 else [0, 0]
    engs = [engine.Engine(d) for d in devs]
    try:
        batches = []
        for i in range(7):
            b, schema = workload.make_hits_batch(3000 + 500 * i, seed=100 + i)
            batches.append(b)
        trs = workload.headline_transformers(workload.counterid_threshold(batches[0], schema))
        pids = [e.plan("public", "hits", schema, trs, {"type": "clickhouse"}) for e in engs]
        plan = po.build_plan("public", "hits", schema, trs)
        workers = [(lambda b, e=e, p=p: e.push_encode(p, b, LZ)) for e, p in zip(engs, pids)]
        d = dispatch.RoundRobinDispatcher(workers)
        try:
            results = list(d.run(iter(batches)))
        finally:
            d.close()
        assert len(results) == len(batches)
        for b, r in zip(batches, results):                      # submission order is preserved
            want = po.push_encode(b, plan, RAW, engs[0].frame_bytes)
            assert r.rows_in == b.nrows and r.rows_out == want.rows_out
            raw, nf = decode_with_liblz4(r.wire, po)
            assert raw == want.raw
    finally:
        for e in engs:
            e.close()


def test_narrow_length_arrays_equal_offsets(eng, po):
    """tf_col.flags TF_COL_LENS8 / 16: uint8 / uint16 per-row lengths instead of uint32 offsets (a host layout that saves PCIe bytes);
    the offsets are rebuilt on the device and every result equals the one of the plain layout — from host memory and from HBM."""
    batch, schema = workload.make_hits_batch(20_000, seed=9)
    trs = workload.headline_transformers(workload.counterid_threshold(batch, schema))
    nb = batch.narrow()
    widths = [getattr(c, "lens_width", 0) for c in nb.columns]
    assert widths.count(1) + widths.count(2) == sum(1 for c in batch.columns if c.type in abi.VAR_TYPES) and nb.input_bytes() < batch.input_bytes() - 3 * 20_000 * 20
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    a = eng.push_encode(pid, batch, RAW); b = eng.push_encode(pid, nb, RAW)
    assert a.wire == b.wire and a.rows_out == b.rows_out and a.errors == b.errors
    # the whole batch in one pinned arena laid out like the device staging: a single DMA, the same result (one and two phases)
    h0 = eng.h2d_bytes(); c = eng.push_encode(pid, nb.pin_arena(), RAW); h1 = eng.h2d_bytes()
    assert c.wire == a.wire and nb.input_bytes() <= h1 - h0 <= nb.input_bytes() + 272 * 5 * len(nb.columns)
    assert eng.push_encode(pid, nb.pin_arena(), RAW, selective=2).wire == a.wire and eng.push_encode(pid, batch.pin_arena(), RAW).wire == a.wire
    assert a.wire == po.push_encode(batch, po.build_plan("public", "hits", schema, trs), RAW).raw
    eng.push_encode_resident(pid, nb.to_device("cuda:0"), RAW)
    st = eng.resident_stats()
    assert eng.resident_fetch(0, st["raw_bytes"]) == a.wire
    # a column with a cell of 300 bytes falls back to uint16 lengths; an all-types batch with nulls
    b2, s2 = all_types_batch(3000, seed=5)
    n2 = b2.narrow()
    assert 2 in [getattr(c, "lens_width", 0) for c in n2.columns] or 1 in [getattr(c, "lens_width", 0) for c in n2.columns]
    p2 = eng.plan("db", "t", s2, [], {"type": "clickhouse"})
    assert eng.push_encode(p2, b2, RAW).wire == eng.push_encode(p2, n2, RAW).wire


@pytest.mark.gpu
def test_two_phase_push_equals_one_phase(eng, po):
    """tfgpu_push_encode_selective: predicate columns first, host gather of the kept rows, the chain over those — the block, the row count and
    the row errors are those of the one-phase call (and of the oracle), from offsets and from narrow lengths, with per-row filter errors."""
    batch, schema = workload.make_hits_batch(60_000, seed=21)
    trs = workload.headline_transformers(workload.counterid_threshold(batch, schema))
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    want = po.push_encode(batch, po.build_plan("public", "hits", schema, trs), RAW)
    for b in (batch, batch.narrow(), batch.narrow().pin()):
        h0 = eng.h2d_bytes()
        one = eng.push_encode(pid, b, RAW); h1 = eng.h2d_bytes()
        two = eng.push_encode(pid, b, RAW, selective=4); h2 = eng.h2d_bytes()
        assert two.wire == one.wire == want.raw and two.rows_out == one.rows_out and two.rows_in == 60_000 and two.errors == one.errors
        assert (h2 - h1) < 0.6 * (h1 - h0)                     # the point of it: fewer bytes over PCIe
    lz = eng.push_encode(pid, batch.narrow(), abi.TF_WIRE_CH_NATIVE_LZ4, selective=0)
    raw, _ = po.ch_decode_frames(lz.wire)
    assert raw == want.raw
    # update / delete kinds make filter_rows fail per row (filter_rows.go:103-107): reported from phase one with the input row index
    kb = abi.Batch(batch.nrows, batch.columns, (np.arange(batch.nrows) % 50 == 7).astype(np.uint8))
    one = eng.push_encode(pid, kb, RAW); two = eng.push_encode(pid, kb, RAW, selective=3)
    assert one.errors and two.errors == one.errors and two.wire == one.wire and two.rows_out == one.rows_out
    # a filter that keeps nothing / everything: phase two sees an empty batch, or the whole one
    for flt in ("c_int64 < -9223372036854775807 AND c_int8 > 100", "c_int8 >= -128"):
        b3, s3 = all_types_batch(20_000, seed=3)
        t3 = [{"filter_rows": {"filter": flt}}]
        p3 = eng.plan("db", "t3", s3, t3, {"type": "clickhouse"})
        a3, c3 = eng.push_encode(p3, b3, RAW), eng.push_encode(p3, b3, RAW, selective=2)
        assert c3.wire == a3.wire and c3.rows_out == a3.rows_out and c3.errors == a3.errors and a3.rows_out in (0, 20_000)
    # all-types batch: nulls, long strings, a predicate on a nullable column
    b2, s2 = all_types_batch(30_000, seed=13)
    t2 = [{"filter_rows": {"filter": "c_int32 > 0 AND n_int16 != NULL"}}]
    p2 = eng.plan("db", "t", s2, t2, {"type": "clickhouse"})
    assert eng.push_encode(p2, b2, RAW, selective=2).wire == eng.push_encode(p2, b2, RAW).wire == po.push_encode(b2, po.build_plan("db", "t", s2, t2), RAW).raw


@pytest.mark.gpu
def test_replace_primary_key_reorders_the_block(eng, po):
    """A composite replace_primary_key puts the key columns first in the result schema: the native block, JSONEachRow and the INSERT column
    list follow that order (the items' values are looked up by name, replace_primary_key.go:70-82)."""
    batch, schema = workload.make_hits_batch(3000, seed=17)
    names = [c["name"] for c in schema]
    keys = [names[40], names[3], names[12]]
    trs = [{"replace_primary_key": {"keys": keys}}, {"filter_rows": {"filter": f"{names[0]} > 0"}}]
    check(eng, po, batch, schema, trs)
    pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    d = eng.describe(pid)
    assert [c["name"] for c in d["result_schema"]][:3] == keys and [c["key"] for c in d["result_schema"]] == [True] * 3 + [False] * (len(names) - 3)
    want = po.push_encode(batch, po.build_plan("public", "hits", schema, trs), abi.TF_WIRE_CH_JSONEACHROW)
    assert eng.push_encode(pid, batch, abi.TF_WIRE_CH_JSONEACHROW).wire == want.raw
