"""Queue Debezium serializer (SURVEY §8 a16): Emitter.EmitKV on columns without a database-specific original_type
(pkg/debezium/emitter_value_converter.go:626-690, emitter_common.go:67-180).

The reference holds no byte-level golden for this path (its pg / mysql canon files go through the database converters), so
the oracle is pinned by (1) the assertions of the reference's own unit tests on it, (2) the message a real Debezium wrote
for the reference's CRUD fixture, restricted to the columns whose pg converter is the identity. The device emitter is then
compared with the oracle byte for byte."""
import json
import os

import numpy as np
import pytest

from transferia_b200 import abi

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "debezium_emit_goldens.json"), encoding="utf-8"))
OPTS = {"ignore_unknown_sources": True, "version": "1.1.2.Final", "topic_prefix": "fullfillment", "database": "pguser", "source_type": "pg"}
TF_E_FATAL_CONFIG, TF_E_FATAL_UNSUPPORTED = -1, -2          # include/tfgpu.h


def _golden_batch():
    schema, cols = [], []
    for c in G["columns"]:
        tf = abi.YT_NAME_TO_TF[c["type"]]
        schema.append({"name": c["name"], "type": c["type"], "key": c["key"], "required": c["required"]})
        if tf == abi.TF_UTF8:
            cols.append(abi.strings_to_column(tf, [c["value"].encode()]))
        else:
            cols.append(abi.fixed_to_column(tf, [c["value"]]))
    meta = {"id": np.array([G["id"]], np.uint32), "lsn": np.array([G["lsn"]], np.uint64), "commit_time": np.array([G["commit_time"]], np.uint64)}
    return abi.Batch(1, cols), schema, meta


def test_oracle_against_real_debezium_message(po):
    """pg/tests/emitter_crud_test.go: the insert fixture, identity-converter columns. Values as the real message holds them
    (doubles compared as numbers: Java prints 3.14E-100), envelope and `source` key sets, constants of the source block."""
    batch, schema, meta = _golden_batch()
    plan = po.build_plan(G["table"][0], G["table"][1], schema, [])
    data, ks, rs, errs = po.debezium_emit(batch, plan, OPTS, meta)
    assert errs == [] and len(ks) == 1
    (key, val), = po.debezium_split(data, ks, rs)
    assert key == b'{"i":1}'
    v = json.loads(val)
    assert sorted(v.keys()) == G["payload_keys"] and v["op"] == G["op"] and v["before"] is None and v["transaction"] is None
    assert list(v.keys()) == sorted(v.keys()) and list(v["after"].keys()) == sorted(v["after"].keys()) and list(v["source"].keys()) == sorted(v["source"].keys())
    for c in G["columns"]:
        m = ('"%s":' % c["name"]).encode()
        at = val.index(m, val.index(b'"after"')) + len(m)
        if c["type"] == "double":
            assert v["after"][c["name"]] == float(c["after_text"])
        else:
            assert val[at:at + len(c["after_text"].encode())] == c["after_text"].encode(), c["name"]
    want = G["source_block"]; got = v["source"]
    assert sorted(got.keys()) == sorted(want.keys())
    for k in ("version", "connector", "name", "snapshot", "db", "schema", "table", "xmin"):
        assert got[k] == want[k], k
    assert got["txId"] == G["id"] and got["lsn"] == G["lsn"] and got["ts_ms"] == G["commit_time"] // 10**6 and v["ts_ms"] == G["commit_time"] // 10**6


def _pg_batch():
    """The canon ChangeItem's columns whose pg: original type the device emitter takes, as strict typed cells."""
    import base64
    schema, cols = [], []
    for c in G["pg_columns"]:
        tf = abi.YT_NAME_TO_TF[c["type"]]
        schema.append({"name": c["name"], "type": c["type"], "key": c["key"], "required": c["required"], "original_type": c["original_type"]})
        k, v = c["kind"], c["cell"]
        if k == "time":
            cols.append(abi.fixed_to_column(tf, [v[0]], None, [v[1]]))
        elif k == "str":
            cols.append(abi.strings_to_column(tf, [v.encode()], tags=[1]) if tf == abi.TF_ANY else abi.strings_to_column(tf, [v.encode()]))
        elif k == "json":
            cols.append(abi.strings_to_column(tf, [v.encode()], tags=[0]))
        elif k == "b64":
            cols.append(abi.strings_to_column(tf, [base64.b64decode(v)]))
        else:
            cols.append(abi.fixed_to_column(tf, [v]))
    meta = {"id": np.array([G["id"]], np.uint32), "lsn": np.array([G["lsn"]], np.uint64), "commit_time": np.array([G["commit_time"]], np.uint64)}
    return abi.Batch(1, cols), schema, meta


def test_oracle_pg_types_against_real_debezium_message(po):
    """pkg/debezium/pg/emitter.go AddPg for 33 columns of the CRUD fixture: the emitted values equal what a real Debezium wrote
    (pg/tests/testdata/emitter_crud_test__debezium_insert.txt); json / jsonb compare as JSON (pg keeps its own spacing), floats as numbers."""
    batch, schema, meta = _pg_batch()
    assert all(po.debezium_pg_form(c) >= 0 for c in schema)
    plan = po.build_plan(G["table"][0], G["table"][1], schema, [])
    opts = {k: v for k, v in OPTS.items() if k != "ignore_unknown_sources"}      # every column carries an original type: the production path
    data, ks, rs, errs = po.debezium_emit(batch, plan, opts, meta)
    assert errs == []
    (key, val), = po.debezium_split(data, ks, rs)
    assert key == b'{"i":1}'
    after = json.loads(val)["after"]
    assert sorted(after) == sorted(c["name"] for c in G["pg_columns"])
    for c in G["pg_columns"]:
        got, want = after[c["name"]], c["after"]
        if c["kind"] == "json":
            assert json.loads(got) == json.loads(want), c["name"]
        elif c["kind"] == "f64":
            assert got == pytest.approx(want, rel=1e-7) and isinstance(got, float), c["name"]
        else:
            assert got == want and type(got) is type(want), (c["name"], got, want)
    assert b'"real_":1.45e-10,' in val and b'"timestamp1":1098181434900,' in val and b'"date_":10599,' in val and b'"j":"{\\"k1\\":\\"v1\\"}"' in val


def test_oracle_pg_forms(po):
    """Branch selection and the special values of AddPg (emitter.go:180-191 NaN / Infinity strings, :104-120 time divider)."""
    F = po.debezium_pg_form
    assert F({"type": "timestamp", "original_type": "pg:timestamp(3) without time zone"}) == 9 and F({"type": "timestamp", "original_type": "pg:timestamp(0) without time zone"}) == 8
    assert F({"type": "timestamp", "original_type": "pg:timestamp(6) with time zone"}) == 10 and F({"type": "utf8", "original_type": "pg:character varying(5)"}) == 4
    assert F({"type": "utf8", "original_type": "pg:integer"}) == -1 and F({"type": "utf8", "original_type": "pg:interval"}) == -1 and F({"type": "any", "original_type": "mysql:json"}) == -1
    schema = [{"name": "d", "type": "double", "original_type": "pg:double precision"}, {"name": "r", "type": "double", "original_type": "pg:real"},
              {"name": "t", "type": "timestamp", "original_type": "pg:timestamp(2) without time zone"}, {"name": "z", "type": "timestamp", "original_type": "pg:timestamp with time zone"},
              {"name": "dd", "type": "date", "original_type": "pg:date"}, {"name": "s", "type": "any", "original_type": "pg:citext"}, {"name": "j", "type": "any", "original_type": "pg:jsonb"}]
    b = abi.Batch(4, [abi.fixed_to_column(abi.TF_DOUBLE, [float("nan"), float("-inf"), float("inf"), 0.1]), abi.fixed_to_column(abi.TF_DOUBLE, [0.1, 1e39, 3.0, 16777217.0]),
                      abi.fixed_to_column(abi.TF_TIMESTAMP, [-1, 0, 1, 253402300800], None, [999999999, 1999, 5000000, 0]), abi.fixed_to_column(abi.TF_TIMESTAMP, [-1, 0, 1, 253402300800], None, [999999999, 0, 5000000, 0]),
                      abi.fixed_to_column(abi.TF_DATE, [-1, 86399, 86400, -86401]), abi.strings_to_column(abi.TF_ANY, [b"<Tom>", b'"q\\u003c"', b"12", None], tags=[1, 0, 0, 0]),
                      abi.strings_to_column(abi.TF_ANY, [b'{"a":[1,"\\u003c"]}', b"plain", b"null", b"[1]"], tags=[0, 1, 0, 0])])
    data, ks, rs, errs = po.debezium_emit(b, po.build_plan("s", "t", schema, []), {"version": "1", "source_type": "pg"})
    kv = po.debezium_split(data, ks, rs)
    a = [json.loads(v)["after"] for _, v in kv]
    assert [x["d"] for x in a] == ["NaN", "-Infinity", "Infinity", 0.1]
    assert a[0]["r"] == 0.1 and b'"r":0.1,' in kv[0][1] and a[2]["r"] == 3 and b'"r":16777216,' in kv[3][1]          # float32(t)
    assert [x["t"] for x in a] == [0, 0, 1005, 253402300800000]            # UnixMicro() / 1000 truncates toward zero (-1 us -> 0)
    assert [x["z"] for x in a] == ["1969-12-31T23:59:59.999999999Z", "1970-01-01T00:00:00Z", "1970-01-01T00:00:01.005Z", "10000-01-01T00:00:00Z"]
    assert [x["dd"] for x in a] == [0, 0, 1, -1]
    assert a[0]["s"] == "<Tom>" and a[1]["s"] == "q<" and a[3]["s"] is None
    assert a[0]["j"] == '{"a":[1,"<"]}' and a[1]["j"] == '"plain"' and a[2]["j"] is None and a[3]["j"] == "[1]"
    assert errs == [(1, 40, 1), (2, 40, 5)]              # float32(1e39) is +Inf; the citext cell of row 2 is not a string


def test_oracle_against_reference_unit_test_assertions(po):
    """emitter_value_converter_test.go:41-79 (schema wrapper on/off, no HTML escaping), mysql/tests/emitter_meta_test.go (file / pos / gtid)."""
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "value", "type": "utf8"}]
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1]), abi.strings_to_column(abi.TF_UTF8, [b"<>!@#$%^&*()_"])])
    plan = po.build_plan("", "", schema, [])
    base = {"ignore_unknown_sources": True, "version": "1.1.2.Final", "topic_prefix": "my_topic", "database": "pguser", "source_type": "pg", "snapshot": True}
    d, ks, rs, _ = po.debezium_emit(b, plan, base)
    (k1, v1), = po.debezium_split(d, ks, rs)
    assert G["substrings"]["html"].encode() in v1 and b'"payload"' not in v1 and b'"payload"' not in k1 and b'"op":"r"' in v1
    d, ks, rs, _ = po.debezium_emit(b, plan, dict(base, key_schema='{"type":"struct"}', val_schema='{"type":"struct","x":1}'))
    (k0, v0), = po.debezium_split(d, ks, rs)
    assert json.loads(k0) == {"payload": {"id": 1}, "schema": {"type": "struct"}} and json.loads(v0)["schema"] == {"type": "struct", "x": 1}
    assert k0.startswith(b'{"payload":') and v0.startswith(b'{"payload":{"after":')
    d, ks, rs, _ = po.debezium_emit(b, plan, dict(base, key_schema_id=7, val_schema_id=0x01020304, drop_keys=False))
    (k2, v2), = po.debezium_split(d, ks, rs)
    assert k2 == b"\x00\x00\x00\x00\x07" + k1 and v2 == b"\x00\x01\x02\x03\x04" + v1          # packer_schema_registry.go:66-76
    d, ks, rs, _ = po.debezium_emit(b, plan, dict(base, drop_keys=True))
    assert list(ks) == [0] and d == v1
    # mysql meta
    schema = [{"name": "pk", "type": "uint32", "key": True}, {"name": "bigint_u", "type": "uint64"}]
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_UINT32, [2]), abi.fixed_to_column(abi.TF_UINT64, [18446744073709551615])])
    tx = b"58c4f6fc-27b5-11ed-b434-0242ac1e0002:2"
    meta = {"lsn": np.array([2000000013747], np.uint64), "txid_offsets": np.array([0, len(tx)], np.uint32), "txid_heap": np.frombuffer(tx, np.uint8)}
    d, ks, rs, _ = po.debezium_emit(b, po.build_plan("", "customers3", schema, []), dict(base, source_type="mysql"), meta)
    (_, v), = po.debezium_split(d, ks, rs)
    for name in ("mysql_file", "mysql_pos", "mysql_gtid"):
        assert G["substrings"][name].encode() in v
    assert b'"bigint_u":18446744073709551615' in v and json.loads(v)["source"]["gtid"] == tx.decode()


def _matrix():
    """Every value form addCommon distinguishes, with the rows that make EmitKV fail."""
    schema = [{"name": "k", "type": "int64", "key": True}, {"name": "f", "type": "float"}, {"name": "d", "type": "double"}, {"name": "y", "type": "string"},
              {"name": "s", "type": "utf8"}, {"name": "b", "type": "boolean"}, {"name": "ts", "type": "timestamp"}, {"name": "dt", "type": "datetime"},
              {"name": "a", "type": "any"}, {"name": "dd", "type": "date"}, {"name": "iv", "type": "interval"}, {"name": "u", "type": "uint64", "key": True}]
    n = 8
    nul = lambda *idx: [i in idx for i in range(n)]
    cols = [abi.fixed_to_column(abi.TF_INT64, [-2**63, 2**63 - 1, 0, 1, 2, 3, 4, 5]),
            abi.fixed_to_column(abi.TF_FLOAT, np.array([1.5, 1e21, 1e-7, 3.4e38, -0.0, 16777216.0, float("inf"), 0.1], np.float32)),
            abi.fixed_to_column(abi.TF_DOUBLE, [1e21, 1e20, 1e-7, 5e-324, -0.0, 0.1, 1.0, float("nan")]),
            abi.strings_to_column(abi.TF_BYTES, [b"", b"\xff", b"ab", b"abc", None, b"\x00\x01\x02\x03", b"x", b"y"]),
            abi.strings_to_column(abi.TF_UTF8, [b"<&>", b'q"\\\n\t\x01', b"\xff\xfe", b"\xe2\x80\xa8", None, "ключ".encode(), b"", b"z"]),
            abi.fixed_to_column(abi.TF_BOOLEAN, [1, 0, 1, 0, 1, 0, 1, 0], nul(3)),
            abi.fixed_to_column(abi.TF_TIMESTAMP, [0, 1_700_000_000, -62167219200, 253402300799, 253402300800, -62167219201, 1, 2], nul(6), [0, 123456789, 0, 999999999, 0, 0, 1000, 0]),
            abi.fixed_to_column(abi.TF_DATETIME, [0, 1, 2, 3, 4, 5, 6, 7], nul(7)),
            abi.strings_to_column(abi.TF_ANY, [b'{"k":"a\\u003cb","n":[1,2]}', b"plain <s>", b'"js\\u0026on"', b"null", None, b"[1,2]", b"12", b"true"], tags=[0, 1, 0, 0, 0, 0, 0, 0]),
            abi.fixed_to_column(abi.TF_DATE, [0] * n, [True] * 7 + [False]),
            abi.fixed_to_column(abi.TF_INTERVAL, [5] * n, [True] * 6 + [False, True]),
            abi.fixed_to_column(abi.TF_UINT64, [2**64 - 1, 0, 1, 2, 3, 4, 5, 6])]
    meta = {"id": np.arange(n, dtype=np.uint32) + 4294967290, "lsn": np.array([0, 1, 10**12 - 1, 10**12, 2**64 - 1, 5, 6, 7], np.uint64),
            "commit_time": np.array([0, 999999, 10**6, 1649273150231781000, 2**63, 2**64 - 1, 7, 8], np.uint64)}
    return abi.Batch(n, cols), schema, meta


def test_oracle_value_forms(po):
    batch, schema, meta = _matrix()
    plan = po.build_plan("public", "t", schema, [])
    data, ks, rs, errs = po.debezium_emit(batch, plan, dict(OPTS, source_type=""), meta)
    kv = po.debezium_split(data, ks, rs)
    assert len(kv) == 8
    assert kv[0][0] == b'{"k":-9223372036854775808,"u":18446744073709551615}'
    assert kv[0][1] == (b'{"after":{"a":"{\\"k\\":\\"a<b\\",\\"n\\":[1,2]}","b":true,"d":1e+21,"dd":null,"dt":"1970-01-01T00:00:00Z","f":1.5,"iv":null,'
                        b'"k":-9223372036854775808,"s":"<&>","ts":"1970-01-01T00:00:00Z","u":18446744073709551615,"y":""},"before":null,"op":"c",'
                        b'"source":{"db":"pguser","name":"fullfillment","snapshot":"false","table":"t","ts_ms":0,"version":"1.1.2.Final"},"transaction":null,"ts_ms":0}')
    v1 = kv[1][1]
    assert b'"a":"plain <s>"' in v1 and b'"d":100000000000000000000,' in v1 and b'"f":1e+21' in v1 and b'"y":"/w=="' in v1 and b'"s":"q\\"\\\\\\n\\t\\u0001"' in v1
    assert b'"ts":"2023-11-14T22:13:20.123456789Z"' in v1
    assert b'"a":"js&on"' in kv[2][1] and b'"s":"\\ufffd\\ufffd"' in kv[2][1] and b'"ts":"0000-01-01T00:00:00Z"' in kv[2][1] and b'"d":1e-7,' in kv[2][1] and b'"f":1e-7,' in kv[2][1]
    assert b'"a":null' in kv[3][1] and b'"s":"\\u2028"' in kv[3][1] and b'"d":5e-324' in kv[3][1] and b'"b":null' in kv[3][1]
    assert b'"ts_ms":1649273150231}' in kv[3][1] and b'"ts_ms":1649273150231,' in kv[3][1]
    # CommitTime >= 2^63: source.ts_ms is unsigned, the payload's goes through time.Unix(...).UnixNano() (int64)
    assert b'"ts_ms":9223372036854,"version"' in kv[4][1] and kv[4][1].endswith(b'"ts_ms":-9223372036854}')
    assert b'"ts_ms":18446744073709,"version"' in kv[5][1] and kv[5][1].endswith(b'"ts_ms":0}')
    # rows EmitKV fails on: year 10000 / year -1, any array / number / bool, +Inf float, NaN double, non-nil date and interval
    # (only the first failing column of a row is reported, in the sorted-key order the encoder walks: a, b, d, dd, dt, f, iv, ...)
    assert errs == [(4, 40, 6), (5, 40, 8), (6, 40, 8), (7, 40, 8)]
    one = [abi.fixed_to_column(abi.TF_FLOAT, np.array([np.inf], np.float32)), abi.fixed_to_column(abi.TF_DOUBLE, [float("nan")]), abi.fixed_to_column(abi.TF_DATE, [0]), abi.fixed_to_column(abi.TF_INTERVAL, [1])]
    for k, typ in enumerate(("float", "double", "date", "interval")):
        sub = abi.Batch(1, [one[k]])
        assert po.debezium_emit(sub, po.build_plan("s", "t", [{"name": "c", "type": typ}], []), OPTS)[3] == [(0, 40, 0)], typ


def test_oracle_kinds_and_chain(po):
    """The chain runs first: filter_rows rejects UPDATE / DELETE rows itself (filter_rows.go:103-107); key columns follow the result schema."""
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "name", "type": "utf8"}, {"name": "x", "type": "int64"}]
    b = abi.Batch(5, [abi.fixed_to_column(abi.TF_INT32, [1, 2, 3, 4, 5]), abi.strings_to_column(abi.TF_UTF8, [b"a", b"b", b"c", b"d", b"e"]),
                      abi.fixed_to_column(abi.TF_INT64, [10, 20, 30, 40, 50])], kinds=np.array([0, 1, 0, 2, 0], np.uint8))
    trs = [{"filter_rows": {"filter": "x > 10"}}, {"mask_field": {"columns": ["name"], "maskFunctionHash": {"userDefinedSalt": "s"}}}]
    plan = po.build_plan("db", "t", schema, trs)
    data, ks, rs, errs = po.debezium_emit(b, plan, OPTS)
    assert errs == [(1, abi.TF_ROWERR_FILTER_KIND, 0), (3, abi.TF_ROWERR_FILTER_KIND, 0)]
    kv = po.debezium_split(data, ks, rs)
    assert [k for k, _ in kv] == [b'{"id":3}', b'{"id":5}']
    after = json.loads(kv[0][1])["after"]
    assert after["x"] == 30 and len(after["name"]) == 64 and after["name"] == po.hmac_hex(b"s", b"c")


def test_oracle_against_typeutil_unit_tests(po):
    """pkg/debezium/typeutil/helpers_test.go: TestGetTimeDivider (:329-375, the timestamp rows), TestSprintfDebeziumTime (:488-496),
    TestLSNToFileAndPos (:482-486) — through the emitter: one row, the pg branches that use those helpers."""
    import calendar, datetime
    F = po.debezium_pg_form
    for p_, want in ((1, 9), (3, 9), (4, 8), (6, 8)):          # divider 1000 -> milliseconds (branch 9), 1 -> microseconds (branch 8)
        assert F({"type": "timestamp", "original_type": f"pg:timestamp({p_}) without time zone"}) == want
    assert F({"type": "timestamp", "original_type": "pg:timestamp without time zone"}) == 8
    sec = calendar.timegm(datetime.datetime(2022, 8, 28, 19, 49, 47).timetuple())
    schema = [{"name": "a", "type": "timestamp", "original_type": "pg:timestamp with time zone", "key": True}, {"name": "b", "type": "timestamp", "original_type": "pg:timestamp with time zone"}]
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_TIMESTAMP, [sec], None, [749906000]), abi.fixed_to_column(abi.TF_TIMESTAMP, [sec], None, [90000000])])
    meta = {"lsn": np.array([2000000013747], np.uint64)}
    data, ks, rs, errs = po.debezium_emit(b, po.build_plan("db", "t", schema, []), {"source_type": "mysql", "version": "1"}, meta)
    (_, val), = po.debezium_split(data, ks, rs)
    v = json.loads(val)
    assert v["after"] == {"a": "2022-08-28T19:49:47.749906Z", "b": "2022-08-28T19:49:47.09Z"}
    assert v["source"]["file"] == "mysql-log.000002" and v["source"]["pos"] == 13747


def test_queue_debezium_batching(po):
    """debezium_multithreading_test.go:10-70 TestMergeWithMaxMessageSize (values {0,0} and {1,1}: one message under a big limit, two
    under limit 1) and random sizes against the literal restatement; the product's host-only function gives the same cuts."""
    from transferia_b200 import engine
    vals = [bytes([0, 0]), bytes([1, 1])]
    assert po.queue_debezium_merge(vals, 999999) == [bytes([0, 0, 1, 1])] and po.queue_debezium_merge(vals, 1) == vals
    assert engine.queue_debezium_batches([2, 2], 999999) == [0, 2] and engine.queue_debezium_batches([2, 2], 1) == [0, 1, 2]
    assert engine.queue_debezium_batches([2, 2], 0) == [0, 1, 2] and engine.queue_debezium_batches([], 10) == [0]
    rng = np.random.default_rng(3)
    for limit in (1, 7, 64, 1000):
        sizes = [int(x) for x in rng.integers(0, 40, 300)]
        values = [bytes([k % 251]) * s for k, s in enumerate(sizes)]
        cuts = engine.queue_debezium_batches(sizes, limit)
        got = [b"".join(values[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        assert got == po.queue_debezium_merge(values, limit), limit


def test_product_host_template_matches_oracle(po):
    """The product's host side of the emitter (libtfgpu.so, no GPU): the branch chosen per column equals the oracle's, and the message
    template — constant text with the per-row fields between — matches every message the oracle writes, field by field."""
    import re
    from transferia_b200 import engine
    batch, schema, meta = _pg_batch()
    schema = schema + [{"name": "zz", "type": "utf8"}]
    batch = abi.Batch(1, batch.columns + [abi.strings_to_column(abi.TF_UTF8, [b"plain"])])
    plan = po.build_plan("public", "basic_types", schema, [])
    tx = b"gt:1"
    meta = dict(meta, txid_offsets=np.array([0, len(tx)], np.uint32), txid_heap=np.frombuffer(tx, np.uint8))
    lsn, ct, rid = int(meta["lsn"][0]), int(meta["commit_time"][0]), int(meta["id"][0])
    field = {3: str(lsn), 4: str(ct // 10**6), 5: str(rid), 6: "%06d" % (lsn // 10**12), 7: str(lsn % 10**12), 8: '"gt:1"', 9: str(ct // 10**6)}
    variants = [{}, {"snapshot": True}, {"drop_keys": True}, {"key_schema": '{"k":"<s>"}', "val_schema": '{"v":1}'}, {"key_schema_id": 3, "val_schema_id": 0x01020304}]      # (ids whose bytes are ASCII: the describe JSON is text)
    for st in ("", "pg", "mysql"):
        for extra in variants:
            opts = dict(OPTS, source_type=st, **extra)
            d = engine.emit_debezium_validate("public", "basic_types", schema, [], opts)
            assert d["forms"] == [po.debezium_pg_form(c) for c in plan.result_schema]
            assert [schema[k]["name"] for k in d["keys"]] == sorted(c["name"] for c in schema if c.get("key"))
            data, ks, rs, errs = po.debezium_emit(batch, plan, opts, meta)
            msg = data[:int(rs[0])].decode("latin-1")
            pat = "".join(re.escape(t.encode("utf-8").decode("latin-1")) + ("(.*)" if code else "") for t, code in d["template"])
            m = re.fullmatch(pat, msg, re.S)
            assert m, (st, extra)
            groups = iter(m.groups())
            for t, code in d["template"]:
                if not code:
                    continue
                g = next(groups)
                if code in field:
                    assert g == field[code], (st, extra, code)
                elif code == 10:          # end of the key message
                    assert g == ""
                elif code == 11:          # `before`: an insert has none
                    assert g == "null"
                elif code == 12:          # op (kindToOp)
                    assert g == ("r" if extra.get("snapshot") else "c")
                else:                     # the key / after object
                    obj = json.loads(g)
                    assert list(obj) == sorted(obj) and (code == 1) == ("zz" in obj)
            # the key message ends where the template says
            key_end = sum(len(t.encode("utf-8")) for t, code in d["template"][:[c for _, c in d["template"]].index(10) + 1]) + (0 if extra.get("drop_keys") else len(b'{"i":1}'))
            assert key_end == int(ks[0]), (st, extra)
    # refusals decided on the host: errUnknownSource, types and (type, column type) pairs left to Go, rewritten pg columns, bad options
    ok = {"name": "i", "type": "int32", "key": True, "original_type": "pg:integer"}
    for sch, trs, opts, rc in (([{"name": "i", "type": "int32"}], [], {"version": "1"}, TF_E_FATAL_CONFIG),
                               ([dict(ok, original_type="pg:interval")], [], OPTS, TF_E_FATAL_UNSUPPORTED), ([dict(ok, original_type="pg:bigint")], [], OPTS, TF_E_FATAL_UNSUPPORTED),
                               ([dict(ok, original_type="mysql:int(11)")], [], OPTS, TF_E_FATAL_UNSUPPORTED), ([ok], [{"convert_to_string": {}}], OPTS, TF_E_FATAL_UNSUPPORTED),
                               ([ok], [{"mask_field": {"columns": ["i"], "maskFunctionHash": {"userDefinedSalt": "s"}}}], {"version": "1"}, TF_E_FATAL_CONFIG),
                               ([ok], [], dict(OPTS, source_type="oracle"), TF_E_FATAL_UNSUPPORTED)):
        with pytest.raises(engine.EngineError) as ei:
            engine.emit_debezium_validate("s", "t", sch, trs, opts)
        assert ei.value.rc == rc, (sch, trs, opts)
    # a masked pg column loses its original type (hmac_hasher.go:41): common path, needs ignore_unknown_sources
    d = engine.emit_debezium_validate("s", "t", [ok], [{"mask_field": {"columns": ["i"], "maskFunctionHash": {"userDefinedSalt": "s"}}}], OPTS)
    assert d["forms"] == [0]


# ----------------------------------------------------------------------------------------------------------- GPU parity
def _same(eng, po, batch, schema, trs, opts, meta, ns="public", name="t"):
    pid = eng.plan(ns, name, schema, trs); plan = po.build_plan(ns, name, schema, trs)
    want = po.debezium_emit(batch, plan, opts, meta)
    got = eng.emit_debezium(pid, batch, opts, meta)
    assert got.errors == want[3], (opts, trs)
    assert list(got.key_sizes) == list(want[1]) and list(got.row_sizes) == list(want[2]), (opts, trs)
    assert got.wire == want[0], (opts, trs)
    return got


@pytest.mark.gpu
def test_device_emitter_equals_oracle(eng, po):
    batch, schema, meta = _golden_batch()
    _same(eng, po, batch, schema, [], OPTS, meta, *G["table"])
    batch, schema, meta = _matrix()
    tx = [b"", b"58c4f6fc-27b5-11ed-b434-0242ac1e0002:2", b"<gt&id>", b"\xff", b"", b"x", b"y", b"z"]
    off = np.zeros(9, np.uint32); np.cumsum([len(t) for t in tx], out=off[1:])
    meta = dict(meta, txid_offsets=off, txid_heap=np.frombuffer(b"".join(tx), np.uint8))
    for st in ("", "pg", "mysql"):
        for extra in ({}, {"snapshot": True}, {"drop_keys": True}, {"key_schema": '{"type":"struct","fields":[]}', "val_schema": '{"type":"struct","name":"<e>"}'},
                      {"key_schema_id": 1, "val_schema_id": 4000000000}):
            _same(eng, po, batch, schema, [], dict(OPTS, source_type=st, **extra), meta)
    _same(eng, po, batch, schema, [], OPTS, None)
    # pg: original types (AddPg branches): the canon fixture and the special values
    batch, schema, meta = _pg_batch()
    _same(eng, po, batch, schema, [], {k: v for k, v in OPTS.items() if k != "ignore_unknown_sources"}, meta, *G["table"])
    schema = [{"name": "d", "type": "double", "original_type": "pg:double precision"}, {"name": "r", "type": "double", "original_type": "pg:real"},
              {"name": "t", "type": "timestamp", "original_type": "pg:timestamp(2) without time zone"}, {"name": "z", "type": "timestamp", "original_type": "pg:timestamp with time zone"},
              {"name": "dd", "type": "date", "original_type": "pg:date"}, {"name": "s", "type": "any", "original_type": "pg:citext"}, {"name": "j", "type": "any", "original_type": "pg:jsonb"},
              {"name": "k", "type": "int64", "original_type": "pg:bigint", "key": True}, {"name": "u", "type": "utf8"}]
    b = abi.Batch(4, [abi.fixed_to_column(abi.TF_DOUBLE, [float("nan"), float("-inf"), float("inf"), 0.1]), abi.fixed_to_column(abi.TF_DOUBLE, [0.1, 1e39, 3.0, 16777217.0]),
                      abi.fixed_to_column(abi.TF_TIMESTAMP, [-1, 0, 1, 253402300800], None, [999999999, 1999, 5000000, 0]), abi.fixed_to_column(abi.TF_TIMESTAMP, [-1, 0, 1, 253402300800], None, [999999999, 0, 5000000, 0]),
                      abi.fixed_to_column(abi.TF_DATE, [-1, 86399, 86400, -86401]), abi.strings_to_column(abi.TF_ANY, [b"<Tom>", b'"q\\u003c"', b"12", None], tags=[1, 0, 0, 0]),
                      abi.strings_to_column(abi.TF_ANY, [b'{"a":[1,"\\u003c"]}', b"plain", b"null", b"[1]"], tags=[0, 1, 0, 0]), abi.fixed_to_column(abi.TF_INT64, [1, 2, 3, 4]),
                      abi.strings_to_column(abi.TF_UTF8, [b"a", None, b"<c>", b""])])
    _same(eng, po, b, schema, [], dict(OPTS, source_type="pg"), None)
    _same(eng, po, b, schema, [{"filter_rows": {"filter": "k > 1"}}], dict(OPTS, source_type="pg", key_schema='{"t":1}', val_schema='{"t":2}'), None)
    # kinds + chain
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "name", "type": "utf8"}, {"name": "x", "type": "int64"}]
    b = abi.Batch(5, [abi.fixed_to_column(abi.TF_INT32, [1, 2, 3, 4, 5]), abi.strings_to_column(abi.TF_UTF8, [b"a", b"b", b"c", b"d", b"e"]),
                      abi.fixed_to_column(abi.TF_INT64, [10, 20, 30, 40, 50])], kinds=np.array([0, 1, 0, 2, 0], np.uint8))
    for trs in ([], [{"filter_rows": {"filter": "x > 10"}}, {"mask_field": {"columns": ["name"], "maskFunctionHash": {"userDefinedSalt": "s"}}}],
                [{"convert_to_string": {"columns": {"includeColumns": ["x", "name"]}}}], [{"rename_tables": {"renameTables": [{"originalName": {"namespace": "public", "name": "t"}, "newName": {"namespace": "ns2", "name": "t<2>"}}]}}]):
        _same(eng, po, b, schema, trs, OPTS, None)


@pytest.mark.gpu
def test_device_emitter_all_types_and_resident(eng, po):
    """The all-types batch (nulls, long strings, NaN, out-of-range years, non-UTF-8 text) with keys, from host and from HBM."""
    from test_gpu_parity import all_types_batch
    batch, schema = all_types_batch(3000, seed=11)
    for c in schema:
        if c["name"] in ("c_int64", "c_utf8"):
            c["key"] = True
    rng = np.random.default_rng(5)
    meta = {"id": rng.integers(0, 2**32, batch.nrows, dtype=np.uint32), "lsn": rng.integers(0, 2**63, batch.nrows, dtype=np.uint64),
            "commit_time": rng.integers(0, 2**62, batch.nrows, dtype=np.uint64)}
    drop_bad = [{"filter_columns": {"columns": {"excludeColumns": ["c_date", "c_interval"]}}}]
    for trs in ([], drop_bad, drop_bad + [{"filter_rows": {"filter": "c_int32 > 0"}}]):
        got = _same(eng, po, batch, schema, trs, OPTS, meta)
    assert got.rows_out > 0
    import torch
    dbatch = batch.to_device("cuda:0")
    dmeta = {k: torch.from_numpy(v.view(np.int32 if v.dtype == np.uint32 else np.int64)).cuda() for k, v in meta.items()}
    pid = eng.plan("public", "t", schema, drop_bad); plan = po.build_plan("public", "t", schema, drop_bad)
    want = po.debezium_emit(batch, plan, OPTS, meta)
    res = eng.emit_debezium(pid, dbatch, OPTS, dmeta)
    assert res.wire == want[0] and list(res.key_sizes) == list(want[1]) and res.errors == want[3]


@pytest.mark.gpu
def test_device_emitter_refusals(eng):
    from transferia_b200.engine import EngineError
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1])])
    # each refusal has the code emit_debezium_validate gives it: UNSUPPORTED keeps the table on the Go emitter
    pid = eng.plan("s", "t", [{"name": "i", "type": "int32", "key": True}], [])
    with pytest.raises(EngineError) as ei:        # errUnknownSource (emitter_value_converter.go:183-191)
        eng.emit_debezium(pid, b, {"version": "1"})
    assert ei.value.rc == TF_E_FATAL_CONFIG
    for col in ({"name": "i", "type": "int32", "key": True, "original_type": "pg:interval"}, {"name": "i", "type": "int32", "key": True, "original_type": "pg:bigint"},
                {"name": "i", "type": "int32", "key": True, "original_type": "mysql:int(11)"}):
        pid = eng.plan("s", "t", [col], [])
        with pytest.raises(EngineError) as ei:
            eng.emit_debezium(pid, b, OPTS)
        assert ei.value.rc == TF_E_FATAL_UNSUPPORTED, col
    pid = eng.plan("s", "t", [{"name": "i", "type": "int32", "key": True, "original_type": "pg:integer"}], [{"convert_to_string": {}}])
    with pytest.raises(EngineError) as ei:        # a transformer rewrote a pg-typed column: AddPg would reject the value
        eng.emit_debezium(pid, b, OPTS)
    assert ei.value.rc == TF_E_FATAL_UNSUPPORTED


# ----------------------------------------------------------------------------------------------------------- update / delete events
GC = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "debezium_crud_goldens.json"), encoding="utf-8"))
KIND = {"insert": abi.TF_KIND_INSERT, "update": abi.TF_KIND_UPDATE, "delete": abi.TF_KIND_DELETE}


def _cell_column(tf, kind, cell):
    import base64
    if cell is None:
        return abi.strings_to_column(tf, [None]) if tf in abi.VAR_TYPES else abi.fixed_to_column(tf, [0], [True])
    if kind == "time":
        return abi.fixed_to_column(tf, [cell[0]], None, [cell[1]])
    if kind == "str":
        return abi.strings_to_column(tf, [cell.encode()], tags=[1]) if tf == abi.TF_ANY else abi.strings_to_column(tf, [cell.encode()])
    if kind == "json":
        return abi.strings_to_column(tf, [cell.encode()], tags=[0])
    if kind == "b64":
        return abi.strings_to_column(tf, [base64.b64decode(cell)])
    return abi.fixed_to_column(tf, [cell])


def _crud_item(it):
    """(batch with kinds, old batch, present column indexes, schema, meta) of one canon ChangeItem of the CRUD fixtures."""
    schema, cols, ocols, present = [], [], [], []
    old = {o["name"]: o for o in it["old"]}
    for k, c in enumerate(it["columns"]):
        tf = abi.YT_NAME_TO_TF[c["type"]]
        schema.append({"name": c["name"], "type": c["type"], "key": c["key"], "required": c["required"], "original_type": c["original_type"]})
        cols.append(_cell_column(tf, c["kind"], c["cell"] if c["present"] else None))
        if c["name"] in old:
            present.append(k); ocols.append(_cell_column(tf, old[c["name"]]["kind"], old[c["name"]]["cell"]))
        else:
            ocols.append(_cell_column(tf, c["kind"], None))
    meta = {"id": np.array([it["id"]], np.uint32), "lsn": np.array([it["lsn"]], np.uint64), "commit_time": np.array([it["commit_time"]], np.uint64)}
    return abi.Batch(1, cols, np.array([KIND[it["kind"]]], np.uint8)), abi.Batch(1, ocols), present, schema, meta


def _same_value(got, want, col):
    if col["kind"] == "json" and got is not None and want is not None:
        return json.loads(got) == json.loads(want)
    if col["kind"] == "f64" and got is not None and want is not None:
        return got == pytest.approx(want, rel=1e-7)
    return got == want and type(got) is type(want)


def test_oracle_update_delete_against_real_debezium_messages(po):
    """emitter_crud_test.go:15-165 and emitter_replica_identity_test.go:17-97: the message count per ChangeItem (1 for a plain update,
    delete event + tombstone for a delete, delete + tombstone + insert for an update that changes its key), the key payloads the Go test
    spells out, and op / before / after of what a real Debezium wrote, over the columns the device emitter takes."""
    opts = {k: v for k, v in OPTS.items() if k != "ignore_unknown_sources"}
    for it in GC["items"]:
        batch, old, present, schema, meta = _crud_item(it)
        plan = po.build_plan(it["table"][0], it["table"][1], schema, [])
        data, ks, rs, errs, ms = po.debezium_emit(batch, plan, opts, meta, old=old, old_present=present, want_msg_sizes=True)
        assert errs == [], it["item"]
        (msgs,) = po.debezium_messages(data, ms)
        want = it["events"]
        if it.get("first_event_only"):
            msgs = msgs[:1]          # that test checks the first event (the delete's tombstone is not in its fixture)
        assert len(msgs) == len(want), (it["item"], len(msgs))
        by_name = {c["name"]: c for c in it["columns"]}
        for (key, val), ev in zip(msgs, want):
            assert json.loads(key) == ev["key"], it["item"]
            if ev["value"] is None:
                assert val is None; continue
            v = json.loads(val)
            assert v["op"] == ev["value"]["op"] and v["transaction"] is None
            for side in ("before", "after"):
                w, g = ev["value"][side], v[side]
                assert (w is None) == (g is None), (it["item"], side)
                if w is not None:
                    assert sorted(g) == sorted(w), (it["item"], side)
                    for n in w:
                        assert _same_value(g[n], w[n], by_name[n]), (it["item"], side, n, g[n], w[n])
            for k in ("connector", "name", "db", "schema", "table", "snapshot"):
                assert v["source"][k] == ev["value"]["source"][k], (it["item"], k)
            assert v["source"]["txId"] == it["id"] and v["source"]["lsn"] == it["lsn"]      # the canon items were captured in another session than the messages


def test_oracle_crud_rules(po):
    """emitKV's branches on a small table: tombstones.on.delete=false, an update without OldKeys (every key compares against nil:
    KeysChanged), hasPreviousValues, a delete's `before` (all columns null + OldKeys), mysql's `before` filled from the row."""
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "name", "type": "utf8"}, {"name": "x", "type": "int64"}]
    b = abi.Batch(4, [abi.fixed_to_column(abi.TF_INT32, [1, 2, 3, 4]), abi.strings_to_column(abi.TF_UTF8, [b"a", b"b", b"c", b"d"]), abi.fixed_to_column(abi.TF_INT64, [10, 20, 30, 40])],
                  kinds=np.array([0, 1, 1, 2], np.uint8))
    old = abi.Batch(4, [abi.fixed_to_column(abi.TF_INT32, [0, 2, 30, 4]), abi.strings_to_column(abi.TF_UTF8, [None, b"B", b"C", b"D"]), abi.fixed_to_column(abi.TF_INT64, [0, 0, 0, 0], [True] * 4)])
    plan = po.build_plan("db", "t", schema, [])
    def run(opts, **kw):
        data, ks, rs, errs, ms = po.debezium_emit(b, plan, dict(OPTS, source_type="", **opts), None, want_msg_sizes=True, **kw)
        assert errs == []
        return [[(k, None if v is None else json.loads(v)) for k, v in row] for row in po.debezium_messages(data, ms)]
    rows = run({}, old=old, old_present=[0, 1])                      # OldKeys = {id, name}: more than the keys -> before on updates
    assert [len(r) for r in rows] == [1, 1, 3, 2]
    assert rows[1][0][0] == b'{"id":2}' and rows[1][0][1]["op"] == "u" and rows[1][0][1]["before"] == {"id": 2, "name": "B"} and rows[1][0][1]["after"] == {"id": 2, "name": "b", "x": 20}
    d, t, i = rows[2]
    assert d[0] == b'{"id":30}' and d[1]["op"] == "d" and d[1]["after"] is None and d[1]["before"] == {"id": 30, "name": "C", "x": None}
    assert t == (b'{"id":30}', None) and i[0] == b'{"id":3}' and i[1]["op"] == "c" and i[1]["before"] is None and i[1]["after"]["name"] == "c"
    assert rows[3][0][1]["op"] == "d" and rows[3][1] == (b'{"id":4}', None)
    assert [len(r) for r in run({"tombstones_on_delete": False}, old=old, old_present=[0, 1])] == [1, 1, 2, 1]
    rows = run({}, old=old, old_present=[0])                         # OldKeys = the key only: no `before` on a plain update
    assert rows[1][0][1]["before"] is None and rows[3][0][1]["before"] == {"id": 4, "name": None, "x": None}
    rows = run({})                                                   # no OldKeys at all: keys from the row, every update counts as key-changing
    assert [len(r) for r in rows] == [1, 3, 3, 2] and rows[1][0][0] == b'{"id":2}' and rows[3][0][1]["before"] == {"id": None, "name": None, "x": None}
    data, ks, rs, errs, ms = po.debezium_emit(b, plan, dict(OPTS, source_type="mysql"), None, old=old, old_present=[0], want_msg_sizes=True)
    assert json.loads(po.debezium_messages(data, ms)[3][0][1])["before"] == {"id": 4, "name": "d", "x": 40}      # mysql: ColumnValues first, OldKeys on top


@pytest.mark.gpu
def test_device_emitter_update_delete_equals_oracle(eng, po):
    """tfgpu_emit_debezium_crud against the oracle, byte for byte: the reference's CRUD fixtures, then a mixed batch over every option."""
    opts = {k: v for k, v in OPTS.items() if k != "ignore_unknown_sources"}
    for it in GC["items"]:
        batch, old, present, schema, meta = _crud_item(it)
        pid = eng.plan(it["table"][0], it["table"][1], schema, []); plan = po.build_plan(it["table"][0], it["table"][1], schema, [])
        want = po.debezium_emit(batch, plan, opts, meta, old=old, old_present=present, want_msg_sizes=True)
        got = eng.emit_debezium(pid, batch, opts, meta, old=old, old_present=present)
        nm = int(want[4][0][0])
        assert got.wire == want[0] and got.errors == want[3] and np.array_equal(got.msg_sizes[:, :1 + 2 * nm], want[4][:, :1 + 2 * nm]), it["item"]
    rng = np.random.default_rng(4); n = 3000
    schema = [{"name": "id", "type": "int64", "key": True}, {"name": "k2", "type": "utf8", "key": True}, {"name": "name", "type": "utf8"}, {"name": "x", "type": "double"},
              {"name": "ts", "type": "timestamp"}, {"name": "j", "type": "any"}]
    ids = rng.integers(0, 50, n); k2 = [b"k%d" % v for v in rng.integers(0, 5, n)]
    def mk(ids_, k2_, salt):
        return abi.Batch(n, [abi.fixed_to_column(abi.TF_INT64, ids_), abi.strings_to_column(abi.TF_UTF8, k2_),
                             abi.strings_to_column(abi.TF_UTF8, [None if (i + salt) % 7 == 0 else b"n<%d>" % (i * salt) for i in range(n)]),
                             abi.fixed_to_column(abi.TF_DOUBLE, rng.random(n) * 1e3, [(i + salt) % 11 == 0 for i in range(n)]),
                             abi.fixed_to_column(abi.TF_TIMESTAMP, rng.integers(0, 2**31, n), None, rng.integers(0, 10**9, n).astype(np.uint32)),
                             abi.strings_to_column(abi.TF_ANY, [b'{"a":%d}' % i for i in range(n)], tags=[0] * n)])
    kinds = rng.integers(0, 3, n).astype(np.uint8)
    b = mk(ids, k2, 1); b.kinds = kinds
    same = rng.random(n) < 0.6
    old = mk(np.where(same, ids, ids + 1), [a if s_ else a + b"x" for a, s_ in zip(k2, rng.random(n) < 0.8)], 3)
    has = (rng.random(n) < 0.9).astype(np.uint8)
    meta = {"id": rng.integers(0, 2**32, n, dtype=np.uint32), "lsn": rng.integers(0, 2**62, n, dtype=np.uint64), "commit_time": rng.integers(0, 2**62, n, dtype=np.uint64)}
    pid = eng.plan("public", "t", schema, []); plan = po.build_plan("public", "t", schema, [])
    for o, present, row_has in (({}, [0, 1], None), ({}, [0, 1, 2, 3, 4, 5], has), ({"tombstones_on_delete": False, "snapshot": True}, [0], has), ({"source_type": "mysql"}, [0, 1, 2], None),
                                ({"key_schema": '{"t":1}', "val_schema": '{"t":2}'}, [1, 2], has), ({"drop_keys": True}, [0, 1], None)):
        oo = dict(OPTS, **o)
        want = po.debezium_emit(b, plan, oo, meta, old=old, old_present=present, old_row_has=row_has, want_msg_sizes=True)
        got = eng.emit_debezium(pid, b, oo, meta, old=old, old_present=present, old_row_has=row_has)
        assert got.errors == want[3] and list(got.row_sizes) == list(want[2]), o
        assert got.wire == want[0], o
        cnt = want[4][:, 0]
        for m in range(3):
            sel = cnt > m
            assert np.array_equal(got.msg_sizes[sel, 1 + 2 * m: 3 + 2 * m], want[4][sel, 1 + 2 * m: 3 + 2 * m]), (o, m)
        assert np.array_equal(got.msg_sizes[:, 0], cnt) and set(cnt.tolist()) >= {1, 2}
    # without OldKeys
    want = po.debezium_emit(b, plan, OPTS, meta, want_msg_sizes=True); got = eng.emit_debezium(pid, b, OPTS, meta)
    assert got.wire == want[0] and np.array_equal(got.msg_sizes[:, 0], want[4][:, 0])


def test_oracle_against_the_serializer_test_messages(po):
    """pkg/serializer/queue/debezium_serializer_test.go:43-145 (TestDebeziumSerializerSnapshot, ...TopicName, ...TopicPrefix): the complete key
    and value messages of one pg item (id 601, LSN 25051056, CommitTime 1643660670333075000, columns id / val `pg:integer`) with the
    include-schema packer, byte for byte — snapshot on (op "r") and off (op "c"), three table names, two topic prefixes. The two schema texts
    are what the shim passes in (the reference caches them per table); the payloads, the source block and the wrapper are computed."""
    schema = [{"name": "id", "type": "int32", "key": True, "original_type": "pg:integer"}, {"name": "val", "type": "int32", "original_type": "pg:integer"}]
    b = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1]), abi.fixed_to_column(abi.TF_INT32, [-8388605])])
    meta = {"id": np.array([601], np.uint32), "lsn": np.array([25051056], np.uint64), "commit_time": np.array([1643660670333075000], np.uint64)}
    for table, prefix, snap in (("snapshot", "__data_transfer_stub", True), ("table0", "__data_transfer_stub", False), ("table1", "__data_transfer_stub", False), ("basic_types15", "my_topic_prefix", False)):
        fq = f"{prefix}.public.{table}"
        key_schema = '{"fields":[{"field":"id","optional":false,"type":"int32"}],"name":"%s.Key","optional":false,"type":"struct"}' % fq
        val_schema = ('{"fields":[{"field":"before","fields":[{"field":"id","optional":false,"type":"int32"},{"field":"val","optional":true,"type":"int32"}],"name":"FQ.Value","optional":true,"type":"struct"},'
                      '{"field":"after","fields":[{"field":"id","optional":false,"type":"int32"},{"field":"val","optional":true,"type":"int32"}],"name":"FQ.Value","optional":true,"type":"struct"},'
                      '{"field":"source","fields":[{"field":"version","optional":false,"type":"string"},{"field":"connector","optional":false,"type":"string"},{"field":"name","optional":false,"type":"string"},{"field":"ts_ms","optional":false,"type":"int64"},'
                      '{"default":"false","field":"snapshot","name":"io.debezium.data.Enum","optional":true,"parameters":{"allowed":"true,last,false"},"type":"string","version":1},{"field":"db","optional":false,"type":"string"},'
                      '{"field":"table","optional":false,"type":"string"},{"field":"lsn","optional":true,"type":"int64"},{"field":"schema","optional":false,"type":"string"},{"field":"txId","optional":true,"type":"int64"},{"field":"xmin","optional":true,"type":"int64"}],'
                      '"name":"io.debezium.connector.postgresql.Source","optional":false,"type":"struct"},{"field":"op","optional":false,"type":"string"},{"field":"ts_ms","optional":true,"type":"int64"},'
                      '{"field":"transaction","fields":[{"field":"id","optional":false,"type":"string"},{"field":"total_order","optional":false,"type":"int64"},{"field":"data_collection_order","optional":false,"type":"int64"}],"optional":true,"type":"struct"}],'
                      '"name":"FQ.Envelope","optional":false,"type":"struct"}').replace("FQ", fq)
        opts = {"version": "1.1.2.Final", "topic_prefix": prefix, "database": "", "source_type": "pg", "snapshot": snap, "key_schema": key_schema, "val_schema": val_schema}
        d, ks, rs, errs = po.debezium_emit(b, po.build_plan("public", table, schema, []), opts, meta=meta)
        (key, val), = po.debezium_split(d, ks, rs)
        assert not errs
        assert key.decode() == '{"payload":{"id":1},"schema":' + key_schema + '}'
        assert val.decode() == ('{"payload":{"after":{"id":1,"val":-8388605},"before":null,"op":"%s","source":{"connector":"postgresql","db":"","lsn":25051056,"name":"%s","schema":"public",'
                                '"snapshot":"%s","table":"%s","ts_ms":1643660670333,"txId":601,"version":"1.1.2.Final","xmin":null},"transaction":null,"ts_ms":1643660670333},"schema":'
                                % ("r" if snap else "c", prefix, "true" if snap else "false", table)) + val_schema + '}'


def test_oracle_pg_time_forms_against_typeutil_tests(po):
    """pkg/debezium/typeutil/helpers_test.go: TestGetTimeDivider (:329-376 — `timestamp(p) without time zone` travels in milliseconds for
    p 1..3, in microseconds for p 4..6 and without a precision) and TestSprintfDebeziumTime (:488-496 — timestamptz text with the trailing
    zeros of the fraction cut) on the emitter oracle."""
    import calendar
    sec = calendar.timegm((2022, 8, 28, 19, 49, 47))

    def emit(ot, ns):
        schema = [{"name": "id", "type": "int32", "key": True, "original_type": "pg:integer"}, {"name": "t", "type": "timestamp", "original_type": ot}]
        b = abi.Batch(1, [abi.fixed_to_column(abi.TF_INT32, [1]), abi.fixed_to_column(abi.TF_TIMESTAMP, [sec], None, [ns])])
        d, ks, rs, errs = po.debezium_emit(b, po.build_plan("public", "t", schema, []), {"version": "1", "topic_prefix": "p", "database": "", "source_type": "pg"})
        (_, v), = po.debezium_split(d, ks, rs)
        assert not errs
        return json.loads(v)["after"]["t"]
    micros = sec * 1_000_000 + 749906
    for p, divider in ((1, 1000), (3, 1000), (4, 1), (6, 1)):
        assert emit(f"pg:timestamp({p}) without time zone", 749906000) == micros // divider
    assert emit("pg:timestamp without time zone", 749906000) == micros
    assert emit("pg:timestamp with time zone", 749906000) == "2022-08-28T19:49:47.749906Z"
    assert emit("pg:timestamp with time zone", 90000000) == "2022-08-28T19:49:47.09Z"
