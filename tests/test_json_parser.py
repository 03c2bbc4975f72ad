"""Generic JSON parser (SURVEY §8 a10): the oracle against the reference's canon data on CPU, the device parser against
the oracle on GPU (lines -> typed columns -> transformer chain -> sink bytes without leaving HBM)."""
import base64
import json
import os

import numpy as np
import pytest

from transferia_b200 import abi

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "json_parser_goldens.json")))

NUM_FIELDS = [{"name": "id", "type": "int8"}, {"name": "number_field", "type": "int64"}, {"name": "float_field", "type": "double"},
              {"name": "obj_field", "type": "any"}, {"name": "array_field", "type": "any"}]            # parser_test.go:132-153
B64_FIELDS = [{"name": "id", "type": "int8"}, {"name": "stringVal", "type": "utf8"}, {"name": "bytesVal", "type": "string"}]   # :234-247


def cell(batch, c, r):
    col = batch.columns[c]
    if col.validity is not None and not (col.validity[r >> 3] >> (r & 7)) & 1:
        return None
    if col.type in abi.VAR_TYPES:
        raw = bytes(col.heap[col.offsets[r]:col.offsets[r + 1]])
        if col.type == abi.TF_ANY:
            return raw.decode() if col.aux[r] == 1 else json.loads(raw)
        return raw
    return col.values[r].item()


def test_number_types_canon(po):
    """TestParserNumberTypes (parser_test.go:129-231): one message per line, both UseNumbersInAny modes."""
    text = G["inputs"]["parser_numbers_test.jsonl"].encode()
    for mode, use in (("UseNumbersFalse", False), ("UseNumbersTrue", True)):
        want = G["canon"]["TestParserNumberTypes"][mode]
        b, errs, lines = po.json_parse(text, NUM_FIELDS, {"use_numbers_in_any": use})
        assert not errs and lines == b.nrows == len(want)
        for r, it in enumerate(want):
            assert it["types"] == ["int8", "int64", "double", "any", "any"]
            got = [cell(b, c, r) for c in range(5)]
            assert got == it["columnvalues"], (mode, got)
    # the spelling Go's encoding/json gives the `any` cells (sorted keys, float64 'f'/'e' switch-over, json.Number verbatim)
    b, _, _ = po.json_parse(text, NUM_FIELDS, {})
    assert bytes(b.columns[3].heap) == b'{"int_field":123123123123123330}'
    assert bytes(b.columns[4].heap) == b"[0,1,2,4,12313.12241632513,-123123.13117532,12345678987654320,-12345678987654320,100000,1e-7]"
    b, _, _ = po.json_parse(text, NUM_FIELDS, {"use_numbers_in_any": True})
    assert bytes(b.columns[4].heap) == b"[0,1,2,4,12313.12241632513,-123123.13117532,12345678987654321,-12345678987654321,1e5,0.0000001]"


def test_do_json_sample(po):
    """TestParser_DoJson (pkg/parsers/tests/generic_parser_test.go:274-296): 36 lines of the json.lb sample give 36 rows and the uint64
    column `version` holds 89488198116272410 + row exactly (values beyond 2^53: the number text, not a float64, is converted)."""
    d = G["do_json"]
    b, errs, lines = po.json_parse(d["input"].encode(), d["fields"], {"add_rest": d["add_rest"], "null_keys_allowed": d["null_keys_allowed"]})
    assert errs == [] and lines == b.nrows == d["rows"]
    vi = [f["name"] for f in d["fields"]].index("version")
    assert [cell(b, vi, r) for r in range(b.nrows)] == [d["version_base"] + r for r in range(b.nrows)]
    assert cell(b, 0, 0) == b"mdbkbeut80vtiba04gid" and cell(b, len(d["fields"]), 0) == {}          # every key is declared: _rest is empty


def test_base64_canon(po):
    """TestBase64Unpack (parser_test.go:233-276): `string` (bytes) cells are base64-decoded, utf8 cells are unescaped."""
    text = G["inputs"]["parse_base64_packed.jsonl"].encode()
    want = G["canon"]["TestBase64Unpack"]
    b, errs, lines = po.json_parse(text, B64_FIELDS, {"unpack_bytes_base64": True})
    assert not errs and b.nrows == len(want) == 2
    for r, it in enumerate(want):
        assert cell(b, 0, r) == it["columnvalues"][0]
        assert cell(b, 1, r).decode() == it["columnvalues"][1]
        assert cell(b, 2, r) == base64.b64decode(it["columnvalues"][2])       # the canon file prints []byte as base64
    # without the option the cell keeps the text
    b, _, _ = po.json_parse(text, B64_FIELDS, {})
    assert cell(b, 2, 0) == b"dGVzdA=="


# ----------------------------------------------------------------------------------------------------------- GPU parity
from transferia_b200 import engine as _engine  # noqa: E402

ALL_FIELDS = [{"name": "i8", "type": "int8"}, {"name": "i64", "type": "int64"}, {"name": "u8", "type": "uint8"}, {"name": "u64", "type": "uint64"},
              {"name": "d", "type": "double"}, {"name": "b", "type": "boolean"}, {"name": "s", "type": "utf8"}, {"name": "y", "type": "string"},
              {"name": "a", "type": "any"}, {"name": "t", "type": "datetime"}]

QUIRK_VALUES = [
    b"null", b"0", b"-1", b"127", b"128", b"-129", b"300", b"1.5", b"1e3", b"1E+2", b"-0", b"0.1", b"123456789012345678", b"1234567890123456789", b"9223372036854775807",
    b"9223372036854775808", b"18446744073709551615", b"18446744073709551616", b"-9223372036854775808", b"12345678765432.23456765432", b"0.8444218515250481",
    b"2.2250738585072014e-308", b"1.7976931348623157e308", b"1e400", b"1e-400", b"4.9e-324", b"1.", b"-1.", b".5", b"-.5", b"-", b"+1", b"1.2.3", b"e", b"1e", b"--1", b"inf", b"-inf", b"nan", b"NaN", b"+Inf",
    b"true", b"false", b'"abc"', b'""', b'"12"', b'"0x1f"', b'"017"', b'"1_000"', b'"-5"', b'"1e2"', b'"1.25"', b'"true"', b'"T"', b'"maybe"', b'"inf"', b'"nan"', b'"+nan"', b'"0x1p-2"',
    b'"a\\nb\\t\\"q\\" \\\\ \\/ \\u0041\\u00e9\\u20ac\\ud83d\\ude00 \\ud83d x \\udc00 \\uZZZZ \\u12"', b'"\\x \\a"', b'"<tag> & \\u2028 \\u0000"', b'"\xd0\xbf\xd1\x80\xd0\xb8\xd0\xb2\xd0\xb5\xd1\x82 \xff\xfe"',
    b'"dGVzdA=="', b'"dGVzdDI="', b'"dGVz\\ndA=="', b'"dGVzdA="', b'"dGVzdA==="', b'"d"', b'"dG"', b'"dG=="', b'"dGV="', b'"dGVzd A=="', b'"4pyTIMOgIGxhIG1vZGU="',
    b'"{\\"k\\":1}"', b'" {}"', b'"null"', b'"nope"', b'"x\\\\\\\\y\\\\z"', b'"[1]"',
    b"{}", b"[]", b'{"z":1,"a":{"y":[1,2,{"q":null}],"x":"s"},"z":2,"\\u0061b":true}', b"[1, 2.50, -3e-7, \"x\", true, false, null, [], {}, [[[]]]]",
    b'{ "sp" : [ 1 ,2 ] , "t" :"a b" }', b'{"n":1e5,"m":0.0000001,"big":123123123123123321,"e21":1e21,"e-7":1e-7}', b'{"bad":1.2.3}', b'{"nn":nan}',
    b"1373838275", b"1373838275.9", b"-1373838275",
]


# decided by the oracle (strtod), left to the host parser by the device: subnormal results, hex floats, underscored float text
HOST_OK = (b"4.9e-324", b'"0x1p-2"', b'"1_000"')


def _lines_for(values, fields):
    out = []
    for v in values:
        out.append(b"{" + b",".join(b'"%s":%s' % (f["name"].encode(), v) for f in fields) + b"}")
    return b"\n".join(out) + b"\n"


def _cmp(eng, po, text, fields, opts=None, msgs=None, name="db", host_ok=()):
    """Device == oracle: same rows, same errors. `host_ok`: values (bytes) whose lines the device may hand to the host parser
    (TF_ROWERR_JSON_HOST) although the oracle decides them; those lines are then replaced by `[]` (a skipped line) and the
    comparison repeated, so every other line is still compared exactly."""
    opts = opts or {}
    schema = _engine.json_result_schema(fields, opts)
    pid = eng.plan(name, "t", schema, [])
    got, gerr, glines = eng.parse_json(pid, text, opts, msgs)
    ref, rerr, rlines = po.json_parse(text, fields, opts, msgs)
    assert glines == rlines
    extra = [e for e in gerr if e not in rerr]
    if extra and host_ok:
        assert all(c == abi.TF_ROWERR_JSON_HOST for _, c, _ in extra) and msgs is None, extra
        lines = text.split(b"\n"); nonempty = [k for k, ln in enumerate(lines) if ln.rstrip(b"\r")]
        for r, _, _ in extra:
            assert any(v in lines[nonempty[r]] for v in host_ok), lines[nonempty[r]]
            lines[nonempty[r]] = b"[]"
        text = b"\n".join(lines)
        got, gerr, glines = eng.parse_json(pid, text, opts, msgs)
        ref, rerr, rlines = po.json_parse(text, fields, opts, msgs)
    assert gerr == rerr, (gerr[:10], rerr[:10])
    from test_gpu_parity import assert_batches_equal
    assert_batches_equal(got, ref)
    return got, gerr


@pytest.mark.gpu
def test_device_json_goldens(eng, po):
    for use in (False, True):
        _cmp(eng, po, G["inputs"]["parser_numbers_test.jsonl"].encode(), NUM_FIELDS, {"use_numbers_in_any": use})
    _cmp(eng, po, G["inputs"]["parse_base64_packed.jsonl"].encode(), B64_FIELDS, {"unpack_bytes_base64": True})
    _cmp(eng, po, G["inputs"]["parse_base64_packed.jsonl"].encode(), B64_FIELDS, {})


@pytest.mark.gpu
def test_device_json_value_matrix(eng, po):
    """Every JSON value shape into every declared type, one column at a time (so a line only fails for that column's reason)."""
    for f in ALL_FIELDS:
        for opts in ({}, {"use_numbers_in_any": True, "unpack_bytes_base64": True}, {"null_keys_allowed": True}):
            for req in (False, True):
                fields = [dict(f, required=req), {"name": "other", "type": "int32"}]
                text = _lines_for(QUIRK_VALUES, [f]) + b'{"other":5}\n{"other":"x","%s":1}\n' % f["name"].encode()
                _cmp(eng, po, text, fields, opts, host_ok=HOST_OK)
    # all columns at once: the first failing column in schema order names the error
    _cmp(eng, po, _lines_for(QUIRK_VALUES, ALL_FIELDS), [dict(f, required=(f["name"] in ("u8", "a"))) for f in ALL_FIELDS], {}, host_ok=HOST_OK)
    _cmp(eng, po, _lines_for(QUIRK_VALUES, ALL_FIELDS), [dict(f, key=(f["name"] == "d")) for f in ALL_FIELDS], {"add_rest": True}, host_ok=HOST_OK)


@pytest.mark.gpu
def test_device_json_lines_and_grammar(eng, po):
    """Line splitting, fastjson's grammar leniencies and errors, duplicate keys, escaped keys, aux columns over several messages."""
    fields = [{"name": "id", "type": "int32", "key": True}, {"name": "s", "type": "utf8"}, {"name": "a", "type": "any"}]
    lines = [b'{"id":1,"s":"x"}', b'', b'  {"id" : 2 , "s":"y" }  ', b'{"id":3,"s":"crlf"}\r', b'\r', b'{"id":4,"id":5,"s":"dup","s":null}', b'{"i\\u0064":6,"s":"esc key"}',
             b'{"id":7,"extra":{"b":2,"a":1},"more":[1,2],"s":"rest","zz":"q","extra":7}', b'[1,2]', b'"str"', b'17', b'{}', b'null', b'{"id":8', b'{"id":9,}', b'{"id":10 "s":1}',
             b'{id:11}', b'{"id":12}x', b'{"id":13} \t', b'{"id":14,"a":tru}', b'{"id":15,"a":[1,]}', b'{"id":16,"a":[1 2]}', b'{"id":17,"s":"unterminated}', b'{"id":18,"a":nul}',
             b'{"id":19,"a":-}', b'{"id":20,"a":-x}', b'{"id":21,"a":+inf}', b'{"s":"no id"}', b'{"id":null}', b'{"id":"22"}', b'{"id":"x"}', b'{"id":2147483648}', b'{"id":"2147483648"}',
             b'{"id":23,"_rest":1}', b'{"id":24,"_offset":5}', b'{"id":25,"a":' + b'[' * 20 + b']' * 20 + b'}', b'{"id":26,"s":' + b'[' * 298 + b']' * 298 + b'}', b'{"id":27,"s":' + b'[' * 299 + b']' * 299 + b'}',
             b'{"id":28,"\\ud83d\\ude00":1,"\xf0\x9f\x98\x80":2,"<":3}', b'{"id":29,"a":{"b":1,"a":2,"b":{"d":1,"c":[{"z":1,"y":2}]}}}', b'\xef\xbb\xbf{"id":30}', b'{"id":31,"s":"tab\tin string"}',
             b'{"id":32,"s":"last line without newline"}']
    text = b"\n".join(lines)
    for opts in ({}, {"add_rest": True}, {"add_rest": True, "add_dedupe_keys": True, "partition": '{"partition":3,"topic":"t/x"}'}, {"add_dedupe_keys": True, "null_keys_allowed": True}):
        _cmp(eng, po, text, fields, opts)
        # several messages: boundaries end lines, _idx restarts, offsets / write times come from the message
        cuts = [0]
        for k in (5, 6, 6, 9, 20, len(lines)):
            cuts.append(len(b"\n".join(lines[:k])) + (1 if k < len(lines) else 0))
        msgs = [(cuts[k + 1], 100 + k, 1_700_000_000 + k, 1000 * k) for k in range(len(cuts) - 1)]
        _cmp(eng, po, text, fields, opts, msgs)
    # a message that ends without '\n' in the middle of the buffer still ends its line
    two = b'{"id":1}{"id":2}\n{"id":3}'
    _cmp(eng, po, two, fields, {"add_dedupe_keys": True}, [(8, 7, 5, 6), (len(two), 8, 9, 10)])
    _cmp(eng, po, b"", fields, {})
    _cmp(eng, po, b"\n\n\r\n", fields, {"add_dedupe_keys": True})


@pytest.mark.gpu
def test_device_json_host_only_classes(eng, po):
    """Lines the device hands to the host parser although the oracle can decide them (documented in include/tfgpu.h)."""
    fields = [{"name": "d", "type": "double"}, {"name": "a", "type": "any"}]
    pid = eng.plan("db", "t", fields, [])
    lines = [b'{"d":1}', b'{"a":' + b'[' * 40 + b']' * 40 + b'}', b'{"d":"' + b'0' * 120 + b'1"}', b'{"d":1}']
    got, gerr, n = eng.parse_json(pid, b"\n".join(lines))
    assert n == 4 and got.nrows == 2 and [(r, c) for r, c, _ in gerr] == [(1, abi.TF_ROWERR_JSON_HOST), (2, abi.TF_ROWERR_JSON_HOST)]


@pytest.mark.gpu
def test_device_json_config2_workload(eng, po):
    """BASELINE configs[1] shape: JSON lines -> parse -> mask_field on one utf8 column -> JSONEachRow and native(+LZ4), fused on the device."""
    from transferia_b200 import workload
    text, fields = workload.make_json_lines(60_000)
    opts = {"add_rest": True, "add_dedupe_keys": True, "partition": '{"partition":0,"topic":"events"}'}
    step = len(text) // 7
    cuts = [text.rfind(b"\n", 0, step * k) + 1 for k in range(1, 7)] + [len(text)]
    msgs = [(c, 1000 + k, 1_700_000_000, 123_000_000 + k) for k, c in enumerate(cuts)]
    got, _ = _cmp(eng, po, text, fields, opts, msgs, name="events")
    assert got.nrows == 60_000
    schema = _engine.json_result_schema(fields, opts)
    trs = [{"mask_field": {"columns": ["user"], "maskFunctionHash": {"userDefinedSalt": "pepper"}}}]
    pid = eng.plan("", "events", schema, trs, {"type": "clickhouse"})
    ref, _, _ = po.json_parse(text, fields, opts, msgs)
    plan = po.build_plan("", "events", schema, trs)
    for fmt in (abi.TF_WIRE_CH_JSONEACHROW, abi.TF_WIRE_CH_NATIVE):
        res = eng.parse_json(pid, text, opts, msgs, wire_fmt=fmt)
        want = po.push_encode(ref, plan, fmt)
        assert res.rows_out == want.rows_out == 60_000 and res.wire == want.raw
    res = eng.parse_json(pid, text, opts, msgs, wire_fmt=abi.TF_WIRE_CH_NATIVE_LZ4)
    raw, _ = po.ch_decode_frames(res.wire)
    assert raw == po.push_encode(ref, plan, abi.TF_WIRE_CH_NATIVE).raw


def _fuzz_lines(n, seed):
    """Random JSON-ish lines: values of every shape under the declared keys, then byte-level mutations of a share of them."""
    rng = np.random.default_rng(seed)
    scal = [b"null", b"true", b"false", b"0", b"-1", b"7", b"255", b"256", b"-129", b"65536", b"4294967296", b"1.5", b"-2.25e3", b"1e-7", b"0.1", b"123456789.125", b"12e", b"1e+2",
            b'""', b'"x"', b'"42"', b'"-7"', b'"1.5"', b'"true"', b'"a\\tb\\u00e9\\\\"', b'"\xd1\x8f\xd0\xb7\xd1\x8b\xd0\xba"', b'"dGVzdA=="', b'"2013-07-15"', b'"q\\"uote"']
    def value(depth=0):
        k = rng.integers(0, 10)
        if k < 6 or depth > 3: return scal[rng.integers(0, len(scal))]
        if k < 8: return b"[" + b",".join(value(depth + 1) for _ in range(rng.integers(0, 4))) + b"]"
        keys = [b"k%d" % rng.integers(0, 5) for _ in range(rng.integers(0, 4))]
        return b"{" + b",".join(b'"' + kk + b'":' + value(depth + 1) for kk in keys) + b"}"
    names = [f["name"].encode() for f in ALL_FIELDS] + [b"extra", b"zz", b"_rest_not"]
    out = []
    for _ in range(n):
        ks = [names[i] for i in rng.permutation(len(names))[: rng.integers(0, len(names))]]
        sp = b" " if rng.random() < 0.2 else b""
        ln = b"{" + (b"," + sp).join(b'"' + kk + b'"' + sp + b":" + sp + value() for kk in ks) + b"}"
        if rng.random() < 0.15 and len(ln) > 2:       # mutate: delete / duplicate / replace one byte
            p = int(rng.integers(0, len(ln))); m = rng.integers(0, 3)
            ln = ln[:p] + ln[p + 1:] if m == 0 else (ln[:p] + ln[p:p + 1] + ln[p:] if m == 1 else ln[:p] + bytes([rng.integers(32, 127)]) + ln[p + 1:])
        if b"\n" in ln: ln = ln.replace(b"\n", b" ")
        out.append(ln)
    return out


def test_oracle_json_fuzz_smoke(po):
    """The oracle itself survives the fuzz corpus (the GPU test compares the device against it line by line)."""
    lines = _fuzz_lines(3000, 5)
    b, errs, n = po.json_parse(b"\n".join(lines), [dict(f) for f in ALL_FIELDS], {"add_rest": True})
    assert n == len([x for x in lines if x.rstrip(b"\r")]) and b.nrows + len(errs) == n and b.nrows > 500


@pytest.mark.gpu
def test_device_json_fuzz(eng, po):
    """Differential fuzz: 40 k random / mutated lines, every option set; the device must agree with the oracle on every line
    (rows, nulls, text bytes, error codes), except lines it hands to the host parser."""
    for seed, opts in ((1, {}), (2, {"add_rest": True, "use_numbers_in_any": True}), (3, {"add_rest": True, "add_dedupe_keys": True, "unpack_bytes_base64": True, "null_keys_allowed": True}),
                       (4, {"add_dedupe_keys": True})):
        lines = _fuzz_lines(10_000, seed)
        fields = [dict(f, required=(f["name"] == "i64" and seed == 4)) for f in ALL_FIELDS]
        text = b"\n".join(lines)
        schema = _engine.json_result_schema(fields, opts)
        pid = eng.plan("db", "fz", schema, [])
        got, gerr, gl = eng.parse_json(pid, text, opts)
        ref, rerr, rl = po.json_parse(text, fields, opts)
        extra = [e for e in gerr if e not in rerr]
        assert gl == rl and all(c == abi.TF_ROWERR_JSON_HOST for _, c, _ in extra) and len(extra) < 200, (extra[:5], [e for e in rerr if e not in gerr][:5])
        if extra:
            nonempty = [k for k, ln in enumerate(lines) if ln.rstrip(b"\r")]
            for r, _, _ in extra: lines[nonempty[r]] = b"[]"
            text = b"\n".join(lines)
            got, gerr, gl = eng.parse_json(pid, text, opts); ref, rerr, rl = po.json_parse(text, fields, opts)
        assert gerr == rerr, ([e for e in gerr if e not in rerr][:5], [e for e in rerr if e not in gerr][:5])
        from test_gpu_parity import assert_batches_equal
        assert_batches_equal(got, ref)
