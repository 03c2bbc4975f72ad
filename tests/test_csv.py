"""CSV path: the oracle against the reference's reader tests (pkg/csv/reader_test.go) on CPU, and the device parser
against the oracle on GPU (tokenise -> typed columns -> transformer chain -> ClickHouse block, no host round trip)."""
import numpy as np
import pytest

from transferia_b200 import abi, workload

S = lambda n: [{"name": f"c{i}", "type": "utf8", "path": str(i)} for i in range(n)]


def cells(batch):
    return [[bytes(c.heap[c.offsets[r]:c.offsets[r + 1]]) for c in batch.columns] for r in range(batch.nrows)]


def test_reader_reference_cases(po):
    """pkg/csv/reader_test.go:13-240 expectations for the single-line reader."""
    b, e, lines, cons = po.csv_parse(b"1, 2, 3\n\t\ta,b,c\n\t\t7,8,9\n", S(3))
    assert cells(b) == [[b"1", b"2", b"3"], [b"a", b"b", b"c"], [b"7", b"8", b"9"]] and lines == 3 and not e
    # "escape char outside of quotes treated as normal char" :85-96
    b, e, _, _ = po.csv_parse(b'a, \\, "c \\" e , f"\n', S(3))
    assert cells(b) == [[b"a", b"\\", b'c \\" e , f']]
    # "no escape char configured" :98-113
    b, e, _, _ = po.csv_parse(b'a, \\, "c \\" e , f"\n', S(4), {"escape": ""})
    assert cells(b) == [[b"a", b"\\", b'"c \\" e', b'f"']]
    # double quotes collapse / disallowed :115-140
    b, e, _, _ = po.csv_parse(b'a, b, "the main ""test"" is this", d\n', S(4))
    assert cells(b)[0][2] == b'the main "test" is this'
    b, e, _, _ = po.csv_parse(b'a, b, "the main ""test"" is this", d\n', S(4), {"double_quote": False})
    assert b.nrows == 0 and e[0][1] == 24
    # an unterminated last line is dropped (reader.go:162-165)
    b, e, lines, cons = po.csv_parse(b"a,b\nc,d", S(2))
    assert cells(b) == [[b"a", b"b"]] and cons == 4
    # a lone quote element is an error (reader.go:293-295)
    b, e, _, _ = po.csv_parse(b'a,"\n', S(2))
    assert b.nrows == 0 and e == [(0, 17, 0)]
    # the reference takes line[lastDelimPosition+1:] for the last element, i.e. line[1:] when there is no delimiter
    b, e, _, _ = po.csv_parse(b"abc\n", S(1))
    assert cells(b) == [[b"bc"]]
    # DoubleQuoteStr is the quote character twice (s3 csv_config.go:141); swapToSingleQuotes turns it into `"` whatever the quote is
    b, e, _, _ = po.csv_parse(b"a,'it''s'\nb,x\"\"y\n", S(2), {"quote": "'"})
    assert cells(b) == [[b"a", b'it"s'], [b"b", b'x""y']] and not e
    b, e, _, _ = po.csv_parse(b"a,'it''s'\nb,x\"\"y\n", S(2), {"quote": "'", "double_quote": False})
    assert cells(b) == [[b"b", b'x""y']] and e == [(0, 24, 0)]
    # no quote character: a line holding `"` fails in readAndDecodeLine (reader.go:185-187), before any other check of the line
    b, e, _, _ = po.csv_parse(b'a,x"y\n"\nb\nc,d\n', S(2), {"quote": ""})
    assert cells(b) == [[b"c", b"d"]] and e == [(0, 25, 0), (1, 25, 0), (2, 16, 0)]


def test_typed_cells_and_errors(po):
    sch = [{"name": "i", "type": "int32", "path": "0"}, {"name": "t", "type": "timestamp", "path": "1"}, {"name": "d", "type": "date", "path": "2"},
           {"name": "f", "type": "double", "path": "3"}, {"name": "b", "type": "boolean", "path": "4"}, {"name": "u", "type": "uint8", "path": "5"},
           {"name": "s", "type": "utf8", "path": "6"}, {"name": "a", "type": "any", "path": "6"}, {"name": "z", "type": "int64", "path": "-1"}]
    data = (b"12,1373838275,2013-07-15,1.5,true,7,x\n"            # plain
            b"010,2013-07-14 21:44:35,2013-07-15,2,0,255,\" q \"\"q\"\" \"\n"   # leading 0 = octal (ParseInt base 0); quoted text with "" inside
            b"-5.000,2013-07-14T21:44:35.5+03:00,2013-07-15,3e2,T,1,\n"        # trimZeroDecimal; RFC3339 with zone
            b"1,1,2013-07-15,1,1,300,x\n"                      # uint8 range error
            b"1,1,2013-02-30,1,1,3,x\n"                        # bad date
            b"1,1,2013-07-15,1,maybe,3,x\n"                    # bad bool
            b"1,1\n"                                           # missing cells
            b"\n")                                             # empty line -> no cells
    b, errs, lines, cons = po.csv_parse(data, sch)
    assert lines == 8 and b.nrows == 3
    assert list(b.columns[0].values) == [12, 8, -5]
    assert list(b.columns[1].values) == [1373838275, 1373838275, 1373827475] and list(b.columns[1].aux) == [0, 0, 500_000_000]
    assert list(b.columns[3].values) == [1.5, 2.0, 300.0] and list(b.columns[4].values) == [1, 0, 1] and list(b.columns[5].values) == [7, 255, 1]
    assert cells(abi.Batch(3, [b.columns[6]])) == [[b"x"], [b' q "q" '], [b""]]
    assert list(b.columns[7].aux) == [1, 1, 1] and list(b.columns[8].values) == [0, 0, 0]
    assert errs == [(3, 19, 0), (4, 21, 0), (5, 20, 0), (6, 16, 0), (7, 16, 0)]
    # null lists and defaults (reader_csv.go:384-405, change_item_builders.go:87-109)
    b, errs, _, _ = po.csv_parse(b"NULL,NULL,NULL\n5,t,z\n", [{"name": "i", "type": "int32", "path": "0"}, {"name": "b", "type": "boolean", "path": "1"}, {"name": "a", "type": "any", "path": "2"}],
                                 {"null_values": ["NULL"], "strings_can_be_null": True})
    assert list(b.columns[0].values) == [0, 5] and list(b.columns[1].values) == [0, 1] and cells(abi.Batch(2, [b.columns[2]])) == [[b"{}"], [b"z"]] and list(b.columns[2].aux) == [0, 1]


def render_hits_csv(batch, schema, rng):
    """hits-shaped batch -> CSV text the way a producer would write it (quotes around text with delimiters / quotes)."""
    import datetime as dt
    rows = []
    cols = []
    for c, sc in zip(batch.columns, schema):
        if c.type in abi.VAR_TYPES:
            vals = []
            for r in range(batch.nrows):
                s = bytes(c.heap[c.offsets[r]:c.offsets[r + 1]])
                if b"," in s or b'"' in s or rng.random() < 0.1:
                    s = b'"' + s.replace(b'"', b'""') + b'"'
                vals.append(s)
            cols.append(vals)
        elif c.type == abi.TF_TIMESTAMP:
            cols.append([dt.datetime.fromtimestamp(int(v), dt.timezone.utc).strftime("%Y-%m-%d %H:%M:%S").encode() for v in c.values])
        elif c.type == abi.TF_DATE:
            cols.append([dt.datetime.fromtimestamp(int(v), dt.timezone.utc).strftime("%Y-%m-%d").encode() for v in c.values])
        else:
            cols.append([str(int(v)).encode() for v in c.values])
    for r in range(batch.nrows):
        rows.append(b",".join(col[r] for col in cols))
    return b"\n".join(rows) + b"\n"


def _assert_equal(a, b):
    from test_gpu_parity import assert_batches_equal
    assert_batches_equal(a, b)


def _col(batch, c):
    col = batch.columns[c]; out = []
    for r in range(batch.nrows):
        if col.validity is not None and not (col.validity[r >> 3] >> (r & 7)) & 1:
            out.append(None)
        elif col.type in abi.VAR_TYPES:
            out.append(bytes(col.heap[col.offsets[r]:col.offsets[r + 1]]))
        else:
            out.append(col.values[r].item())
    return out


def test_s3_reader_value_rule_cases(po):
    """pkg/providers/s3/reader/registry/csv/reader_csv_test.go: TestParseNullValues (:304-355), TestParseBooleanValue (:394-432) and
    TestParseDateValue case 1 / 4 (:357-392), at the level of the whole reader (a leading key column keeps the tested cell away from the
    reader's first-element quirk). A null value becomes abstract.DefaultValue of the column (change_item_builders.go:88-109)."""
    S2 = lambda t: [{"name": "k", "type": "utf8", "path": "0"}, {"name": "v", "type": t, "path": "1"}]
    nulls = {"strings_can_be_null": True, "quoted_strings_can_be_null": True, "null_values": ["NULL", "NA"]}
    b, e, _, _ = po.csv_parse(b'1,"NULL"\n2,"notnull"\n3,NULL\n4,notnull\n5,NA\n', S2("utf8"), nulls)
    assert _col(b, 1) == [b"", b"notnull", b"", b"notnull", b""] and not e                 # cases 1-4, 6: "" is DefaultValue(utf8)
    b, e, _, _ = po.csv_parse(b'1,"NULL"\n2,NULL\n', S2("utf8"), {"null_values": ["NULL", "NA"]})
    assert _col(b, 1) == [b"NULL", b"NULL"]                                                # case 5: both switches off
    bools = {"strings_can_be_null": True, "null_values": ["NULL", "NA"], "true_values": ["true", "yes", "1"], "false_values": ["false", "no", "0"]}
    b, e, _, _ = po.csv_parse(b"1,NULL\n2,true\n3,false\n4,TRUE\n5,random\n6,yes\n7,no\n", S2("boolean"), bools)
    assert _col(b, 1) == [0, 1, 0, 1, 1, 0] and e == [(4, 20, 0)]        # NULL -> false, lists, strconv.ParseBool("TRUE"); "random" stays a string and fails the cast
    # TestConstructCI (:168-233): a one-element row against a two-column schema (the line "ttrue" reads as the single element "true",
    # see the reader quirk above): included as DefaultValue with IncludeMissingColumns, "missing row element" otherwise
    ci = [{"name": "test-first-column", "type": "boolean", "path": "0"}, {"name": "test-missing-row-column", "type": "utf8", "path": "1"}]
    b, e, _, _ = po.csv_parse(b"ttrue\n", ci, {"include_missing_columns": True})
    assert [_col(b, 0), _col(b, 1)] == [[1], [b""]] and not e
    b, e, _, _ = po.csv_parse(b"ttrue\n", ci)
    assert b.nrows == 0 and e == [(0, 16, 0)]
    b, e, _, _ = po.csv_parse(b"true,this is a test string\n", ci)
    assert [_col(b, 0), _col(b, 1)] == [[1], [b"this is a test string"]] and not e
    b, e, _, _ = po.csv_parse(b"1,2024-03-22\n2,2024/03/22\n", S2("date"))
    assert _col(b, 1) == [1711065600] and [x[0] for x in e] == [1]      # yyyy-mm-dd parses; a text no parser takes stays a string


@pytest.mark.gpu
def test_device_csv_equals_oracle_on_hits(eng, po):
    """BASELINE configs[4] shape: hits-shaped CSV -> parse -> cast -> ClickHouse native block, all on the device."""
    rng = np.random.default_rng(3)
    batch, schema = workload.make_hits_batch(20_000, seed=11)
    schema = [dict(c, path=str(i)) for i, c in enumerate(schema)]
    text = render_hits_csv(batch, schema, rng)
    pid = eng.plan("public", "hits", schema, [], {"type": "clickhouse"})
    got, gerr, consumed = eng.parse_csv(pid, text)
    ref, rerr, lines, rcons = po.csv_parse(text, schema)
    assert consumed == rcons == len(text) and gerr == rerr == [] and got.nrows == ref.nrows == batch.nrows
    _assert_equal(got, ref)
    # the parsed cells are the values the batch was rendered from (round trip): quoting is undone
    names = [c["name"] for c in schema]
    assert np.array_equal(got.columns[names.index("watchid")].values, batch.columns[names.index("watchid")].values)
    assert np.array_equal(got.columns[names.index("eventtime")].values, batch.columns[names.index("eventtime")].values)
    # fused: CSV -> filter_rows -> ClickHouse block + LZ4, vs oracle(parse) -> oracle(push_encode)
    k = workload.counterid_threshold(batch, schema)
    trs = workload.headline_transformers(k)
    pid2 = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
    res, _ = eng.parse_csv(pid2, text, wire_fmt=abi.TF_WIRE_CH_NATIVE)
    want = po.push_encode(ref, po.build_plan("public", "hits", schema, trs), abi.TF_WIRE_CH_NATIVE)
    assert res.rows_out == want.rows_out and res.wire == want.raw
    res_lz, _ = eng.parse_csv(pid2, text, wire_fmt=abi.TF_WIRE_CH_NATIVE_LZ4)
    raw, _ = po.ch_decode_frames(res_lz.wire)
    assert raw == want.raw


@pytest.mark.gpu
def test_device_csv_cases_and_errors(eng, po):
    cases = [
        (b"1, 2, 3\n\t\ta,b,c\n\t\t7,8,9\n", S(3), None),
        (b'a, \\, "c \\" e , f"\n', S(3), None), (b'a, \\, "c \\" e , f"\n', S(4), {"escape": ""}),
        (b'a, b, "the main ""test"" is this", d\n', S(4), None), (b'a, b, "the main ""test"" is this", d\n', S(4), {"double_quote": False}),
        (b"a,b\nc,d", S(2), None), (b'a,"\nx,y\n', S(2), None), (b"abc\n\n\r\nq\n", S(1), {"include_missing_columns": True}),
        (b"h1;h2\n1;\xc2\xa0 spaced \xe3\x80\x80\n", S(2), {"delimiter": ";", "skip_lines": 1}), (b"", S(2), None), (b"no newline", S(1), None),
        (b"a,'it''s'\nb,x\"\"y\nc,'''',''\nd,'x''''\n", S(2), {"quote": "'"}), (b"a,'it''s'\nb,x\"\"y\n", S(2), {"quote": "'", "double_quote": False}),
        (b"k,'it''s',x\"\"y," + b",".join(b"%d" % f for f in range(260)) + b"\n", S(3), {"quote": "'"}),      # 263 fields: the sequential path
        (b'a,x"y\n"\nb\nc,d\n"h",1\nq,r\n', S(2), {"quote": "", "skip_lines": 1}),
    ]
    sch = [{"name": "i", "type": "int32", "path": "0"}, {"name": "t", "type": "timestamp", "path": "1"}, {"name": "d", "type": "date", "path": "2"},
           {"name": "f", "type": "double", "path": "3"}, {"name": "b", "type": "boolean", "path": "4"}, {"name": "u", "type": "uint8", "path": "5"},
           {"name": "s", "type": "utf8", "path": "6"}, {"name": "a", "type": "any", "path": "6"}, {"name": "z", "type": "int64", "path": "-1"},
           {"name": "g", "type": "float", "path": "3"}, {"name": "dt", "type": "datetime", "path": "1"}, {"name": "n", "type": "uint64", "path": "0"}]
    data = (b"12,2013-07-14 21:44:35,2013-07-15,1.5,true,7,x\n010,2013-07-14 21:44:35,2013-07-15,2,0,255,\" q \"\"q\"\" \"\n"
            b"5.000,2013-07-14T21:44:35.5+03:00,2013-07-15,3e2,T,1,\n1,1,2013-07-15,1,1,300,x\n1,2013-07-14 21:44:35,2013-02-30,1,1,3,x\n"
            b"1,2013-07-14 21:44:35,2013-07-15,1,maybe,3,x\n1,1\n\n-3,2013-07-14 21:44:35,2013-07-15,1,1,3,x\n0x1f,2013-07-14 21:44:35,2013-07-15,1e400,1,3,x\n"
            b"99999999999,2013-07-14 21:44:35,2013-07-15,0.1234567890123456789,1,3,x\n1_0,2013-07-14 21:44:35,2013-07-15,nan,1,3,x\n")
    cases.append((data, sch, None))
    cases.append((b"NULL,NULL,NULL\n5,t,z\n'NULL',f,\"NULL\"\n", [{"name": "i", "type": "int32", "path": "0"}, {"name": "b", "type": "boolean", "path": "1"}, {"name": "a", "type": "any", "path": "2"}],
                  {"null_values": ["NULL"], "strings_can_be_null": True}))
    cases.append((b"NULL,x\n'NULL',y\n", [{"name": "s", "type": "utf8", "path": "0"}, {"name": "t", "type": "string", "path": "1"}], {"null_values": ["NULL"], "quoted_strings_can_be_null": True}))
    for text, schema, opts in cases:
        pid = eng.plan("db", "t", schema, [])
        got, gerr, consumed = eng.parse_csv(pid, text, opts)
        ref, rerr, lines, rcons = po.csv_parse(text, schema, opts)
        assert consumed == rcons, text
        assert [(r, c) for r, c, _ in gerr] == [(r, c) for r, c, _ in rerr], (text, gerr, rerr)
        _assert_equal(got, ref)


def test_malformed_row_is_a_row_level_error(po):
    """pkg/providers/s3/reader/registry/csv/data_error_matrix_test.go:113-160 (TestCSVMalformedRow_DataPolicies): `1\\nnot_int\\n` into one int64
    column gives row-level failures (`_unparsed` items under UnparsedPolicyContinue; Fail / Retry turn the same row error into a fatal /
    retriable error of the whole read: the provider's policy, not the parser's). The reference test only asks for > 0 unparsed rows — and in
    fact BOTH rows fail there: without a delimiter splitString takes line[lastDelimPosition+1:] = line[1:] for the only element
    (pkg/csv/reader.go:262), so "1" reads as "" as well. With a second column the first row parses."""
    sch1 = [{"name": "v", "type": "int64", "path": "0"}]
    b, errs, lines, cons = po.csv_parse(b"1\nnot_int\n", sch1)
    assert lines == 2 and b.nrows == 0 and cons == 10 and errs == [(0, 18, 0), (1, 18, 0)]          # TF_ROWERR_CSV_BAD_INT twice
    b, errs, lines, cons = po.csv_parse(b"1,x\nnot_int,y\n", sch1 + [{"name": "s", "type": "utf8", "path": "1"}])
    assert b.nrows == 1 and list(b.columns[0].values) == [1] and errs == [(1, 18, 0)]
    # TestCSVEmptySample: an empty object yields no rows at all (the `_unparsed` item there is the reader's empty-sample marker)
    b, errs, lines, cons = po.csv_parse(b"", sch1)
    assert b.nrows == 0 and not errs and lines == 0 and cons == 0
