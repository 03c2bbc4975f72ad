"""CSV parser: every way the device tokenises a line, and device-resident input.

k_csv_pass1 tokenises a line in one of three ways: a CTA stages 32 lines in shared memory (tiles up to CSV_TILE_BYTES = 28672 bytes,
schemas reading at most CSV_TF = 250 fields, element boundaries in a table of 250 entries); a warp per line reads it from global
memory (longer tiles, wider schemas; a table of CSV_MAXF = 512 boundaries); one thread walks the line sequentially (lines with more
delimiters than the active table holds). The tests here build inputs on both sides of each of those limits and compare the device
with the oracle, the three paths with each other, and device-memory input with host input.

On the CPU, a short restatement of the S3 reader's single-line mode (pkg/csv/reader.go ReadLine / splitString / sanitizeElement,
reader_csv.go's missing-cell rule) written from the Go semantics checks the oracle on a fuzz corpus of utf8 cells."""
import numpy as np
import pytest

from transferia_b200 import abi

# ------------------------------------------------------------------------------------------------ the restatement (CPU)
# unicode.IsSpace: \t \n \v \f \r, space, U+0085, U+00A0 and the White_Space runes above Latin-1 (str.isspace also takes \x1c-\x1f)
GO_SPACE = frozenset([0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F, 0x205F, 0x3000])
RUNE_ERROR = 0xFFFD


def go_decode_rune(b: bytes, i: int):
    """utf8.DecodeRune(b[i:]) -> (rune, width): an invalid or truncated encoding is (U+FFFD, 1), as `for range` sees it."""
    c = b[i]
    if c < 0x80:
        return c, 1
    n = 2 if 0xC2 <= c <= 0xDF else 3 if 0xE0 <= c <= 0xEF else 4 if 0xF0 <= c <= 0xF4 else 0
    if n and i + n <= len(b):
        try:
            return ord(b[i:i + n].decode("utf-8")), n        # strict: no surrogates, no overlong forms, nothing above U+10FFFF
        except UnicodeDecodeError:
            pass
    return RUNE_ERROR, 1


def go_decode_last_rune(b: bytes):
    """utf8.DecodeLastRune: back up to the last rune-start byte (at most 4 bytes), decode from there; it must end at len(b)."""
    end = len(b)
    if b[end - 1] < 0x80:
        return b[end - 1], 1
    start, lim = end - 1, max(0, end - 4)
    start -= 1
    while start >= lim and (b[start] & 0xC0) == 0x80:
        start -= 1
    start = max(start, 0)
    r, w = go_decode_rune(b, start)
    return (r, w) if start + w == end else (RUNE_ERROR, 1)


def go_trim_space(b: bytes) -> bytes:
    i = 0
    while i < len(b):
        r, w = go_decode_rune(b, i)
        if r not in GO_SPACE:
            break
        i += w
    j = len(b)
    while j > i:
        r, w = go_decode_last_rune(b[i:j])
        if r not in GO_SPACE:
            break
        j -= w
    return b[i:j]


class ReadError(Exception):
    def __init__(self, code):
        self.code = code


def go_sanitize(el: bytes, o: dict) -> bytes:
    """sanitizeElement: TrimSpace, unquote, swapToSingleQuotes with DoubleQuoteStr = quote + quote."""
    el = go_trim_space(el)
    q = o["quote"]
    if not q:
        return el
    if len(el) == 1 and el[0] == q:
        raise ReadError(17)                                         # an element of only one quote
    if len(el) >= 2 and el[0] == q and el[-1] == q:
        el = el[1:-1]
    pair = bytes([q, q])
    if not o["double_quote"]:
        if pair in el:
            raise ReadError(abi.TF_ROWERR_CSV_DQ_DISABLED)
        return el
    return el.replace(pair, b'"')


def go_split_string(line: bytes, o: dict):
    """splitString: runes as `for index, char := range line` yields them; the escape skips the next rune inside quotes only."""
    out, prev, inq, last, prev_d, i = [], 0, False, 0, 0, 0
    while i < len(line):
        r, w = go_decode_rune(line, i)
        if o["escape"] and o["escape"] == prev and inq:
            prev = r; i += w
            continue
        if o["quote"] and r == o["quote"]:
            inq = not inq; prev = r; i += w
            continue
        if r == o["delimiter"] and not inq:
            last = i
            out.append(go_sanitize(line[prev_d:last], o))
            prev_d = last + 1
        prev = r; i += w
    out.append(go_sanitize(line[last + 1:], o))        # line[lastDelimPosition+1:]: line[1:] when no delimiter was seen
    return out


def _go_opts(opts):
    opts = opts or {}
    ch = lambda k, d: ord(opts.get(k, d)) if opts.get(k, d) else 0
    return {"delimiter": ch("delimiter", ","), "quote": ch("quote", '"'), "escape": ch("escape", "\\"), "double_quote": opts.get("double_quote", True),
            "include_missing": bool(opts.get("include_missing_columns")), "skip": int(opts.get("skip_lines", 0))}


def go_read_csv(data: bytes, paths, opts=None):
    """The S3 CSV reader over one chunk, utf8 columns at `paths`: (rows of cell bytes, [(data line, code, 0)], lines, consumed)."""
    o = _go_opts(opts)
    rows, errs, pos, ln, consumed = [], [], 0, 0, 0
    while True:
        nl = data.find(b"\n", pos)
        if nl < 0:
            break                                             # an unterminated tail is dropped (reader.go:162-165)
        line = data[pos:nl + 1]; pos = consumed = nl + 1
        k = ln; ln += 1
        if k < o["skip"]:
            continue
        r = k - o["skip"]
        try:
            if not o["quote"] and b'"' in line:
                raise ReadError(abi.TF_ROWERR_CSV_QUOTING_DISABLED)    # readAndDecodeLine: errQuotingDisabled
            cells = [] if line == b"\n" else go_split_string(line, o)
            row = []
            for p in paths:                                   # constructCI: a missing element, or DefaultValue("") with IncludeMissingColumns
                if p >= len(cells) and not o["include_missing"]:
                    raise ReadError(16)
                row.append(cells[p] if p < len(cells) else b"")
        except ReadError as e:
            errs.append((r, e.code, 0))
            continue
        rows.append(row)
    return rows, errs, max(ln - o["skip"], 0), consumed


def cells(batch):
    return [[bytes(c.heap[c.offsets[r]:c.offsets[r + 1]]) for c in batch.columns] for r in range(batch.nrows)]


U = lambda paths: [{"name": f"c{i}", "type": "utf8", "path": str(p)} for i, p in enumerate(paths)]


def test_restatement_pinned_by_reader_tests():
    """The pkg/csv/reader_test.go cases of test_csv.py::test_reader_reference_cases, through the restatement."""
    P = lambda n: list(range(n))
    assert go_read_csv(b"1, 2, 3\n\t\ta,b,c\n\t\t7,8,9\n", P(3))[:3] == ([[b"1", b"2", b"3"], [b"a", b"b", b"c"], [b"7", b"8", b"9"]], [], 3)
    assert go_read_csv(b'a, \\, "c \\" e , f"\n', P(3))[0] == [[b"a", b"\\", b'c \\" e , f']]
    assert go_read_csv(b'a, \\, "c \\" e , f"\n', P(4), {"escape": ""})[0] == [[b"a", b"\\", b'"c \\" e', b'f"']]
    assert go_read_csv(b'a, b, "the main ""test"" is this", d\n', P(4))[0][0][2] == b'the main "test" is this'
    assert go_read_csv(b'a, b, "the main ""test"" is this", d\n', P(4), {"double_quote": False})[:2] == ([], [(0, 24, 0)])
    assert go_read_csv(b"a,b\nc,d", P(2))[0::3] == ([[b"a", b"b"]], 4)
    assert go_read_csv(b'a,"\n', P(2))[:2] == ([], [(0, 17, 0)])
    assert go_read_csv(b"abc\n", P(1))[0] == [[b"bc"]]
    # DoubleQuoteStr follows the quote character; quoting disabled rejects any '"'
    assert go_read_csv(b"a,'it''s'\n", P(2), {"quote": "'"})[0] == [[b"a", b'it"s']]
    assert go_read_csv(b'a,x""y\n', P(2), {"quote": "'"})[0] == [[b"a", b'x""y']]
    assert go_read_csv(b'a,x"y\nb,c\n', P(2), {"quote": ""})[:2] == ([[b"b", b"c"]], [(0, 25, 0)])
    # TrimSpace is unicode.IsSpace, not str.isspace; an invalid byte is one U+FFFD rune
    assert go_trim_space(b"\x1c a \xc2\x85") == b"\x1c a" and go_trim_space(b"\xe2\x80\x80\xc2\xa0x\xe3\x80\x80") == b"x"
    assert go_trim_space(b"x\x85") == b"x\x85" and go_trim_space(b"x\xc2") == b"x\xc2" and go_trim_space(b"x\xe2\xc2\x85 ") == b"x\xe2"


# structural bytes the parser branches on, weighted up; typed cells so that conversions succeed as well as fail
_STRUCT = [b",", b";", b"\t", b" ", b"|", b'"', b"'", b"\\", b"\r", b"\x00", b"\xc2\xa0", b"\xe3\x80\x80", b"\xe2\x80\x8a", b"\xc2\x85", b"\xc2", b"\xff",
           b'""', b"''", b'"""', b"'''", b"\\\\", b"\\\"", b"\\'", b"\x1c"]
_TYPED = [b"12", b"-7", b"0x1f", b"010", b"99999999999", b"1_0", b"true", b"F", b"yes", b"no", b"NULL", b"\\N", b"1373838275", b"2013-07-14 21:44:35",
          b"2013-07-14T21:44:35.5+03:00", b"2013-02-30", b"1.5", b"3e2", b"-0.25", b"1e400", b"nan", b"", b"x", b"abc"]


_FIELD_OK = {3: [b"12", b"-7", b"0x1f", b"010", b" 5 "], 4: [b"true", b"0", b"F", b"yes", b"no"], 5: [b"1373838275", b"2013-07-14 21:44:35", b"2013-07-14T21:44:35.5+03:00"],
             6: [b"1.5", b"3e2", b"-0.25", b"7"]}


def fuzz_text(n, seed, delim=b",", quote=b'"', double_quote=True):
    """n lines of mostly 6..10 cells (typed tokens, or short runs of structural bytes and letters, sometimes quoted or padded), mostly joined
    by `delim`, sometimes by another delimiter; a share end in '\r'; the text may end in an unterminated line. Most lines lose their '"'
    when there is no quote character, and their doubled quotes when double_quote is off, so that not every line is an error row."""
    rng = np.random.default_rng(seed)
    pool = _STRUCT + [bytes([c]) for c in b"abcXYZ019"]
    seps = [b",", b";", b"\t", b" ", b"|"]
    text = []
    for _ in range(n):
        nf = int(rng.integers(6, 11)) if rng.random() < 0.8 else int(rng.integers(0, 6))
        parts = []
        for f in range(nf):
            k = rng.random()
            if f in _FIELD_OK and k < 0.75:        # fields 3-6 mostly hold what MIXED reads there, so that whole rows convert
                c = _FIELD_OK[f][rng.integers(0, len(_FIELD_OK[f]))]
            elif k < 0.45:
                c = _TYPED[rng.integers(0, len(_TYPED))]
            else:
                c = b"".join(pool[int(rng.integers(0, len(pool)))] for _ in range(rng.integers(0, 7)))
            if rng.random() < 0.25 and quote:
                c = quote + c + quote
            if rng.random() < 0.15:
                c = b" " + c + b"\t"
            parts.append(c)
        ln = (delim if rng.random() < 0.85 else seps[int(rng.integers(0, 5))]).join(parts)
        if rng.random() < 0.05:
            ln += b"\r"
        if not quote and rng.random() < 0.85:
            ln = ln.replace(b'"', b"'")
        if quote and not double_quote and rng.random() < 0.85:
            ln = ln.replace(quote * 2, quote)
        text.append(ln.replace(b"\n", b" "))
    return b"\n".join(text) + (b"\n" if rng.random() < 0.5 else b"\ntail,without,newline")


CPU_CONFIGS = [({}, b","), ({"quote": "'"}, b","), ({"delimiter": ";", "quote": "'", "double_quote": False}, b";"), ({"quote": ""}, b","), ({"delimiter": "\t", "quote": "", "escape": ""}, b"\t"),
               ({"delimiter": ";", "escape": ""}, b";"), ({"delimiter": " ", "escape": '"'}, b" "), ({"delimiter": "|", "quote": "'", "escape": "|"}, b"|"),
               ({"double_quote": False, "include_missing_columns": True}, b","), ({"include_missing_columns": True, "skip_lines": 5}, b",")]


@pytest.mark.parametrize("k", range(len(CPU_CONFIGS)))
def test_oracle_equals_restatement_fuzz(po, k):
    """The oracle against the restatement on 3000 fuzz lines per config (utf8 cells): rows, error codes, consumed, lines."""
    opts, delim = CPU_CONFIGS[k]
    text = fuzz_text(3000, 100 + k, delim, opts.get("quote", '"').encode(), opts.get("double_quote", True))
    paths = [0, 1, 2, 0, 5]
    rows, errs, lines, consumed = go_read_csv(text, paths, opts)
    b, e, l2, c2 = po.csv_parse(text, U(paths), opts)
    assert (l2, c2) == (lines, consumed)
    assert e == errs, ([x for x in e if x not in errs][:5], [x for x in errs if x not in e][:5])
    assert cells(b) == rows
    assert len(rows) > 100 and len(errs) >= 10


# ------------------------------------------------------------------------------------------------ device against oracle (GPU)
MIXED = [{"name": "s0", "type": "utf8", "path": "0"}, {"name": "s1", "type": "string", "path": "1"}, {"name": "a2", "type": "any", "path": "2"},
         {"name": "s0b", "type": "utf8", "path": "0"}, {"name": "i3", "type": "int32", "path": "3"}, {"name": "b4", "type": "boolean", "path": "4"},
         {"name": "t5", "type": "timestamp", "path": "5"}, {"name": "d6", "type": "double", "path": "6"}, {"name": "z", "type": "int64", "path": "-1"},
         {"name": "a1", "type": "any", "path": "1"}, {"name": "far", "type": "utf8", "path": "9"}]

GPU_CONFIGS = [({}, b","), ({"delimiter": ";", "quote": "'", "escape": ""}, b";"), ({"delimiter": "\t", "quote": "", "include_missing_columns": True}, b"\t"),
               ({"delimiter": " ", "escape": '"', "include_missing_columns": True}, b" "), ({"delimiter": "|", "quote": "'", "escape": "|", "include_missing_columns": True}, b"|"),
               ({"double_quote": False, "include_missing_columns": True}, b","), ({"quote": "'", "double_quote": False}, b","),
               ({"null_values": ["NULL", "", "\\N"], "strings_can_be_null": True, "true_values": ["yes"], "false_values": ["no"], "include_missing_columns": True}, b","),
               ({"quote": "'", "null_values": ["NULL", "x"], "quoted_strings_can_be_null": True, "include_missing_columns": True, "skip_lines": 7}, b","),
               ({"quote": "", "escape": "", "null_values": ["NULL"], "strings_can_be_null": True, "skip_lines": 2}, b",")]


def dev_vs_oracle(eng, po, text, schema, opts=None):
    from test_gpu_parity import assert_batches_equal
    pid = eng.plan("db", "t", schema, [])
    got, gerr, consumed = eng.parse_csv(pid, text, opts)
    ref, rerr, lines, rcons = po.csv_parse(bytes(text) if not isinstance(text, bytes) else text, schema, opts)
    assert consumed == rcons
    assert [(r, c) for r, c, _ in gerr] == [(r, c) for r, c, _ in rerr], ([x for x in gerr if x not in rerr][:5], [x for x in rerr if x not in gerr][:5])
    assert got.nrows == ref.nrows
    if ref.nrows:         # (an empty batch may leave an `any` column's tags unallocated)
        assert_batches_equal(got, ref)
    return got, gerr


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(GPU_CONFIGS)))
def test_device_csv_fuzz(eng, po, k):
    """Seeded differential fuzz, 20 k lines per config, mixed schema (text / any / a second column on a used path / typed / default /
    a path most lines lack): the whole batch, the error codes and consumed agree with the oracle."""
    opts, delim = GPU_CONFIGS[k]
    text = fuzz_text(20_000, 200 + k, delim, opts.get("quote", '"').encode(), opts.get("double_quote", True))
    schema = MIXED if opts.get("include_missing_columns") else MIXED[:-1]      # without the switch, lines lacking field 9 are all errors
    got, gerr = dev_vs_oracle(eng, po, text, schema, opts)
    assert got.nrows > 500 and len(gerr) > 100


def _line(nd, delim=b",", cell=lambda f: b"%d" % f):
    return delim.join(cell(f) for f in range(nd + 1)) + b"\n"


@pytest.mark.gpu
def test_device_csv_path_boundaries(eng, po):
    """Inputs built to land on a known side of each limit of k_csv_pass1 / the newline index / the offset scan."""
    sch = [{"name": "i", "type": "int32", "path": "0"}, {"name": "s", "type": "utf8", "path": "1"}, {"name": "t", "type": "any", "path": "2"}]
    # a tile of 32 lines of exactly CSV_TILE_BYTES (staged) and one byte more (warp per line); quoted pairs inside
    for total in (28672, 28673):
        body = [b'%d,"p""q",' % r for r in range(32)]
        fill = total - sum(len(x) + 1 for x in body)
        lines = [x + b"x" * (fill // 32 + (1 if r < fill % 32 else 0)) + b"\n" for r, x in enumerate(body)]
        tile = b"".join(lines); assert len(tile) == total
        dev_vs_oracle(eng, po, tile + tile[:200].rsplit(b"\n", 1)[0] + b"\n", sch)
    cell = lambda f: b"'a''b'" if f == 7 else b"%d" % f if 240 <= f < 260 else b""      # short lines: 32 of them stay within one staged tile
    for hi, opts in ((249, {"quote": "'"}), (251, {"quote": "'", "include_missing_columns": True})):
        # paths up to 249: 250 fields read, staged; up to 251: warp per line. Lines with more boundaries than the table holds go sequential.
        wide = [{"name": f"w{p}", "type": "utf8" if p % 2 else "int32", "path": str(p)} for p in range(hi - 3, hi + 1)] + [{"name": "q", "type": "utf8", "path": "7"}]
        text = b"".join(_line(nd, cell=cell) for nd in (249, 250, 251, 252, 600, 0, 248) * 6)
        got, gerr = dev_vs_oracle(eng, po, text, wide, opts)
        assert got.nrows >= 24 and b'a"b' in bytes(got.columns[-1].heap)
    # a schema reading field 250: warp path for every tile; CSV_MAXF = 512 boundaries, then sequential
    w250 = [{"name": "a", "type": "utf8", "path": "250"}, {"name": "b", "type": "int32", "path": "245"}, {"name": "q", "type": "utf8", "path": "7"}]
    text = b"".join(_line(nd, cell=cell) for nd in (512, 513, 1000, 251, 300) * 8)
    got, _ = dev_vs_oracle(eng, po, text, w250, {"quote": "'"})
    assert got.nrows == 40
    # one line over 65535 bytes with a text cell over 64 KiB, among short lines
    big = b"1," + b"\"" + b"y" * 70_000 + b"\"\"z\"" + b",t\n"
    dev_vs_oracle(eng, po, b"0,a,b\n" * 40 + big + b"2,c,d\n" * 40, sch)
    # quote / escape bytes around the slab edges (line offsets 30-33 and 62-65): escape at lane 31 then a quote at lane 0, runs of escapes
    rng = np.random.default_rng(7)
    pieces = [b'"', b"\\", b",", b"a", b"\\\\", b'\\"', b'""']
    edge = []
    for _ in range(3000):
        ln = bytearray(b"k" * 70)
        for at in (int(rng.integers(28, 35)), int(rng.integers(60, 67)), int(rng.integers(0, 70))):
            p = pieces[int(rng.integers(0, len(pieces)))]
            ln[at:at + len(p)] = p
        ln[int(rng.integers(1, 20))] = ord(",")
        edge.append(bytes(ln[:int(rng.integers(40, 70))]))
    edge += [b"a," + b"x" * 28 + b'"\\' + b'"' + b"y" * 30 + b'\\"' + b'",z', b'a,"' + b"\\" * 61 + b'",b', b'a,"' + b"\\" * 62 + b'",b', b'a,' + b'"' * 63 + b",b"]
    text = b"\n".join(edge) + b"\n"
    esch = U([0, 1])
    for opts in ({}, {"escape": '"'}, {"escape": ","}, {"include_missing_columns": True}):
        got, _ = dev_vs_oracle(eng, po, text, esch, opts)
        assert got.nrows > 1000
        dev_vs_oracle(eng, po, text, esch + [{"name": "far", "type": "utf8", "path": "300"}], dict(opts, include_missing_columns=True))     # the same lines, warp per line
    # texts of 8191 / 8192 / 8193 bytes, with a newline as the last byte of the first 8 KiB newline-count block
    for n in (8191, 8192, 8193):
        body = (b"1,ab,c\n" * (8192 // 7))[:8191] + b"\n"
        text = (body + b"3,x,y\n")[:n] if n != 8191 else body[:8190] + b"\n"
        dev_vs_oracle(eng, po, text, sch)
    # 4095 / 4096 / 4097 rows (the offsets scan works in chunks of 4096)
    for n in (4095, 4096, 4097):
        dev_vs_oracle(eng, po, b"".join(b"%d,%s,q\n" % (r, b"v" * (r % 13)) for r in range(n)), sch)
    # skip_lines equal to and larger than the line count
    for skip in (5, 6, 50):
        got, gerr = dev_vs_oracle(eng, po, b"1,a,b\n" * 5 + b"tail", sch, {"skip_lines": skip})
        assert got.nrows == 0 and gerr == []


def outcome(batch, errs, nlines):
    """Per data line: ("err", code) or the bytes of each cell (text, or value + aux)."""
    bad = {r: c for r, c, _ in errs}
    out, k = [], 0
    for ln in range(nlines):
        if ln in bad:
            out.append(("err", bad[ln])); continue
        row = []
        for c in batch.columns:
            if c.type in abi.VAR_TYPES:
                row.append(bytes(c.heap[c.offsets[k]:c.offsets[k + 1]]) + (bytes([c.aux[k]]) if c.aux is not None else b""))
            else:
                w = np.asarray(c.values).itemsize
                row.append(np.asarray(c.values).view(np.uint8)[k * w:(k + 1) * w].tobytes() + (np.asarray(c.aux)[k].tobytes() if c.aux is not None else b""))
        out.append(tuple(row)); k += 1
    assert k == batch.nrows
    return out


@pytest.mark.gpu
def test_device_csv_paths_agree(eng, po):
    """The same random lines through the staged tiles, through tiles pushed onto the warp path by one long neighbour line, and under a
    schema that reads field 300 (warp path everywhere): every shared column byte-identical, the same errors. No oracle involved."""
    opts = {"include_missing_columns": True, "quote": "'", "null_values": ["NULL"], "strings_can_be_null": True}
    lines = fuzz_text(8000, 31, b",", b"'").split(b"\n")[:-1]
    n = len(lines)
    pid_a = eng.plan("db", "t", MIXED, [])
    a, ea, _ = eng.parse_csv(pid_a, b"\n".join(lines) + b"\n", opts)
    want = outcome(a, ea, n)
    long_line = b"L," + b"w" * 30_000
    mixed = []
    for k in range(0, n, 31):
        mixed.append(long_line); mixed.extend(lines[k:k + 31])
    b, eb, _ = eng.parse_csv(pid_a, b"\n".join(mixed) + b"\n", opts)
    got_b = [x for k, x in enumerate(outcome(b, eb, len(mixed))) if k % 32]
    assert got_b == want
    pid_c = eng.plan("db", "t", MIXED + [{"name": "p300", "type": "utf8", "path": "300"}], [])
    c, ec, _ = eng.parse_csv(pid_c, b"\n".join(lines) + b"\n", opts)
    got_c = [x if x[0] == "err" else x[:-1] for x in outcome(c, ec, n)]
    assert got_c == want
    assert a.nrows > 1000 and len(ea) > 100


# ------------------------------------------------------------------------------------------------ device-resident input (GPU)
def _device_copies(text):
    """`text` in HBM at every offset 0..15 from a 256-byte aligned allocation."""
    import torch
    buf = torch.zeros(len(text) + 32, dtype=torch.uint8, device="cuda:0")
    src = torch.frombuffer(bytearray(text), dtype=torch.uint8) if text else torch.zeros(0, dtype=torch.uint8)
    for off in range(16):
        buf.zero_()
        buf[off:off + len(text)].copy_(src)
        yield off, buf[off:off + len(text)]


@pytest.mark.gpu
def test_device_resident_input(eng, po):
    """CSV, JSON lines and Debezium bytes in device memory, at every alignment: the same result as from host memory, byte for byte."""
    from test_gpu_parity import assert_batches_equal
    from test_csv import render_hits_csv
    from transferia_b200 import engine, workload
    # CSV: a hits-shaped text, and a text whose first tile holds typed cells
    batch, hs = workload.make_hits_batch(3000, seed=5)
    hs = [dict(c, path=str(i)) for i, c in enumerate(hs)]
    typed = [{"name": "i", "type": "int32", "path": "0"}, {"name": "t", "type": "timestamp", "path": "1"}, {"name": "f", "type": "double", "path": "2"},
             {"name": "b", "type": "boolean", "path": "3"}, {"name": "s", "type": "utf8", "path": "4"}, {"name": "g", "type": "float", "path": "2"}]
    ttext = b"".join(b'%d,2013-07-14 21:44:%02d,%d.25,%s,"s""%d"\n' % (r, r % 60, r, b"true" if r % 3 else b"0", r) for r in range(100)) + b"x,1,1,1,1\n"
    for text, schema in ((render_hits_csv(batch, hs, np.random.default_rng(3)), hs), (ttext, typed)):
        pid = eng.plan("db", "t", schema, [])
        want, werr, wcons = eng.parse_csv(pid, text)
        assert want.nrows > 90
        for off, t in _device_copies(text):
            got, gerr, cons = eng.parse_csv(pid, t)
            assert (gerr, cons) == (werr, wcons), off
            assert_batches_equal(got, want)
        pid2 = eng.plan("db", "t", schema, [], {"type": "clickhouse"})
        wres, _ = eng.parse_csv(pid2, text, wire_fmt=abi.TF_WIRE_CH_NATIVE)
        for off, t in _device_copies(text):
            res, _ = eng.parse_csv(pid2, t, wire_fmt=abi.TF_WIRE_CH_NATIVE)
            assert res.wire == wres.wire and res.rows_out == wres.rows_out, off
    # JSON lines (test_json_parser's workload shape, several messages)
    text, fields = workload.make_json_lines(3000)
    opts = {"add_rest": True, "add_dedupe_keys": True, "partition": '{"partition":0,"topic":"events"}'}
    cuts = [text.rfind(b"\n", 0, len(text) // 3 * k) + 1 for k in (1, 2)] + [len(text)]
    msgs = [(c, 10 + k, 1_700_000_000, k) for k, c in enumerate(cuts)]
    pid = eng.plan("", "events", engine.json_result_schema(fields, opts), [])
    want, werr, wl = eng.parse_json(pid, text, opts, msgs)
    for off, t in _device_copies(text):
        got, gerr, gl = eng.parse_json(pid, t, opts, msgs)
        assert (gerr, gl) == (werr, wl), off
        assert_batches_equal(got, want)
    # Debezium (test_debezium's message shapes)
    from test_debezium import _shape_msgs
    schema_text, dmsgs = _shape_msgs()
    data = b"".join(dmsgs); ends = np.cumsum([len(x) for x in dmsgs]).tolist()
    pid = eng.plan("public", "t", engine.debezium_table_schema(schema_text), [])
    want, werr, wmeta = eng.parse_debezium(pid, data, ends, schema_text)
    for off, t in _device_copies(data):
        got, gerr, meta = eng.parse_debezium(pid, t, ends, schema_text)
        assert gerr == werr, off
        assert_batches_equal(got, want)
        assert all(np.array_equal(meta[k], wmeta[k]) for k in wmeta), off
