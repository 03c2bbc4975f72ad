"""gzip / zlib output of the batch serializers (TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB, the S3 sink's OutputEncoding).

CPU: the oracle's strict inflater against CPython zlib, its refusals, and the host stream helper that joins several results into
one gzip member / zlib stream. GPU: the device containers decode (strict inflater, CPython, pyarrow) to exactly the text of the
same call without the flag, on the serializer goldens, a hits-shaped batch and crafted texts that aim at the chunk edges, the
match lengths, the block choice and the code-length limit."""
import ctypes
import ctypes.util
import gzip
import json
import os
import random
import struct
import zlib

import pytest

from transferia_b200 import abi

SER_JSON, SER_CSV, F_NL, F_AAS = abi.TF_WIRE_SER_JSON, abi.TF_WIRE_SER_CSV, abi.TF_WIRE_F_CLOSING_NEWLINE, abi.TF_WIRE_F_ANY_AS_STRING
GZ, ZL = abi.TF_WIRE_F_GZIP, abi.TF_WIRE_F_ZLIB
CHUNK = 16384                      # the engine's chunk size (include/tfgpu.h)
GZIP_HDR, ZLIB_HDR = bytes.fromhex("1f8b08000000000000ff"), bytes.fromhex("789c")


def _wrap(body: bytes, text: bytes, container: int) -> bytes:
    """A raw DEFLATE body (sync-flushed) in the engine's container layout."""
    if container == GZ:
        return GZIP_HDR + body + b"\x03\x00" + struct.pack("<II", zlib.crc32(text), len(text) & 0xffffffff)
    return ZLIB_HDR + body + b"\x03\x00" + struct.pack(">I", zlib.adler32(text))


def _sync_body(text: bytes, level: int = 6) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    return (c.compress(text) + c.flush(zlib.Z_SYNC_FLUSH)) if text else b""


def _libz():
    path = ctypes.util.find_library("z") or "libz.so.1"
    L = ctypes.CDLL(path)
    for fn in ("crc32_combine64", "adler32_combine64"):
        getattr(L, fn).restype = ctypes.c_ulong
        getattr(L, fn).argtypes = [ctypes.c_ulong, ctypes.c_ulong, ctypes.c_int64]
    return L


# ------------------------------------------------------------------------------------------------------------------- CPU

@pytest.fixture(scope="module")
def inf():
    """The oracle's strict inflater (oracle/inflate.hpp)."""
    from oracle import pyinflate
    pyinflate.build()
    return pyinflate


def test_strict_inflater_agrees_with_zlib(inf):
    """Every level 0-9, raw / zlib / gzip wbits, texts of 0..300 bytes (text and runs), with and without sync flushes."""
    rng = random.Random(5)
    conts = ((-15, inf.INFLATE_RAW), (15, inf.INFLATE_ZLIB), (31, inf.INFLATE_GZIP))
    for size in range(0, 301):
        kind = size % 3
        text = bytes(rng.randrange(256) for _ in range(size)) if kind == 0 else (b"abcabcabd" * 40)[:size] if kind == 1 else \
            bytes(rng.choice(b"eeeetaoin \n") for _ in range(size))
        for level in range(10):
            for wbits, cont in conts:
                c = zlib.compressobj(level, zlib.DEFLATED, wbits)
                if size % 2:        # sync flushes inside the stream
                    data = c.compress(text[: size // 2]) + c.flush(zlib.Z_SYNC_FLUSH) + c.compress(text[size // 2:]) + c.flush()
                else:
                    data = c.compress(text) + c.flush()
                got, err, _ = inf.inflate(data, cont)
                assert err is None and got == text, (size, level, wbits, err)


def test_strict_inflater_refuses_broken_streams(inf):
    text = b"hello, hello, hello world\n" * 20
    good = _wrap(_sync_body(text), text, GZ)
    assert inf.inflate(good, inf.INFLATE_GZIP, CHUNK)[0] == text
    # over-subscribed code: dynamic block whose code-length code gives three symbols one bit each
    # BFINAL=1, BTYPE=10 (dynamic), HLIT=0, HDIST=0, HCLEN=0 (4 code-length codes: 16, 17, 18, 0 each 1 bit)
    v, n = 0, 0
    for val, nb in ((1, 1), (2, 2), (0, 5), (0, 5), (0, 4), (1, 3), (1, 3), (1, 3), (1, 3)):
        v |= val << n; n += nb
    over = v.to_bytes((n + 7) // 8, "little") + b"\x00" * 4
    assert inf.inflate(over, inf.INFLATE_RAW)[1] == "code-length code: over-subscribed code"
    # distance too far back: fixed block, literal 'a', then length 3 distance 2
    v, n = 0, 0
    def put(val, nb, rev=False):
        nonlocal v, n
        if rev:
            val = int(format(val, "0%db" % nb)[::-1], 2)
        v |= val << n; n += nb
    put(1, 1); put(1, 2); put(0x30 + ord("a"), 8, True); put(1, 7, True); put(1, 5, True); put(0, 7, True)
    far = v.to_bytes((n + 7) // 8, "little")
    assert inf.inflate(far, inf.INFLATE_RAW)[1] == "distance too far back"
    # bad NLEN
    assert inf.inflate(b"\x01\x05\x00\xfa\xfe" + b"abcde", inf.INFLATE_RAW)[1] == "stored LEN / NLEN disagree"
    assert inf.inflate(b"\x01\x05\x00\xfa\xff" + b"abcde", inf.INFLATE_RAW)[0] == b"abcde"
    # missing final block, trailing byte, wrong CRC / ISIZE / Adler
    body = _sync_body(text)
    assert inf.inflate(GZIP_HDR + body + struct.pack("<II", zlib.crc32(text), len(text)), inf.INFLATE_GZIP)[0] is None
    assert inf.inflate(good + b"\x00", inf.INFLATE_GZIP)[1] == "bytes behind the trailer"
    assert inf.inflate(GZIP_HDR + body + b"\x03\x00" + struct.pack("<II", zlib.crc32(text) ^ 1, len(text)), inf.INFLATE_GZIP)[1] == "CRC-32 mismatch"
    assert inf.inflate(GZIP_HDR + body + b"\x03\x00" + struct.pack("<II", zlib.crc32(text), len(text) + 1), inf.INFLATE_GZIP)[1] == "ISIZE mismatch"
    zgood = _wrap(body, text, ZL)
    assert inf.inflate(zgood, inf.INFLATE_ZLIB, CHUNK)[0] == text
    assert inf.inflate(zgood[:-1] + bytes([zgood[-1] ^ 1]), inf.INFLATE_ZLIB)[1] == "Adler-32 mismatch"
    # the layout promises: exact header, the final block empty behind a marker, no distance before its chunk, markers at chunk ends
    assert inf.inflate(gzip.compress(text), inf.INFLATE_GZIP)[0] == text
    assert inf.inflate(gzip.compress(text), inf.INFLATE_GZIP, CHUNK)[1].startswith("gzip header is not")
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    unflushed = c.compress(text) + c.flush()          # data in the final block
    assert "layout" in inf.inflate(GZIP_HDR + unflushed + struct.pack("<II", zlib.crc32(text), len(text)), inf.INFLATE_GZIP, CHUNK)[1]
    two = text[:100] * 2          # one compressor across a marker at 100 bytes: the second half refers back into the first
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    across = c.compress(two[:100]) + c.flush(zlib.Z_SYNC_FLUSH) + c.compress(two[100:]) + c.flush(zlib.Z_SYNC_FLUSH)
    assert inf.inflate(_wrap(across, two, GZ), inf.INFLATE_GZIP)[0] == two
    assert inf.inflate(_wrap(across, two, GZ), inf.INFLATE_GZIP, 100)[1] == "layout: a distance reaches before its chunk"
    assert inf.inflate(_wrap(_sync_body(two), two, GZ), inf.INFLATE_GZIP, 100)[1] == "layout: a chunk runs past its size without a sync-flush marker"
    pieces = _sync_body(two[:100], 0) + _sync_body(two[100:], 0)
    assert inf.inflate(_wrap(pieces, two, GZ), inf.INFLATE_GZIP, 100)[0] == two
    assert inf.inflate(_wrap(pieces, two, GZ), inf.INFLATE_GZIP, 150)[1] == "layout: a sync-flush marker not at a chunk end"


def test_stream_helper_joins_results(inf):
    """Bodies of zlib.compressobj(wbits=-15) + Z_SYNC_FLUSH in the engine's layout join into one member / stream that gzip, zlib and
    the strict inflater decode to the concatenation, empty pieces included; framing that does not match is refused."""
    from transferia_b200 import engine
    rng = random.Random(3)
    pieces = [b"", b"a,b\n" * 1000, bytes(rng.randrange(256) for _ in range(5000)), b"", b"x\n", json.dumps({"k": list(range(300))}).encode()]
    for cont, dec in ((GZ, gzip.decompress), (ZL, zlib.decompress)):
        s = engine.DeflateStream(cont)
        out = b"".join(s.append(_wrap(_sync_body(p), p, cont), len(p)) for p in pieces) + s.close()
        want = b"".join(pieces)
        assert dec(out) == want
        assert inf.inflate(out, inf.INFLATE_GZIP if cont == GZ else inf.INFLATE_ZLIB)[0] == want
        assert out.startswith(GZIP_HDR if cont == GZ else ZLIB_HDR)
        # nothing appended: an empty member / stream
        e = engine.DeflateStream(cont)
        assert dec(e.close()) == b""
        # refusals: the other container, a truncated result, a wrong final block, an ISIZE that is not raw_len, a body without its marker
        p = pieces[1]; good = _wrap(_sync_body(p), p, cont)
        other = _wrap(_sync_body(p), p, ZL if cont == GZ else GZ)
        r = engine.DeflateStream(cont)
        for bad, raw_len in ((other, len(p)), (good[:-1], len(p)), (good[:len(good) - 6 if cont == ZL else len(good) - 10] + b"\x01\x00" + good[-4 if cont == ZL else -8:], len(p)),
                             (_wrap(_sync_body(p)[:-5], p, cont), len(p)), (good[:5], len(p))):
            with pytest.raises(engine.EngineError):
                r.append(bad, raw_len)
        if cont == GZ:
            with pytest.raises(engine.EngineError):
                r.append(good, len(p) + 1)
        assert dec(r.append(good, len(p)) + r.close()) == p      # a refusal leaves the stream as it was
    with pytest.raises(engine.EngineError):
        engine.DeflateStream(GZ | ZL)


def test_stream_helper_combines_like_libz():
    """The trailer's CRC-32 / Adler-32 are libz's crc32_combine64 / adler32_combine64 of the pieces' values, lengths above 2^32 included."""
    from transferia_b200 import engine
    Z = _libz()
    rng = random.Random(11)
    body = _sync_body(b"q")        # any sync-flushed body: only the trailers are combined here
    for _ in range(40):
        a, b = rng.getrandbits(32), rng.getrandbits(32)
        la, lb = rng.choice([1, 7, 65521, 1 << 31, (1 << 32) + 5, (1 << 40) + 3, rng.getrandbits(45)]), rng.choice([1, 65520, (1 << 32) - 1, 1 << 33, rng.getrandbits(50)])
        s = engine.DeflateStream(GZ)
        s.append(GZIP_HDR + body + b"\x03\x00" + struct.pack("<II", a, la & 0xffffffff), la)
        s.append(GZIP_HDR + body + b"\x03\x00" + struct.pack("<II", b, lb & 0xffffffff), lb)
        crc, isize = struct.unpack("<II", s.close()[-8:])
        assert crc == Z.crc32_combine64(Z.crc32_combine64(0, a, la), b, lb) and isize == (la + lb) & 0xffffffff
        a, b = rng.randrange(65521) | rng.randrange(65521) << 16, rng.randrange(65521) | rng.randrange(65521) << 16
        s = engine.DeflateStream(ZL)
        s.append(ZLIB_HDR + body + b"\x03\x00" + struct.pack(">I", a), la)
        s.append(ZLIB_HDR + body + b"\x03\x00" + struct.pack(">I", b), lb)
        (ad,) = struct.unpack(">I", s.close()[-4:])
        assert ad == Z.adler32_combine64(Z.adler32_combine64(1, a, la), b, lb)


# ------------------------------------------------------------------------------------------------------------------- GPU

def _check(inf, res, plain, cont):
    """The container decodes through the strict inflater (with the layout checks), CPython and pyarrow to the plain call's text."""
    got, err, info = inf.inflate(res.wire, inf.INFLATE_GZIP if cont == GZ else inf.INFLATE_ZLIB, CHUNK)
    assert err is None, err
    assert got == plain.wire
    assert (gzip.decompress(res.wire) if cont == GZ else zlib.decompress(res.wire)) == plain.wire
    if cont == GZ:          # pyarrow's gzip codec (it has no zlib-container codec)
        import pyarrow as pa
        with pa.CompressedInputStream(pa.BufferReader(res.wire), "gzip") as f:
            assert f.read() == plain.wire
    assert res.raw_len == plain.raw_len == len(plain.wire)
    assert res.rows_in == plain.rows_in and res.rows_out == plain.rows_out and res.errors == plain.errors
    assert getattr(res, "row_sizes", None) == getattr(plain, "row_sizes", None)
    assert info["markers"] == (len(plain.wire) + CHUNK - 1) // CHUNK
    return info


def _bound(text_len, cont):
    return text_len + 10 * ((text_len + CHUNK - 1) // CHUNK) + (10 + 2 + 8 if cont == GZ else 2 + 2 + 4)


def _golden_cases():
    G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "serializer_goldens.json"), encoding="utf-8"))
    import importlib.util
    spec = importlib.util.spec_from_file_location("_ser", os.path.join(os.path.dirname(__file__), "test_serializers.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return [(c["schema"], m.case_batch(c)) for c in G["cases"]]


FLAGS = (0, F_NL, F_AAS)


@pytest.mark.gpu
def test_device_parity(eng, inf):
    """Serializer goldens and a hits-shaped batch (after filter_rows): SER_JSON / SER_CSV x GZIP / ZLIB x {-, CLOSING_NEWLINE, ANY_AS_STRING}."""
    from transferia_b200 import workload
    cases = _golden_cases()
    batch, schema = workload.make_hits_batch(60000, seed=4)
    k = workload.counterid_threshold(batch, schema)
    cases.append((schema, batch, workload.headline_transformers(k)))
    for case in cases:
        schema, b = case[0], case[1]
        trs = case[2] if len(case) > 2 else []
        pid = eng.plan("s", "t", schema, trs)
        for base in (SER_JSON, SER_CSV):
            for fl in FLAGS:
                if base == SER_CSV and fl:
                    continue
                plain = eng.push_encode(pid, b, base | fl)
                for cont in (GZ, ZL):
                    res = eng.push_encode(pid, b, base | fl | cont)
                    _check(inf, res, plain, cont)
                    assert len(res.wire) <= _bound(len(plain.wire), cont)
                    if len(case) > 2:        # the two-phase path of a filtering plan
                        _check(inf, eng.push_encode(pid, b, base | fl | cont, selective=0), plain, cont)


@pytest.mark.gpu
def test_device_parity_parsers(eng, inf):
    """parse_csv, parse_json and parse_debezium with a compressed serializer format == the same call without the flag."""
    from transferia_b200 import engine, workload
    text, fields = workload.make_json_lines(20000)
    opts = {"add_rest": True, "add_dedupe_keys": True, "partition": '{"partition":0,"topic":"events"}'}
    jschema = engine.json_result_schema(fields, opts)
    pid = eng.plan("", "events", jschema, [])
    for base in (SER_JSON, SER_CSV):
        plain = eng.parse_json(pid, text, opts, None, wire_fmt=base)
        for cont in (GZ, ZL):
            _check(inf, eng.parse_json(pid, text, opts, None, wire_fmt=base | cont), plain, cont)
    data, ends, schema_text, table = workload.make_debezium_messages(5000)
    dschema = engine.debezium_table_schema(schema_text)
    pid = eng.plan(table[0], table[1], dschema, workload.debezium_transformers())
    for base in (SER_JSON, SER_CSV):
        plain, _ = eng.parse_debezium(pid, data, ends, schema_text, schema_registry=True, schema_id=7, wire_fmt=base)
        for cont in (GZ, ZL):
            res, _ = eng.parse_debezium(pid, data, ends, schema_text, schema_registry=True, schema_id=7, wire_fmt=base | cont)
            _check(inf, res, plain, cont)
    cschema = [{"name": "a", "type": "int64", "path": "0"}, {"name": "b", "type": "utf8", "path": "1"}, {"name": "c", "type": "double", "path": "2"}]
    rng = random.Random(2)
    ctext = "".join(f"{rng.randrange(-10**9, 10**9)},w{rng.randrange(10**6)} x,{rng.random() * 1e3:.3f}\n" for _ in range(30000)).encode()
    pid = eng.plan("", "c", cschema, [{"filter_rows": {"filter": "a > 0"}}])
    for base in (SER_JSON, SER_CSV):
        plain, _ = eng.parse_csv(pid, ctext, wire_fmt=base)
        for cont in (GZ, ZL):
            res, _ = eng.parse_csv(pid, ctext, wire_fmt=base | cont)
            _check(inf, res, plain, cont)


def _text_push(eng, pid, text, fmt):
    """One utf8 column through SER_CSV writes each value + '\\n': the text is controlled byte for byte (no , \" \\r \\n, no leading space)."""
    vals = text.split(b"\n")
    assert vals[-1] == b"" and all(v and v[:1] not in (b" ", b"\xc2") and not (set(v) & set(b',"\r\n')) and v != b"\\." for v in vals[:-1])
    b = abi.Batch(len(vals) - 1, [abi.strings_to_column(abi.TF_UTF8, vals[:-1])])
    return eng.push_encode(pid, b, fmt)


def _lines(body: bytes, width: int = 60) -> bytes:
    """body cut into values of `width` bytes, each followed by '\\n'."""
    return b"".join(body[i:i + width] + b"\n" for i in range(0, len(body), width))


@pytest.mark.gpu
def test_device_crafted_texts(eng, inf):
    pid = eng.plan("s", "t", [{"name": "v", "type": "utf8"}], [])
    rng = random.Random(17)
    letters = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"

    def rand_text(n):        # letters + '\n' every 60 bytes: few repeats of 4 bytes
        return _lines(bytes(rng.choice(letters) for _ in range(n * 60 // 61 + 1)))[:n - 1] + b"\n" if n > 1 else b""

    def run(text, conts=(GZ, ZL)):
        plain = _text_push(eng, pid, text, SER_CSV)
        assert plain.wire == text
        infos = []
        for cont in conts:
            res = _text_push(eng, pid, text, SER_CSV | cont)
            infos.append(_check(inf, res, plain, cont))
            assert len(res.wire) <= _bound(len(text), cont)
            infos[-1]["size"] = len(res.wire)
        return infos

    # 0 rows, the smallest texts, fixed Huffman for a short chunk
    for cont in (GZ, ZL):
        res = eng.push_encode(pid, abi.Batch(0, [abi.strings_to_column(abi.TF_UTF8, [])]), SER_CSV | cont)
        assert inf.inflate(res.wire, inf.INFLATE_GZIP if cont == GZ else inf.INFLATE_ZLIB, CHUNK)[0] == b""
        assert res.wire == (GZIP_HDR + b"\x03\x00" + bytes(8) if cont == GZ else ZLIB_HDR + b"\x03\x00" + b"\x00\x00\x00\x01")
    info = run(b"a\n")[0]
    assert info["fixed"] == 2 and info["dynamic"] == 0 and info["stored"] == 0          # the chunk's fixed block + the final block
    run(b"ab\nab\n")
    # chunk size - 1, + 0, + 1, several chunks, more than 1000 chunks
    for n in (CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5, 1001 * CHUNK + 7):
        run(rand_text(n))
    # 3-byte repeats only (too short for a match): every 4-gram of the body is unique
    db = bytearray(); seen = set()
    while len(db) < 3 * CHUNK:
        c = rng.choice(b"abcdefgh")
        if len(db) >= 3 and bytes(db[-3:]) + bytes([c]) in seen:
            c = rng.choice(letters)
        db.append(c)
        if len(db) >= 4:
            seen.add(bytes(db[-4:]))
    run(_lines(bytes(db), 2000))
    # matches of 4, 258 and 259 bytes at distances up to the chunk edge
    for mlen in (4, 258, 259):
        for dist in (1000, CHUNK // 2, CHUNK - 2 * mlen - 100):
            body = bytearray(bytes(rng.choice(letters) for _ in range(2 * CHUNK)))
            seg = bytes(rng.choice(b"#$%&()*+-./") for _ in range(mlen))
            for base in (10, CHUNK + 30):
                body[base:base + mlen] = seg; body[base + dist:base + dist + mlen] = seg
            run(bytes(body) + b"\n")
    # random bytes (every value but \r \n: the CSV writer quotes the values with , or "): incompressible, so stored blocks, and no
    # more than the stored overhead
    vals = [bytes(rng.choice([x for x in range(256) if x not in (10, 13)]) for _ in range(4000)) for _ in range(21)]
    b = abi.Batch(len(vals), [abi.strings_to_column(abi.TF_UTF8, vals)])
    plain = eng.push_encode(pid, b, SER_CSV)
    for cont in (GZ, ZL):
        res = eng.push_encode(pid, b, SER_CSV | cont)
        info = _check(inf, res, plain, cont)
        assert info["stored"] >= 5 and info["dynamic"] == 0 and len(res.wire) <= _bound(len(plain.wire), cont)
    # runs: "abc\n" repeated. The greedy parse codes every chunk as 4 literals + 63 matches of 258 + one of 126 (distance 4), which
    # fixed Huffman alone codes in 3 + 4 * 8 + 63 * (8 + 5) + (8 + 4 + 5) + 7 = 878 bits: with the marker at most 115 bytes a chunk.
    text = b"abc\n" * (8 * CHUNK // 4)
    for info, cont in zip(run(text), (GZ, ZL)):
        assert info["size"] <= (10 + 2 + 8 if cont == GZ else 8) + 8 * 115, info
    # skewed frequencies: 156 common bytes about 95 times each (random order: next to no repeats of 4 bytes, so they stay literals) and
    # a tail of 14 bytes with Fibonacci counts 1, 1, 2, .. 377. Unlimited, that literal histogram needs a 13-bit code; the limit is
    # not reached (a text that needs more than 15 bits from literals alone repeats its frequent bytes, and matches absorb them)
    common = [x for x in range(0x21, 0x7f) if x not in b',"'] + list(range(0x80, 0xc0))
    fib = [1, 1]
    while len(fib) < 14:
        fib.append(fib[-1] + fib[-2])
    pool = bytearray(bytes(common) * 95)
    for k, c in enumerate(range(0xc3, 0xc3 + 14)):
        pool += bytes([c]) * fib[k]
    rng.shuffle(pool)
    infos = run(_lines(bytes(pool), 200))
    assert all(i["dynamic"] == 1 and i["max_len"] >= 13 for i in infos), infos
    # stale bytes: a large push, then a small one on the same engine
    run(rand_text(4 * CHUNK + 99))
    run(b"zz\nyy\n")


@pytest.mark.gpu
def test_device_pushes_joined_by_the_stream_helper(eng, inf):
    from transferia_b200 import engine, workload
    _, schema = workload.make_hits_batch(10, seed=8)
    pid = eng.plan("s", "t", schema, [])
    texts, outs = [], {GZ: [], ZL: []}
    for seed in (1, 2, 3):
        b, _ = workload.make_hits_batch(3000 * seed, seed=seed)
        texts.append(eng.push_encode(pid, b, SER_JSON | F_NL).wire)
        for cont in (GZ, ZL):
            r = eng.push_encode(pid, b, SER_JSON | F_NL | cont)
            outs[cont].append((r.wire, r.raw_len))
    for cont, dec in ((GZ, gzip.decompress), (ZL, zlib.decompress)):
        s = engine.DeflateStream(cont)
        joined = b"".join(s.append(w, n) for w, n in outs[cont]) + s.close()
        assert dec(joined) == b"".join(texts)
        assert inf.inflate(joined, inf.INFLATE_GZIP if cont == GZ else inf.INFLATE_ZLIB)[0] == b"".join(texts)


@pytest.mark.gpu
def test_device_refusals(eng):
    from transferia_b200 import engine, workload
    batch, schema = workload.make_hits_batch(100)
    pid = eng.plan("s", "t", schema, [], {"type": "clickhouse"})
    for fmt in (SER_JSON | GZ | ZL, SER_CSV | GZ | ZL, abi.TF_WIRE_CH_NATIVE | GZ, abi.TF_WIRE_CH_NATIVE_LZ4 | ZL, abi.TF_WIRE_CH_JSONEACHROW | GZ):
        with pytest.raises(engine.EngineError) as ei:
            eng.push_encode(pid, batch, fmt)
        assert ei.value.rc == -2 and "wire format not implemented" in str(ei.value)


@pytest.mark.gpu
def test_sink_push_delivers_the_container(eng, inf):
    from transferia_b200 import rows, sink, workload
    batch, schema = workload.make_hits_batch(2000, seed=6)
    items = rows.items_from_batch(batch)
    plain = eng.push_encode(eng.plan("public", "hits", schema, []), batch, SER_JSON)
    s = sink.Sink(eng, wire_fmt=SER_JSON | GZ)
    s.push(rows.RowsImage(items, [("public", "hits", schema)]))
    ev = [e for e in s.events if e["type"] == sink.EV_ROWS]
    assert len(ev) == 1 and gzip.decompress(ev[0]["wire"]) == plain.wire and ev[0]["raw_len"] == len(plain.wire)
    assert inf.inflate(ev[0]["wire"], inf.INFLATE_GZIP, CHUNK)[0] == plain.wire
    s.close()
