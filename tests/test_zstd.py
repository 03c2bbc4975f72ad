"""zstd of the ClickHouse JSONEachRow text on the device (TF_WIRE_F_ZSTD, include/tfgpu.h).

CPU: the oracle's strict decoder (oracle/zstd_dec.hpp, written from RFC 8878) against libzstd on frames libzstd made, one hand-built
bad frame per refusal rule, and the host helper that puts the INSERT line in front of a device frame (tfgpu_zstd_prefix).
GPU: every entry point that takes TF_WIRE_CH_JSONEACHROW gives, with the flag, one frame in the engine's layout that decodes (oracle
with the layout checks, libzstd, pyarrow) to exactly the bytes of the same call without it; crafted texts at the encoder's edges;
ratio floors that fail without the entropy stages; refusals of the flag where it does not apply."""
import ctypes as C
import random

import pytest

from transferia_b200 import abi

CHUNK = 16384
JER, ZSTD = abi.TF_WIRE_CH_JSONEACHROW, abi.TF_WIRE_F_ZSTD
HDR = 14


@pytest.fixture(scope="module")
def zd():
    from oracle import pyzstd_dec
    pyzstd_dec.build()
    return pyzstd_dec


class _Lib:
    def __init__(self):
        L = C.CDLL("libzstd.so.1")
        L.ZSTD_createCCtx.restype = C.c_void_p
        L.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        L.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]; L.ZSTD_CCtx_setParameter.restype = C.c_size_t
        L.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]; L.ZSTD_compress2.restype = C.c_size_t
        L.ZSTD_compressBound.argtypes = [C.c_size_t]; L.ZSTD_compressBound.restype = C.c_size_t
        L.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]; L.ZSTD_decompress.restype = C.c_size_t
        L.ZSTD_isError.argtypes = [C.c_size_t]; L.ZSTD_isError.restype = C.c_uint
        self.L = L

    def compress(self, data, level, checksum=False, window_log=0):
        L = self.L; cx = L.ZSTD_createCCtx()
        try:
            L.ZSTD_CCtx_setParameter(cx, 100, level); L.ZSTD_CCtx_setParameter(cx, 201, int(checksum))
            if window_log:
                L.ZSTD_CCtx_setParameter(cx, 101, window_log)
            cap = L.ZSTD_compressBound(len(data)); out = C.create_string_buffer(cap)
            n = L.ZSTD_compress2(cx, out, cap, data, len(data))
            assert not L.ZSTD_isError(n)
            return out.raw[:n]
        finally:
            L.ZSTD_freeCCtx(cx)

    def decompress(self, frame, n):
        out = C.create_string_buffer(max(1, n))
        got = self.L.ZSTD_decompress(out, n, frame, len(frame))
        assert not self.L.ZSTD_isError(got), "libzstd refused the frame"
        return out.raw[:got]


@pytest.fixture(scope="module")
def lz():
    return _Lib()


def _texts(rng):
    words = [b"alpha", b"beta", b"\xd0\xbf\xd1\x80\xd0\xb8", b"gamma", b"0123", b'{"k":', b"\n"]
    text = b"".join(rng.choice(words) + bytes([rng.randrange(32, 127)]) for _ in range(60000))
    return {"text": text, "random": bytes(rng.randrange(256) for _ in range(150000)),
            "runs": b"".join(bytes([rng.randrange(256)]) * rng.randrange(1, 3000) for _ in range(200)), "one run": b"\x07" * 300000}


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_strict_decoder_agrees_with_libzstd(zd, lz):
    """Frames libzstd made at levels -5..19, with and without its checksum, decode to their content; small sizes on every level."""
    rng = random.Random(3)
    big = _texts(rng)
    seen = {}
    for level in range(-5, 20):
        for cs in (False, True):
            for name, data in big.items():
                f = lz.compress(data, level, cs)
                out, err, info = zd.decode(f)
                assert err is None and out == data, (level, cs, name, err)
                for k, v in info.items():
                    seen[k] = seen.get(k, 0) + v
            for n in range(0, 301, 1 if level in (-5, 1, 19) else 37):
                data = bytes(rng.choice(b"abcab\x80\xff") for _ in range(n))
                out, err, _ = zd.decode(lz.compress(data, level, cs))
                assert err is None and out == data, (level, cs, n, err)
    # windowed frames with several blocks (the small window keeps them apart), besides single-segment ones
    for name, data in big.items():
        out, err, _ = zd.decode(lz.compress(data, 3, True, window_log=10))
        assert err is None and out == data, (name, err)
    # the forms the decoder must know all occurred
    for k in ("raw", "rle", "compressed", "huf_literals", "fse_weights", "fse_tables", "predefined_tables", "rle_tables"):
        assert seen[k] > 0, (k, seen)


class _Bits:
    """Forward LSB-first bit writer; close() adds the end marker of a backward-read stream."""
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, v, n):
        self.v |= v << self.n; self.n += n

    def close(self, marker=True):
        if marker:
            self.put(1, 1)
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _hdr(content, wd=0x28, fhd=0xC0):
    return bytes([0x28, 0xB5, 0x2F, 0xFD, fhd, wd]) + content.to_bytes(8, "little")


def _blk(body, btype, last, size=None):
    h = (last & 1) | (btype << 1) | ((len(body) if size is None else size) << 3)
    return h.to_bytes(3, "little") + body


def _raw_lits(lits):
    assert len(lits) < 32
    return bytes([len(lits) << 3]) + lits


def _one_seq(ll, ml, ofv, extra_bits=0, marker=True):
    """Sequences section of one sequence, all three tables in RLE_Mode (no state bits): LL / OF / ML codes, then the extra bits."""
    llc = ll if ll < 16 else None
    assert llc is not None and 3 <= ml <= 34
    ofc = ofv.bit_length() - 1
    b = _Bits()
    b.put(0, 0)                         # LL extra (code < 16: none)
    b.put(0, 0)                         # ML extra (code < 32: none)
    b.put(ofv - (1 << ofc), ofc)
    b.put(0, extra_bits)
    return bytes([1, (1 << 6) | (1 << 4) | (1 << 2), llc, ofc, ml - 3]) + b.close(marker)


def test_strict_decoder_refusals(zd, lz):
    rng = random.Random(9)
    data = bytes(rng.randrange(97, 100) for _ in range(5000))
    good = lz.compress(data, 3, True)
    assert zd.decode(good)[0] == data

    def refused(frame, what):
        out, err, _ = zd.decode(frame)
        assert out is None and what in err, (what, err)

    refused(good[:4] + bytes([good[4] | 8]) + good[5:], "reserved bit")
    refused(good[:-1] + bytes([good[-1] ^ 1]), "checksum")
    refused(good + b"\x00", "trailing bytes")
    lits = b"abcdefgh"
    seq = _one_seq(len(lits), 4, 5 + 3)         # copies "defg" from 5 back
    ok = _hdr(12) + _blk(_raw_lits(lits) + seq, 2, 1)
    assert zd.decode(ok)[0] == b"abcdefghdefg"
    refused(_hdr(13) + ok[HDR:], "Frame_Content_Size")
    refused(_hdr(12) + _blk(b"", 3, 1), "reserved block type")
    refused(_hdr(1025, wd=0x00) + _blk(bytes(1025), 0, 1), "Block_Maximum_Size")        # 1 KiB window: 1 KiB blocks
    refused(_hdr(12) + _blk(_raw_lits(lits) + _one_seq(8, 4, 9 + 3), 2, 1), "before the content start")
    # an offset past a 1 KiB window, in a block that stays within it
    far = _hdr(1100 + 8 + 4, wd=0x00) + _blk(bytes(550), 0, 0) + _blk(bytes(550), 0, 0) + _blk(_raw_lits(lits) + _one_seq(8, 4, 1105 + 3), 2, 1)
    refused(far, "beyond the window")
    refused(_hdr(12) + _blk(_raw_lits(lits) + _one_seq(8, 4, 8, extra_bits=3), 2, 1), "bits left over")
    noend = _raw_lits(lits) + _one_seq(8, 4, 8)[:-1] + b"\x00"
    refused(_hdr(12) + _blk(noend, 2, 1), "end marker")
    # Huffman weights 3, 1 (+ the implied last): 4 + 1 = 5 leaves 3, not a power of two
    tree = bytes([127 + 2, 0x31])
    body = tree + b"\x01"
    lhdr = (2 | (0 << 2) | (4 << 4) | (len(body) << 14)).to_bytes(3, "little")
    refused(_hdr(4) + _blk(lhdr + body + b"\x00", 2, 1), "power of two")
    # an FSE-compressed literal-length table with accuracy log 10 (the limit is 9)
    refused(_hdr(12) + _blk(_raw_lits(lits) + bytes([1, 2 << 6 | 1 << 4 | 1 << 2, 5]), 2, 1), "accuracy log")
    # the engine's layout: a repeat code whose offset the block did not set (offset value 1 with literals: the first repeat offset)
    rep = _hdr(12) + _blk(_raw_lits(lits) + _one_seq(8, 4, 1), 2, 1)
    assert zd.decode(rep)[0] == lits + b"hhhh"
    out, err, _ = zd.decode(rep, CHUNK)
    assert out is None and ("repeat code" in err or "layout" in err), err


def _engine_frame(chunks):
    """A frame in the engine's layout made of raw blocks, one per chunk (the last one marked)."""
    body = b"".join(_blk(c, 0, k == len(chunks) - 1) for k, c in enumerate(chunks)) if chunks else _blk(b"", 0, 1)
    return _hdr(sum(map(len, chunks))) + body


def test_prefix_helper(zd, lz):
    import pyarrow as pa
    from transferia_b200 import engine
    rng = random.Random(5)
    for plen, tlen in ((0, 0), (40, 0), (0, 100), (70, 3 * CHUNK + 5), (70000, 2 * CHUNK)):
        prefix = b"INSERT INTO `db`.`t` FORMAT JSONEachRow\n"[:plen] + bytes(rng.randrange(256) for _ in range(max(0, plen - 41)))
        text = bytes(rng.randrange(256) for _ in range(tlen))
        frame = _engine_frame([text[i:i + CHUNK] for i in range(0, tlen, CHUNK)])
        assert zd.decode(frame, CHUNK)[0] == text
        head = engine.zstd_prefix(prefix, frame)
        whole = head + frame[HDR:]
        want = prefix + text
        assert zd.decode(whole)[0] == want
        assert lz.decompress(whole, len(want)) == want
        with pa.CompressedInputStream(pa.BufferReader(whole), "zstd") as f:
            assert f.read() == want
    frame = _engine_frame([b"abc"])
    for broken in (frame[:-1], frame + b"\x00", b"\x28\xb5\x2f\xfd\xe0" + frame[5:], frame[:5] + b"\x30" + frame[6:],
                   frame[:HDR] + _blk(b"abc", 0, 0), frame[:HDR] + _blk(b"", 3, 1)):
        with pytest.raises(engine.EngineError):
            engine.zstd_prefix(b"x", broken)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _check(zd, lz, res, plain, chunk=CHUNK):
    """The result decodes through the oracle (layout checked), libzstd and pyarrow to the plain call's bytes; everything else is
    the plain call's."""
    import pyarrow as pa
    out, err, info = zd.decode(res.wire, chunk)
    assert err is None, err
    assert out == plain.wire
    assert lz.decompress(res.wire, len(plain.wire)) == plain.wire
    with pa.CompressedInputStream(pa.BufferReader(res.wire), "zstd") as f:
        assert f.read() == plain.wire
    assert res.raw_len == plain.raw_len == len(plain.wire)
    assert res.rows_in == plain.rows_in and res.rows_out == plain.rows_out and res.errors == plain.errors
    assert getattr(res, "row_sizes", None) == getattr(plain, "row_sizes", None)
    assert len(res.wire) <= HDR + len(plain.wire) + 3 * max(1, (len(plain.wire) + chunk - 1) // chunk)
    info["size"] = len(res.wire)
    return info


@pytest.mark.gpu
def test_device_parity(eng, zd, lz):
    """A filtered hits-shaped batch through push_encode (one and two phases), parse_json with mask_field, parse_csv, parse_debezium."""
    from transferia_b200 import engine, workload
    batch, schema = workload.make_hits_batch(60000, seed=4)
    k = workload.counterid_threshold(batch, schema)
    pid = eng.plan("public", "hits", schema, workload.headline_transformers(k), {"type": "clickhouse"})
    plain = eng.push_encode(pid, batch, JER)
    info = _check(zd, lz, eng.push_encode(pid, batch, JER | ZSTD), plain)
    assert info["huf_literals"] > 0 and info["compressed"] > 0
    _check(zd, lz, eng.push_encode(pid, batch, JER | ZSTD, selective=0), plain)
    text, fields = workload.make_json_lines(20000)
    opts = {"add_rest": True, "add_dedupe_keys": True, "partition": '{"partition":0,"topic":"events"}'}
    jschema = engine.json_result_schema(fields, opts)
    jtrs = [{"mask_field": {"columns": ["user"], "maskFunctionHash": {"userDefinedSalt": "pepper"}}}]
    jpid = eng.plan("", "events", jschema, jtrs, {"type": "clickhouse"})
    _check(zd, lz, eng.parse_json(jpid, text, opts, None, wire_fmt=JER | ZSTD), eng.parse_json(jpid, text, opts, None, wire_fmt=JER))
    data, ends, schema_text, table = workload.make_debezium_messages(5000)
    dpid = eng.plan(table[0], table[1], engine.debezium_table_schema(schema_text), workload.debezium_transformers(), {"type": "clickhouse"})
    plain, _ = eng.parse_debezium(dpid, data, ends, schema_text, schema_registry=True, schema_id=7, wire_fmt=JER)
    res, _ = eng.parse_debezium(dpid, data, ends, schema_text, schema_registry=True, schema_id=7, wire_fmt=JER | ZSTD)
    _check(zd, lz, res, plain)
    cschema = [{"name": "a", "type": "int64", "path": "0"}, {"name": "b", "type": "utf8", "path": "1"}, {"name": "c", "type": "double", "path": "2"}]
    rng = random.Random(2)
    ctext = "".join(f"{rng.randrange(-10**9, 10**9)},w{rng.randrange(10**6)} x,{rng.random() * 1e3:.3f}\n" for _ in range(30000)).encode()
    cpid = eng.plan("", "c", cschema, [{"filter_rows": {"filter": "a > 0"}}], {"type": "clickhouse"})
    plain, _ = eng.parse_csv(cpid, ctext, wire_fmt=JER)
    res, _ = eng.parse_csv(cpid, ctext, wire_fmt=JER | ZSTD)
    _check(zd, lz, res, plain)


@pytest.mark.gpu
def test_device_ratio_floors(eng, zd, lz):
    """The hits-shaped text: Huffman-coded literals and FSE-compressed sequence tables are what reach these ratios (raw literals or
    predefined tables alone fall below them), and the history before each chunk is used."""
    from transferia_b200 import workload
    batch, schema = workload.make_hits_batch(30000, seed=1)
    pid = eng.plan("public", "hits", schema, [], {"type": "clickhouse"})
    plain = eng.push_encode(pid, batch, JER)
    info = _check(zd, lz, eng.push_encode(pid, batch, JER | ZSTD), plain)
    ratio = len(plain.wire) / info["size"]
    print("hits JSONEachRow ratio", round(ratio, 3), info)
    assert info["fse_tables"] > 0 and info["huf_literals"] > 0 and info["fse_weights"] > 0
    # 6.61 on an H100 with this encoder; raw literals (no Huffman stage) give 5.61 and sequence tables held to Predefined_Mode 6.21
    assert ratio >= 6.0, ("literals left raw?", ratio)
    assert ratio >= 6.4, ("sequence tables held to Predefined_Mode?", ratio)


def _text_push(eng, pid, vals):
    b = abi.Batch(len(vals), [abi.strings_to_column(abi.TF_UTF8, [v if isinstance(v, bytes) else v.encode() for v in vals])])
    return eng.push_encode(pid, b, JER), eng.push_encode(pid, b, JER | ZSTD)


@pytest.mark.gpu
def test_device_crafted_texts(eng, zd, lz):
    pid = eng.plan("s", "t", [{"name": "v", "type": "utf8"}], [], {"type": "clickhouse"})
    rng = random.Random(17)
    letters = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"

    def run(vals):
        plain, res = _text_push(eng, pid, vals)
        return _check(zd, lz, res, plain), plain

    def rand_vals(nbytes, width=60):      # each row {"v":"<width letters>"}\n is width + 9 bytes
        n = max(1, nbytes // (width + 9))
        return ["".join(rng.choice(letters) for _ in range(width)) for _ in range(n)]

    # 0 rows: one empty last raw block
    b = abi.Batch(0, [abi.strings_to_column(abi.TF_UTF8, [])])
    res = eng.push_encode(pid, b, JER | ZSTD)
    assert res.wire == bytes([0x28, 0xB5, 0x2F, 0xFD, 0xC0, 0x28]) + bytes(8) + b"\x01\x00\x00"
    assert zd.decode(res.wire, CHUNK)[0] == b""
    run(["a"])                                 # shorter than a match... of the text's own bytes
    run(["ab", "ab"])
    # chunk size - 1 / + 0 / + 1 (rows of 69 bytes plus a tail row sized to land there), several chunks, more than 1000 chunks
    for n in (CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5):
        vals = rand_vals(n - 40)
        rest = n - sum(len(v) + 9 for v in vals) - 9
        vals.append("q" * rest)
        info, plain = run(vals)
        assert len(plain.wire) == n
    info, plain = run(rand_vals(1001 * CHUNK + 7))
    assert info["compressed"] + info["raw"] + info["rle"] >= 1001
    # 3-byte repeats only: every 4-gram of the body is unique
    db = []; seen = set()
    while len(db) < 3 * CHUNK:
        c = rng.choice("abcdefgh")
        if len(db) >= 3 and "".join(db[-3:]) + c in seen:
            c = rng.choice(letters)
        db.append(c)
        if len(db) >= 4:
            seen.add("".join(db[-4:]))
    body = "".join(db)
    run([body[i:i + 2000] for i in range(0, len(body), 2000)])
    # a chunk whose only matches lie in the chunk before it: chunk 1 repeats chunk 0's letters
    first = "".join(rng.choice(letters) for _ in range(CHUNK - 10))
    info, plain = run([first, first])
    assert info["size"] < 0.65 * len(plain.wire), info
    # repeats just inside and just beyond the 16 KiB history of a chunk
    seg = "".join(rng.choice(letters) for _ in range(3000))
    for gap in (CHUNK - 3000 - 20, CHUNK + 200):
        filler = "".join(rng.choice(letters) for _ in range(gap))
        run([seg + filler + seg])
    # matches and literal runs at the LL / ML code boundaries (16, 24, 64, 128, ... bytes)
    for m in (3, 4, 5, 34, 35, 36, 66, 67, 130, 131, 258, 259, 1026, 1027, 4098, 4099):
        s = "".join(rng.choice(letters) for _ in range(m))
        lit = "".join(rng.choice(letters) for _ in range(m))
        run([s + lit + s + "".join(rng.choice(letters) for _ in range(m % 64)) + s])
    # literal sections of at most and of more than 1023 bytes (1 and 4 Huffman streams)
    for n in (900, 1000, 1100, 5000):
        run(["".join(rng.choice("abcdefghij") for _ in range(n))])
    # incompressible bytes (the writer passes every byte but the ones JSON escapes as it is): raw blocks within 3 bytes per chunk
    # plus the header
    plain_bytes = [x for x in range(256) if x not in b'"\\\n\r\t\b\f']
    vals = [bytes(rng.choice(plain_bytes) for _ in range(3000)) for _ in range(12)]
    info, plain = run(vals)
    assert info["raw"] >= 1 and info["size"] <= HDR + len(plain.wire) + 3 * ((len(plain.wire) + CHUNK - 1) // CHUNK)
    # a single-byte run (RLE blocks for the chunks inside it)
    info, _ = run(["z" * (5 * CHUNK)])
    assert info["rle"] >= 3, info
    # (nearly) all 256 byte values, skewed so that Huffman pays: symbols past 128 need FSE-compressed Huffman weights
    skew = bytes(plain_bytes) + b"etaoinshrdlu" * 40
    vals = [bytes(rng.choice(skew) for _ in range(200)) for _ in range(400)]
    info, _ = run(vals)
    assert info["fse_weights"] >= 1, info
    # a skewed histogram: 60 frequent letters and a Fibonacci tail that wants codes past 11 bits
    pool = list(letters) * 60
    fib = [1, 1]
    while len(fib) < 16:
        fib.append(fib[-1] + fib[-2])
    for k, c in enumerate("!#$%&()*+,-./:;<"):
        pool += [c] * fib[k]
    rng.shuffle(pool)
    body = "".join(pool)
    run([body[i:i + 200] for i in range(0, len(body), 200)])
    # stale bytes: a large push, then a small one on the same engine
    run(rand_vals(4 * CHUNK + 99))
    run(["zz", "yy"])


@pytest.mark.gpu
def test_device_prefix_and_sink(eng, zd, lz):
    """The INSERT line in front of a device frame through the helper, and tfgpu_sink_push with the flag."""
    import pyarrow as pa
    from transferia_b200 import engine, rows, sink, workload
    batch, schema = workload.make_hits_batch(5000, seed=6)
    pid = eng.plan("public", "hits", schema, [], {"type": "clickhouse"})
    plain = eng.push_encode(pid, batch, JER)
    res = eng.push_encode(pid, batch, JER | ZSTD)
    line = b"INSERT INTO `public`.`hits` SETTINGS input_format_null_as_default=1 FORMAT JSONEachRow\n"
    whole = engine.zstd_prefix(line, res.wire) + res.wire[HDR:]
    assert zd.decode(whole)[0] == line + plain.wire
    assert lz.decompress(whole, len(line) + len(plain.wire)) == line + plain.wire
    with pa.CompressedInputStream(pa.BufferReader(whole), "zstd") as f:
        assert f.read() == line + plain.wire
    items = rows.items_from_batch(batch)
    s = sink.Sink(eng, wire_fmt=JER | ZSTD)
    s.push(rows.RowsImage(items, [("public", "hits", schema)]))
    ev = [e for e in s.events if e["type"] == sink.EV_ROWS]
    s.close()
    s2 = sink.Sink(eng, wire_fmt=JER)
    s2.push(rows.RowsImage(items, [("public", "hits", schema)]))
    ev2 = [e for e in s2.events if e["type"] == sink.EV_ROWS]
    s2.close()
    assert len(ev) == len(ev2) == 1 and ev[0]["raw_len"] == len(ev2[0]["wire"])
    out, err, _ = zd.decode(ev[0]["wire"], CHUNK)
    assert err is None and out == ev2[0]["wire"]
    assert lz.decompress(ev[0]["wire"], len(out)) == out


@pytest.mark.gpu
def test_device_refusals(eng):
    from transferia_b200 import engine, workload
    batch, schema = workload.make_hits_batch(100)
    pid = eng.plan("s", "t", schema, [], {"type": "clickhouse"})
    for fmt in (abi.TF_WIRE_CH_NATIVE | ZSTD, abi.TF_WIRE_CH_NATIVE_LZ4 | ZSTD, abi.TF_WIRE_SER_JSON | ZSTD, abi.TF_WIRE_SER_CSV | ZSTD,
                abi.TF_WIRE_DEBEZIUM | ZSTD, JER | ZSTD | abi.TF_WIRE_F_GZIP, JER | ZSTD | abi.TF_WIRE_F_ZLIB):
        with pytest.raises(engine.EngineError) as ei:
            eng.push_encode(pid, batch, fmt)
        assert ei.value.rc == -2 and "wire format not implemented" in str(ei.value)
