"""The LZ4 frame kernels (k_lz4_frames, k_frame_seal) on frames crafted to hit their structure: 60-byte parse segments,
1024-position match rounds, the end-of-block rules, the length-extension steps, the continuation of long matches, the
CityHash paths of the seal and the look-back over many frames.

The harness pushes one required UInt8 column. Its native block is a fixed header (block info, column and row counts,
name "a", type "UInt8", custom-serialization byte: 18 bytes + varint(rows)) followed by the column's bytes verbatim, so
a test controls every byte of every frame through the public ABI. Every push is checked in full (Harness.push): frame
walk and header fields, each checksum against the oracle's CityHash128, each block through the strict oracle decoder
and stock liblz4 back to the oracle's block. On top of that, cases whose output is fixed by the format alone (no match
possible) are compared byte for byte, and long runs must compress to one sequence per frame."""
import ctypes as C
import os
import struct
import sys
from dataclasses import dataclass

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cityhash_independent  # noqa: E402

from transferia_b200 import abi, engine  # noqa: E402

pytestmark = pytest.mark.gpu
LZ, RAW = abi.TF_WIRE_CH_NATIVE_LZ4, abi.TF_WIRE_CH_NATIVE
SCHEMA = [{"name": "a", "type": "uint8", "required": True}]
SEG, ROUND = 60, 1024                       # parse segment and match-finding round of k_lz4_frames
# multiples of 16 in [1024, 15360]; 1040, 1264, 4112, 9232 and 15344 are multiples of neither 60 nor 1024, so every full frame
# of theirs ends in a partial round and a partial segment
FRAME_SIZES = [1024, 1040, 1264, 4112, 9232, 15344, 15360]


def uvarint(n: int) -> bytes:
    out = b""
    while n >= 0x80:
        out += bytes([(n & 0x7F) | 0x80]); n >>= 7
    return out + bytes([n])


def lz_ext(n: int) -> bytes:
    """LZ4 length-extension bytes of a literal run of n bytes (or of a match of n + 4)."""
    if n < 15:
        return b""
    n -= 15
    return b"\xff" * (n // 255) + bytes([n % 255])


def literal_block(raw: bytes) -> bytes:
    """The only LZ4 block of raw when no match is possible: one token, its extension bytes, the literals."""
    return bytes([min(len(raw), 15) << 4]) + lz_ext(len(raw)) + raw


def has_repeat4(b: bytes) -> bool:
    if len(b) < 5:
        return False
    a = np.frombuffer(b, dtype=np.uint8).astype(np.uint32)
    g = a[:-3] | (a[1:-2] << 8) | (a[2:-1] << 16) | (a[3:] << 24)
    return len(np.unique(g)) != len(g)


def unique_bytes(rng, n: int, prefix: bytes = b"") -> bytes:
    """n seeded random bytes such that no 4-byte sequence occurs twice in prefix + them (redrawn on a hit)."""
    for _ in range(100):
        b = bytes(rng.integers(0, 256, n, dtype=np.uint8))
        if not has_repeat4(prefix + b):
            return b
    raise AssertionError("no 4-gram-unique draw")


def periodic(unit: bytes, n: int) -> bytes:
    return (unit * (n // len(unit) + 1))[:n]


@dataclass
class Frame:
    off: int        # offset in the wire buffer
    cs: int         # compressed-size field: LZ4 block + 9, the length the checksum covers
    raw: bytes
    block: bytes


class Harness:
    def __init__(self, po, eng):
        self.po, self.eng, self.F = po, eng, eng.frame_bytes
        self.pid = eng.plan("db", "t", SCHEMA, [], {"type": "clickhouse"})
        self.plan = po.build_plan("db", "t", SCHEMA, [])
        self.lz = C.CDLL("liblz4.so.1")
        one = po.push_encode(self.batch(b"\x00"), self.plan, RAW).raw
        assert len(one) == 20 and one[9] == 1 and one[-1] == 0      # [9 bytes][varint rows = 1][9 bytes][the one value]
        self.hdr_pre, self.hdr_post = one[:9], one[10:19]

    @staticmethod
    def batch(payload: bytes) -> abi.Batch:
        return abi.Batch(len(payload), [abi.fixed_to_column(abi.TF_UINT8, np.frombuffer(payload, dtype=np.uint8))])

    def header(self, rows: int) -> bytes:
        return self.hdr_pre + uvarint(rows) + self.hdr_post

    def payload_len(self, block_len: int) -> int:
        """Rows whose block is block_len bytes long."""
        for v in (1, 2, 3, 4):
            p = block_len - 18 - v
            if p >= 0 and len(uvarint(p)) == v:
                return p
        raise ValueError(f"no native block of {block_len} bytes")

    def compose(self, block_len: int, body) -> bytes:
        """Payload of a block_len-byte block: body(header) returns the bytes behind the header."""
        hdr = self.header(self.payload_len(block_len))
        p = body(hdr)
        assert len(hdr) + len(p) == block_len
        return p

    def push(self, payload: bytes):
        """One push through the engine, checked in full; returns (native block, frames)."""
        po, F = self.po, self.F
        b = self.batch(payload)
        ref = po.push_encode(b, self.plan, RAW).raw
        assert ref == self.header(len(payload)) + payload, "the harness's block layout"
        got = self.eng.push_encode(self.pid, b, LZ)
        wire, frames, pos = got.wire, [], 0
        while pos < len(wire):
            k = len(frames)
            assert pos + 25 <= len(wire) and wire[pos + 16] == 0x82, f"frame {k}: header"
            cs, rs = struct.unpack_from("<II", wire, pos + 17)
            assert rs == min(F, len(ref) - k * F) > 0, f"frame {k}: raw size {rs}"
            assert 9 <= cs and pos + 16 + cs <= len(wire), f"frame {k}: compressed size {cs}"
            raw, blk = ref[k * F: k * F + rs], wire[pos + 25: pos + 16 + cs]
            assert struct.unpack_from("<QQ", wire, pos) == po.cityhash128(wire[pos + 16: pos + 16 + cs]), f"frame {k}: checksum"
            assert po.lz4_decompress(blk, rs) == raw, f"frame {k} of {F} B: the strict decoder rejects the block or decodes another one"
            dst = C.create_string_buffer(rs)
            assert self.lz.LZ4_decompress_safe(blk, dst, len(blk), rs) == rs and dst.raw == raw, f"frame {k}: liblz4"
            frames.append(Frame(pos, cs, raw, blk))
            pos += 16 + cs
        assert pos == len(wire) == sum(16 + f.cs for f in frames)
        assert len(frames) == got.n_frames == -(-len(ref) // F)
        return ref, frames


@pytest.fixture(scope="module")
def harness(po, eng):
    """Harness per frame size; the engines of the non-default sizes are made here and closed at the end of the module."""
    made = {}

    def get(F):
        if F not in made:
            made[F] = Harness(po, eng if F == eng.frame_bytes else engine.Engine(0, F))
        return made[F]
    yield get
    for h in made.values():
        if h.eng is not eng:
            h.eng.close()


def literal_only_payload(h: Harness, rng, block_len: int) -> bytes:
    """A block in which no 4-byte sequence occurs twice within a frame (frame 0 counts its header): no match is possible."""
    def body(hdr):
        out = hdr
        while len(out) < block_len:
            start = len(out) - len(out) % h.F
            out += unique_bytes(rng, min(block_len, start + h.F) - len(out), out[start:])
        return out[len(hdr):]
    return h.compose(block_len, body)


# ---------------------------------------------------------------------------------------------------------------- a
@pytest.mark.parametrize("F", FRAME_SIZES)
def test_literal_only_frames_exact(harness, F):
    """No match possible: every frame's block is exactly token + extension bytes + literals. Last-frame lengths sit at the
    literal-length steps (15, 270, 525, 780), run through every residue mod 60 (so mod 4 and 16), and blocks end one byte
    before, on and behind a frame boundary. Pins put_ext for literals, the carry of trailing literals over every segment and
    warp of a frame, and copy_lit at every source and destination alignment."""
    h = harness(F)
    rng = np.random.default_rng(F)
    lasts = [1, 2, 3, 4, 5, 14, 15, 16, 269, 270, 271, 524, 525, 526, 779, 780, 781] + list(range(600, 660)) + [F - 1, F]
    blocks = [F + L for L in lasts] + [k * F + d for k in (2, 3) for d in (-1, 0, 1)]
    for n in blocks:
        ref, frames = h.push(literal_only_payload(h, rng, n))
        for k, fr in enumerate(frames):
            assert fr.block == literal_block(fr.raw), f"block of {n} B, frame {k} ({len(fr.raw)} B) is not the literal-only block"


# ---------------------------------------------------------------------------------------------------------------- b
@pytest.mark.parametrize("F", [1024, 1040, 15344])
def test_tiny_last_frames(harness, F):
    """Last frames of 1..13 bytes of repetitive content: below 13 bytes a block has no match, so it is [len << 4] + bytes."""
    h = harness(F)
    for fill in (b"\x00", b"ab"):
        for L in range(1, 14):
            ref, frames = h.push(h.compose(F + L, lambda hdr: periodic(fill, F + L - len(hdr))))
            last = frames[-1]
            assert len(last.raw) == L
            if L <= 12:
                assert last.block == bytes([L << 4]) + last.raw, f"last frame of {L} B"


# ---------------------------------------------------------------------------------------------------------------- c
def end_sweep_frames(rng, L):
    """Last-frame contents of L bytes that offer a match at every position near the end."""
    pre = unique_bytes(rng, 5)
    out = [pre + b"\x07" * (L - 5)]                                      # a constant run to the last byte
    for p in (3, 5, 6, 7, 12):                                           # periodic runs to the last byte
        out.append(pre + periodic(unique_bytes(rng, p), L - 5))
    base = bytearray(unique_bytes(rng, L))
    for s in range(max(0, L - 16), L - 3):                              # one 4..8-byte repeat starting at each of L-16 .. L-4
        m = min(4 + (s + L) % 5, L - s)
        if s < m:
            continue
        f = bytearray(base)
        src = int(rng.integers(0, s - m + 1))
        f[s: s + m] = f[src: src + m]
        out.append(bytes(f))
    return out


def end_sweep_cases():
    cases = [(1040, 13, 140)] + [(F, F - 70, F) for F in (1040, 4112, 15344)]
    cases += [(4112, 2040, 2056), (9232, 8184, 8200)]                    # last frames ending around a round boundary
    return cases


@pytest.mark.parametrize("F,lo,hi", end_sweep_cases())
def test_end_of_block_sweep(harness, F, lo, hi):
    """Last-frame lengths L in [lo, hi], each with content that offers matches up to the last byte: constant and periodic
    runs, and unique bytes with one short repeat at each of L-16 .. L-4 (both parities). Every block must keep the LZ4
    end-of-block rules (the strict decoder in Harness.push): last 5 bytes literals, no match starting in the last 12."""
    h = harness(F)
    rng = np.random.default_rng(lo * 7 + F)
    for L in range(lo, hi + 1):
        for last in end_sweep_frames(rng, L):
            h.push(h.compose(F + L, lambda hdr: bytes(F - len(hdr)) + last))


# ---------------------------------------------------------------------------------------------------------------- d
def copy_in(f: bytearray, dst: int, src: int, n: int):
    for i in range(n):          # byte by byte: an overlapping copy repeats, as an LZ4 match does
        f[dst + i] = f[src + i]


def pattern_frames(rng, F):
    """Frames (F bytes each) aimed at the structure of k_lz4_frames."""
    out = []
    for p in (1, 2, 3, 4, 5, 6, 7, 8, 9, 12, 13, 16, 60, 61, 64, 120):      # runs: overlapping copies, the 4 / 8-back test,
        unit = unique_bytes(rng, p)                                      # table candidates, continuation over pure segments
        out += [periodic(unit, F), unique_bytes(rng, 7) + periodic(unit, F - 7)]
    u = unique_bytes(rng, F)
    for m in (16, 64, 256, F // 2):                                      # large offsets: the frame's start copied to its end
        out.append(u[:F - m] + u[:m])
    out.append(u[:F // 2] + u[:F - F // 2])                              # one match over half the frame

    def ending_at(ends, mlen):                                           # unique bytes with copies that end exactly at `ends`
        f = bytearray(unique_bytes(rng, F))
        for e in ends:
            if e - mlen >= 64 and e <= F:
                s = e - mlen
                copy_in(f, s, int(rng.integers(0, s - mlen // 2)), mlen)
        return bytes(f)
    for d in range(-3, 4):                                               # ... on, 1-3 bytes before and behind segment ends
        out.append(ending_at([SEG * k + d for k in range(3, F // SEG, 3)], 100))
        out.append(ending_at([ROUND * k + d for k in range(1, F // ROUND + 1)], 300))
    for q in (40, 41, 42, 43):                                           # backward extension that reaches the frame start:
        f = bytearray(unique_bytes(rng, F))                              # the copy's source is at 0 and zeros in front of both
        f[q - 2: q] = b"\0\0"; f[0:1] = b"\0"
        copy_in(f, q, 0, 48)
        out.append(bytes(f))
    for e1 in (301, 302, 303, 304):                                      # backward extension that reaches the previous match's end:
        f = bytearray(unique_bytes(rng, F))                              # the bytes in front of the second copy also agree
        copy_in(f, e1 - 40, e1 - 40 - 170, 40)
        a = 20
        f[a: a + 8] = f[e1 - 8: e1]
        copy_in(f, e1, a + 8, 40)
        out.append(bytes(f))
    for gap in (15, 270, 525):                                           # literal runs at the length-extension steps
        f, dic = bytearray(unique_bytes(rng, F)), 600
        for s in range(dic, F - 40, 24 + gap):
            copy_in(f, s, int(rng.integers(0, dic - 24)), 24)
        out.append(bytes(f))
    for mls in ((18, 19, 20), (272, 273, 274, 275)):                     # match lengths at the length-extension steps
        f, s, i = bytearray(unique_bytes(rng, F)), 600, 0
        while s + mls[i % len(mls)] + 9 < F:
            m = mls[i % len(mls)]
            copy_in(f, s, int(rng.integers(0, 600 - min(m, 300))), m)
            s += m + 9; i += 1
        out.append(bytes(f))
    return out


def mixed_frames(rng, F, n):
    """n frames cut from one stream of chunks: unique bytes, a copy of an earlier span at a random distance, a constant."""
    f = bytearray()
    while len(f) < n * F:
        kind, m = int(rng.integers(0, 3)), int(rng.integers(1, 400))
        if kind == 0 or len(f) < 8:
            f += bytes(rng.integers(0, 256, m, dtype=np.uint8))
        elif kind == 1:
            src = len(f) - int(rng.integers(1, min(len(f), 70000)))
            f += bytes(m); copy_in(f, len(f) - m, src, m)
        else:
            f += bytes([int(rng.integers(0, 256))]) * m
    return bytes(f[:n * F])


@pytest.mark.parametrize("F", FRAME_SIZES)
def test_structure_patterns(harness, F):
    """Runs of many periods, large offsets, matches ending on and around segment and round boundaries, backward extension
    up to the frame start and up to the previous match, literal runs and match lengths at the extension steps, then a
    seeded mix of 200 frames. The check is the full one of Harness.push."""
    h = harness(F)
    rng = np.random.default_rng(100 + F)
    pats = pattern_frames(rng, F)
    h.push(h.compose(F * (len(pats) + 1) - 37, lambda hdr: bytes(F - len(hdr)) + b"".join(pats)[:-37]))
    h.push(h.compose(200 * F + 333, lambda hdr: mixed_frames(rng, F, 201)[len(hdr): 200 * F + 333]))


# ---------------------------------------------------------------------------------------------------------------- e
RATIO_SLACK = 24      # an H100 80GB HBM3 (400 W power limit) gives at most F/255 + 18 bytes on these frames, at every size tested


@pytest.mark.parametrize("F", FRAME_SIZES)
def test_ratio_floor_of_runs(harness, F):
    """Constant frames and runs of period 1, 2, 4 and 8 compress to one sequence per frame: at most F/255 + RATIO_SLACK bytes.

    Why the bound holds: in such a run every even position >= 8 gets a candidate 4 or 8 bytes back from the run test of
    the match-finding round, which involves no race between threads. So the walker of every segment finds a match at its
    first position that reaches the segment end; the continuation merges those pieces into the match that started in the
    first segment, and the frame is one sequence (a few literals, one match of about F bytes whose length takes F/255
    extension bytes) plus the 5 literals of the end. One sequence per segment instead, which is what the kernel emits
    when the continuation is lost, takes at least 3 bytes (token, offset) per 60-byte segment, 3F/60 bytes: 768 bytes
    for a 15360-byte frame against the bound's 84."""
    h = harness(F)
    rng = np.random.default_rng(200 + F)
    units = [b"\x00", b"\xab", unique_bytes(rng, 2), unique_bytes(rng, 4), unique_bytes(rng, 8)]
    content = bytes(F) + b"".join(periodic(u, F) * 2 for u in units) + bytes(100)
    ref, frames = h.push(h.compose(len(content), lambda hdr: content[len(hdr):]))
    sizes = [len(fr.block) for fr in frames[1:-1]]
    assert max(sizes) <= F // 255 + RATIO_SLACK, f"run frames of {F} B compress to {sizes} B"


# ---------------------------------------------------------------------------------------------------------------- f
def test_seal_sweep(harness):
    """k_frame_seal at every hashed length from 11 to 612 and every alignment of the frame in the wire buffer.

    F = 1040: an incompressible frame takes 16 + 9 + 1046 = 1071 wire bytes, 15 mod 16, so k = 1..16 such frames in front of
    the last one put it at every offset mod 16 (the wire buffer comes from cudaMalloc, so that is the hashed body's offset
    mod 16, `bsh` in the kernel). The last frame holds L unique bytes, hashed length cs = L + 1 + ext(L) + 9. The sweep
    covers the generic path (cs < 160) and the 128-byte-block path with its tail loop at every remainder 0..127 behind 1-3
    blocks, with the tail window at 0 (cs - 16 <= 272) and behind it."""
    F = 1040
    h = harness(F)
    rng = np.random.default_rng(5)
    seen = set()
    for L in range(1, 601):
        last = unique_bytes(rng, L)
        for j in (0, 8):
            k = 1 + (L + j) % 16
            def body(hdr):
                out = hdr + unique_bytes(rng, F - len(hdr), hdr)
                out += b"".join(unique_bytes(rng, F) for _ in range(k - 1))
                return out[len(hdr):] + last
            ref, frames = h.push(h.compose(k * F + L, body))
            assert [f.cs for f in frames[:-1]] == [1055] * k
            fr = frames[-1]
            assert fr.block == literal_block(last) and fr.cs == L + 1 + len(lz_ext(L)) + 9
            seen.add((fr.cs, fr.off % 16))
            hashed = b"\x82" + struct.pack("<II", fr.cs, L) + fr.block      # the device's checksum equals the oracle's (Harness.push)
            assert cityhash_independent.cityhash128(hashed) == h.po.cityhash128(hashed), f"cs {fr.cs}"
    cs_seen = {cs for cs, _ in seen}
    reachable = {L + 1 + len(lz_ext(L)) + 9 for L in range(1, 601)}
    assert cs_seen == reachable and min(cs_seen) == 11 and max(cs_seen) >= 600
    for bsh in range(16):
        assert any(cs < 160 and b == bsh for cs, b in seen) and any(cs >= 160 and b == bsh for cs, b in seen), bsh


# ---------------------------------------------------------------------------------------------------------------- g
def test_stale_bytes_behind_the_block(harness):
    """Staging loads up to 15 bytes behind the last frame, and the engine's buffers only grow: what a larger earlier push
    left there must not leak into a block. Each large push is followed by a smaller one whose end is not 16-aligned,
    with content the stale bytes would continue (a constant run, a period-7 run: both pushes' payloads start alike) and
    with literal-only content that must still come out byte-exact."""
    F = 1040
    h = harness(F)
    rng = np.random.default_rng(9)
    big = 16000                                  # same varint length as the small blocks: the stale bytes continue the run
    for unit in (b"\x00", unique_bytes(rng, 7)):
        run = periodic(unit, big)
        for r in range(1, 16, 2):
            n = 5 * F + 16 * 3 + r               # not 16-aligned, ends inside a round and a segment
            h.push(run)
            h.push(run[:h.payload_len(n)])
    for r in (1, 6, 11, 15):
        h.push(periodic(b"\x00", big))
        ref, frames = h.push(literal_only_payload(h, rng, 3 * F + 100 + r))
        for fr in frames:
            assert fr.block == literal_block(fr.raw)


# ---------------------------------------------------------------------------------------------------------------- h
def test_many_frames(harness):
    """More than 1000 frames of mixed content at F = 1024: frame sizes vary, so the decoupled look-back of every frame sums
    a long, uneven prefix; every frame sits where the sizes in front of it put it (Harness.push's walk)."""
    F = 1024
    h = harness(F)
    rng = np.random.default_rng(13)
    n = 1100 * F + 517
    ref, frames = h.push(h.compose(n, lambda hdr: mixed_frames(rng, F, 1101)[len(hdr): n]))
    assert len(frames) == 1101 and len({f.cs for f in frames}) > 100
