"""Decimal text -> binary floating point, on the device and in the oracle, against correctly rounded references.

Entry points (one literal per row, or per cell for number_to_float):
  strconv.ParseFloat(s, 64)  d_go_parse_float + d_eisel_lemire   JSON string cell -> double, number_to_float
  fastfloat.ParseBestEffort  d_ff_best                           JSON number -> double and -> canonical `any` text
  CSV Clinger fast path      d_parse_float                       CSV double / float columns (float: ParseFloat(s, 32))
References: CPython float() for ParseFloat(s, 64) (correctly rounded, ties to even, like Go); glibc strtof for ParseFloat(s, 32),
itself cross-checked against exact Fraction rounding; the oracle for fastfloat bit for bit, with fastfloat's own structure
checked independently (fall-back rows equal float(text), integer-only rows equal float(int(text))); encoding/json's float layout
built from repr()'s shortest digits. A row the device hands to the host must be exactly a row the documented hand-off rule
predicts (include/tfgpu.h, DESIGN §3): Eisel-Lemire declines or the truncated mantissa's two bounds disagree, a subnormal result,
hex or underscored text — computed here with the Eisel-Lemire prototype scripts/el_proto.py."""
import base64
import ctypes
import ctypes.util
import functools
import math
import os
import random
import re
import struct
import sys
import time
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

from transferia_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import el_proto  # noqa: E402

CSRC = os.path.join(ROOT, "transferia_b200", "csrc")
GO_NAN = 0x7FF8000000000001          # math.NaN()
DBL_MAX = (2 ** 53 - 1) * 2 ** 971
MIN_NORMAL = Fraction(1, 2 ** 1022)


def b64(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def next_up(x):
    return math.nextafter(x, math.inf)


# ------------------------------------------------------------------------------------------------ references
_libc = ctypes.CDLL(ctypes.util.find_library("c"))
_libc.strtof.restype = ctypes.c_float
_libc.strtof.argtypes = [ctypes.c_char_p, ctypes.c_void_p]


def strtof_bits(s):
    """ParseFloat(s, 32) for plain decimal text: glibc strtof (correctly rounded, ties to even)."""
    return struct.unpack("<I", struct.pack("<f", _libc.strtof(s.encode(), None)))[0]


def f32_round_bits(fr):
    """Exact round-to-nearest-even of a rational to binary32 (the cross-check of strtof)."""
    if fr == 0:
        return 0
    sign = 0x80000000 if fr < 0 else 0
    a = abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)
    sc = a / Fraction(2) ** (e - 23)
    q, r = divmod(sc.numerator, sc.denominator)
    if 2 * r > sc.denominator or (2 * r == sc.denominator and q & 1):
        q += 1
    if q == 1 << 24:
        q >>= 1; e += 1
    if e + 127 >= 255:
        return sign | 0x7F800000
    return sign | (((e + 127) << 23) | (q - (1 << 23)) if q >= 1 << 23 else q)


def go_json_float(x):
    """encoding/json's float64 text: shortest digits ('f', or 'e' below 1e-6 / from 1e21, with e-07 -> e-7), from repr()."""
    if x == 0:
        return "-0" if math.copysign(1, x) < 0 else "0"
    mant, _, ex = repr(abs(x)).partition("e")
    ip, _, fp = mant.partition(".")
    if fp == "0":
        fp = ""
    raw = ip + fp
    point = len(ip) + int(ex or 0) - (len(raw) - len(raw.lstrip("0")))       # value = 0.digits * 10^point
    digits = raw.lstrip("0").rstrip("0")
    sign = "-" if x < 0 else ""
    if abs(x) < 1e-6 or abs(x) >= 1e21:
        e = point - 1
        m = digits[0] + ("." + digits[1:] if len(digits) > 1 else "")
        return sign + (f"{m}e-{-e}" if -10 < e < 0 else f"{m}e{'-' if e < 0 else '+'}{abs(e):02d}")
    if point <= 0:
        return sign + "0." + "0" * -point + digits
    if point >= len(digits):
        return sign + digits + "0" * (point - len(digits))
    return sign + digits[:point] + "." + digits[point:]


# ------------------------------------------------------------------------------------------------ the hand-off rule
def go_parse_path(s):
    """strconv.ParseFloat(s, 64) as the device decides it (readFloat, atof64exact, the u64 integer path, Eisel-Lemire with the
    man+1 check for truncated mantissas, decimal's dp cut-offs). Returns (path, el): path names the `return` taken; for a
    decided Eisel-Lemire result el = (the table row it read, the prototype's bits), else None."""
    if not s:
        return "syntax_empty", None
    t, sign = s, False
    if t[0] in "+-":
        t, sign = t[1:], True
    if t.lower() in ("inf", "infinity"):
        return "special_inf", None
    if not sign and t.lower() == "nan":
        return "special_nan", None
    i = 1 if s[0] in "+-" else 0
    n = len(s)
    if i + 2 < n and s[i] == "0" and s[i + 1] in "xX":
        k, dig, dot = i + 2, False, False
        while k < n:
            c = s[k]
            if c == "_":
                return "host_hex_underscore", None
            if c == ".":
                if dot:
                    break
                dot = True; k += 1; continue
            if c.isdigit() or c.lower() in "abcdef":
                dig = True; k += 1; continue
            break
        if not dig or k >= n or s[k].lower() != "p":
            return "syntax_hex", None
        return "host_hex", None
    man = nd = ndm = dp = 0
    sawdot = sawdigits = trunc = False
    while i < n:
        c = s[i]
        if c == "_":
            return "host_underscore", None
        if c == ".":
            if sawdot:
                break
            sawdot, dp = True, nd
        elif "0" <= c <= "9":
            sawdigits = True
            if c == "0" and nd == 0:
                dp -= 1
            else:
                nd += 1
                if ndm < 19:
                    man = man * 10 + int(c); ndm += 1
                elif c != "0":
                    trunc = True
        else:
            break
        i += 1
    if not sawdigits:
        return "syntax_nodigits", None
    if not sawdot:
        dp = nd
    if i < n and s[i] in "eE":
        i += 1
        if i >= n:
            return "syntax_exp_end", None
        es = 1
        if s[i] == "+":
            i += 1
        elif s[i] == "-":
            es = -1; i += 1
        if i >= n or not s[i].isdigit():
            return "syntax_exp_digit", None
        e = 0
        while i < n and (s[i].isdigit() or s[i] == "_"):
            if s[i] == "_":
                return "host_exp_underscore", None
            if e < 10000:
                e = e * 10 + int(s[i])
            i += 1
        dp += e * es
    if i != n:
        return "syntax_trailing", None
    if man == 0:
        return "zero", None
    exp = dp - ndm
    if not trunc and man >> 53 == 0:
        f = float(man)
        if exp == 0:
            return "exact_int", None
        if 0 < exp <= 37:
            if exp <= 22:
                return "exact_mul", None
            if f * float(10 ** (exp - 22)) <= 1e15:
                return "exact_mul2", None
        elif -22 <= exp < 0:
            return "exact_div", None
    if not trunc and 0 <= exp <= 19 and man * 10 ** exp < 1 << 64:
        return "u64", None
    b0, ok0 = el_proto.el64(man, exp)
    if ok0:
        if not trunc:
            return "el", (exp, b0)
        b1, ok1 = el_proto.el64(man + 1, exp)
        if ok1 and b0 == b1:
            return "el_trunc", (exp, b0)
    if dp > 310:
        return "overflow", None
    if dp < -330:
        return "underflow", None
    return "host_trunc_disagree" if trunc and ok0 else "host_el_declined", None


GO_RETURNS = {"syntax_empty", "special_inf", "special_nan", "host_hex_underscore", "syntax_hex", "host_hex", "host_underscore", "syntax_nodigits",
              "syntax_exp_end", "syntax_exp_digit", "host_exp_underscore", "syntax_trailing", "zero", "exact_int", "exact_mul", "exact_mul2", "exact_div",
              "u64", "el", "el_trunc", "overflow", "underflow", "host_trunc_disagree", "host_el_declined"}


def go_host(path):
    return path.startswith("host")


def ff_path(s):
    """fastfloat.ParseBestEffort's branch for a JSON number: 'slow' (the strconv fall-back: more than 18 characters before the
    fraction, sign included; 17 characters from the first digit to the fraction's end; an exponent above 300), 'int' (digits only),
    'fast' (fraction / exponent through math.Pow10)."""
    n = len(s); i = 1 if s[0] == "-" else 0; j = i
    while i < n and s[i].isdigit():
        i += 1
        if i > 18:
            return "slow"
    if i >= n:
        return "int"
    if s[i] == ".":
        i += 1
        while i < n and s[i].isdigit():
            i += 1
            if i - j >= 17:
                return "slow"
    if i < n and s[i] in "eE":
        i += 1
        if s[i] in "+-":
            i += 1
        e = 0
        while i < n and s[i].isdigit():
            e = e * 10 + int(s[i]); i += 1
            if e > 300:
                return "slow"
    return "fast"


def csv_fast(s):
    """The CSV fast path's domain (<= 15 significant digits, |exp10| <= 22 after the point shift, or a zero): otherwise the row is
    TF_ROWERR_CSV_UNSUPPORTED and the host's strconv takes it."""
    m = re.fullmatch(r"[+-]?(\d*)(?:\.(\d*))?(?:[eE]([+-]?\d+))?", s)
    ip, fp, ex = m.group(1), m.group(2) or "", m.group(3)
    digits = (ip + fp).lstrip("0")
    if not digits.strip("0"):
        return True
    return len(digits) <= 15 and -22 <= int(ex or 0) - len(fp) <= 22


REQUIRED_D = [{"name": "d", "type": "double", "required": True}]     # a ParseVal error fails the row instead of leaving a null
JSON_NUMBER = re.compile(r"-?(0|[1-9]\d*)(\.\d+)?([eE][+-]?\d+)?")


# ------------------------------------------------------------------------------------------------ corpus
def q_range():
    """Eisel-Lemire rows that can give a normal double for a mantissa of at most 19 digits: the largest mantissa reaches the
    smallest normal, the mantissa 1 stays at or below DBL_MAX."""
    lo = next(q for q in range(-400, 0) if (10 ** 19 - 1) * Fraction(10) ** q >= MIN_NORMAL)
    hi = max(q for q in range(0, 400) if 10 ** q <= DBL_MAX)
    return lo, hi


def _spell(rng, digits, e10):
    k = rng.randrange(4)
    if k == 0:
        return f"{digits}e{e10}"
    if k == 1:
        return f"{digits[0]}.{digits[1:]}e{e10 + len(digits) - 1}" if len(digits) > 1 else f"{digits}E{e10:+d}"
    if k == 2 and -40 < e10 < 0:
        p = len(digits) + e10
        return f"{digits[:p]}.{digits[p:]}" if p > 0 else "0." + "0" * -p + digits
    if k == 2 and 0 <= e10 < 30:
        return digits + "0" * e10
    return f"-{digits}e{e10}"


def _rand_digits(rng, nd):
    return str(rng.randrange(10 ** (nd - 1), 10 ** nd))


def _double_digits(x):
    """Exact decimal expansion of a positive dyadic rational (a double, a midpoint of two): (digit string, exponent)."""
    fr = Fraction(x)
    k = fr.denominator.bit_length() - 1
    assert fr.denominator == 1 << k
    D = str(fr.numerator * 5 ** k); e10 = -k
    s = D.rstrip("0")
    return s, e10 + len(D) - len(s)


def _cuts(D, e10, lens):
    out = []
    for L in lens:
        if L >= len(D):
            continue
        head = int(D[:L]); e = e10 + len(D) - L
        for d in (-1, 0, 1):
            out.append(f"{head + d}e{e}")
    return out


@functools.lru_cache(maxsize=None)
def corpus():
    """[(class, literal)], deterministic."""
    rng = random.Random(20261016)
    out = []
    add = lambda cls, xs: out.extend((cls, x) for x in xs)
    qlo, qhi = q_range()
    # every Eisel-Lemire row: 19-digit (incl. the largest), 17-digit and short mantissas; 17+ digits exceed 2^53, so rows in [-22, 37]
    # reach Eisel-Lemire too
    rows = []
    for q in range(qlo, qhi + 1):
        ms = ["9999999999999999999", "1000000000000000001"] + [_rand_digits(rng, 19) for _ in range(10)] + [_rand_digits(rng, 17) for _ in range(8)]
        ms += [_rand_digits(rng, rng.randint(1, 4)) for _ in range(4)]
        rows += [_spell(rng, m, q) for m in ms]
        rows += [f"{_rand_digits(rng, 22)}e{q - 3}" for _ in range(4)]     # truncated to 19 digits, still row q (the only way to row 0)
    add("el_rows", rows)
    # shortest repr of random doubles over every binary exponent, and of the doubles around each power of ten
    sh = []
    for e2 in range(1, 2047):
        for _ in range(150):
            x = f64((e2 << 52) | rng.getrandbits(52))
            sh.append(repr(x) if rng.random() < 0.8 else repr(-x))
    for q in range(-323, 309):
        x = float(f"1e{q}")
        for k in range(-2, 3):
            y = x
            for _ in range(abs(k)):
                y = math.nextafter(y, math.inf if k > 0 else 0.0)
            if y:
                sh.append(repr(y))
    add("shortest", sh)
    # near-halfway: the exact midpoint of two adjacent doubles cut to 19, 20, 25 and 30 digits, +-1 in the last digit
    hw = []
    for _ in range(35000):
        x = f64((rng.randint(1, 2045) << 52) | rng.getrandbits(52))
        D, e10 = _double_digits((Fraction(x) + Fraction(next_up(x))) / 2)
        hw += _cuts(D, e10, (19, 20, 25, 30))
    for _ in range(2000):          # the full midpoint text, when short enough for a message cell
        x = f64((rng.randint(900, 1200) << 52) | rng.getrandbits(52))
        D, e10 = _double_digits((Fraction(x) + Fraction(next_up(x))) / 2)
        if len(D) < 400:
            hw.append(f"{D}e{e10}")
    add("halfway", hw)
    # the exact path's edges
    ex = []
    for m in (2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1):
        for e in range(-25, 41):
            ex.append(f"{m}e{e}")
    for e in (-23, -22, 22, 23, 37, 38):
        ex += [f"{_rand_digits(rng, rng.randint(1, 16))}e{e}" for _ in range(200)]
    for e in range(23, 38):
        edge = 10 ** 15 // 10 ** (e - 22)        # man * 10^(e-22) around 1e15
        ex += [f"{edge + d}e{e}" for d in (-1, 0, 1) if edge + d > 0]
        ex += [f"{rng.randrange(1, 2 ** 53)}e{e}" for _ in range(2000)]
    add("exact_edges", ex)
    # the u64 integer path: 19-digit mantissas times 10^0..19 on both sides of 2^64, and integers half-way between doubles
    it = []
    for e in range(0, 20):
        lim = (2 ** 64 - 1) // 10 ** e
        for m in (lim - 1, lim, lim + 1):
            if m > 0:
                it.append(f"{m}e{e}")
        it += [f"{rng.randrange(max(1, lim // 10), lim * 10 + 10)}e{e}" for _ in range(200)]
    for _ in range(5000):
        x = float(rng.randrange(2 ** 53, 2 ** 64))
        it.append(str((int(x) + int(next_up(x))) // 2))
    add("int_edges", it)
    # the range's edges
    rg = ["4.9406564584124654e-324", "5e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.2250738585072009e-308",
          "2.2250738585072014e-308", "2.2250738585072011e-308", "2.2250738585072019e-308", "2.225073858507201e-308",
          "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "-1.7976931348623159e308", "1.8e308",
          "1e309", "1e310", "1e311", "1e-331", "1e-332", "1e-333", "1" + "0" * 309, "1" + "0" * 310, "9" * 311,
          "0." + "0" * 329 + "1", "0." + "0" * 330 + "1", "0." + "0" * 331 + "1", "1234567890123456789e-349", "1234567890123456789e-350",
          "1234567890123456789e291", "1234567890123456789e292", "1e99999", "1e-99999", "-1e99999", "-1e-99999", "1e999999999999", "0e99999"]
    for k in range(1, 2050, 7):
        rg.append(repr(f64(k)))                                   # subnormals
    add("range_edges", rg)
    # fastfloat: integer parts of 17-19 characters with and without '-', fractions reaching 16 / 17 characters, exponents 300 / 301,
    # negative exponents (math.Pow10 divides, fastfloat multiplies by the quotient)
    ff = []
    for nd in (16, 17, 18, 19):
        for _ in range(300):
            d = _rand_digits(rng, nd)
            ff += [d, "-" + d]
    for ip in range(1, 17):
        for fl in range(1, 18 - ip):
            for _ in range(60):
                s = _rand_digits(rng, ip) + "." + "".join(rng.choice("0123456789") for _ in range(fl))
                ff.append(s if rng.random() < 0.5 else "-" + s)
    for e in ("300", "301", "-300", "-301", "0300", "+300", "+301"):
        ff += [f"{_rand_digits(rng, rng.randint(1, 3))}.{_rand_digits(rng, 2)}e{e}" for _ in range(50)]
    for _ in range(40000):
        ip = _rand_digits(rng, rng.randint(1, 8)); fp = _rand_digits(rng, rng.randint(1, 16 - len(ip)))
        ff.append(f"{ip}.{fp}e-{rng.randint(1, 300)}")
    add("fastfloat", ff)
    # CSV float32: the <= 15-digit decimals nearest the midpoint above a random float32 in every binade of [1e-22, 1e37], exact
    # midpoints, and cells just outside the fast path
    cv = ["0.00364231679122895", "9.88259625955834e-6", "633014029798867000", "6.33014029798867e17", "3.54756748566783e+25", "2.06239255692255e+35",
          "16777217", "16777219", "-16777217", "1.6777217e7", "16777217.000", "8388608.5", "8388609.5", "33554434", "33554438"]
    for b in range(-73, 123):
        for _ in range(40):
            x = float(np.float32((1 + rng.random()) * 2.0 ** b))
            y = float(np.nextafter(np.float32(x), np.float32(np.inf)))
            mid = (Fraction(x) + Fraction(y)) / 2
            if not (Fraction(1, 10 ** 22) <= mid <= 10 ** 37):
                continue
            D, e10 = _double_digits(mid)
            for L in (15, 14, 13, 9):
                if L < len(D):
                    head = int(D[:L]) + (int(D[L]) >= 5); e = e10 + len(D) - L
                    cv += [f"{head + d}e{e}" for d in (-1, 0, 1)]
    for _ in range(3000):                                             # exact midpoints with <= 15 digits: binades 2^13 .. 2^49
        k = rng.randint(13, 49)
        x = float(np.float32((1 + rng.random()) * 2.0 ** k))
        y = float(np.nextafter(np.float32(x), np.float32(np.inf)))
        D, e10 = _double_digits((Fraction(x) + Fraction(y)) / 2)
        if len(D) <= 15:
            cv.append(_spell(rng, D, e10))
    cv += ["1234567890123456", "1e23", "1e-23", "12345678901234.5e9", "1.5e23", "3.5e38", "1e39", "-3.4028236e38", "3.4028235e38",
           "999999999999999e22", "1e-22", "0.0000000000000000000001", "1e-45", "1.4e-45"]
    add("csv", cv)
    return out


QUIRKS = [      # ParseFloat(s, 64), stated by hand: ("ok", value) / ("syntax", None) / ("host", Go's value), for a JSON string cell
    ("+1.5", "ok", 1.5), ("-1.5", "ok", -1.5), ("inf", "ok", math.inf), ("Inf", "ok", math.inf), ("+INF", "ok", math.inf),
    ("-infinity", "ok", -math.inf), ("Infinity", "ok", math.inf), ("+iNfInItY", "ok", math.inf), ("nan", "ok", math.nan), ("NaN", "ok", math.nan),
    ("NAN", "ok", math.nan), ("+nan", "syntax", None), ("-NaN", "syntax", None), ("infinit", "syntax", None), ("infinityx", "syntax", None),
    ("1.", "ok", 1.0), ("-1.", "ok", -1.0), (".5", "ok", 0.5), ("-.5", "ok", -0.5), (".", "syntax", None), ("-", "syntax", None), ("", "syntax", None),
    ("1.2.3", "syntax", None), ("1_000.5", "host", 1000.5), ("1e1_0", "host", 1e10), ("0x1p-2", "host", 0.25), ("-0x1.8p1", "host", -3.0),
    ("0x_1p0", "host", 1.0), ("0x1", "syntax", None), ("0x", "syntax", None), ("0xp1", "syntax", None), ("1e", "syntax", None), ("1e+", "syntax", None),
    ("e5", "syntax", None), ("1e0000000000000000000000005", "ok", 1e5), ("1e-00000000000000000000000005", "ok", 1e-5),
    ("00000000000000000000000001.5", "ok", 1.5), ("1.5 ", "syntax", None), (" 1.5", "syntax", None), ("-0", "ok", -0.0), ("0e-5", "ok", 0.0),
]


@functools.lru_cache(maxsize=None)
def paths():
    return [go_parse_path(s) for _, s in corpus()]


def _stats(tag, classes, host):
    by = Counter(classes); hc = Counter(c for c, h in zip(classes, host) if h)
    print(f"{tag}: " + ", ".join(f"{c} {by[c]} (host {hc[c]})" for c in sorted(by)))


# ------------------------------------------------------------------------------------------------ CPU: tables
def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_eisel_lemire_table_from_definition():
    """el_tables.cuh: for q in [EL_QMIN, EL_QMAX] the 128-bit mantissa of 10^q, normalised to a set top bit, rounded down."""
    src = _read("el_tables.cuh")
    qmin = int(re.search(r"#define EL_QMIN \((-?\d+)\)", src).group(1)); qmax = int(re.search(r"#define EL_QMAX \((-?\d+)\)", src).group(1))
    rows = [(int(lo, 16), int(hi, 16)) for lo, hi in re.findall(r"\{0x([0-9a-f]{16})ull, 0x([0-9a-f]{16})ull\}", src)]
    assert (qmin, qmax) == (-348, 347) and len(rows) == qmax - qmin + 1
    lo, hi = q_range()
    assert qmin <= lo and hi <= qmax and (lo, hi) == (-326, 308)
    for q, (tlo, thi) in zip(range(qmin, qmax + 1), rows):
        v = Fraction(10) ** q
        k = 127 - (v.numerator.bit_length() - v.denominator.bit_length())        # v * 2^k in [2^127, 2^128)
        m = v * Fraction(2) ** k
        if m < 2 ** 127:
            m *= 2
        elif m >= 2 ** 128:
            m /= 2
        want = m.numerator // m.denominator
        assert want >> 127 == 1 and (thi << 64 | tlo) == want, q


def test_ryu_tables_from_definition():
    """ryu_tables.cuh: POW5_INV_SPLIT[i] = floor(2^j / 5^i) + 1 with j = bitlen(5^i) - 1 + 125; POW5_SPLIT[i] = the top 125 bits of 5^i."""
    src = _read("ryu_tables.cuh")
    inv_src, spl_src = src.split("RYU_POW5_SPLIT")
    pairs = lambda t: [int(lo) | int(hi) << 64 for lo, hi in re.findall(r"\{(\d+)u, (\d+)u\}", t)]
    inv, spl = pairs(inv_src), pairs(spl_src)
    assert len(inv) == 342 and len(spl) == 326
    for i, v in enumerate(inv):
        p = 5 ** i
        assert v == (1 << (p.bit_length() - 1 + 125)) // p + 1, i
    for i, v in enumerate(spl):
        p = 5 ** i; sh = p.bit_length() - 125
        assert v == (p >> sh if sh >= 0 else p << -sh) and v.bit_length() == 125, i


# ------------------------------------------------------------------------------------------------ CPU: the corpus itself
def test_corpus_covers_the_parser():
    """Computed from the corpus alone: every Eisel-Lemire row of the reachable q range is read by a decided literal, the
    truncation check decides both ways, and every `return` of d_go_parse_float is reached (the quirk table supplies the syntax ones)."""
    c = corpus(); ps = paths()
    assert len(c) > 900_000
    lo, hi = q_range()
    used = {el[0] for _, el in ps if el}
    assert set(range(lo, hi + 1)) <= used, sorted(set(range(lo, hi + 1)) - used)[:10]
    kinds = Counter(p for p, _ in ps)
    assert kinds["el_trunc"] > 1000 and kinds["host_trunc_disagree"] > 1000, kinds
    reached = set(kinds) | {go_parse_path(s)[0] for s, _, _ in QUIRKS}
    assert reached == GO_RETURNS, (GO_RETURNS - reached, reached - GO_RETURNS)
    _stats("classes", [k for k, _ in c], [go_host(p) for p, _ in ps])
    print("paths:", dict(sorted(kinds.items())))


def test_references_agree():
    """strtof against exact Fraction rounding, the Eisel-Lemire prototype against float() wherever it decides, and the quirk table."""
    c = corpus(); rng = random.Random(7)
    sample = [s for k, s in c if k == "csv"] + [s for _, s in rng.sample(c, 20000)]
    for s in sample:
        assert strtof_bits(s) == f32_round_bits(Fraction(s)), s
    for (_, s), (p, el) in zip(c, paths()):
        if el:
            assert el[1] == b64(abs(float(s))), (s, p, hex(el[1]))
    for s, kind, v in QUIRKS:
        p, _ = go_parse_path(s)
        assert (kind == "host") == go_host(p) and (kind == "syntax") == p.startswith("syntax"), (s, p)
        if kind != "syntax" and s.lower().lstrip("+-") not in ("nan",) and not s.startswith(("0x", "-0x")) and "_" not in s:
            assert float(s) == v or (math.isnan(v) and math.isnan(float(s))), s


# ------------------------------------------------------------------------------------------------ CPU: the oracle against the references
def _json_lines(lits, quoted):
    q = '"' if quoted else ""
    return "\n".join('{"d":%s%s%s}' % (q, s, q) for s in lits).encode() + b"\n"


def _split_rows(n, errs, vals):
    """Row errors [(row, code, col)] + the values of the rows without one, in order -> {row: ("err", code) | ("v", value)}."""
    err = {r: c for r, c, _ in errs}
    ok = [r for r in range(n) if r not in err]
    assert len(ok) == len(vals)
    out = {r: ("err", c) for r, c in err.items()}
    out.update({r: ("v", v) for r, v in zip(ok, vals)})
    return out


def _want64(s):
    """ParseFloat(s, 64) of plain decimal text: (bits, None) or (None, "range")."""
    x = float(s)
    return (None, "range") if math.isinf(x) else (b64(x), None)


def test_oracle_json_string_cells_equal_float(po):
    lits = [s for _, s in corpus()]
    b, errs, n = po.json_parse(_json_lines(lits, True), REQUIRED_D)
    got = _split_rows(n, errs, b.columns[0].values.view(np.uint64).tolist())
    for r, s in enumerate(lits):
        bits, err = _want64(s)
        assert got[r] == (("err", abi.TF_ROWERR_JSON_PARSEVAL) if err else ("v", bits)), (s, got[r])


def test_oracle_json_numbers_fastfloat_structure(po):
    lits = [s for _, s in corpus() if JSON_NUMBER.fullmatch(s)]
    b, errs, n = po.json_parse(_json_lines(lits, False), [{"name": "d", "type": "double"}])
    assert not errs and n == len(lits)
    vals = b.columns[0].values.tolist()
    seen = Counter()
    for s, v in zip(lits, vals):
        k = ff_path(s); seen[k] += 1
        if k == "slow":
            assert v == float(s) and math.copysign(1, v) == math.copysign(1, float(s)), (s, v)
        elif k == "int":
            assert v == float(int(s)), (s, v)
    assert min(seen.values()) > 1000, seen


@pytest.mark.parametrize("tf", ["double", "float"])
def test_oracle_csv_float_cells(po, tf):
    """CSV double: float(cell); CSV float: ParseFloat(cell, 32) = strtof, one rounding (the five cells that fail through the double
    included); cells outside the fast path are TF_ROWERR_CSV_UNSUPPORTED."""
    lits = [s for _, s in corpus() if len(s) < 60]
    text = "".join(f"{s},x\n" for s in lits).encode()
    b, errs, _, _ = po.csv_parse(text, [{"name": "v", "type": tf, "path": "0"}, {"name": "k", "type": "utf8", "path": "1"}])
    vals = b.columns[0].values.view(np.uint64 if tf == "double" else np.uint32).tolist()
    got = _split_rows(len(lits), errs, vals)
    for r, s in enumerate(lits):
        if not csv_fast(s):
            assert got[r] == ("err", abi.TF_ROWERR_CSV_UNSUPPORTED), (s, got[r])
        else:
            assert got[r] == ("v", b64(float(s)) if tf == "double" else strtof_bits(s)), (s, got[r])
    if tf == "float":
        five = {"0.00364231679122895": 0x3b6eb3ef, "9.88259625955834e-6": 0x3725cd6d, "6.33014029798867e17": 0x5d0c8eaf,
                "3.54756748566783e+25": 0x69eac221, "2.06239255692255e+35": 0x7a1ee185, "16777217": 0x4b800000}
        for s, bits in five.items():
            assert got[lits.index(s)] == ("v", bits), s
        assert got[lits.index("633014029798867000")] == ("err", abi.TF_ROWERR_CSV_UNSUPPORTED)       # 18 digits: trailing zeros count


def test_oracle_strictify_string_to_float32(po):
    """cast.ToFloat32E(string) = ParseFloat(s, 32): one rounding, and a range error (a cast error) beyond the float32 range."""
    c = corpus(); rng = random.Random(3)
    sample = [s for k, s in c if k == "csv"] + [s for _, s in rng.sample(c, 5000)]
    for s in sample:
        rc, out = po.strictify_value("string", s, abi.TF_FLOAT)
        want = strtof_bits(s)
        if want & 0x7FFFFFFF == 0x7F800000:
            assert rc == 1, (s, rc, out)
        else:
            assert rc == 0 and out["go"] == "float32" and struct.unpack("<I", struct.pack("<f", float(out["v"])))[0] == want, (s, out, hex(want))
    for s, rc_want in (("3.4028235e38", 0), ("3.40282356e38", 0), ("3.4028236e38", 1), ("-3.4028236e38", 1), ("1e39", 1), ("-1e39", 1), ("1e-50", 0), ("inf", 0), ("1e400", 1), ("x", 1)):
        assert po.strictify_value("string", s, abi.TF_FLOAT)[0] == rc_want, s


# ------------------------------------------------------------------------------------------------ GPU: the device against the references
def _timed(label, fn):
    t0 = time.perf_counter(); r = fn(); print(f"{label}: {time.perf_counter() - t0:.2f} s"); return r


@pytest.mark.gpu
def test_device_json_string_cells_parsefloat64(eng):
    """JSON string cell -> double: d_go_parse_float. Every row is float(text) (or the range error), or TF_ROWERR_JSON_HOST exactly
    where the hand-off rule says so."""
    c = corpus(); lits = [s for _, s in c] + [s for s, _, _ in QUIRKS]
    pid = eng.plan("db", "t", REQUIRED_D, [])
    b, errs, n = _timed("device json string cells", lambda: eng.parse_json(pid, _json_lines(lits, True)))
    assert n == len(lits)
    got = _split_rows(n, errs, b.columns[0].values.view(np.uint64).tolist())
    host = []
    for r, s in enumerate(lits):
        p, _ = go_parse_path(s)
        host.append(go_host(p) or len(s) > 96)          # a string cell longer than 96 bytes is never converted on the device
        if host[-1]:
            assert got[r] == ("err", abi.TF_ROWERR_JSON_HOST), (s, p, got[r])
        elif p.startswith("syntax") or p == "overflow":
            assert got[r] == ("err", abi.TF_ROWERR_JSON_PARSEVAL), (s, p, got[r])
        elif p == "special_nan":
            assert got[r] == ("v", GO_NAN), (s, got[r])
        else:
            assert got[r] == ("v", b64(float(s))), (s, p, got[r], hex(b64(float(s))))
    _stats("json string cells", [k for k, _ in c] + ["quirks"] * len(QUIRKS), host)


@pytest.mark.gpu
def test_device_json_numbers_fastfloat(eng, po):
    """JSON number -> double (d_ff_best), -> the canonical `any` text and -> datetime (the double's |x| cut to int64 seconds, as
    amd64 converts: out of range gives INT64_MIN): the oracle bit for bit, fall-back rows equal float(text),
    integer-only rows float(int(text)); host rows exactly the fall-back rows the hand-off rule gives to the host (plus, for the
    `any` text, ±Inf, which encoding/json cannot write)."""
    lits = [s for _, s in corpus() if JSON_NUMBER.fullmatch(s)]
    fields = [{"name": "d", "type": "double"}, {"name": "a", "type": "any"}, {"name": "t", "type": "datetime"}]
    text = "\n".join('{"d":%s,"a":%s,"t":%s}' % (s, s, s) for s in lits).encode()
    pid = eng.plan("db", "t", fields, [])
    b, errs, n = _timed("device json numbers", lambda: eng.parse_json(pid, text))
    ref, rerr, rn = po.json_parse(text, fields)
    assert n == rn == len(lits)
    got = _split_rows(n, errs, list(range(b.nrows)))
    want = _split_rows(n, rerr, list(range(ref.nrows)))
    dv = b.columns[0].values.view(np.uint64); a = b.columns[1]
    rv = ref.columns[0].values.view(np.uint64); ra = ref.columns[1]
    dt, rt = b.columns[2].values.view(np.int64), ref.columns[2].values.view(np.int64)
    host = []
    for r, s in enumerate(lits):
        k = ff_path(s)
        if want[r][0] == "err":          # the oracle too hands a line to the host when its `any` cell would be ±Inf
            assert want[r] == ("err", abi.TF_ROWERR_JSON_HOST) and math.isinf(float(s)), (s, want[r])
            assert got[r] == want[r], (s, got[r])
            host.append(True)
            continue
        j = want[r][1]; x = f64(int(rv[j]))
        if k == "slow":
            assert x == float(s) and math.copysign(1, x) == math.copysign(1, float(s)), s
        elif k == "int":
            assert x == float(int(s)), s
        h = k == "slow" and go_host(go_parse_path(s)[0])
        host.append(h)
        if h:
            assert got[r] == ("err", abi.TF_ROWERR_JSON_HOST), (s, k, got[r])
            continue
        assert got[r][0] == "v", (s, got[r])
        i = got[r][1]
        assert int(dv[i]) == int(rv[j]), (s, hex(int(dv[i])), hex(int(rv[j])))
        gtext = bytes(a.heap[a.offsets[i]:a.offsets[i + 1]]); rtext = bytes(ra.heap[ra.offsets[j]:ra.offsets[j + 1]])
        assert gtext == rtext == go_json_float(x).encode(), (s, gtext, rtext)
        ax = abs(x)
        assert int(dt[i]) == int(rt[j]) == (int(ax) if ax < 2.0 ** 63 else -(1 << 63)), (s, int(dt[i]), int(rt[j]))
    _stats("json numbers", [ff_path(s) for s in lits], host)


@pytest.mark.gpu
@pytest.mark.parametrize("tf", ["double", "float"])
def test_device_csv_float_cells(eng, tf):
    """CSV double: float(cell); CSV float: strtof(cell), rounded once (the five cells above and exact midpoints such as 16777217
    included); outside the fast path TF_ROWERR_CSV_UNSUPPORTED, never a stored value — float32 overflow included."""
    c = corpus()
    lits = [s for _, s in c if len(s) < 60]
    schema = [{"name": "v", "type": tf, "path": "0"}, {"name": "k", "type": "utf8", "path": "1"}]
    pid = eng.plan("db", "t", schema, [])
    text = "".join(f"{s},x\n" for s in lits).encode()
    b, errs, consumed = _timed(f"device csv {tf}", lambda: eng.parse_csv(pid, text))
    assert consumed == len(text)
    got = _split_rows(len(lits), errs, b.columns[0].values.view(np.uint64 if tf == "double" else np.uint32).tolist())
    host = []
    for r, s in enumerate(lits):
        fast = csv_fast(s); host.append(not fast)
        if not fast:
            assert got[r] == ("err", abi.TF_ROWERR_CSV_UNSUPPORTED), (s, got[r])
        else:
            want = b64(float(s)) if tf == "double" else strtof_bits(s)
            assert got[r] == ("v", want), (s, got[r], hex(want))
    for s in ("3.5e38", "1e39", "-3.4028236e38", "1e-45", "1e23", "1234567890123456"):
        assert got[lits.index(s)] == ("err", abi.TF_ROWERR_CSV_UNSUPPORTED), s
    _stats(f"csv {tf}", [k for k, s in c if len(s) < 60], host)


@pytest.mark.gpu
def test_device_number_to_float_cells(eng):
    """number_to_float over `any` cells holding one literal each: encoding/json's float64 text of float(literal); a literal that
    overflows keeps its text; TF_ROWERR_N2F_HOST exactly where the hand-off rule says so."""
    c = corpus()
    lits = [s for _, s in c if JSON_NUMBER.fullmatch(s)]
    n = len(lits)
    schema = [{"name": "id", "type": "int32", "key": True}, {"name": "a", "type": "any"}]
    batch = abi.Batch(n, [abi.fixed_to_column(abi.TF_INT32, list(range(n))), abi.strings_to_column(abi.TF_ANY, [s.encode() for s in lits])])
    pid = eng.plan("db", "t", schema, [{"number_to_float_transformer": {}}], {"type": "clickhouse"})
    out, errs = _timed("device number_to_float", lambda: eng.push_columns(pid, batch))
    a = out.columns[1]
    got = _split_rows(n, errs, [bytes(a.heap[a.offsets[i]:a.offsets[i + 1]]) for i in range(out.nrows)])
    host = []
    for r, s in enumerate(lits):
        p, _ = go_parse_path(s); host.append(go_host(p))
        if go_host(p):
            assert got[r] == ("err", abi.TF_ROWERR_N2F_HOST), (s, p, got[r])
            continue
        x = float(s)
        assert got[r] == ("v", (s if math.isinf(x) else go_json_float(x)).encode()), (s, got[r])
    _stats("number_to_float", [k for k, s in c if JSON_NUMBER.fullmatch(s)], host)


def _vsd(s):
    """A decimal literal as io.debezium.data.VariableScaleDecimal: (base64 of the unscaled integer's minimal big-endian two's
    complement, scale, the decimal text the receiver's Base64ToNumeric gives it, the byte count), or None for an exponent too far out
    to write that way."""
    m = re.fullmatch(r"([+-]?)(\d*)(?:\.(\d*))?(?:[eE]([+-]?\d+))?", s)
    fp = m.group(3) or ""
    u = int((m.group(2) + fp) or "0"); e = int(m.group(4) or 0) - len(fp)
    if e > 0:
        if e > 400:
            return None
        u *= 10 ** e; e = 0
    u = -u if m.group(1) == "-" else u
    scale = -e
    if scale > 10 ** 4:
        return None
    raw = u.to_bytes((u if u >= 0 else ~u).bit_length() // 8 + 1, "big", signed=True)
    digits = str(abs(u)) if u else ""
    if not digits:
        text = "0"
    elif scale == 0:
        text = digits
    else:
        digits = digits.rjust(scale + 1, "0") if scale > len(digits) else digits
        text = digits[:len(digits) - scale] + "." + digits[len(digits) - scale:]
    return base64.b64encode(raw).decode(), scale, ("-" if u < 0 else "") + text, len(raw)


@pytest.mark.gpu
def test_device_debezium_double_and_variable_scale_decimal(eng):
    """Debezium `double` fields (a JSON number through d_go_parse_float) and VariableScaleDecimal fields (Base64ToNumeric text, then
    d_go_parse_float), in schema-registry frames, one literal per message. double: float(text), DBZ_UNPARSED on a syntax or range
    error, DBZ_HOST exactly where the hand-off rule says so. VariableScaleDecimal: float() of the receiver's text, DBZ_HOST exactly
    where the rule says so or where the value is wider than the device converts (more than 32 bytes, scale above 200, text over 256
    bytes)."""
    from transferia_b200 import engine
    c = corpus()
    fr = lambda p: b"\x00" + (7).to_bytes(4, "big") + p
    st = '{"type":"struct","fields":[{"type":"struct","fields":[%s],"optional":true,"field":"before"},{"type":"struct","fields":[%s],"optional":true,"field":"after"}]}'
    cases = {
        "double": ('{"type":"double","optional":true,"field":"x"}', [(k, s) for k, s in c if JSON_NUMBER.fullmatch(s)]),
        "vsd": ('{"type":"struct","fields":[],"optional":true,"name":"io.debezium.data.VariableScaleDecimal","version":1,"field":"x"}',
                [(k, s) for k, s in c if _vsd(s)]),
    }
    for name, (field, rows) in cases.items():
        schema_text = st % (field, field)
        if name == "double":
            msgs = [fr(b'{"after":{"x":%s},"op":"c"}' % s.encode()) for _, s in rows]
        else:
            enc = [_vsd(s) for _, s in rows]
            msgs = [fr(b'{"after":{"x":{"scale":%d,"value":"%s"}},"op":"c"}' % (scale, b.encode())) for b, scale, _, _ in enc]
        data = b"".join(msgs); ends = np.cumsum([len(x) for x in msgs]).tolist()
        pid = eng.plan("public", "t", engine.debezium_table_schema(schema_text), [])
        got, errs, meta = _timed(f"device debezium {name}", lambda: eng.parse_debezium(pid, data, ends, schema_text, schema_registry=True, schema_id=7))
        sel = list(meta["selection"]); vals = got.columns[0].values.view(np.uint64)
        assert len(sel) == got.nrows and len(sel) + len(errs) == len(msgs) and all(col == 0 for _, _, col in errs)
        res = {r: ("err", code) for r, code, _ in errs}
        res.update({int(r): ("v", int(v)) for r, v in zip(sel, vals)})
        host = []
        for r, (_, s) in enumerate(rows):
            if name == "double":
                p = go_parse_path(s)[0]
                h = go_host(p)
                want = ("err", abi.TF_ROWERR_DBZ_HOST) if h else ("err", abi.TF_ROWERR_DBZ_UNPARSED) if p == "overflow" or p.startswith("syntax") else ("v", b64(float(s)))
            else:
                _, scale, text, nbytes = enc[r]
                h = nbytes > 32 or scale > 200 or len(text) > 256
                if not h:
                    p = go_parse_path(text)[0]
                    h = go_host(p) or p == "overflow"
                want = ("err", abi.TF_ROWERR_DBZ_HOST) if h else ("v", b64(float(text)))
            host.append(h)
            assert res[r] == want, (name, s, res[r], want)
        _stats(f"debezium {name}", [k for k, _ in rows], host)
