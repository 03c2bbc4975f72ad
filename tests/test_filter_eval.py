"""filter_rows row evaluation at the value edges: the device (k_filter / eval_term) and the oracle (match_value) against a Python
restatement of FilterRowsTransformer.Apply / matchItem / matchExpression / matchValue (pkg/transformer/registry/filter_rows/
filter_rows.go:99-383, util.go:47-107) written from the Go, not from either C++ implementation.

The parsed terms come from the product's describe JSON, so the filter grammar is not restated here a second time; Suitable
(checkColumnSuitable, filter_rows.go:489-519) is, to know which filter_rows steps the plan keeps."""
import functools
import math
import random

import numpy as np
import pytest

from transferia_b200 import abi, engine

TF_E_FATAL_CONFIG, TF_E_FATAL_UNSUPPORTED = -1, -2
KIND, OVERFLOW, TYPEPAIR = abi.TF_ROWERR_FILTER_KIND, abi.TF_ROWERR_FILTER_OVERFLOW, abi.TF_ROWERR_FILTER_TYPEPAIR
INSERT, UPDATE, DELETE = abi.TF_KIND_INSERT, abi.TF_KIND_UPDATE, abi.TF_KIND_DELETE
# filter.OperatorType (library/go/yandex/cloud/filter/filters.go:12-23) and the describe JSON's literal kinds
EQ, NE, LT, LE, GT, GE, IN, NOTIN, MATCH, NOTMATCH = range(10)
LV_INT, LV_FLOAT, LV_BOOL, LV_STRING, LV_TIME, LV_NULL, LV_LIST = 1, 2, 3, 4, 5, 6, 16
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1

NUMERIC = ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float", "double")
TEXT = ("utf8", "string", "any")
TIMES = ("date", "datetime", "timestamp")


# ----------------------------------------------------------------------------- the restatement
# A column value is the Go value a typed column carries (typesystem/values/type_checkers.go): ("nil",), ("int", i) for every
# integer type but uint64, ("uint64", u), ("float64", f), ("float32", f) (f: the float32 value, exactly), ("bool", b),
# ("string", bytes), ("bytes", bytes), ("time", sec, nsec), ("duration", ns), ("opaque", text) (an `any` value that is not a string).

class RowError(Exception):
    def __init__(self, code):
        super().__init__(code)
        self.code = code


def to_int64e(v):
    """toInt64E (util.go:47-79): every Go integer type; a uint64 above MaxInt64 is errIntOverflow. None: not an integer."""
    if v[0] == "int":
        return v[1]
    if v[0] == "uint64":
        if v[1] > I64_MAX:
            raise RowError(OVERFLOW)
        return v[1]
    return None


PARSE_FLOAT = object()      # cast.ToFloat64E of a Go string is strconv.ParseFloat: the plan refuses numeric literals on text columns


def to_float64e(v):
    """spf13/cast v1.7.1 ToFloat64E for the Go types of typed columns. None: an error (time.Duration, time.Time, []byte, JSON trees)."""
    k = v[0]
    if k in ("float64", "float32"):
        return v[1]                                   # float64(float32) widens exactly
    if k in ("int", "uint64"):
        return float(v[1])                            # float64(int): round to nearest even, as Python's int -> float
    if k == "bool":
        return 1.0 if v[1] else 0.0
    if k == "nil":
        return 0.0
    if k == "string":
        return PARSE_FLOAT
    return None


def go_trunc(f):
    return f if math.isinf(f) or math.isnan(f) else float(math.trunc(f))


def go_f2i64(f):
    """int64(float64) on amd64 (CVTTSD2SQ): truncation, and 0x8000000000000000 for NaN and everything outside the int64 range."""
    return int(f) if -2.0 ** 63 <= f < 2.0 ** 63 else I64_MIN


def set_contains(values, x):
    """set.Set[interface{}].Contains: a Go map lookup, so == semantics: NaN is never found, -0 finds 0."""
    return any(y == x for y in values)


def ordered(a, b, op):
    """matchOrderedValue / matchBytesValue (filter_rows.go:367-401): no ~ / !~ there, an error instead."""
    if op == EQ: return a == b
    if op == NE: return a != b
    if op == LT: return a < b
    if op == LE: return a <= b
    if op == GT: return a > b
    if op == GE: return a >= b
    raise RowError(TYPEPAIR)


def unix_micro(sec, nsec):
    """time.Time.UnixMicro: sec*1e6 + nsec/1e3 in int64 arithmetic (nsec is never negative, so the division floors)."""
    return (sec * 10 ** 6 + nsec // 1000 + 2 ** 63) % 2 ** 64 - 2 ** 63


def match_value(v, op, vtype, lit):
    """matchValue (filter_rows.go:180-365). Errors are RowError(TF_ROWERR_*)."""
    base, is_list = vtype & 15, bool(vtype & LV_LIST)
    is_set = op in (IN, NOTIN)
    in_set = lambda c: c if op == IN else not c
    int1 = to_int64e(v)                               # the overflow error comes before any literal is looked at (:190-197)
    is_int1 = int1 is not None
    float1 = None if is_int1 else to_float64e(v)
    is_float1 = float1 is not None
    if base in (LV_INT, LV_FLOAT):
        assert float1 is not PARSE_FLOAT, "numeric literal against a Go string: the plan refuses it"
    if base == LV_INT:                                # :213-241
        if is_int1:
            return in_set(int1 in lit) if is_set else ordered(int1, lit, op)
        if is_float1:
            if is_set:
                return in_set(go_f2i64(float1) in lit) if go_trunc(float1) == float1 else False
            return ordered(float1, float(lit), op)
    elif base == LV_FLOAT:                            # :243-267
        if is_int1 or is_float1:
            x = float(int1) if is_int1 else float1
            return in_set(set_contains(lit, x)) if is_set else ordered(x, lit, op)
    elif base == LV_BOOL:                             # :269-285 (a bool list is refused when the transformer is built)
        assert not is_list
        if v[0] == "bool":
            return ordered(int(v[1]), int(lit), op)
    elif base == LV_STRING:                           # :287-328
        if not is_list and v[0] == "bytes":
            if op == MATCH: return lit in v[1]        # bytes.Contains
            if op == NOTMATCH: return lit not in v[1]
            return ordered(v[1], lit, op)             # bytes.Compare: bytewise
        if v[0] in ("bytes", "string"):
            s = v[1]
            if op == MATCH: return lit in s           # strings.Contains
            if op == NOTMATCH: return lit not in s
            return in_set(s in lit) if is_set else ordered(s, lit, op)
    elif base == LV_TIME:                             # :330-351
        assert v[0] != "string", "stringToTime: the plan refuses time literals on text columns"
        if v[0] == "time":
            um = unix_micro(v[1], v[2])
            return in_set(um in lit) if is_set else ordered(um, lit, op)
    elif base == LV_NULL:                             # :353-358
        if op == EQ: return v[0] == "nil"
        if op == NE: return v[0] != "nil"
    raise RowError(TYPEPAIR)                          # :364 "Unsupported type pair"


def match_expression(terms, match):
    """matchExpression (:150-177): AND; a false term ends it before the terms after it are evaluated."""
    for t in terms:
        if not match(t):
            return False
    return True


def match_item(exprs, match):
    """matchItem (:137-148): OR over `filters`; the first error ends the row, a matched expression skips the rest."""
    for e in exprs:
        if match_expression(e, match):
            return True
    return False


def run_chain(steps, kind, match):
    """One ChangeItem through the chain: (kept, (code, step index) or None). SkipEvents.Apply (filter/skip_events.go:52-62) and
    FilterRowsTransformer.Apply (filter_rows.go:99-130): update / delete rows are an error of the filter_rows step."""
    for si, st in enumerate(steps):
        if st["type"] == "skip_events":
            if kind in st["kinds"]:
                return False, None
            continue
        if kind in (UPDATE, DELETE):
            return False, (KIND, si)
        try:
            if not match_item(st["exprs"], match):
                return False, None
        except RowError as e:
            return False, (e.code, si)
    return True, None


def literal(t):
    """The literal of a describe JSON term. A float literal is printed with %.17g, which keeps every finite double (the grammar
    refuses the rest, as strconv.ParseFloat does); -0.0 comes back as 0, which no comparison and no Go map lookup tells apart."""
    base = t["vtype"] & 15
    conv = {LV_INT: int, LV_TIME: int, LV_FLOAT: float, LV_BOOL: bool, LV_STRING: bytes.fromhex, LV_NULL: lambda x: None}[base]
    return [conv(x) for x in t["value"]] if t["vtype"] & LV_LIST else conv(t["value"])


def suitable(kind, is_list, typ):
    """checkColumnSuitable (filter_rows.go:489-519) for a literal kind of the generator."""
    if is_list:
        return kind in ("int", "float", "str", "time")
    return {"bool": typ == "boolean", "int": typ in NUMERIC, "float": typ in NUMERIC, "str": typ in TEXT, "time": typ in TIMES,
            "null": True}[kind]


class Restated:
    """The restatement over one batch: column values as distinct Go values + a per-row index, so that every term is evaluated once
    per distinct value of its column."""

    def __init__(self, values, kinds):
        self.n = len(kinds)
        self.kinds = [int(k) for k in kinds]
        self.distinct, self.idx = [], []
        for col in values:
            keys, d, ix = {}, [], []
            for v in col:
                key = repr(v)                          # repr keeps -0.0 / NaN apart from 0.0 / each other
                if key not in keys:
                    keys[key] = len(d); d.append(v)
                ix.append(keys[key])
            self.distinct.append(d); self.idx.append(ix)
        self.memo = {}

    def term_results(self, t):
        if id(t) not in self.memo:
            lit, res = literal(t), []
            for v in self.distinct[t["col"]]:
                try:
                    res.append(1 if match_value(v, t["op"], t["vtype"], lit) else 0)
                except RowError as e:
                    res.append(-e.code)
            self.memo[id(t)] = (res, self.idx[t["col"]], t)          # (t: keeps the id taken)
        return self.memo[id(t)]

    def apply(self, steps):
        """(kept rows, [(row, code, step)]). Rows with the same kind and the same values in the columns the terms read have the
        same outcome: the chain runs once per such signature."""
        cols = sorted({t["col"] for st in steps for e in st.get("exprs", ()) for t in e})
        outcome = {}
        kept, errors = [], []
        for r in range(self.n):
            sig = (self.kinds[r],) + tuple(self.idx[c][r] for c in cols)
            if sig not in outcome:
                def match(t):
                    res, ix, _ = self.term_results(t)
                    x = res[ix[r]]
                    if x < 0:
                        raise RowError(-x)
                    return x == 1
                outcome[sig] = run_chain(steps, self.kinds[r], match)
            ok, err = outcome[sig]
            if ok:
                kept.append(r)
            elif err:
                errors.append((r, err[0], err[1]))
        return kept, errors

    def encode_errors(self, kept, errors):
        """What a ClickHouse wire format adds: update / delete rows that survive the chain come back as TF_ROWERR_SINK_KIND_HOST."""
        extra = [(r, abi.TF_ROWERR_SINK_KIND_HOST, 0xff) for r in kept if self.kinds[r] != INSERT]
        return [r for r in kept if self.kinds[r] == INSERT], sorted(errors + extra)


def chain_steps(trs, describe):
    """The restatement's steps: skip_events from the config, filter_rows terms from the describe JSON."""
    steps = []
    for tr, d in zip(trs, describe["steps"]):
        (ttype, cfg), = tr.items()
        assert d["type"] == ttype
        if ttype == "skip_events":
            steps.append({"type": ttype, "kinds": {{"insert": INSERT, "update": UPDATE, "delete": DELETE}[e] for e in cfg["events"]}})
        else:
            assert not d["pass_all"]
            steps.append({"type": ttype, "exprs": d["exprs"]})
    return steps


# ----------------------------------------------------------------------------- pinned by filter_rows_test.go

def _golden_value(case, x):
    go = case["go"]
    if go == "mixed":
        return ("uint64" if x[0] == "uint64" else "int", x[1])
    if go == "int": return ("int", x)
    if go == "float64": return ("float64", x)
    if go == "bool": return ("bool", x)
    if go == "string": return ("string", x.encode())
    if go == "bytes": return ("bytes", x.encode())
    import datetime as dt
    us = (dt.datetime.fromisoformat(x) - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(microseconds=1)
    return ("time", us // 10 ** 6, (us % 10 ** 6) * 1000)


def test_restatement_reproduces_reference_filter_cases(goldens):
    """Every filter_rows_test.go case, on the Go values the Go test feeds (float64 even for the float column): kept rows and errors."""
    assert len(goldens["filter_rows"]) == 45
    for case in goldens["filter_rows"]:
        schema = [{"name": "column", "type": case["type"], "key": True, "required": False}]
        trs = [{"filter_rows": {"filter": case["filter"]}}]
        d = engine.plan_validate("db", "table", schema, trs)
        rs = Restated([[_golden_value(case, x) for x in case["input"]]], [INSERT] * len(case["input"]))
        kept, errors = rs.apply(chain_steps(trs, d))
        val = (lambda x: x[1]) if case["go"] == "mixed" else (lambda x: x)
        assert [val(case["input"][r]) for r in kept] == case["expected"], case["name"]
        assert len(errors) == case["errors"], case["name"]
        if case.get("error_code"):
            assert {c for _, c, _ in errors} == {case["error_code"]}, case["name"]


# ----------------------------------------------------------------------------- the edge-value batch

def _int_edges(lo, hi):
    cand = [lo, lo + 1, hi - 1, hi, 0, 1, -1, 15, -16, 2 ** 53, -2 ** 53, 2 ** 53 + 1, -(2 ** 53 + 1)]
    return sorted({x for x in cand if lo <= x <= hi})


F64_EDGES = [math.nan, math.inf, -math.inf, 0.0, -0.0, 2.0 ** 63, -2.0 ** 63, 1e19, -1e19, 5e-324, 0.1, 0.5, 1.5, -0.5, -1.5, 1.0, -1.0,
             2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 63 - 1024, 1.7976931348623157e308, 127.0, 255.0]
F32_EDGES = [float(np.float32(x)) for x in (0.1, 3.4e38, math.nan, -0.0, 0.0, math.inf, -math.inf, 0.5, 1.5, 2.0 ** 63, 1e19, -1e19,
                                            16777217.0, 1.0, -1.0, 1e-45, 3.4028234663852886e38)]
STR_EDGES = [b"", b"a", b"ab", b"abc", b"b", b"A", b"~", b"\x80", b"\xff", b"a\xff", b"\xc3\xa9", b'"', b"'", b"it's \"q\"", b"://",
             b"http://x.y/", b"\x00", b"\x00a"]
TIME_EDGES = [(0, 0), (0, 999), (0, 1000), (0, 1999), (-1, 0), (-1, 999), (-1, 999999000), (-1, 999999999), (-86400, 500),
              (1577836800, 0), (1577836800, 123456000), (1577836800, 123456789), (1577836800, 123455999), (1577836799, 999999999),
              (1577836799, 999999000), (4291747199, 0), (-2208988800, 1)]
ANY_EDGES = [(1, b""), (1, b"a"), (1, b"://"), (1, b"\xff"), (0, b'{"k":1}'), (0, b"1"), (0, b'"a"'), (0, b"")]
EDGES = {
    **{t: _int_edges(int(np.iinfo(t).min), int(np.iinfo(t).max)) for t in ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32")},
    "uint64": [0, 1, 2 ** 53, 2 ** 53 + 1, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1],
    "double": F64_EDGES, "float": F32_EDGES, "boolean": [False, True], "utf8": STR_EDGES, "string": STR_EDGES,
    "date": TIME_EDGES, "datetime": TIME_EDGES, "timestamp": TIME_EDGES, "interval": [0, 1, -1, 1000, I64_MAX, I64_MIN], "any": ANY_EDGES,
}


def go_value(typ, x):
    """The Go value of one cell of a typed column (None = nil)."""
    if x is None: return ("nil",)
    if typ == "uint64": return ("uint64", x)
    if typ in NUMERIC[:7]: return ("int", x)
    if typ == "double": return ("float64", x)
    if typ == "float": return ("float32", float(np.float32(x)))
    if typ == "boolean": return ("bool", bool(x))
    if typ == "utf8": return ("string", x)
    if typ == "string": return ("bytes", x)
    if typ == "any": return ("string", x[1]) if x[0] == 1 else ("opaque", x[1])
    if typ in TIMES: return ("time", x[0], x[1])
    return ("duration", x)


def make_column(typ, vals):
    tf = abi.YT_NAME_TO_TF[typ]
    nulls = [v is None for v in vals]
    if typ in ("utf8", "string"):
        return abi.strings_to_column(tf, vals)
    if typ == "any":
        return abi.strings_to_column(tf, [None if v is None else v[1] for v in vals], tags=[0 if v is None else v[0] for v in vals])
    if typ in TIMES:
        return abi.fixed_to_column(tf, [0 if v is None else v[0] for v in vals], nulls, nanos=[0 if v is None else v[1] for v in vals])
    return abi.fixed_to_column(tf, [0 if v is None else v for v in vals], nulls)


def make_batch(spec, kinds=None):
    """spec: [(name, type, required, values)] -> (Batch, schema, Restated)."""
    n = len(spec[0][3])
    kinds = np.zeros(n, dtype=np.uint8) if kinds is None else np.asarray(kinds, dtype=np.uint8)
    schema = [{"name": nm, "type": typ, "required": req, "key": False} for nm, typ, req, _ in spec]
    batch = abi.Batch(n, [make_column(typ, vals) for _, typ, _, vals in spec], kinds)
    return batch, schema, Restated([[go_value(typ, x) for x in vals] for _, typ, _, vals in spec], kinds)


def edge_spec(n, seed=11):
    """A row id, then every type twice: required (c_<type>) and nullable (n_<type>), each cell drawn from the type's edge values;
    the first rows walk the edge list so that each value occurs."""
    rng = np.random.default_rng(seed)
    spec = [("rid", "int64", True, list(range(n)))]
    for typ, edges in EDGES.items():
        for req in (True, False):
            ix = rng.integers(0, len(edges), n)
            ix[:min(n, len(edges))] = np.arange(min(n, len(edges)))
            vals = [edges[i] for i in ix]
            if not req:
                vals = [None if z else v for v, z in zip(vals, rng.random(n) < 0.15)]
            spec.append((("c_" if req else "n_") + typ, typ, req, vals))
    return spec


def edge_kinds(n, seed=11):
    rng = np.random.default_rng(seed + 1)
    u = rng.random(n)
    return np.where(u < 0.02, UPDATE, np.where(u < 0.04, DELETE, INSERT)).astype(np.uint8)


# ----------------------------------------------------------------------------- the filter generator

INT_LITS = ["-9223372036854775808", "9223372036854775807", "0", "1", "-1", "127", "-128", "255", "9007199254740992", "9007199254740993",
            "-9007199254740993", "4294967295", "2147483647", "15"]
FLOAT_LITS = ["0.1", "-0.0", "0.0", "0.5", "1.5", "-1.5", "1.0", "10000000000000000000.0", "-10000000000000000000.0",
              "9223372036854775808.0", "9223372036854775807.0", "9007199254740993.0", "0.10000000149011612",
              "340000000000000000000000000000000000000.0", "127.0"]
STR_LITS = ['""', '"a"', "'ab'", '"abc"', '"b"', '"\\xff"', '"\\x80"', '"a\\xff"', '"~"', '"://"', "'it\\'s'", '"\\"q\\""', '"\\""', '"http"', '"\\x00"']
TIME_LITS = ["1970-01-01T00:00:00Z", "1970-01-01T00:00:00.000001Z", "1969-12-31T23:59:59.999999Z", "1969-12-31T23:59:59Z", "1970-01-01",
             "2020-01-01", "2020-01-01T00:00:00.123456Z", "2020-01-01T03:00:00.123456+03:00", "2019-12-31T23:59:59.999999Z",
             "2105-12-31T23:59:59Z", "1969-12-31T00:00:00Z"]
BOOL_LITS = ["true", "false", "TRUE"]
LITS = {"int": INT_LITS, "float": FLOAT_LITS, "str": STR_LITS, "time": TIME_LITS, "bool": BOOL_LITS}
OPS = ["=", "!=", "<", "<=", ">", ">=", "~", "!~"]


def _kinds_for(typ):
    if typ in NUMERIC: return ["int", "float", "null"]
    if typ == "boolean": return ["bool", "null", "int", "float"]
    if typ in TEXT: return ["str", "null"]
    if typ in TIMES: return ["time", "null"]
    return ["null", "int"]


class FilterGen:
    """Random chains over a schema: AND chains, `filters` OR lists, two filter_rows steps, skip_events before or after. Each
    transformer comes with the (literal kind, list?, column type) of its terms, to restate Suitable and the plan's refusals."""

    def __init__(self, schema, seed):
        self.rnd = random.Random(seed)
        self.cols = [(c["name"], c["type"]) for c in schema if c["name"] != "rid"]

    def term(self):
        rnd = self.rnd
        name, typ = rnd.choice(self.cols)
        kind = rnd.choice(_kinds_for(typ) if rnd.random() < 0.8 else ["int", "float", "str", "bool", "null", "time"])
        if kind == "null":
            return f"{name} {rnd.choice(['=', '!='])} {rnd.choice(['NULL', 'null', 'NIL'])}", (kind, False, typ)
        if kind != "bool" and rnd.random() < 0.35:
            items = ", ".join(rnd.choice(LITS[kind]) for _ in range(rnd.randint(1, 4)))
            return f"{name} {rnd.choice(['IN', 'NOT IN', 'not in', 'in'])} ({items})", (kind, True, typ)
        return f"{name} {rnd.choice(OPS)} {rnd.choice(LITS[kind])}", (kind, False, typ)

    def conj(self):
        terms = [self.term() for _ in range(self.rnd.randint(1, 3))]
        return " AND ".join(t for t, _ in terms), [k for _, k in terms]

    def filter_rows(self):
        if self.rnd.random() < 0.3:
            fs = [self.conj() for _ in range(self.rnd.randint(2, 3))]
            return {"filter_rows": {"filters": [f for f, _ in fs]}}, [k for _, ks in fs for k in ks]
        f, ks = self.conj()
        return {"filter_rows": {"filter": f}}, ks

    def chain(self):
        rnd = self.rnd
        trs = [self.filter_rows()]
        if rnd.random() < 0.25:
            trs.append(self.filter_rows())
        if rnd.random() < 0.25:
            ev = rnd.sample(["update", "delete", "insert"], rnd.choice([1, 1, 2]))
            trs.insert(rnd.choice([0, len(trs)]), ({"skip_events": {"events": ev}}, []))
        return trs


def plan_case(schema, chain):
    """(transformers, describe, restated steps) of an accepted plan; None when the product refuses it (TF_E_FATAL_UNSUPPORTED)."""
    trs = [tr for tr, _ in chain]
    kept = [tr for tr, ks in chain if all(suitable(*k) for k in ks)]          # Suitable drops a transformer, it does not fail
    refused = any((k in ("int", "float") and typ in ("utf8", "any")) or (k == "time" and lst and typ in TEXT)
                  for tr, ks in chain if all(suitable(*x) for x in ks) for k, lst, typ in ks)
    try:
        d = engine.plan_validate("db", "t", schema, trs, {"type": "clickhouse"})
    except engine.EngineError as ex:
        assert ex.rc == TF_E_FATAL_UNSUPPORTED and refused, (trs, ex)
        return None
    assert not refused, trs
    assert [s["type"] for s in d["steps"]] == [next(iter(tr)) for tr in kept], trs
    return trs, d, chain_steps(kept, d)


N_EDGE_ROWS = 3000
N_CHAINS = 2600


@functools.lru_cache(maxsize=None)
def corpus():
    """The edge batch and the accepted plans of the generator on a fixed seed, with the restatement's result of each."""
    spec = edge_spec(N_EDGE_ROWS)
    batch, schema, rs = make_batch(spec, edge_kinds(N_EDGE_ROWS))
    gen = FilterGen(schema, seed=2024)
    cases, refused = [], 0
    for _ in range(N_CHAINS):
        c = plan_case(schema, gen.chain())
        if c is None:
            refused += 1
            continue
        trs, d, steps = c
        cases.append((trs, steps, rs.apply(steps)))
    return batch, schema, rs, cases, refused


def test_generator_is_mostly_accepted_and_reaches_every_outcome():
    batch, schema, rs, cases, refused = corpus()
    assert len(cases) >= 2000 and refused < 0.2 * N_CHAINS, (len(cases), refused)
    codes = {c for _, _, (_, errs) in cases for _, c, _ in errs}
    assert codes == {KIND, OVERFLOW, TYPEPAIR}, codes
    kept = [len(k) for _, _, (k, _) in cases]
    assert sum(0 < k < batch.nrows for k in kept) > 0.3 * len(cases)
    assert sum(len(steps) > 1 for _, steps, _ in cases) > 300
    assert sum(any(len(s.get("exprs", ())) > 1 for s in steps) for _, steps, _ in cases) > 300


def _rid(out):
    return out.columns[0].values.tolist() if out.nrows else []


def test_oracle_matches_restatement_on_edge_corpus(po):
    """The CPU oracle (push_columns) against the restatement: kept rows and (row, code, step) errors of every accepted plan."""
    batch, schema, rs, cases, _ = corpus()
    bad = []
    for trs, steps, (kept, errors) in cases:
        out, errs = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
        if _rid(out) != kept or sorted(errs) != errors:
            bad.append(trs)
    assert not bad, (len(bad), bad[:5])


# ----------------------------------------------------------------------------- directed cases
# (name, [(type, values)] as columns c0, c1, ..., transformers, kept rows, errors). Each names the rule it pins.

F32_01 = float(np.float32(0.1))
DIRECTED = [
    # int64(float64) of amd64 (CVTTSD2SQ) in IN / NOT IN against an int list: out of range is 0x8000000000000000, not a saturated value
    ("f2i_in_int64_min_double", [("double", [1e19, -1e19, 2.0 ** 63, math.inf, -math.inf, 2.0 ** 63 - 1024, -2.0 ** 63])],
     "c0 IN (-9223372036854775808)", [0, 1, 2, 3, 4, 6], []),
    ("f2i_in_int64_max_double", [("double", [1e19, 2.0 ** 63, math.inf, 2.0 ** 63 - 1024])], "c0 IN (9223372036854775807)", [], []),
    ("f2i_not_in_int64_min_double", [("double", [1e19, 2.0 ** 63, math.inf, -math.inf, 2.0 ** 63 - 1024, 1.5])],
     "c0 NOT IN (-9223372036854775808)", [4], []),
    ("f2i_not_in_int64_max_double", [("double", [1e19, 2.0 ** 63, math.inf, 2.0 ** 63 - 1024])], "c0 NOT IN (9223372036854775807)", [0, 1, 2, 3], []),
    ("f2i_in_int64_min_float", [("float", [1e19, 2.0 ** 63, math.inf, -math.inf, 3.4e38, 16777217.0])], "c0 IN (-9223372036854775808)", [0, 1, 2, 3, 4], []),
    ("f2i_in_int64_max_float", [("float", [1e19, 2.0 ** 63, math.inf, 3.4e38])], "c0 IN (9223372036854775807)", [], []),
    ("f2i_not_in_int64_max_float", [("float", [1e19, 2.0 ** 63, math.inf, 3.4e38, 16777217.0])], "c0 NOT IN (9223372036854775807, 16777216)", [0, 1, 2, 3], []),
    # float32 is widened to float64: float32(0.1) is not the literal 0.1
    ("f32_0.1_eq_literal", [("float", [0.1, 0.5])], "c0 = 0.1", [], []),
    ("f32_0.1_eq_its_float64", [("float", [0.1, 0.5])], "c0 = 0.10000000149011612", [0], []),
    ("f32_0.1_in_literal", [("float", [0.1])], "c0 IN (0.1, 0.2)", [], []),
    # NaN: every ordered operator false but !=; not found in a float set; never an integer, so IN and NOT IN an int list are false
    ("nan_eq", [("double", [math.nan])], "c0 = 1.5", [], []),
    ("nan_ne", [("double", [math.nan])], "c0 != 1.5", [0], []),
    ("nan_lt", [("double", [math.nan])], "c0 < 1.5", [], []),
    ("nan_le", [("double", [math.nan])], "c0 <= 1", [], []),
    ("nan_gt", [("double", [math.nan])], "c0 > -1.5", [], []),
    ("nan_ge", [("double", [math.nan])], "c0 >= -1", [], []),
    ("nan_ne_int", [("float", [math.nan])], "c0 != 1", [0], []),
    ("nan_in_float_list", [("double", [math.nan])], "c0 IN (1.5, 0.0)", [], []),
    ("nan_not_in_float_list", [("double", [math.nan])], "c0 NOT IN (1.5)", [0], []),
    ("nan_in_int_list", [("double", [math.nan])], "c0 IN (0)", [], []),
    ("nan_not_in_int_list", [("float", [math.nan])], "c0 NOT IN (0)", [], []),
    ("nan_match", [("double", [math.nan])], "c0 ~ 1.5", [], [(0, TYPEPAIR, 0)]),
    # -0 is 0 for == and for a Go map
    ("neg_zero_in_int_list", [("double", [-0.0])], "c0 IN (0)", [0], []),
    ("neg_zero_in_float_list", [("float", [-0.0])], "c0 IN (0.0)", [0], []),
    ("neg_zero_not_in", [("double", [-0.0, 0.0])], "c0 NOT IN (-0.0)", [], []),
    ("fraction_not_in_int_list", [("double", [0.5, 2.0])], "c0 NOT IN (7)", [1], []),
    # toInt64E: a uint64 above MaxInt64 is an overflow error whatever the literal, `= NULL` included
    ("u64_2p63_eq_null", [("uint64", [2 ** 63, 2 ** 63 - 1])], "c0 = NULL", [], [(0, OVERFLOW, 0)]),
    ("u64_max_ne_null", [("uint64", [2 ** 64 - 1, None])], "c0 != NULL", [], [(0, OVERFLOW, 0)]),
    ("u64_2p63_string_list", [("uint64", [2 ** 63, 1])], "c0 IN ('a')", [], [(0, OVERFLOW, 0), (1, TYPEPAIR, 0)]),
    ("u64_2p63_minus_1_float", [("uint64", [2 ** 63 - 1])], "c0 = 9223372036854775808.0", [0], []),
    # float64(int64) rounds: 2^53+1 equals the float literal 2^53
    ("int_2p53_plus_1_vs_float", [("int64", [2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2])], "c0 = 9007199254740992.0", [0, 1], []),
    ("int_2p53_plus_1_vs_int", [("int64", [2 ** 53, 2 ** 53 + 1])], "c0 = 9007199254740993", [1], []),
    # AND stops at a false term; OR stops at the first error or the first match
    ("error_after_false_term", [("int64", [1, 9])], "c0 > 5 AND c0 IN ('a')", [], [(1, TYPEPAIR, 0)]),
    ("error_in_first_filter", [("int64", [1])], {"filters": ["c0 IN ('a')", "c0 = 1"]}, [], [(0, TYPEPAIR, 0)]),
    ("match_before_erroring_filter", [("int64", [1, 2])], {"filters": ["c0 = 1", "c0 IN ('a')"]}, [0], [(1, TYPEPAIR, 0)]),
    # ~ / !~ exist for strings only: matchOrderedValue refuses them
    ("match_int", [("int32", [1, 2])], "c0 ~ 1", [], [(0, TYPEPAIR, 0), (1, TYPEPAIR, 0)]),
    ("notmatch_float", [("double", [1.5])], "c0 !~ 1.5", [], [(0, TYPEPAIR, 0)]),
    ("match_bool", [("boolean", [True, False])], "c0 ~ true", [], [(0, TYPEPAIR, 0), (1, TYPEPAIR, 0)]),
    ("match_time", [("timestamp", [(0, 0)])], "c0 !~ 1970-01-01", [], [(0, TYPEPAIR, 0)]),
    ("match_u64_overflow_first", [("uint64", [2 ** 63])], "c0 ~ 1", [], [(0, OVERFLOW, 0)]),
    # cast.ToFloat64E: bool is 1 / 0 and nil is 0 against int / float lists; Duration, time and []byte are refused
    ("bool_in_int_list", [("boolean", [True, False, None])], "c0 IN (1)", [0], []),
    ("nil_is_zero", [("boolean", [True, False, None])], "c0 IN (0.0)", [1, 2], []),
    ("nil_int_gt", [("int16", [None, 5])], "c0 > -1 AND c0 < 1", [0], []),
    ("duration_in_list", [("interval", [0, None])], "c0 IN (0)", [1], [(0, TYPEPAIR, 0)]),
    ("time_in_int_list", [("date", [(0, 0)])], "c0 IN (0)", [], [(0, TYPEPAIR, 0)]),
    ("bytes_in_int_list", [("string", [b"1"])], "c0 IN (1)", [], [(0, TYPEPAIR, 0)]),
    ("nil_vs_string", [("utf8", [None, b"a"])], "c0 >= 'a'", [1], [(0, TYPEPAIR, 0)]),
    # strings: bytewise order, bytes.Contains, an empty needle
    ("bytes_order_high_bit", [("string", [b"\xff", b"z", b"\x80a"])], "c0 > 'z'", [0, 2], []),
    ("utf8_order_prefix", [("utf8", [b"ab", b"a", b"", b"abc"])], "c0 < 'ab'", [1, 2], []),
    ("contains_empty", [("utf8", [b"", b"x"])], "c0 ~ ''", [0, 1], []),
    ("contains_high_bit", [("string", [b"a\xffb", b"ab"])], 'c0 ~ "\\xff"', [0], []),
    ("string_list_exact", [("string", [b"a", b"a\x00", b""])], "c0 IN ('a', '')", [0, 2], []),
    # any: a string tag is a Go string, anything else an opaque value
    ("any_tags", [("any", [(1, b"x://"), (0, b"x://"), None])], "c0 ~ '://'", [0], [(1, TYPEPAIR, 0), (2, TYPEPAIR, 0)]),
    ("any_null", [("any", [(1, b""), (0, b"{}"), None])], "c0 = NULL", [2], []),
    # time as UnixMicro: nanoseconds below 1000 truncate, before 1970 too
    ("time_negative_nanos", [("timestamp", [(-1, 999999999), (-1, 999999000), (-1, 999998999)])], "c0 = 1969-12-31T23:59:59.999999Z", [0, 1], []),
    ("time_sub_micro", [("datetime", [(0, 999), (0, 1000), (-1, 999999999)])], "c0 <= 1970-01-01T00:00:00Z", [0, 2], []),
    ("time_list", [("date", [(1577836800, 123456789), (1577836800, 123457000)])], "c0 IN (2020-01-01T00:00:00.123456Z)", [0], []),
    # kinds: update / delete rows are errors of filter_rows, unless skip_events dropped them first
    ("kind_errors", [("int8", [1, 1, 1])], "c0 = 1", [0], [(1, KIND, 0), (2, KIND, 0)]),
]
DIRECTED_KINDS = {"kind_errors": [INSERT, UPDATE, DELETE]}


def directed_case(case):
    name, cols, flt, keep, errs = case
    n = len(cols[0][1])
    spec = [("rid", "int64", True, list(range(n)))] + [(f"c{i}", typ, all(v is not None for v in vals), vals) for i, (typ, vals) in enumerate(cols)]
    batch, schema, rs = make_batch(spec, DIRECTED_KINDS.get(name))
    trs = [{"filter_rows": flt if isinstance(flt, dict) else {"filter": flt}}]
    return batch, schema, rs, trs, keep, sorted(errs)


@pytest.mark.parametrize("case", DIRECTED, ids=[c[0] for c in DIRECTED])
def test_directed_restatement_and_oracle(po, case):
    batch, schema, rs, trs, keep, errs = directed_case(case)
    d = engine.plan_validate("db", "t", schema, trs, {"type": "clickhouse"})
    assert rs.apply(chain_steps(trs, d)) == (keep, errs)
    out, oerrs = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
    assert (_rid(out), sorted(oerrs)) == (keep, errs)


def test_skip_events_around_filter_rows(po):
    """skip_events before filter_rows drops update / delete rows without an error; after it, filter_rows has already refused them."""
    spec = edge_spec(64)
    kinds = [INSERT, UPDATE, DELETE, INSERT] * 16
    batch, schema, rs = make_batch(spec, kinds)
    f = {"filter_rows": {"filter": "c_int8 != 0"}}
    for trs, n_err in (([{"skip_events": {"events": ["update", "delete"]}}, f], 0), ([f, {"skip_events": {"events": ["update", "delete"]}}], 32),
                       ([{"skip_events": {"events": ["update"]}}, f], 16)):
        d = engine.plan_validate("db", "t", schema, trs, {"type": "clickhouse"})
        kept, errors = rs.apply(chain_steps(trs, d))
        assert len(errors) == n_err and all(c == KIND for _, c, _ in errors)
        out, oerrs = po.push_columns(batch, po.build_plan("db", "t", schema, trs))
        assert (_rid(out), sorted(oerrs)) == (kept, errors)


def test_float_literal_out_of_range_is_a_syntax_error(po):
    """strconv.ParseFloat (grammar.go Float.delayedParse) refuses a literal beyond the float64 range (ErrRange): no ±Inf literal."""
    schema = [{"name": "d", "type": "double"}]
    for lit in ("1" + "0" * 400 + ".0", "-" + "9" * 309 + ".5"):
        with pytest.raises(engine.EngineError) as ei:
            engine.plan_validate("db", "t", schema, [{"filter_rows": {"filter": f"d > {lit}"}}])
        assert ei.value.rc == TF_E_FATAL_CONFIG
        with pytest.raises(po.FilterSyntaxError):
            po.build_plan("db", "t", schema, [{"filter_rows": {"filter": f"d IN (1.0, {lit})"}}])
    big = "1" + "0" * 308 + ".0"                                   # 1e308: in range
    d = engine.plan_validate("db", "t", schema, [{"filter_rows": {"filter": f"d < {big}"}}])
    assert d["steps"][0]["exprs"][0][0]["value"] == 1e308


# ----------------------------------------------------------------------------- on the device

def _device_columns(eng, batch, schema, trs):
    pid = eng.plan("db", "t", schema, trs, {"type": "clickhouse"})
    out, errs = eng.push_columns(pid, batch)
    return pid, _rid(out), sorted(errs)


@pytest.mark.gpu
@pytest.mark.parametrize("case", DIRECTED, ids=[c[0] for c in DIRECTED])
def test_directed_on_device(eng, po, case):
    batch, schema, rs, trs, keep, errs = directed_case(case)
    pid, kept, got = _device_columns(eng, batch, schema, trs)
    assert (kept, got) == (keep, errs)
    ref = po.push_encode(batch, po.build_plan("db", "t", schema, trs), abi.TF_WIRE_CH_NATIVE, eng.frame_bytes)
    enc = eng.push_encode(pid, batch, abi.TF_WIRE_CH_NATIVE)
    assert enc.wire == ref.raw and sorted(enc.errors) == sorted(ref.errors) == rs.encode_errors(keep, errs)[1]


@pytest.mark.gpu
def test_device_matches_restatement_and_oracle_on_edge_corpus(eng, po):
    """Every accepted plan of the corpus on the device: push_columns against the restatement, push_encode (native, no LZ4) against
    the oracle's block and the restatement's rows and errors."""
    batch, schema, rs, cases, _ = corpus()
    bad = []
    for trs, steps, (kept, errors) in cases:
        pid, got_kept, got_errs = _device_columns(eng, batch, schema, trs)
        enc = eng.push_encode(pid, batch, abi.TF_WIRE_CH_NATIVE)
        ref = po.push_encode(batch, po.build_plan("db", "t", schema, trs), abi.TF_WIRE_CH_NATIVE, eng.frame_bytes)
        ekept, eerrs = rs.encode_errors(kept, errors)
        if (got_kept, got_errs) != (kept, errors) or enc.wire != ref.raw or enc.rows_out != len(ekept) or sorted(enc.errors) != eerrs:
            bad.append(trs)
    assert not bad, (len(bad), bad[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 4097])
def test_device_row_counts_around_blocks_and_warps(eng, po, n):
    """k_filter runs 256-thread blocks and counts kept / failed rows by warp ballots: ragged tails of both, on 300 plans."""
    spec = edge_spec(n, seed=n)
    batch, schema, rs = make_batch(spec, edge_kinds(n, seed=n))
    gen = FilterGen(schema, seed=n)
    done = 0
    while done < 300:
        c = plan_case(schema, gen.chain())
        if c is None:
            continue
        trs, d, steps = c
        kept, errors = rs.apply(steps)
        pid, got_kept, got_errs = _device_columns(eng, batch, schema, trs)
        assert (got_kept, got_errs) == (kept, errors), trs
        if done % 10 == 0:
            enc = eng.push_encode(pid, batch, abi.TF_WIRE_CH_NATIVE)
            ref = po.push_encode(batch, po.build_plan("db", "t", schema, trs), abi.TF_WIRE_CH_NATIVE, eng.frame_bytes)
            assert enc.wire == ref.raw and sorted(enc.errors) == rs.encode_errors(kept, errors)[1], trs
        done += 1


@pytest.mark.gpu
def test_device_resident_input(eng, po):
    """push_encode_resident over the edge batch in HBM: rows, error count and native block of 40 plans."""
    batch, schema, rs, cases, _ = corpus()
    dbatch = batch.to_device("cuda:0")
    for trs, steps, (kept, errors) in cases[:40]:
        pid = eng.plan("db", "t", schema, trs, {"type": "clickhouse"})
        eng.push_encode_resident(pid, dbatch, abi.TF_WIRE_CH_NATIVE)
        st = eng.resident_stats()
        ekept, eerrs = rs.encode_errors(kept, errors)
        assert st["rows_out"] == len(ekept) and st["n_errors"] == len(eerrs), trs
        ref = po.push_encode(batch, po.build_plan("db", "t", schema, trs), abi.TF_WIRE_CH_NATIVE, eng.frame_bytes).raw
        assert eng.resident_fetch(0, st["raw_bytes"]) == ref, trs
