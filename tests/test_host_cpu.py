"""CPU-side tests of the product's host logic: the C-ABI library loads and exports every declared symbol,
the host plan builder (filter grammar, Suitable/ResultSchema, ClickHouse types) agrees with the oracle's
restatement, batch dealing for N GPUs, and the engine refuses to run without a device (no CPU fallback)."""
import json
import os
import re
import subprocess
import sys
import ctypes as C

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from transferia_b200 import abi, dispatch, engine, workload


def test_library_exports_every_declared_symbol():
    """Every function the headers declare has one prototype in the binding's table of its header, with the header's parameter count, and
    the library exports it with that prototype applied."""
    from transferia_b200 import sink
    hdr = "".join(open(os.path.join(ROOT, "include", h)).read() for h in sorted(os.listdir(os.path.join(ROOT, "include"))) if h.endswith(".h"))
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(tfgpu_\w+)\s*\(", hdr))
    bound = set(engine.EXPORTED_SYMBOLS) | set(sink.SINK_SYMBOLS)
    assert declared == bound, declared ^ bound
    L = engine.load_library()
    for name in declared:
        assert hasattr(L, name), name
    assert L.tfgpu_version().decode().startswith("tfgpu ") and b"sm_90a" in L.tfgpu_version()
    proto = r"^\s*(?:const\s+)?\w+(?:\s*\*)?\s+(tfgpu_\w+)\s*\(([^;{]*?)\)\s*;"
    for h, table in (("tfgpu.h", abi.TFGPU_H_PROTOTYPES), ("tfgpu_sink.h", abi.TFGPU_SINK_H_PROTOTYPES)):
        text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", h)).read(), flags=re.S)
        params = dict(re.findall(proto, text, flags=re.M | re.S))
        assert set(params) == set(re.findall(r"\b(tfgpu_\w+)\s*\(", text)) == set(table), (h, set(params) ^ set(table))
        for name, args in params.items():
            n = 0 if args.strip() in ("", "void") else args.count(",") + 1
            assert len(table[name][1]) == n, (name, table[name][1], args)
    assert abi.PROTOTYPES == {**abi.TFGPU_H_PROTOTYPES, **abi.TFGPU_SINK_H_PROTOTYPES}
    for name, (restype, argtypes) in abi.PROTOTYPES.items():
        f = getattr(L, name)
        assert f.restype is restype and list(f.argtypes) == argtypes, name


def test_library_is_sm90a_native():
    import shutil
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([tool, "-lelf", engine.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(engine.EngineError) as ei:
        engine.Engine(0)
    assert ei.value.rc == engine.TF_E_FATAL_NODEVICE and not ei.value.retriable


def test_product_does_not_import_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "transferia_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle|pyoracle|liboracle|#include\s+\"[^\"]*oracle", src, flags=re.M), f


def _terms_from_describe(d):
    out = []
    for st in d["steps"]:
        if st["type"] == "filter_rows":
            out.append([[(t["col"], t["op"], t["vtype"], t["value"]) for t in e] for e in st["exprs"]])
    return out


def _oracle_terms(plan, po):
    out = []
    for st in plan.steps:
        if st["kind"] != "filter_rows":
            continue
        exprs = []
        for e in st["exprs"]:
            row = []
            for col, t in e:
                base = t.vtype & 15
                enc = lambda v: (v.hex() if base == po.LV_STRING else (None if base == po.LV_NULL else v))
                val = [enc(x) for x in t.value] if t.vtype & po.LV_LIST else enc(t.value)
                row.append((col, t.op, t.vtype, val))
            exprs.append(row)
        out.append(exprs)
    return out


def test_plan_matches_oracle_on_reference_filters(po, goldens):
    """Every filter string of filter_rows_test.go through the product's C++ grammar vs the oracle's."""
    for case in goldens["filter_rows"]:
        schema = [{"name": "column", "type": case["type"], "key": True, "required": False}]
        trs = [{"filter_rows": {"filter": case["filter"]}}]
        d = engine.plan_validate("db", "table", schema, trs, {"type": "clickhouse"})
        plan = po.build_plan("db", "table", schema, trs)
        assert _terms_from_describe(d) == _oracle_terms(plan, po), case["name"]


def test_plan_headline_and_result_schema(po):
    schema = workload.hits_schema()
    trs = workload.headline_transformers(1234) + [{"mask_field": {"columns": ["userid", "url"], "maskFunctionHash": {"userDefinedSalt": "s"}}}]
    d = engine.plan_validate("public", "hits", schema, trs, {"type": "clickhouse"})
    plan = po.build_plan("public", "hits", schema, trs)
    assert [c["type"] for c in d["result_schema"]] == [c["type"] for c in plan.result_schema]
    assert [c["name"] for c in d["result_schema"]] == [c["name"] for c in schema]
    assert d["sink"]["columns"] == [po.ch_type(c) for c in plan.result_schema]
    assert [s["type"] for s in d["steps"]] == ["filter_rows", "mask_field"]
    assert d["steps"][1]["cols"] == plan.steps[1]["cols"]
    masked = [c for c in d["result_schema"] if c["name"] in ("userid", "url")]
    assert all(c["type"] == "utf8" and c["original_type"] == "" for c in masked)


def test_plan_suitable_rules():
    schema = [{"name": "colstr", "type": "utf8"}, {"name": "colint", "type": "int32"}]
    # filter_rows_test.go "Compare different types": not Suitable -> transformer dropped from the plan
    d = engine.plan_validate("db", "table", schema, [{"filter_rows": {"filter": 'colstr > 10 AND colint = "str"'}}])
    assert d["steps"] == []
    # missing column -> not Suitable
    assert engine.plan_validate("db", "table", schema[:1], [{"filter_rows": {"filter": 'colstr = "s" AND colint > 4'}}])["steps"] == []
    # table include / exclude (transformer_common.go:9-33: matches `db.table` or `"db"."table"`)
    t = {"filter_rows": {"tables": {"includeTables": ["^db\\.table$"]}, "filter": "colint > 4"}}
    assert len(engine.plan_validate("db", "table", schema, [t])["steps"]) == 1
    assert engine.plan_validate("db", "other", schema, [t])["steps"] == []
    # MatchAnyTableNameVariant: ANY variant passing the filter is enough, so an exclude that only hits the quoted
    # form does not exclude the table, one that hits both forms does
    t2 = {"filter_rows": {"tables": {"excludeTables": ['^"db"\\."table"$']}, "filter": "colint > 4"}}
    assert len(engine.plan_validate("db", "table", schema, [t2])["steps"]) == 1
    t3 = {"filter_rows": {"tables": {"excludeTables": ["table"]}, "filter": "colint > 4"}}
    assert engine.plan_validate("db", "table", schema, [t3])["steps"] == []
    # mask_field with no matching column is not Suitable (hmac_hasher.go:76-89)
    assert engine.plan_validate("db", "table", schema, [{"mask_field": {"columns": ["nope"], "maskFunctionHash": {"userDefinedSalt": "x"}}}])["steps"] == []


def test_plan_config_errors_are_fatal():
    schema = [{"name": "c", "type": "int32"}]
    for trs in ([{"filter_rows": {"filter": 'c = str"'}}], [{"filter_rows": {"filter": "c IN 5"}}],
                [{"filter_rows": {"filter": "c > 1", "filters": ["c > 2"]}}], [{"no_such_transformer": {}}]):
        with pytest.raises(engine.EngineError) as ei:
            engine.plan_validate("db", "t", schema, trs)
        assert ei.value.rc < 0
    with pytest.raises(engine.EngineError):
        engine.plan_validate("db", "t", [{"name": "c", "type": "decimal"}], [])


def test_partition_rows():
    for n in (0, 1, 7, 8, 1000003):
        for w in (1, 2, 3, 8):
            parts = dispatch.partition_rows(n, w)
            assert parts[0][0] == 0 and parts[-1][1] == n and all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
            sizes = [hi - lo for lo, hi in parts]
            assert max(sizes) - min(sizes) <= 1


def test_round_robin_dispatcher_keeps_order():
    import time, random
    seen = [[] for _ in range(3)]

    def mk(i):
        def w(b):
            time.sleep(random.random() * 0.01); seen[i].append(b); return b * 10
        return w
    d = dispatch.RoundRobinDispatcher([mk(i) for i in range(3)])
    assert list(d.run(range(50))) == [b * 10 for b in range(50)]
    assert seen[0] == list(range(0, 50, 3)) and seen[1] == list(range(1, 50, 3))
    d.close()


def test_batch_slice_equals_oracle_on_parts(po):
    """Row-sharding invariant used for N GPUs: the kept-row count over shards sums to the whole batch's."""
    batch, schema = workload.make_hits_batch(3000)
    trs = workload.headline_transformers(workload.counterid_threshold(batch, schema))
    plan = po.build_plan("public", "hits", schema, trs)
    whole = po.push_encode(batch, plan, abi.TF_WIRE_CH_NATIVE)
    parts = [po.push_encode(batch.slice(lo, hi), plan, abi.TF_WIRE_CH_NATIVE) for lo, hi in dispatch.partition_rows(batch.nrows, 4)]
    assert sum(p.rows_out for p in parts) == whole.rows_out


_GLOO_WORKER = r'''
import os, sys, json
sys.path.insert(0, sys.argv[1])
import torch, torch.distributed as dist
from transferia_b200 import abi, dispatch, workload
from oracle import pyoracle as po
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
batch, schema = workload.make_hits_batch(4000)
trs = workload.headline_transformers(workload.counterid_threshold(batch, schema))
plan = po.build_plan("public", "hits", schema, trs)
lo, hi = dispatch.partition_rows(batch.nrows, world)[rank]
res = po.push_encode(batch.slice(lo, hi), plan, abi.TF_WIRE_CH_NATIVE)
t = torch.tensor([res.rows_out, hi - lo], dtype=torch.int64)
dist.all_reduce(t)
if rank == 0:
    whole = po.push_encode(batch, plan, abi.TF_WIRE_CH_NATIVE)
    print(json.dumps({"sum_rows_out": int(t[0]), "sum_rows_in": int(t[1]), "whole_rows_out": whole.rows_out, "nrows": batch.nrows}))
dist.destroy_process_group()
'''


def test_two_rank_gloo_sharding(tmp_path):
    """world_size-2 run of the N>1 path on CPU (gloo): shards by rank, no data-path collective, the only
    exchange is the result count (what bench.py all-reduces)."""
    script = tmp_path / "w.py"; script.write_text(_GLOO_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29611", str(script), ROOT], capture_output=True, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    line = [l for l in p.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    assert d["sum_rows_in"] == d["nrows"] and d["sum_rows_out"] == d["whole_rows_out"]


def test_plan_filter_columns_skip_events_rename(po):
    """filter_columns_transformer.go:215-236, skip_events.go:52-66, rename.go:46-67 — plan-level agreement with the oracle."""
    schema = [{"name": "id", "type": "int32", "key": True, "required": True}, {"name": "a", "type": "utf8"}, {"name": "b", "type": "int64"}, {"name": "secret", "type": "utf8"}]
    trs = [
        {"skip_events": {"events": ["delete", "truncate"]}},
        {"rename_tables": {"renameTables": [{"originalName": {"nameSpace": "db", "name": "t"}, "newName": {"nameSpace": "dst", "name": "t2"}}]}},
        {"filter_rows": {"tables": {"includeTables": ["^db\\.t$"]}, "filter": "b > 5"}},     # Suitable by the original id, but Apply sees dst.t2
        {"filter_columns": {"columns": {"excludeColumns": ["^secret$"]}}},
        {"filter_rows": {"filter": "secret = 'x'"}},                                          # column gone -> not Suitable
        {"mask_field": {"columns": ["a"], "maskFunctionHash": {"userDefinedSalt": "s"}}},
    ]
    d = engine.plan_validate("db", "t", schema, trs, {"type": "clickhouse"})
    plan = po.build_plan("db", "t", schema, trs)
    assert d["result_table"] == "dst.t2" and plan.result_table == ("dst", "t2")
    assert d["out_cols"] == plan.out_cols == [0, 1, 2]
    assert [s["type"] for s in d["steps"]] == [s["kind"] for s in plan.steps] == ["skip_events", "rename_tables", "filter_rows", "filter_columns", "mask_field"]
    assert d["steps"][2]["pass_all"] is True and plan.steps[2]["pass_all"] is True
    assert d["steps"][0]["kind_mask"] == plan.steps[0]["kind_mask"] == 4
    assert [c["name"] for c in d["result_schema"]] == ["id", "a", "b"] and d["result_schema"][1]["type"] == "utf8"
    # a primary key cannot be dropped: the transformer is simply not Suitable
    d2 = engine.plan_validate("db", "t", schema, [{"filter_columns": {"columns": {"includeColumns": ["^a$"]}}}])
    assert d2["steps"] == [] and d2["out_cols"] == [0, 1, 2, 3]
    assert po.build_plan("db", "t", schema, [{"filter_columns": {"columns": {"includeColumns": ["^a$"]}}}]).out_cols == [0, 1, 2, 3]


def test_bench_reference_arm_line(tmp_path):
    """`bench.py --impl reference` (the CPU port of the path, no GPU): one JSON line with the contract's keys, the same metric / unit as the
    GPU arm, an e2e block without copies and a cpu_baseline describing the run."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--rows", "20000", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300, cwd=root)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "rows/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and "workload" in d["config"]


def test_plan_fuzz_product_vs_oracle(po):
    """Random transformer chains over a mixed schema: the product's C++ plan builder (libtfgpu.so, host only) and the oracle's Python
    restatement of transformation.AddTablePlan must agree on which transformers are Suitable, on the columns each one touches, on the
    result schema and on the surviving columns — or both must refuse the chain."""
    import random
    rnd = random.Random(20240923)
    types = ["int8", "int16", "int32", "int64", "uint8", "uint32", "uint64", "float", "double", "boolean", "string", "utf8", "any", "date", "datetime", "timestamp", "interval"]
    names = ["id", "a", "b", "c_x", "c_y", "ts", "payload", "n1", "n2", "flag"]
    agreed = refused = 0
    for it in range(1500):
        ncol = rnd.randint(2, len(names))
        schema = [{"name": names[k], "type": rnd.choice(types), "key": k == 0, "required": rnd.random() < 0.3} for k in range(ncol)]
        ints = [c["name"] for c in schema if c["type"] in ("int8", "int16", "int32", "int64", "uint8", "uint32", "uint64")]

        def cols_cfg():
            k = rnd.random()
            pool = [c["name"] for c in schema] + ["^c_", "nope", "^n"]
            if k < 0.25:
                return {}
            if k < 0.65:
                return {"includeColumns": rnd.sample(pool, rnd.randint(1, 3))}
            return {"excludeColumns": rnd.sample(pool, rnd.randint(1, 2))}

        def tables_cfg():
            k = rnd.random()
            return {} if k < 0.6 else ({"includeTables": ["^db\\.t$"]} if k < 0.8 else {"excludeTables": ["^db\\.t$"]} if k < 0.9 else {"includeTables": ["other"]})

        chain = []
        for _ in range(rnd.randint(1, 4)):
            k = rnd.choice(["filter_rows", "skip_events", "filter_columns", "rename_tables", "mask_field", "convert_to_string", "convert_to_datetime", "number_to_float_transformer", "sharder_transformer", "replace_primary_key"])
            if k == "replace_primary_key":
                chain.append({k: {"tables": tables_cfg(), "keys": rnd.sample([c["name"] for c in schema] + ["nope"], rnd.randint(1, 3))}})
            elif k == "filter_rows":
                if not ints:
                    continue
                chain.append({k: {"tables": tables_cfg(), "filter": f"{rnd.choice(ints)} > {rnd.randint(-5, 5)}"}})
            elif k == "skip_events":
                chain.append({k: {"tables": tables_cfg(), "events": rnd.sample(["insert", "update", "delete"], rnd.randint(1, 2))}})
            elif k == "filter_columns":
                chain.append({k: {"tables": tables_cfg(), "columns": cols_cfg()}})
            elif k == "rename_tables":
                chain.append({k: {"renameTables": [{"originalName": {"nameSpace": "db", "name": "t"}, "newName": {"nameSpace": "db2", "name": "u"}}]}})
            elif k == "mask_field":
                chain.append({k: {"tables": tables_cfg(), "columns": rnd.sample([c["name"] for c in schema] + ["nope"], rnd.randint(1, 2)), "maskFunctionHash": {"userDefinedSalt": "s"}}})
            elif k == "convert_to_string":
                chain.append({k: {"tables": tables_cfg(), "columns": cols_cfg(), "convert_to_bytes": rnd.random() < 0.3}})
            elif k == "convert_to_datetime":
                chain.append({k: {"tables": tables_cfg(), "columns": cols_cfg()}})
            elif k == "number_to_float_transformer":
                chain.append({k: {"tables": tables_cfg()}})
            else:
                chain.append({k: {"tables": tables_cfg(), "columns": cols_cfg(), "shardsCount": str(rnd.randint(1, 9))}})
        if not chain:
            continue
        try:
            d = engine.plan_validate("db", "t", schema, chain)
        except engine.EngineError:
            d = None
        try:
            plan = po.build_plan("db", "t", schema, chain)
        except (NotImplementedError, ValueError):
            plan = None
        if d is None:
            # combinations the device does not model (a column rewritten twice, a filter behind a mask of its column, ...) may be refused
            # by the product only; the oracle applies steps one after another and has no such limits
            refused += 1
            continue
        assert plan is not None, chain
        agreed += 1
        # (a number_to_float that is Suitable but touches nothing — no `any` column left, or the table was renamed away from its filter —
        # keeps its place in the chain on both sides; only the product lists it)
        dsteps = [s for s in d["steps"] if not (s["type"] == "number_to_float_transformer" and not s["cols"])]
        psteps = [s for s in plan.steps if not (s["kind"] == "number_to_float" and not s["cols"])]
        assert [s["type"] for s in dsteps] == [{"number_to_float": "number_to_float_transformer", "sharder": "sharder_transformer"}.get(s["kind"], s["kind"]) for s in psteps], (schema, chain)
        assert [c["name"] for c in d["result_schema"]] == [c["name"] for c in plan.result_schema], (schema, chain)
        assert [c["type"] for c in d["result_schema"]] == [c["type"] for c in plan.result_schema], (schema, chain)
        assert [bool(c["key"]) for c in d["result_schema"]] == [bool(c.get("key")) for c in plan.result_schema], (schema, chain)
        assert d["out_cols"] == plan.out_cols, (schema, chain)
        assert d["result_table"] == ".".join(x for x in plan.result_table if x), (schema, chain)
        for ds, ps in zip(dsteps, psteps):
            if "cols" in ds and "cols" in ps:
                assert ds["cols"] == ps["cols"], (ds, ps, chain)
    assert agreed > 900 and refused < 600, (agreed, refused)


def test_filter_grammar_fuzz_product_vs_oracle(po):
    """Random filter_rows expressions (every operator, literal kind, list, quoting style, AND chains, several `filters`) through the
    product's C++ grammar and the oracle's Python restatement of the yandex-cloud filter grammar: same terms or both a syntax error."""
    import random
    rnd = random.Random(7)
    cols = {"i": "int64", "u": "uint32", "d": "double", "s": "utf8", "y": "string", "b": "boolean", "t": "timestamp", "dt": "date"}
    schema = [{"name": n, "type": t, "key": n == "i"} for n, t in cols.items()]

    def lit(kind):
        if kind == "int":
            return str(rnd.choice([0, 1, -1, 42, 2**31, -2**63, 2**63 - 1, 2**64 - 1, 10**20, -10**20]))
        if kind == "float":
            return rnd.choice(["1.5", "-0.25", "10.0", "1e3", "2.5E-3", ".5", "5.", "1e400", "-1e-400", "00.1"])
        if kind == "str":
            body = rnd.choice(["str", "", "a b", "☺", "it''s", 'say \\"hi\\"', "x\\\\y", "tab\\tq", "%like%", "O'Neil", 'dq"in'])
            q = rnd.choice(['"', "'"])
            return q + body + q
        if kind == "bool":
            return rnd.choice(["true", "false", "TRUE", "False"])
        if kind == "null":
            return rnd.choice(["NULL", "null", "Null"])
        return rnd.choice(["1990-07-22T00:00:00+04:00", "2003-04-17T10:19:00.001+03:00", "2020-01-01T00:00:00Z", "2020-01-01", "2020-13-01T00:00:00Z", "1970-01-01T00:00:00.123456789Z"])

    kinds = ["int", "float", "str", "bool", "null", "time"]
    ops = ["=", "!=", "<", "<=", ">", ">=", "~", "!~", "IN", "NOT IN", "in", "not in"]
    same = errs = 0
    for it in range(6000):
        terms = []
        for _ in range(rnd.randint(1, 3)):
            col, op = rnd.choice(list(cols)), rnd.choice(ops)
            if op.upper().endswith("IN"):
                k = rnd.choice(kinds)
                val = "(" + rnd.choice([", ", ",", " , "]).join(lit(k if rnd.random() < 0.85 else rnd.choice(kinds)) for _ in range(rnd.randint(1, 4))) + ")"
                if rnd.random() < 0.05:
                    val = lit(k)                                   # IN without a list: a syntax error
            else:
                val = lit(rnd.choice(kinds))
            terms.append(f"{col}{rnd.choice([' ', '  '])}{op}{rnd.choice([' ', ''])}{val}" if op in ("=", "!=", "<", "<=", ">", ">=", "~", "!~") else f"{col} {op} {val}")
        flt = rnd.choice([" AND ", " and ", " And "]).join(terms)
        if rnd.random() < 0.03:
            flt += rnd.choice([" AND", " OR i = 1", ")", " i"])       # broken tails
        cfg = {"filter": flt} if rnd.random() < 0.8 else {"filters": [flt, "i > 0"]}
        trs = [{"filter_rows": cfg}]
        try:
            d = engine.plan_validate("db", "t", schema, trs)
        except engine.EngineError as ex:
            d = ex
        try:
            plan = po.build_plan("db", "t", schema, trs)
        except Exception as ex:          # FilterSyntaxError / ValueError from the grammar
            plan = ex
        if isinstance(d, engine.EngineError) and d.rc == -2 and not isinstance(plan, Exception):
            continue                     # valid for the grammar, but a comparison the device does not implement (TF_E_FATAL_UNSUPPORTED)
        if isinstance(d, Exception) or isinstance(plan, Exception):
            assert isinstance(d, Exception) and isinstance(plan, Exception), (flt, d, plan)
            errs += 1
            continue
        assert _terms_from_describe(d) == _oracle_terms(plan, po), flt
        same += 1
    assert same > 1800 and errs > 50, (same, errs)


def test_replace_primary_key_plan_reference_cases(po):
    """registry/replace_primary_key/replace_primary_key_test.go:37-84: Suitable needs every new key in the schema; ResultSchema puts a
    composite key's columns first, in the order given, as the only primary keys; a single key only flips the flags."""
    def sch(cols):
        return [{"name": n, "type": "string", "key": k} for n, k in cols]
    tr = [{"replace_primary_key": {"keys": ["col1", "col2"]}}]
    cases = [([("col1", False), ("col2", False), ("col3", False)], True), ([("col2", True), ("col1", False), ("col3", True)], True),
             ([("col1", False), ("col3", False)], False), ([("col3", False), ("col1", True)], False)]
    for cols, suitable in cases:
        d = engine.plan_validate("", "t", sch(cols), tr)
        o = po.build_plan("", "t", sch(cols), tr)
        got = [(c["name"], c["key"]) for c in d["result_schema"]]
        assert got == [(c["name"], c["key"]) for c in o.result_schema]
        assert d["out_cols"] == o.out_cols
        if suitable:
            assert got[:2] == [("col1", True), ("col2", True)] and all(not k for _, k in got[2:]) and len(d["steps"]) == 1
        else:
            assert got == cols and d["steps"] == []
    one = engine.plan_validate("", "t", sch(cases[1][0]), [{"replace_primary_key": {"keys": ["col3"]}}])
    assert [(c["name"], c["key"]) for c in one["result_schema"]] == [("col2", False), ("col1", False), ("col3", True)] and one["out_cols"] == [0, 1, 2]
    with pytest.raises(engine.EngineError) as ei:                      # NewReplacePrimaryKeyTransformer: the same key twice
        engine.plan_validate("", "t", sch(cases[0][0]), [{"replace_primary_key": {"keys": ["key1", "key1"]}}])
    assert ei.value.rc == -1
    with pytest.raises(ValueError):
        po.build_plan("", "t", sch(cases[0][0]), [{"replace_primary_key": {"keys": ["key1", "key1"]}}])
    # a table filter that does not match leaves the schema alone
    d = engine.plan_validate("public", "t", sch(cases[0][0]), [{"replace_primary_key": {"keys": ["col2"], "tables": {"includeTables": ["^public.other$"]}}}])
    assert d["steps"] == [] and not any(c["key"] for c in d["result_schema"])


def test_transformation_test_multiple_transformers(po):
    """pkg/transformer/transformation_test.go:29-111 (TestMultipleTransformers): replace_primary_key [field2, field1] followed by
    filter_columns [field2, field1, field4] over four key columns -> TableSchema {field2 key, field1 key, field4 not key}; the control item and
    the insert both reach the sink (2 items). The item's values stay addressed by column NAME (the reference keeps ColumnNames / ColumnValues in
    item order, ["test", 2, "{}"]): in the columnar result every output column carries its own input column (out_cols)."""
    schema = [{"name": "field1", "type": "utf8", "key": True}, {"name": "field2", "type": "int64", "key": True},
              {"name": "field3", "type": "double", "key": True}, {"name": "field4", "type": "utf8", "key": True}]
    trs = [{"replace_primary_key": {"keys": ["field2", "field1"], "tables": {"includeTables": ["test_table"]}}},
           {"filter_columns": {"tables": {"includeTables": ["test_table"]}, "columns": {"includeColumns": ["field2", "field1", "field4"]}}}]
    d = engine.plan_validate("", "test_table", schema, trs)
    o = po.build_plan("", "test_table", schema, trs)
    want = [("field2", True), ("field1", True), ("field4", False)]
    assert [(c["name"], c["key"]) for c in d["result_schema"]] == want == [(c["name"], bool(c.get("key"))) for c in o.result_schema]
    assert d["out_cols"] == [1, 0, 3] == o.out_cols and [s["type"] for s in d["steps"]] == ["replace_primary_key", "filter_columns"]
    # through Sinker.Push: the init_load_table item travels alone, then the row — 2 items at the sink, as the reference asserts
    from transferia_b200 import rows, sink
    from transferia_b200.rows import ChangeItem, go
    s = sink.Sink()        # (the always-on middleware alone: the chain itself is checked above and on the device in tests/test_gpu_parity.py)
    s.push(rows.RowsImage([ChangeItem(rows.KIND_INIT_TABLE_LOAD, 0), ChangeItem(rows.KIND_INSERT, 0, [go.string("test"), go.int64(2), go.float64(1.23), go.string("{}")])],
                          [("", "test_table", schema)]))
    assert [e["n_items"] for e in s.events] == [1, 1] and s.stats()["change_items_pushed"] == 2
    s.close()


def test_headers_are_plain_c(tmp_path):
    """The boundary is a C ABI: both headers compile as C99 (`gcc -std=c99 -pedantic`), and the struct sizes the Python binding assumes are the
    ones the C compiler lays out."""
    src = tmp_path / "hdr.c"
    src.write_text('#include <stdio.h>\n#include "tfgpu.h"\n#include "tfgpu_sink.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(tf_col), sizeof(tf_batch), sizeof(tf_item), sizeof(tf_rows), sizeof(tf_table),'
                   ' sizeof(tf_sink_event), sizeof(tf_sink_stats)); return 0; }\n')
    exe = tmp_path / "hdr"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [C.sizeof(abi.TfCol), C.sizeof(abi.TfBatch), C.sizeof(abi.TfItem), C.sizeof(abi.TfRows), C.sizeof(abi.TfTable), C.sizeof(abi.TfSinkEvent), C.sizeof(abi.TfSinkStats)]
    assert got == want, (got, want)


def test_c_example_compiles_links_and_refuses_without_a_device(tmp_path):
    """examples/push_clickhouse.c — plain C99 against the two headers, linked against libtfgpu.so: every symbol it uses resolves; without a GPU
    the program stops at tfgpu_engine_create (no CPU fallback)."""
    exe = tmp_path / "push_clickhouse"
    subprocess.run(["gcc", "-std=c99", "-D_POSIX_C_SOURCE=200809L", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "push_clickhouse.c"), "-L", os.path.dirname(engine.LIB_PATH), "-ltfgpu", "-o", str(exe)], check=True)
    import torch
    if torch.cuda.is_available():
        return
    r = subprocess.run([str(exe)], capture_output=True, text=True, env=dict(os.environ, LD_LIBRARY_PATH=os.path.dirname(engine.LIB_PATH)))
    assert r.returncode == 1 and "no CPU fallback" in r.stderr


def test_name_filter_reference_cases(po):
    """registry/filter/filter_test.go:9-33 (TestFilter): empty filter, exclude only, include + exclude, exclude wins over include, a bad regexp
    is a construction error — through convert_to_string's column filter (the same filter.Filter) in the product's plan and the oracle's."""
    schema = [{"name": n, "type": "int32"} for n in ("include", "exclude", "other", "any_value")]
    def converted(cols_cfg):
        trs = [{"convert_to_string": {"columns": cols_cfg}}]
        d = engine.plan_validate("", "t", schema, trs); o = po.build_plan("", "t", schema, trs)
        got = [c["name"] for c in d["result_schema"] if c["type"] == "utf8"]
        assert got == [c["name"] for c in o.result_schema if c["type"] == "utf8"]
        return got
    assert converted({}) == ["include", "exclude", "other", "any_value"]
    assert converted({"excludeColumns": ["exclude"]}) == ["include", "other", "any_value"]
    assert converted({"includeColumns": ["include"], "excludeColumns": ["exclude"]}) == ["include"]
    assert converted({"includeColumns": ["include", "other.*"], "excludeColumns": [".*other.*"]}) == ["include"]
    with pytest.raises(engine.EngineError) as ei:
        engine.plan_validate("", "t", schema, [{"convert_to_string": {"columns": {"includeColumns": ["include", "*"], "excludeColumns": [".*other.*"]}}}])
    assert ei.value.rc == -1
    # the expressions are Go's (regexp.Compile), not ECMAScript's: \z, \A, POSIX classes, named groups; what the library's engine does not
    # carry is an unsupported plan, not a silently different match
    def product_only(cols_cfg):
        d = engine.plan_validate("", "t", schema, [{"convert_to_string": {"columns": cols_cfg}}])
        return [c["name"] for c in d["result_schema"] if c["type"] == "utf8"]
    assert product_only({"includeColumns": [r"\Aother\z"]}) == ["other"]
    assert product_only({"includeColumns": [r"^[[:lower:]]+_[[:alpha:]]+$"]}) == ["any_value"]
    assert product_only({"includeColumns": [r"^(?P<stem>in|ex)clude$"]}) == ["include", "exclude"]
    assert product_only({"includeColumns": ["(?i)^INCLUDE$"]}) == ["include"]
    with pytest.raises(engine.EngineError) as ei:
        product_only({"includeColumns": [r"^\pL+$"]})
    assert ei.value.rc == -2


def test_skip_events_and_rename_reference_cases():
    """registry/filter/skip_events_test.go (TestSkipEvents): table1 with delete / truncate / drop_table skipped -> init_load, done_load, insert and
    update remain, in order; table2 is not Suitable. registry/rename/rename_test.go (TestRenameTableTransformer): public.objects_0 ->
    service.objects, public.objects untouched. Both through Sinker.Push (kinds and table names are host decisions)."""
    from transferia_b200 import rows, sink
    from transferia_b200.rows import ChangeItem, go
    K = rows
    schema = [{"name": "id", "type": "int32"}]
    kinds = [K.KIND_DROP_TABLE, K.KIND_TRUNCATE, K.KIND_INIT_TABLE_LOAD, K.KIND_DONE_TABLE_LOAD, K.KIND_INSERT, K.KIND_UPDATE, K.KIND_DELETE]
    items = [ChangeItem(k, t, [go.int32(i)] if k <= 2 else None) for t in (0, 1) for i, k in enumerate(kinds)]
    s = sink.Sink(transformers=[{"skip_events": {"tables": {"includeTables": ["table1"]}, "events": ["delete", "truncate", "drop_table"]}}])
    s.push(rows.RowsImage(items, [("", "table1", schema), ("", "table2", schema)]))
    per_table = {0: [], 1: []}
    for e in s.events:
        per_table[e["table"]] += [items[i].kind for i in e["items"]]
    assert per_table[0] == [K.KIND_INIT_TABLE_LOAD, K.KIND_DONE_TABLE_LOAD, K.KIND_INSERT, K.KIND_UPDATE] and per_table[1] == kinds
    s.close()
    ren = {"rename_tables": {"renameTables": [{"originalName": {"nameSpace": "public", "name": "objects_0"}, "newName": {"nameSpace": "service", "name": "objects"}},
                                              {"originalName": {"nameSpace": "public", "name": "objects_1"}, "newName": {"nameSpace": "service", "name": "objects"}}]}}
    s = sink.Sink(transformers=[ren])
    s.push(rows.RowsImage([ChangeItem(K.KIND_INSERT, 0, [go.int32(1)]), ChangeItem(K.KIND_INSERT, 1, [go.int32(2)]), ChangeItem(K.KIND_DDL, 1)],
                          [("public", "objects", schema), ("public", "objects_0", schema)]))
    assert [e["out"] for e in s.events] == [("public", "objects"), ("service", "objects"), ("service", "objects")]
    s.close()
