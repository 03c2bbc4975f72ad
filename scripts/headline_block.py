"""Writes the native block of the bench.py headline step (1 M rows, seed workload.SEED, watchid filter at 28 % kept), computed by the
CPU oracle, to a file: the input of scripts/lz4_model.cpp.  python scripts/headline_block.py OUT.bin [rows]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from transferia_b200 import abi, workload
from oracle import pyoracle as po
import bench

out = sys.argv[1]
rows = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
batch, schema = bench.make_batch(rows, workload.SEED)
k = workload.headline_threshold(batch, schema)
plan = po.build_plan("public", "hits", schema, workload.headline_transformers_watchid(k))
res = po.push_encode(batch, plan, abi.TF_WIRE_CH_NATIVE)
with open(out, "wb") as f:
    f.write(res.raw)
print(f"rows {rows} -> {res.rows_out} kept, block {len(res.raw)} B -> {out}")
