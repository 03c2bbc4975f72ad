"""Profiling aid (GPU): share of k_lz4_frames cycles per phase on the bench.py headline workload (watchid filter, 28 % of the
rows kept), plus per-kernel event times. TFGPU_LIB_PATH selects a build variant.  python scripts/lz4_phases.py [rows]"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transferia_b200 import abi, engine, workload
import bench

PHASES = ("stage", "match", "parse+continuation", "scan", "emit", "resolve+flush of the previous frame")   # counter k = LZ_PHASE(k)

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
batch, schema = bench.make_batch(rows, workload.SEED)
k = workload.headline_threshold(batch, schema); trs = workload.headline_transformers_watchid(k)
eng = engine.Engine(0)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); eng.set_stream(stream.cuda_stream)
pid = eng.plan("public", "hits", schema, trs, {"type": "clickhouse"})
d = batch.to_device("cuda:0")
for _ in range(3): eng.push_encode_resident(pid, d, abi.TF_WIRE_CH_NATIVE_LZ4)
torch.cuda.synchronize()
eng.lz4_phases(True)
eng.profile_enable(True)
acc = {}
for _ in range(5):
    eng.push_encode_resident(pid, d, abi.TF_WIRE_CH_NATIVE_LZ4)
    for kk in eng.profile_read(): acc[kk["name"]] = acc.get(kk["name"], 0) + kk["ms"] / 5
ph = eng.lz4_phases(True); tot = sum(ph) or 1
st = eng.resident_stats()
print(json.dumps({"kernels_ms": {n: round(v, 4) for n, v in sorted(acc.items(), key=lambda kv: -kv[1])}, "step_ms": round(sum(acc.values()), 4),
                  "lz4_phase_share": {PHASES[i]: round(ph[i] / tot, 3) for i in range(len(PHASES))},
                  "selectivity": st["rows_out"] / rows, "lz4_ratio": st["raw_bytes"] / max(1, st["wire_bytes"]), "lib": engine.LIB_PATH}))
