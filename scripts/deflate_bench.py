"""Device DEFLATE of the batch serializers' row text (TF_WIRE_F_GZIP / TF_WIRE_F_ZLIB) on a hits-shaped batch held in device memory.

For SER_JSON and SER_CSV, each without and with GZIP (and with ZLIB), it reports:
  - per-kernel CUDA-event times of one push (the mean over --reps pushes after --warmup);
  - the uncompressed text rate of the deflate kernels (text bytes / (k_deflate_chunks + k_deflate_finish));
  - the bytes copied device -> host (the result bytes) with and without compression;
  - the compression ratio beside CPython zlib levels 1 and 6 on the same text, and the single-core CPU time of zlib level 6
    (CPython's zlib, not Go's compress/flate, which is not measured here);
  - the card's name and power limit, read in the same run.
Prints one JSON object.   python scripts/deflate_bench.py [--rows 1000000] [--reps 5] [--warmup 2]"""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from transferia_b200 import abi, engine, workload  # noqa: E402

DEFLATE_KERNELS = ("k_deflate_chunks", "k_deflate_finish")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    batch, schema = workload.make_hits_batch(a.rows)
    dbatch = batch.to_device("cuda:0")
    eng = engine.Engine(0)
    pid = eng.plan("public", "hits", schema, [])
    out = {"card": card, "rows": a.rows, "formats": {}}
    for name, base in (("SER_JSON", abi.TF_WIRE_SER_JSON), ("SER_CSV", abi.TF_WIRE_SER_CSV)):
        text = eng.push_encode(pid, dbatch, base).wire
        row = {"text_bytes": len(text)}
        for cname, flag in (("plain", 0), ("gzip", abi.TF_WIRE_F_GZIP), ("zlib", abi.TF_WIRE_F_ZLIB)):
            for _ in range(a.warmup):
                eng.push_encode(pid, dbatch, base | flag, copy_bytes=False)
            acc, wall, d2h = {}, 0.0, 0
            for _ in range(a.reps):
                eng.profile_enable(True)
                t0 = time.perf_counter()
                res = eng.push_encode(pid, dbatch, base | flag, copy_bytes=False)      # returns after the result bytes landed on the host
                wall += time.perf_counter() - t0
                for k in eng.profile_read():
                    acc[k["name"]] = acc.get(k["name"], 0.0) + k["ms"]
                eng.profile_enable(False)
                d2h = res.wire_len
            kern = {k: round(v / a.reps, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])}
            r = {"kernel_ms": kern, "call_ms": round(1e3 * wall / a.reps, 3), "d2h_bytes": d2h}
            if flag:
                dms = sum(kern.get(k, 0.0) for k in DEFLATE_KERNELS)
                r["deflate_ms"] = round(dms, 4)
                r["deflate_text_GBps"] = round(len(text) / (dms * 1e-3) / 1e9, 2) if dms else None
                r["ratio"] = round(len(text) / d2h, 3)
            row[cname] = r
        for lvl in (1, 6):
            t0 = time.perf_counter(); z = zlib.compress(text, lvl); dt = time.perf_counter() - t0
            row[f"cpython_zlib_level{lvl}"] = {"ratio": round(len(text) / len(z), 3), "cpu_s_one_core": round(dt, 3),
                                               "text_MBps_one_core": round(len(text) / dt / 1e6, 1)}
        out["formats"][name] = row
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
