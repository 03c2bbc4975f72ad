"""Device zstd of the ClickHouse JSONEachRow text (TF_WIRE_F_ZSTD) on a hits-shaped batch held in device memory.

JSONEachRow without and with the flag, it reports:
  - per-kernel CUDA-event times of one push (the mean over --reps pushes after --warmup) and the text rate of each zstd kernel
    (text bytes / kernel time);
  - the bytes copied device -> host (the result bytes) and the whole-call time, with and without the flag;
  - the device's ratio beside libzstd levels 1 and -1 on the same text (one CPU core, with its time);
  - the card's name, power limit and SM clock, read in the same run.
Prints one JSON object.   python scripts/zstd_bench.py [--rows 1000000] [--reps 5] [--warmup 2]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from transferia_b200 import abi, engine, workload  # noqa: E402

ZSTD_KERNELS = ("k_zstd_chunks", "k_zstd_finish")


def libzstd(text, level):
    L = C.CDLL("libzstd.so.1")
    L.ZSTD_compressBound.argtypes = [C.c_size_t]; L.ZSTD_compressBound.restype = C.c_size_t
    L.ZSTD_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]; L.ZSTD_compress.restype = C.c_size_t
    cap = L.ZSTD_compressBound(len(text)); out = C.create_string_buffer(cap)
    t0 = time.perf_counter(); n = L.ZSTD_compress(out, cap, text, len(text), level); dt = time.perf_counter() - t0
    return {"ratio": round(len(text) / n, 3), "cpu_s_one_core": round(dt, 3), "text_MBps_one_core": round(len(text) / dt / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    batch, schema = workload.make_hits_batch(a.rows)
    dbatch = batch.to_device("cuda:0")
    eng = engine.Engine(0)
    pid = eng.plan("public", "hits", schema, [], {"type": "clickhouse"})
    text = eng.push_encode(pid, dbatch, abi.TF_WIRE_CH_JSONEACHROW).wire
    out = {"card": card, "rows": a.rows, "text_bytes": len(text)}
    for cname, flag in (("plain", 0), ("zstd", abi.TF_WIRE_F_ZSTD)):
        fmt = abi.TF_WIRE_CH_JSONEACHROW | flag
        for _ in range(a.warmup):
            eng.push_encode(pid, dbatch, fmt, copy_bytes=False)
        acc, wall, d2h = {}, 0.0, 0
        for _ in range(a.reps):
            eng.profile_enable(True)
            t0 = time.perf_counter()
            res = eng.push_encode(pid, dbatch, fmt, copy_bytes=False)      # returns after the result bytes landed on the host
            wall += time.perf_counter() - t0
            for k in eng.profile_read():
                acc[k["name"]] = acc.get(k["name"], 0.0) + k["ms"]
            eng.profile_enable(False)
            d2h = res.wire_len
        kern = {k: round(v / a.reps, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])}
        r = {"kernel_ms": kern, "call_ms": round(1e3 * wall / a.reps, 3), "d2h_bytes": d2h}
        if flag:
            r["kernel_text_GBps"] = {k: round(len(text) / (kern[k] * 1e-3) / 1e9, 2) for k in ZSTD_KERNELS if kern.get(k)}
            zms = sum(kern.get(k, 0.0) for k in ZSTD_KERNELS)
            r["zstd_ms"] = round(zms, 4)
            r["zstd_text_GBps"] = round(len(text) / (zms * 1e-3) / 1e9, 2) if zms else None
            r["ratio"] = round(len(text) / d2h, 3)
        out[cname] = r
    for lvl in (1, -1):
        out[f"libzstd_level{lvl}"] = libzstd(text, lvl)
    out["card_after"] = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"],
                                       capture_output=True, text=True).stdout.strip()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
