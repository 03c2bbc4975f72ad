"""The String-column kernels of the headline step (k_str_sizes, k_encode_str_plain) on the bench.py workload.

The batch, filter and call are bench.py's: a seeded 1 M-row ClickBench-shaped batch resident in device memory,
`watchid > K AND url ~ '://'` with K set for 28 % kept rows, tfgpu_push_encode_resident to the native block + LZ4.
It reports:
  - each kernel's CUDA-event time from the per-kernel profile (eng.profile_read()) of every one of --pushes pushes
    after --warmup: median, min and max;
  - the algorithmic bytes of each kernel, computed from the batch: per kept row and String column the `sel` entry (4 B)
    and the two heap offsets (8 B) both kernels gather, the payload k_encode_str_plain reads and the block bytes
    (LEB128 length + payload) it writes;
  - the achieved GB/s (algorithmic bytes / median time) beside the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s,
    a figure for the card and not one reached;
  - the card's name and power limit and the SM clock sampled while the pushes ran.
Prints one JSON object.   python scripts/str_encode_bench.py [--rows 1000000] [--pushes 50] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import ClockSampler, make_batch  # noqa: E402

KERNELS = ("k_str_sizes", "k_encode_str_plain")
DATASHEET_HBM_GBS = 3350.0       # H100 SXM data sheet, HBM3


def string_bytes(batch, schema, k):
    """Kept-row count and the algorithmic bytes of the String columns under the headline filter (same rule as bench.py's)."""
    names = [c["name"] for c in schema]
    wid = np.asarray(batch.columns[names.index("watchid")].values)
    url = np.asarray(batch.columns[names.index("url")].offsets).astype(np.int64)
    sel = np.flatnonzero((wid > k) & (np.diff(url) > 0))          # every non-empty generated URL contains "://"
    payload = block = ncols = 0
    for c in batch.columns:
        if c.offsets is None:
            continue
        L = np.diff(np.asarray(c.offsets).astype(np.int64))[sel]
        if c.validity is not None:
            L = np.where(np.unpackbits(np.asarray(c.validity), bitorder="little")[sel] > 0, L, 0)
        vl = np.ones_like(L)
        for lim in (1 << 7, 1 << 14, 1 << 21, 1 << 28):
            vl += L >= lim
        payload += int(L.sum()); block += int((L + vl).sum()); ncols += 1
    gather = 12 * len(sel) * ncols                                  # sel[j] + offsets[r], offsets[r + 1]
    return len(sel), ncols, {"k_str_sizes": {"read": gather, "written": 0},
                             "k_encode_str_plain": {"read": gather + payload, "written": block}}, payload, block


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--pushes", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if a.pushes < 1:
        raise SystemExit("--pushes must be at least 1")
    import torch
    from transferia_b200 import abi, engine, workload
    if not torch.cuda.is_available():
        raise SystemExit("str_encode_bench.py: no CUDA device (the engine has no CPU path)")
    card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    batch, schema = make_batch(a.rows, workload.SEED)
    k = workload.headline_threshold(batch, schema)
    n_kept, ncols, alg, payload, block = string_bytes(batch, schema, k)
    eng = engine.Engine(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    pid = eng.plan("public", "hits", schema, workload.headline_transformers_watchid(k), {"type": "clickhouse"})
    dbatch = batch.to_device("cuda:0")
    for _ in range(a.warmup):
        eng.push_encode_resident(pid, dbatch, abi.TF_WIRE_CH_NATIVE_LZ4)
    rows_out = eng.resident_stats()["rows_out"]
    if rows_out != n_kept:
        raise SystemExit(f"str_encode_bench.py: the engine kept {rows_out} rows, the byte count assumes {n_kept}")
    times = {n: [] for n in KERNELS}
    sampler = ClockSampler(0); sampler.start(); sampler.mark_start()
    eng.profile_enable(True)
    for _ in range(a.pushes):
        eng.push_encode_resident(pid, dbatch, abi.TF_WIRE_CH_NATIVE_LZ4)
        prof = eng.profile_read()
        for n in KERNELS:
            times[n].append(sum(x["ms"] for x in prof if x["name"] == n))
    eng.profile_enable(False)
    sampler.mark_end(); sampler.stop_flag = True; sampler.join(timeout=2)
    out = {"card": card, "clocks": sampler.result(), "lib": engine.LIB_PATH, "rows": a.rows, "kept_rows": n_kept,
           "string_columns": ncols, "payload_bytes": payload, "block_bytes": block, "pushes": a.pushes,
           "peak_basis": "3.35 TB/s: H100 SXM data-sheet HBM3 bandwidth, not a measured peak", "kernels": {}}
    for n in KERNELS:
        t = np.asarray(times[n])
        med = float(np.median(t))
        byt = alg[n]["read"] + alg[n]["written"]
        gbs = byt / (med * 1e-3) / 1e9
        out["kernels"][n] = {"ms_median": round(med, 4), "ms_min": round(float(t.min()), 4), "ms_max": round(float(t.max()), 4),
                             "alg_bytes_read": alg[n]["read"], "alg_bytes_written": alg[n]["written"],
                             "achieved_GBps": round(gbs, 1), "share_of_datasheet_hbm": round(gbs / DATASHEET_HBM_GBS, 3)}
    both = sum(out["kernels"][n]["ms_median"] for n in KERNELS)
    out["both_ms_median_sum"] = round(both, 4)
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
