"""How libtfgpu.so launches its kernels: each kernel is declared once in its family header (kernels_*.cuh) and launched from tfgpu.cu
only through TF_LAUNCH (launch.hpp), which counts the launch (tfgpu_engine_launch_count, bench `gpu_launches`) and, with profiling on,
records it under the kernel's own name (tfgpu_profile_read, bench `roofline`). The profile holds every launch of the last call that
launched anything.

On the CPU: the kernels defined, declared, compiled into the library and launched are the same set, and no other launch path is
left. On the device: every entry point's count and profile agree, and the headline step launches its ten kernels in order."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from transferia_b200 import abi, engine, workload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "transferia_b200", "csrc")
KERNEL = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s+)?(\w+)\s*\(")


def _src(name):
    return open(os.path.join(CSRC, name), encoding="utf-8").read()


def _kernels():
    """(defined, declared): the __global__ functions of kernels_*.cuh defined under a TF_KERNELS_* guard, and declared outside them."""
    defined, declared = [], []
    for f in sorted(os.listdir(CSRC)):
        if not (f.startswith("kernels_") and f.endswith(".cuh")):
            continue
        guards = []                 # one entry per open #if: is it a TF_KERNELS_* guard
        for line in _src(f).splitlines():
            s = line.strip()
            if s.startswith("#if"):
                guards.append(s.startswith("#ifdef TF_KERNELS_"))
            elif s.startswith("#endif"):
                guards.pop()
            m = KERNEL.search(s)
            if not m:
                continue
            if s.endswith(";"):
                assert not any(guards), (f, s)
                declared.append(m.group(1))
            else:
                assert any(guards) and "{" in s, (f, s)
                defined.append(m.group(1))
    assert len(set(defined)) == len(defined) and len(set(declared)) == len(declared)
    return set(defined), set(declared)


def test_every_kernel_is_declared_once_and_built():
    defined, declared = _kernels()
    assert defined == declared
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    # the device functions of the library (-res-usage lists the same ones as -sass, without disassembling them)
    out = subprocess.run([tool, "-res-usage", engine.LIB_PATH], capture_output=True, text=True, check=True).stdout
    built = {m.group(2)[:int(m.group(1))] for m in re.finditer(r"Function _ZN3tfk(\d+)(\w+):", out)}
    assert len(re.findall(r"Function ", out)) == len(built)          # every one is a tfk kernel
    assert built == declared


def test_every_kernel_is_launched_by_tf_launch():
    _, declared = _kernels()
    assert set(re.findall(r"\bTF_LAUNCH\(e, (\w+),", _src("tfgpu.cu"))) == declared


def test_no_launch_path_besides_the_launcher():
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".hpp")) and f != "launch.hpp":
            src = _src(f)
            for token in ("<<<", "launch_k_", "prof_begin(", "launches++"):
                assert token not in src, (f, token)


# ----------------------------------------------------------------------------------------------------------- device
DBZ_OPTS = {"ignore_unknown_sources": True, "version": "1.1.2.Final", "topic_prefix": "p", "database": "db", "source_type": "pg"}


@pytest.fixture
def peng(eng):
    eng.profile_enable(True)
    yield eng
    eng.profile_enable(False)


def _profiled(eng, call):
    """Runs one entry-point call; its launches are exactly what the profile lists, and a call that launches nothing keeps it."""
    _, declared = _kernels()
    n0 = eng.launch_count()
    call()
    prof = eng.profile_read()
    names = [k["name"] for k in prof]
    assert eng.launch_count() - n0 == len(prof) > 0, names
    assert set(names) <= declared, names
    eng.resident_stats()
    assert eng.profile_read() == prof
    return names


def _text_batch(n, kinds=None):
    rng = np.random.default_rng(5)
    words = [b"x" * int(k) for k in rng.integers(0, 40, n)]
    return abi.Batch(n, [abi.fixed_to_column(abi.TF_INT64, np.arange(n)), abi.strings_to_column(abi.TF_UTF8, words)], kinds)


TEXT_SCHEMA = [{"name": "id", "type": "int64", "key": True}, {"name": "s", "type": "utf8"}]


@pytest.mark.gpu
def test_every_entry_point_counts_what_it_profiles(peng):
    import torch
    eng = peng
    sink = eng.plan("public", "t", TEXT_SCHEMA, [], {"type": "clickhouse"})
    plain = eng.plan("public", "t", TEXT_SCHEMA, [])
    lz = abi.TF_WIRE_CH_NATIVE_LZ4
    # TF_COL_LENS8 lengths become offsets on the device
    names = _profiled(eng, lambda: eng.push_encode(sink, _text_batch(3000).narrow(), lz))
    assert {"k_widen_lens", "k_offsets_sum", "k_offsets_chunks", "k_offsets_write", "k_lz4_frames"} <= set(names), names
    # no rows: the offsets of a TF_COL_LENS8 column come from the one-pass scan
    z = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    empty = abi.Batch(0, [abi.Column(abi.TF_INT64, values=z), abi.Column(abi.TF_UTF8, offsets=z, heap=z, lens_width=1)], mem=abi.TF_MEM_DEVICE)
    assert "k_csv_offsets" in _profiled(eng, lambda: eng.push_encode(sink, empty, lz))
    # row errors are collected on the device: update / delete rows at a sink
    kinds = np.zeros(3000, np.uint8); kinds[::7] = 1
    got = {}
    names = _profiled(eng, lambda: got.setdefault("r", eng.push_encode(sink, _text_batch(3000, kinds), abi.TF_WIRE_CH_NATIVE)))
    assert got["r"].errors and "k_collect_errors" in names
    # two phases: the filter of phase one, then the whole chain over the kept rows
    batch, schema = workload.make_hits_batch(10000)
    hpid = eng.plan("public", "hits", schema, workload.headline_transformers(workload.counterid_threshold(batch, schema)), {"type": "clickhouse"})
    assert _profiled(eng, lambda: eng.push_encode(hpid, batch, lz, selective=0)).count("k_filter") == 2
    assert "k_layout_columnar" in _profiled(eng, lambda: eng.push_columns(hpid, batch))
    assert "k_measure" in _profiled(eng, lambda: eng.measure(batch))
    names = _profiled(eng, lambda: eng.push_encode(plain, _text_batch(3000), abi.TF_WIRE_SER_JSON | abi.TF_WIRE_F_GZIP))
    assert {"k_json_sizes", "k_json_write", "k_deflate_chunks", "k_deflate_finish"} <= set(names), names
    # the parsers
    cpid = eng.plan("db", "t", [{"name": "i", "type": "int32", "path": "0"}, {"name": "s", "type": "utf8", "path": "1"}], [])
    assert "k_csv_pass2" in _profiled(eng, lambda: eng.parse_csv(cpid, b"1,a\n2,bb\n3,\n"))
    text, fields = workload.make_json_lines(500)
    jpid = eng.plan("", "events", engine.json_result_schema(fields, {}), [])
    assert "k_json_pass2" in _profiled(eng, lambda: eng.parse_json(jpid, text, {}))
    data, ends, schema_text, table = workload.make_debezium_messages(500)
    dpid = eng.plan(table[0], table[1], engine.debezium_table_schema(schema_text), workload.debezium_transformers(), {"type": "clickhouse"})
    assert "k_dbz_pass2" in _profiled(eng, lambda: eng.parse_debezium(dpid, data, ends, schema_text, schema_registry=True, schema_id=7, wire_fmt=lz))
    assert "k_json_write" in _profiled(eng, lambda: eng.emit_debezium(plain, _text_batch(300), DBZ_OPTS))


@pytest.mark.gpu
def test_profile_holds_one_call(peng):
    eng = peng
    pid = eng.plan("db", "t", [{"name": "i", "type": "int32", "path": "0"}, {"name": "s", "type": "utf8", "path": "1"}], [])
    text = b"".join(b"%d,v%d\n" % (i, i) for i in range(5000))
    first = _profiled(eng, lambda: eng.parse_csv(pid, text))
    assert _profiled(eng, lambda: eng.parse_csv(pid, text)) == first


@pytest.mark.gpu
def test_headline_step_launch_sequence(peng):
    """DESIGN.md §4: the headline step (filter_rows -> native block -> LZ4 frames, device resident) is these ten launches."""
    eng = peng
    batch, schema = workload.make_hits_batch(20000)
    k = workload.headline_threshold(batch, schema)
    pid = eng.plan("public", "hits", schema, workload.headline_transformers_watchid(k), {"type": "clickhouse"})
    dbatch = batch.to_device("cuda:0")
    names = _profiled(eng, lambda: eng.push_encode_resident(pid, dbatch, abi.TF_WIRE_CH_NATIVE_LZ4))
    assert names == ["k_filter", "k_scan_blockcnt", "k_compact_sel", "k_str_sizes", "k_layout_scan", "k_layout_finish",
                     "k_encode_fixed", "k_encode_str_plain", "k_lz4_frames", "k_frame_seal"]
