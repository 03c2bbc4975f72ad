#!/bin/bash
# Host-side C++ (row transposer, sink push / dispatcher, ClickHouse writer, plan validation and queue batchers) under AddressSanitizer + UBSan:
# the four host translation units are built with g++ into a library of their own, the device entry points of tfgpu.h are stubbed (they answer
# TF_E_FATAL_NODEVICE), and the CPU tests that drive the host code (fuzzers included) run against it.
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd); OUT=${1:-/tmp/tfhost_asan}; mkdir -p "$OUT"
CSRC="$ROOT/transferia_b200/csrc"
HOST_TUS=("$CSRC/host_rows.cu" "$CSRC/host_sink.cu" "$CSRC/host_chwire.cu" "$CSRC/host_plan.cu" "$CSRC/host_deflate.cu" "$CSRC/host_zstd.cu")
python - "$ROOT" "$OUT" "$CSRC/host_plan.cu" "$CSRC/host_deflate.cu" "$CSRC/host_zstd.cu" <<'PY'
import re, sys
root, out, host_defs = sys.argv[1], sys.argv[2], sys.argv[3:]
hdr = re.sub(r"/\*.*?\*/", "", open(root + "/include/tfgpu.h").read(), flags=re.S)
protos = re.findall(r"^\s*((?:const\s+)?[\w]+(?:\s*\*)?)\s+(tfgpu_\w+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.M | re.S)
real = set(n for f in host_defs for n in re.findall(r"^(?:int|void) (tfgpu_\w+)\(", open(f).read(), flags=re.M))     # defined by host_plan.cu / host_deflate.cu, compiled below
lines = ['#include "%s/include/tfgpu.h"' % root, 'extern "C" {']
for ret, name, args in protos:
    if name in real:
        continue
    ret = ret.strip(); body = "{}" if ret == "void" else ("{ return TF_E_FATAL_NODEVICE; }" if ret == "int" else "{ return 0; }")
    lines.append("%s %s(%s) %s" % (ret, name, " ".join(args.split()), body))
open(out + "/stubs.cpp", "w").write("\n".join(lines) + "\n}\n")
PY
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -fPIC -shared -I/usr/local/cuda/include \
    -x c++ "${HOST_TUS[@]}" "$OUT/stubs.cpp" -o "$OUT/libtfhost_asan.so" -L/usr/local/cuda/lib64 -lcudart
cd "$ROOT"
TFGPU_LIB_PATH="$OUT/libtfhost_asan.so" LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" \
    ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 \
    python -m pytest tests/test_rows.py tests/test_sink_push.py tests/test_ch_wire.py tests/test_host_cpu.py tests/test_regex_replace.py -q -m "not gpu" -p no:cacheprovider \
    -k "not exports and not sm90a and not no_cpu_fallback and not gloo and not bench_reference and not c_example"
# the deflate stream helper (host_deflate.cu)
TFGPU_LIB_PATH="$OUT/libtfhost_asan.so" LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" \
    ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 \
    python -m pytest tests/test_deflate.py -q -m "not gpu" -p no:cacheprovider -k "stream_helper"
# the zstd prefix helper (host_zstd.cu)
TFGPU_LIB_PATH="$OUT/libtfhost_asan.so" LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" \
    ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 \
    python -m pytest tests/test_zstd.py -q -m "not gpu" -p no:cacheprovider -k "prefix"
# the queue serializer batchers (host_plan.cu)
TFGPU_LIB_PATH="$OUT/libtfhost_asan.so" LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" \
    ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 \
    python -m pytest tests/test_serializers.py tests/test_debezium_emit.py -q -m "not gpu" -p no:cacheprovider -k "queue_json_batching or queue_debezium_batching"
# the threaded parts (worker pool of the transposer / gather / column-wise replace, dispatcher lanes and its delivery gate) under ThreadSanitizer
g++ -std=c++17 -O1 -g -fsanitize=thread -fno-omit-frame-pointer -fPIC -shared -I/usr/local/cuda/include \
    -x c++ "${HOST_TUS[@]}" "$OUT/stubs.cpp" -o "$OUT/libtfhost_tsan.so" -L/usr/local/cuda/lib64 -lcudart
TFGPU_LIB_PATH="$OUT/libtfhost_tsan.so" LD_PRELOAD="$(gcc -print-file-name=libtsan.so)" TSAN_OPTIONS="halt_on_error=1 report_signal_unsafe=0" \
    python -m pytest tests/test_rows.py tests/test_sink_push.py tests/test_regex_replace.py -q -m "not gpu" -p no:cacheprovider -k "dispatcher or two_pools or host_gather or transposer_fuzz or strict_single or replace_steps or mixed_text or inverse_transposer or under_the_dispatcher"
