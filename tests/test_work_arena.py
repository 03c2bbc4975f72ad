"""Who may touch the engine's work arena (`e->work` in tfgpu.cu). The checksum kernel of an LZ4 batch (k_frame_seal) keeps running
into the next call and reads the frame sizes and offsets that run_chain laid out there (DESIGN.md §4). So only run_chain, which joins
that kernel whenever it lays the arena out differently, and tfgpu_measure, which joins it first, may write there. Anything else must
use an arena of its own."""
import os
import re

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "transferia_b200", "csrc", "tfgpu.cu")
DEFINITION = re.compile(r"^[A-Za-z_].*?\b(\w+)\s*\(")       # a function definition starts in column 0; its name precedes the first '('


def test_only_run_chain_and_measure_touch_the_work_arena():
    users, func = set(), None
    for line in open(SRC, encoding="utf-8"):
        m = DEFINITION.match(line)
        if m and not line.rstrip().endswith(";"):
            func = m.group(1)
        if re.search(r"\be->work\b", line) and not line.lstrip().startswith("//"):
            users.add(func)
    assert users == {"run_chain", "tfgpu_measure"}, users
