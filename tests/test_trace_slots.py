"""The trace-slot names of the kernel (enum TraceSlot, TRACE_SLOTS and TRACE_TILES in fm_kernel.cuh) and of
flashmoe_b200/trace_slots.py, which the trace scripts read the stamps by, are the same names with the same columns."""
import os
import re

from flashmoe_b200 import trace_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "flashmoe_b200", "csrc", "fm_kernel.cuh")


def header_slots():
    src = open(HEADER).read()
    enum = re.search(r"enum TraceSlot : int \{(.*?)\};", src, re.S)
    assert enum, "enum TraceSlot not found in fm_kernel.cuh"
    slots = {m.group(1): int(m.group(2)) for m in re.finditer(r"\bTRACE_(\w+)\s*=\s*(\d+)\s*,", enum.group(1))}
    for name in ("SLOTS", "TILES"):
        m = re.search(rf"constexpr int TRACE_{name} = (\d+);", src)
        assert m, f"TRACE_{name} not found in fm_kernel.cuh"
        slots[name] = int(m.group(1))
    return slots


def python_slots():
    return {k: v for k, v in vars(trace_slots).items() if k.isupper() and isinstance(v, int)}


def test_trace_slots_match_the_kernel():
    hdr = header_slots()
    assert len(hdr) == 16 + 7 + 2   # phase slots 0-15, seven per-tile bases, SLOTS and TILES
    assert python_slots() == hdr


def test_trace_slots_layout():
    s = header_slots()
    phases = sorted(v for k, v in s.items() if k not in ("SLOTS", "TILES") and not k.startswith("TILE_"))
    assert phases == list(range(16))
    bases = sorted(v for k, v in s.items() if k.startswith("TILE_"))
    assert bases == [16 + s["TILES"] * i for i in range(7)]
    assert bases[-1] + s["TILES"] == s["SLOTS"] == 128
