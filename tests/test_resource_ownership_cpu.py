"""Every device buffer, pinned buffer, event and stream of the library has an owner in csrc/internal.cuh (DevArray,
HostPinned, PooledArray, CallBuffers, Events, Stream, Resident).  This scan keeps it so: no source outside internal.cuh
calls the runtime's allocator or creates or destroys events and streams (the buffer pool of ctx.cu releases through
mem_free too), and the hand-written allocation macros of the old context create stay gone."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pymbar_b200", "csrc")
SCAFFOLD = "internal.cuh"

RAW_CALLS = re.compile(
    r"\b(cudaMalloc\w*|cudaHostAlloc|cudaFree\w*|cudaEventCreate\w*|cudaEventDestroy|cudaStreamCreate\w*|"
    r"cudaStreamDestroy)\s*\(")
OLD_MACROS = re.compile(r"#\s*define\s+(ALLOC|CREATE_CUDA|AUG_CUDA)\b")
TOKENS = re.compile(r'"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'|//[^\n]*|/\*.*?\*/', re.S)


def sources():
    names = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))
    assert SCAFFOLD in names
    return names


def strip_comments(src):
    """Comments become blanks (newlines kept, so line numbers hold); string and character literals stay."""
    def keep(m):
        t = m.group(0)
        return t if t[0] in "\"'" else re.sub(r"[^\n]", " ", t)

    return TOKENS.sub(keep, src)


@pytest.mark.parametrize("name", [n for n in sources() if n != SCAFFOLD])
def test_no_raw_resource_calls(name):
    src = strip_comments(open(os.path.join(CSRC, name)).read())
    hits = [f"{name}:{src.count(chr(10), 0, m.start()) + 1}: {m.group(1)}" for m in RAW_CALLS.finditer(src)]
    assert not hits, "raw allocation, free, event or stream calls outside the scaffold:\n" + "\n".join(hits)


def test_old_allocation_macros_are_gone():
    for name in sources():
        m = OLD_MACROS.search(strip_comments(open(os.path.join(CSRC, name)).read()))
        assert not m, f"{name} defines {m.group(1)}"


def test_scan_sees_the_scaffold():
    """The scan is live: the scaffold holds the raw calls it forbids everywhere else."""
    scaffold = strip_comments(open(os.path.join(CSRC, SCAFFOLD)).read())
    for call in ("cudaMalloc", "cudaHostAlloc", "cudaFree", "cudaFreeHost", "cudaEventCreateWithFlags",
                 "cudaEventDestroy", "cudaStreamCreateWithFlags", "cudaStreamDestroy"):
        assert re.search(r"\b" + call + r"\s*\(", scaffold), call
    assert strip_comments('a = "//x"; // c\nb; /* d */') == 'a = "//x";     \nb;        '
