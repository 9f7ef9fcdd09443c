"""CPU test: the streaming decode kernel keeps its per-thread state in registers.

Every `k_decode_stream` instantiation runs 512 threads with one CTA per SM, which caps a thread at 128 registers. A value
that does not fit goes to local memory, and in this kernel such reloads miss L1 (the dynamic shared-memory plan leaves
little of it) and put an L2 round trip into every phase of the token. The built library must show no stack frame and no
LDL / STL in those functions."""
import re
import subprocess

from nano_b200 import build as nb_build

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"

# Q80 with 64-element groups (no preset model uses it) still spills two words around the prologue's poll loop.
ALLOWED_STACK = {(0x80, 4, 2): 8, (0x80, 4, 4): 8}
ALLOWED_LOCAL_OPS = {(0x80, 4, 2): 4, (0x80, 4, 4): 4}


def _inst(name):
    m = re.search(r"k_decode_streamILi(\d+)ELi(\d+)ELi(\d+)E", name)
    return tuple(int(x) for x in m.groups()) if m else None


def test_stream_kernel_has_no_stack_frame():
    out = subprocess.run([CUOBJDUMP, "-res-usage", nb_build.ENGINE_SO], capture_output=True, text=True, check=True).stdout
    stack = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.match(r"\s*Function (\S+):", line)
        if m and _inst(m.group(1)):
            st = re.search(r"STACK:(\d+)", lines[i + 1])
            stack[_inst(m.group(1))] = int(st.group(1))
    assert len(stack) == 12, sorted(stack)
    bad = {k: v for k, v in stack.items() if v > ALLOWED_STACK.get(k, 0)}
    assert not bad, f"stack bytes per thread: {bad}"


def test_stream_kernel_sass_has_no_local_memory_access():
    out = subprocess.run([CUOBJDUMP, "-sass", nb_build.ENGINE_SO], capture_output=True, text=True, check=True).stdout
    count, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = _inst(m.group(1))
            if cur:
                count[cur] = 0
            continue
        if cur and re.search(r"\b(LDL|STL)\b", line):
            count[cur] += 1
    assert len(count) == 12, sorted(count)
    bad = {k: v for k, v in count.items() if v > ALLOWED_LOCAL_OPS.get(k, 0)}
    assert not bad, f"LDL/STL instructions: {bad}"
