"""kernel_construct's register and local-memory budget, read from the compiler (no GPU needed).

The builder runs 4 blocks of 256 threads per SM, so 64 registers per thread. Whatever does not fit goes to local
memory, and with 4 x 37 KB of shared memory per SM the spill traffic leaves L1 and costs an L2 round trip per access in
a kernel that already waits on L2. This file compiles construct.cu exactly as simlod_b200/build.py compiles the shipped
cubin and pins the budget: ptxas's report for the kernel and its out-of-line helpers, and, through the line table of the
SASS, no local-memory access in the per-point loops.
"""
import os
import re
import shutil
import subprocess

import pytest

from simlod_b200 import build as B

SRC = os.path.join(B.CSRC, "construct.cu")

# Functions that still use local memory, each with its ceiling (stack frame, spill stores, spill loads in bytes, as
# ptxas reports them) and the reason; every other function must report none. A ceiling only goes down.
LOCAL_MEMORY_CEILING = {
    # the per-thread leaf cache (leaf word, 64-bit key) and the tile index: loaded on every first-visit point, stored on
    # every cache miss, and the same in the legacy re-walk. A shared-memory leaf cache removes those accesses but
    # measures slower (DESIGN.md §4).
    "kernel_construct": ((64, 112, 160), "the leaf cache of the first-visit and legacy re-walk loops lives in local memory"),
    "countGlobal": ((0, 32, 24), "cold (once per leaf per pass): the refused-split undo keeps more values than the call ABI leaves it"),
}

# per-point loops: (function, first line of the loop inside the function) -> no LDL / STL may map to the loop's lines.
# Not listed: the first-visit tile loop of passItems, walk's leaf-cache check and the legacy re-walk, where the leaf
# cache is in local memory (see kernel_construct's ceiling above).
HOT_LOOPS = [
    ("walk", "for (;;) {"),                                    # the descent through the first-child table
    ("sampleUp", "for (;;) {"),                                # the upward probes, three atomics in flight
    ("passItems", "for (; base < numListed; base += stride) {"),  # the listed re-walk
    ("passItems", "for (; g < numGranules; g += gStride) {"),  # the spilled-point re-walk
    ("insertAll", "for (;;) {"),                               # the insertion tiles
]


def _nvcc_or_skip():
    if not os.path.exists(B.NVCC) or shutil.which("nvdisasm", path=os.path.join(B.CUDA, "bin")) is None:
        pytest.skip("CUDA toolkit (nvcc, nvdisasm) not found")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    _nvcc_or_skip()
    cubin = str(tmp_path_factory.mktemp("construct") / "construct.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("construct", []) + ["-cubin", "-o", cubin, SRC]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return cubin, res.stdout


def _functions(log):
    """ptxas -v: {function (demangled base name): {stack, stores, loads}}, plus the kernel's register count"""
    out, regs = {}, None
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        mangled = m.group(1)
        mm = re.match(r"_Z(\d+)", mangled)
        name = mangled[len(mm.group(0)):][:int(mm.group(1))] if mm else mangled
        out[name] = dict(stack=int(m.group(2)), stores=int(m.group(3)), loads=int(m.group(4)))
    m = re.search(r"Compiling entry function 'kernel_construct'.*?Used (\d+) registers", log, re.S)
    if m:
        regs = int(m.group(1))
    return out, regs


def test_kernel_fits_64_registers(compiled):
    _, log = compiled
    funcs, regs = _functions(log)
    assert regs is not None, log
    assert regs <= 64, "kernel_construct uses %d registers: 4 blocks of 256 threads per SM need <= 64" % regs
    assert "kernel_construct" in funcs


def test_local_memory_budget(compiled):
    _, log = compiled
    funcs, _ = _functions(log)
    helpers = set(funcs) - {"kernel_construct"}
    assert helpers >= {"splitRound", "allocateChunks", "insertAll", "recordVoxelShared"}, sorted(funcs)
    bad = {}
    for name, r in funcs.items():
        ceiling = LOCAL_MEMORY_CEILING.get(name, ((0, 0, 0), None))[0]
        if any(v > c for v, c in zip((r["stack"], r["stores"], r["loads"]), ceiling)):
            bad[name] = r
    assert not bad, "local memory in kernel_construct or its out-of-line helpers: %r" % bad


def _body_lines(lines, func, loop_head):
    """1-based line range of the loop that starts with `loop_head` inside the definition of `func`"""
    start = next(i for i, l in enumerate(lines) if re.search(r"\b%s\s*\(" % func, l) and "__device__" in l)
    i = start
    while loop_head not in lines[i]:
        i += 1
    depth = 0
    for j in range(i, len(lines)):
        depth += lines[j].count("{") - lines[j].count("}")
        if depth <= 0:
            return i + 1, j + 1
    raise AssertionError("unbalanced braces after %s: %s" % (func, loop_head))


def test_hot_loops_touch_no_local_memory(compiled):
    cubin, _ = compiled
    sass = subprocess.run([os.path.join(B.CUDA, "bin", "nvdisasm"), "-g", "-c", cubin], stdout=subprocess.PIPE, text=True, check=True).stdout
    with open(SRC) as f:
        lines = f.read().split("\n")
    ranges = [(f, h) + _body_lines(lines, f, h) for f, h in HOT_LOOPS]
    hits = {}
    cur = None
    for l in sass.split("\n"):
        m = re.search(r'//## File ".*?([^/"]+)", line (\d+)', l)
        if m:
            cur = (m.group(1), int(m.group(2)))
            continue
        if cur and cur[0] == "construct.cu" and re.search(r"\b(LDL|STL)(\.\w+)*\b", l):
            for f, h, a, b in ranges:
                if a <= cur[1] <= b:
                    hits.setdefault("%s: %s" % (f, h), []).append(cur[1])
    assert not hits, "local-memory accesses in per-point loops (source lines): %r" % hits
