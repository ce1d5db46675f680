"""What the POA sweep's plane accesses compile to, checked on the SASS of every CTA class (no GPU needed).

A row of the DP planes is chunk-major (poa_types.h: DpState): one 16-byte chunk per thread, so a warp's chunk store or load covers
512 contiguous bytes. That only pays off when each chunk is one 128-bit instruction. Split into four 32-bit stores, every store
spans the same 4 lines, and the L1 store path handles four times the line requests. NVVM has split such stores in this kernel
before, so the instructions the helpers st4 / ld4cg produce are pinned here, together with t128's spill budget."""
import os
import re
import shutil
import subprocess

import pytest

from cactus_b200 import build as B

SRC = os.path.join(B.CSRC, "poa_kernel.cu")
CLASSES = (32, 64, 128, 256, 640, 1024)
NVDISASM = os.path.join(os.path.dirname(B.NVCC), "nvdisasm")
# t128 (the 2 kbp class) at the time the plane stores became 128-bit: more spill traffic would land inside the row loop
T128_SPILL_STORES, T128_SPILL_LOADS = 180, 212

pytestmark = pytest.mark.skipif(not (shutil.which(B.NVCC) and shutil.which(NVDISASM)), reason="needs nvcc and nvdisasm")


def helper_lines(name):
    """1-based source lines of the device helper `name` in poa_kernel.cu (a one-liner, or up to its closing brace in column 0)"""
    lines = open(SRC).read().split("\n")
    start = next(i for i, s in enumerate(lines) if re.search(r"__device__ __forceinline__ \S+ %s\(" % name, s))
    end = start if lines[start].rstrip().endswith("}") else lines.index("}", start)
    return set(range(start + 1, end + 2))


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    d = tmp_path_factory.mktemp("sweep_sass")
    cubin = str(d / "poa_kernel.cubin")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-cubin", "-x", "cu", SRC, "-o", cubin], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([NVDISASM, "-gi", cubin], capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


def kernel_instructions(sass, kernel):
    """(opcode, every (file, line) of the instruction's inlining chain) for every instruction of `kernel`"""
    out, cur, fresh, inside = [], set(), True, False
    for s in sass.split("\n"):
        m = re.match(r"\s*\.section\s+\.text\.(\w+),", s)
        if m:
            inside = m.group(1) == kernel
            continue
        if not inside:
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', s)
        if m:
            if fresh:                              # a new block of line info: one line per inlined frame
                cur = set()
            cur.add((os.path.basename(m.group(1)), int(m.group(2))))
            fresh = False
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)", s)
        if m:
            out.append((m.group(1), cur))
            fresh = True
    assert out, "no SASS found for %s" % kernel
    return out


def ops_of(instrs, lines, prefix):
    return [op for op, chain in instrs if op.startswith(prefix) and any(f == "poa_kernel.cu" and n in lines for f, n in chain)]


@pytest.mark.parametrize("T", CLASSES)
def test_plane_chunks_are_128_bit_accesses(compiled, T):
    instrs = kernel_instructions(compiled[0], "poa_msa_kernel_t%d" % T)
    stores = ops_of(instrs, helper_lines("st4"), "STG")
    # row 0, the three masking modes of row_pass2 and the padding blocks: 8 chunk stores each
    assert len(stores) >= 40, stores
    assert all(op.startswith("STG.E.128") for op in stores), sorted(set(stores))
    loads = ops_of(instrs, helper_lines("ld4cg"), "LDG")
    assert len(loads) >= 8, loads
    assert all(op.startswith("LDG.E.128") for op in loads), sorted(set(loads))


def test_t128_spills_stay_within_budget(compiled):
    log = compiled[1]
    m = re.search(r"Function properties for poa_msa_kernel_t128\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert m, log
    assert int(m.group(1)) <= T128_SPILL_STORES and int(m.group(2)) <= T128_SPILL_LOADS, m.group(0)
