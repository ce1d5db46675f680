"""What the POA sweep's row loop compiles to, checked on the SASS (no GPU needed).

A row takes a few thousand SM clocks and issues under half of them; what it waits on is memory. Two things keep that off the
loop: no local memory (spill reloads of loop invariants would run on every row and can miss L1), and a predecessor two rows
back (every substitution bubble and deletion makes such rows) read from the ring of the last two rows in shared memory rather
than from L2. The ring's chunks are 128-bit shared-memory accesses, a warp's access 512 contiguous bytes; the 1024-thread
class, whose two rows do not fit its shared memory, has no ring."""
import os
import subprocess

import pytest

from cactus_b200 import build as B
from test_sweep_sass import NVDISASM, SRC, helper_lines, kernel_instructions, ops_of

RING_CLASSES = (32, 64, 128, 256, 640)

pytestmark = pytest.mark.skipif(not (os.path.exists(B.NVCC) and os.path.exists(NVDISASM)), reason="needs nvcc and nvdisasm")


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    cubin = str(tmp_path_factory.mktemp("ring_sass") / "poa_kernel.cubin")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-cubin", "-x", "cu", SRC, "-o", cubin], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return subprocess.run([NVDISASM, "-gi", cubin], capture_output=True, text=True, check=True).stdout


def row_loop_lines():
    """1-based source lines of dp_sweep's row loop, from its `for` to the function's `return cells;`"""
    lines = open(SRC).read().split("\n")
    start = next(i for i, s in enumerate(lines) if "for (int r = 1; r < R; ++r)" in s)
    end = next(i for i in range(start, len(lines)) if lines[i].strip() == "return cells;")
    return set(range(start + 1, end + 2))


def test_t128_row_loop_has_no_local_memory(sass):
    instrs = kernel_instructions(sass, "poa_msa_kernel_t128")
    loop = row_loop_lines()
    assert ops_of(instrs, loop, "STG"), "row loop not found in the SASS"
    local = ops_of(instrs, loop, "LDL") + ops_of(instrs, loop, "STL")
    assert not local, local


@pytest.mark.parametrize("T", RING_CLASSES)
def test_ring_chunks_are_128_bit_shared_accesses(sass, T):
    instrs = kernel_instructions(sass, "poa_msa_kernel_t%d" % T)
    stores = ops_of(instrs, helper_lines("sts4"), "STS")
    # row 0 and the three masking modes of row_pass2: 8 chunk stores each
    assert len(stores) >= 32, stores
    assert all(op.startswith("STS.128") for op in stores), sorted(set(stores))
    # a predecessor at r - 2: row 0 (with its E sentinel) and any other row, 8 chunk loads each
    loads = ops_of(instrs, helper_lines("lds4"), "LDS")
    assert len(loads) >= 16, loads
    assert all(op.startswith("LDS.128") for op in loads), sorted(set(loads))


def test_t1024_has_no_ring(sass):
    instrs = kernel_instructions(sass, "poa_msa_kernel_t1024")
    assert not ops_of(instrs, helper_lines("sts4"), "STS")
    assert not ops_of(instrs, helper_lines("lds4"), "LDS")
