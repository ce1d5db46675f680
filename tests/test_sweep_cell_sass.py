"""What the POA sweep issues per DP cell in its common row, checked on the SASS of the 2 kbp class (no GPU needed).

With the plane accesses 128-bit and the row loop free of local memory, a row whose columns all lie inside the band is integer
arithmetic: `row_pass1` (score lookup, H' = max(M + s, E1, E2), the thread's F-scan aggregate) and `row_pass2` (F1 / F2, H, the E
values of the next rows, the D word, the stores). Each thread sweeps 16 cells per row, so the instructions the compiler emits at
the two call sites of the unmasked passes, over 16, are the sweep's per-cell cost. Neither pass forms per-column gap offsets
k * e (an IMAD by a gap extension per cell): the F states run their recurrence inside a thread, and the score table's entry
address is one PRMT."""
import os
import re

import pytest

from cactus_b200 import build as B
from test_sweep_sass import NVDISASM, SRC, kernel_instructions
from test_sweep_ring_sass import sass  # noqa: F401  (the module's compiled SASS fixture)

pytestmark = pytest.mark.skipif(not (os.path.exists(B.NVCC) and os.path.exists(NVDISASM)), reason="needs nvcc and nvdisasm")

CPT = 16
# instructions per cell at the two call sites of t128's unmasked passes, at the time the F states left "A space" inside a thread
PASS1_PER_CELL, PASS2_PER_CELL, TOTAL_PER_CELL = 7.5, 16.5, 23.5


def call_site(pattern):
    """the 1-based source line in dp_sweep that calls `pattern`"""
    lines = open(SRC).read().split("\n")
    hits = [i + 1 for i, s in enumerate(lines) if pattern in s and "__device__" not in s]
    assert len(hits) == 1, (pattern, hits)
    return hits[0]


def ops_at(instrs, line):
    return [op for op, chain in instrs if ("poa_kernel.cu", line) in chain]


@pytest.fixture(scope="module")
def passes(sass):  # noqa: F811
    instrs = kernel_instructions(sass, "poa_msa_kernel_t128")
    p1 = ops_at(instrs, call_site("row_pass1<false>("))
    p2 = ops_at(instrs, call_site("row_pass2<0, RING_NT>("))
    assert p1 and p2, "unmasked passes not found in the SASS"
    return p1, p2


def test_t128_common_row_instructions_per_cell(passes):
    p1, p2 = passes
    n1, n2 = len(p1) / CPT, len(p2) / CPT
    assert n1 <= PASS1_PER_CELL and n2 <= PASS2_PER_CELL and n1 + n2 <= TOTAL_PER_CELL, (n1, n2)


def test_t128_passes_multiply_nothing_per_cell(passes):
    # IMAD.IADD is an add and IMAD.MOV / IMAD.U32 a move (ptxas places them on the FMA pipe); IMAD.X / .WIDE / .SHL are the
    # stores' 64-bit address arithmetic, a few per row. A plain IMAD per cell is what forming k * e per column (or a scaled
    # table index) costs; what is left is per row (j0 * e of the two planes, a chunk stride)
    for ops in passes:
        mul = [op for op in ops if op in ("IMAD", "IMAD.HI")]
        assert len(mul) < CPT // 4, mul


def test_t128_score_lookup_is_prmt_and_lds(passes):
    p1, _ = passes
    # one shared-memory load per cell, its address one PRMT; no shift / mask of packed query codes
    assert p1.count("LDS") == CPT, p1
    assert sum(op.startswith("PRMT") for op in p1) == CPT, p1
    assert not [op for op in p1 if re.match(r"(SHF|LOP3|BFE)\b", op)], p1
