"""The POA kernel's graph phases where the graph does not fit the CTA's shared-memory scratch: with BARB200_SCRATCH_KB=0 each class
gets only its sweep's ring (t32: 8 KB, so the far-row families' larger graphs take the global-memory forms of the order splice and
the topological sort while the smaller ones stay on chip) or none at all (t1024 has no ring: every phase takes its global-memory
form). Every MSA and cell count must equal the oracle's (tests/test_graph_phases_cpu.py checks which form a graph takes)."""
import pytest

import test_gpu_far_rows as F


@pytest.mark.gpu
@pytest.mark.parametrize("threads", (32, 1024))
def test_far_rows_with_minimal_scratch(oracle_built, monkeypatch, threads):
    monkeypatch.setenv("BARB200_SCRATCH_KB", "0")
    F.run_and_compare(threads, 511)
