"""The read families of test_gpu_far_rows.py really give the sweep the rows that test is about (no GPU needed).

The host build of the product's graph code (tests/hosttest) aligns each family as the kernel does, and pred_rows.cpp counts the
predecessors of every row of every sweep. The GPU test reads a predecessor at r - 2 from the shared-memory ring and older ones
from global memory, so the families must contain predecessors at r - 2, at r - 3 and far beyond, row 0 as a predecessor of row 2,
and 3- and 4-way bubbles, under each of the test's parameter sets."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import _reflib as R
import test_gpu_far_rows as F

HOSTTEST = os.path.join(R.ROOT, "tests", "hosttest")

pytestmark = pytest.mark.skipif(not shutil.which("g++"), reason="needs g++")


@pytest.fixture(scope="module")
def pred_rows_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pred_rows") / "libpred_rows.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-pthread", "-fopenmp", "-x", "c++",
                           "-o", so, os.path.join(HOSTTEST, "pred_rows.cpp"), os.path.join(R.ROOT, "cactus_b200", "csrc", "pecan_plan.cpp")])
    lib = C.CDLL(so)
    lib.pred_rows_counts.restype = C.POINTER(C.c_longlong)
    return so, lib


def counts_of(lib, so, jobs, p, monkeypatch):
    """predecessor counts over every sweep of every job (pred_rows.cpp: PredRowCounts)"""
    monkeypatch.setattr(R, "HOSTTEST_SO", so)
    lib.pred_rows_reset()
    for job in jobs:
        R.hosttest_poa_msa_trace(job, p)
    c = np.ctypeslib.as_array(lib.pred_rows_counts(), shape=(1 + 65 + 1 + 5,)).copy()
    return dict(rows=int(c[0]), dist=c[1:66], row0_at_row2=int(c[66]), npre=c[67:72])


@pytest.mark.parametrize("name", sorted(F.PARAMS))
@pytest.mark.parametrize("n", (511, 2000))
def test_families_have_far_predecessors(pred_rows_lib, monkeypatch, name, n):
    so, lib = pred_rows_lib
    jobs = F.families(np.random.default_rng(2024 + n), n)      # the jobs test_gpu_far_rows.cases(n) runs
    c = counts_of(lib, so, jobs, F.PARAMS[name], monkeypatch)
    d = c["dist"]
    assert c["rows"] > 0 and d[1] > 0
    assert d[2] > 0, "no predecessor at r - 2 (the ring)"
    assert d[3] > 0, "no predecessor at r - 3 (global memory)"
    assert d[40:].sum() > 0, "no predecessor far back (long insertions)"
    assert c["row0_at_row2"] > 0, "row 2 never has row 0 as a predecessor"
    assert c["npre"][3] > 0 and c["npre"][4] > 0, "no 3- or 4-way bubble"
