"""The shared-memory forms of the POA kernel's graph phases (cactus_b200/csrc/graph_phases.cuh: the fusion's order splice, and the
edge sort + max_remain + row tables of the topological sort) give exactly what the serial forms give, with no GPU.

tests/hosttest/graph_phases.cpp runs them after every fusion of the host build's incremental-order pipeline, the CTA's threads one
after the other, and fails the job on any difference from hosttest's incremental_order (the spliced order), graph_bfs_remain
(remain; this also checks that the first out edge after the edge sort is the first heaviest one) and graph_build_rows (every
RowRec and pre_row entry). The jobs: the golden vectors, random read families, and the far-row families of test_gpu_far_rows.py.
The kernel takes these forms only where the graph fits its scratch; with a scratch too small it keeps the global-memory forms,
and the counts below show which form each fusion took."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import _golden as G
import _reflib as R
import test_gpu_far_rows as F
from _synth import family

HOSTTEST = os.path.join(R.ROOT, "tests", "hosttest")

pytestmark = pytest.mark.skipif(not shutil.which("g++"), reason="needs g++")


@pytest.fixture(scope="module")
def phases_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("graph_phases") / "libgraph_phases.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-pthread", "-fopenmp", "-x", "c++",
                           "-o", so, os.path.join(HOSTTEST, "graph_phases.cpp"), os.path.join(R.ROOT, "cactus_b200", "csrc", "pecan_plan.cpp")])
    lib = C.CDLL(so)
    lib.graph_phases_config.argtypes = [C.c_int, C.c_int]
    lib.graph_phases_stats.restype = C.POINTER(C.c_longlong)
    return so, lib


def jobs():
    out = [(c["seqs"], R.cactus_params(**c["params"])) for c in G.poa_cases()]
    rng = np.random.default_rng(80)
    for _ in range(30):
        K = int(rng.integers(2, 16))
        L = int(rng.choice([5, 20, 60, 150, 300, 800]))
        kw = dict(sub=float(rng.choice([0.0, 0.02, 0.08, 0.2, 0.4])), ins=float(rng.choice([0, 0.005, 0.03, 0.1])),
                  dele=float(rng.choice([0, 0.005, 0.03, 0.1])), nfrac=float(rng.choice([0, 0, 0.01])))
        seqs = family(rng, K, L, sort=bool(rng.random() < 0.7), **kw)
        p = R.cactus_params() if rng.random() < 0.5 else R.cactus_params(
            wb=int(rng.choice([0, 5, 10, 30, 100])), wf=float(rng.choice([0.0, 0.01, 0.02, 0.1])), progressive=int(rng.integers(0, 2)))
        out.append((seqs, p))
    far = F.families(np.random.default_rng(2024 + 511), 511)
    for p in F.PARAMS.values():
        out += [(job, p) for job in far]
    return out


def run_all(lib, so, monkeypatch, scr_bytes, threads):
    monkeypatch.setattr(R, "HOSTTEST_SO", so)
    monkeypatch.setenv("HOSTTEST_INCREMENTAL_ORDER", "1")
    lib.graph_phases_config(scr_bytes, threads)
    for seqs, p in jobs():
        R.hosttest_poa_msa_trace(seqs, p)            # asserts job status 0: no difference from the serial forms
    s = np.ctypeslib.as_array(lib.graph_phases_stats(), shape=(5,)).copy()
    assert s[4] == 0
    return dict(splice_smem=int(s[0]), splice_global=int(s[1]), topo_smem=int(s[2]), topo_global=int(s[3]))


@pytest.mark.parametrize("threads", (32, 128))
def test_shared_memory_forms_equal_serial_forms(phases_lib, monkeypatch, threads):
    so, lib = phases_lib
    c = run_all(lib, so, monkeypatch, 1 << 22, threads)
    assert c["splice_smem"] > 0 and c["topo_smem"] > 0 and c["splice_global"] == 0 and c["topo_global"] == 0, c


def test_scratch_too_small_keeps_global_forms(phases_lib, monkeypatch):
    so, lib = phases_lib
    c = run_all(lib, so, monkeypatch, 0, 128)
    assert c["splice_smem"] == 0 and c["topo_smem"] == 0 and c["splice_global"] > 0 and c["topo_global"] > 0, c
    # t32's scratch (10 KB): small graphs fit, the far-row families' larger ones do not
    c = run_all(lib, so, monkeypatch, 10 * 1024, 32)
    assert min(c.values()) > 0, c
