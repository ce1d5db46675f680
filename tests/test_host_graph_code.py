"""CPU check of the product's __host__ __device__ code (cactus_b200/csrc/poa_graph.cuh: graph fusion, topological
sort, edge sort, max_remain, row tables, MSA rank/fill, traceback) and of its host guide tree (guide_tree.cpp), compiled
by tests/hosttest for the host and compared with the oracle on seeded inputs and with the golden vectors. The CUDA DP
sweep is stood in for by a scalar emulation of the kernel's row formulation; the real kernel is tested under -m gpu."""
import numpy as np

import _golden as G
import _reflib as R
from _synth import family, gapped_family
from test_oracle_vs_ref import assert_same_trace


def test_hosttest_golden():
    for c in G.poa_cases():
        p = R.cactus_params(**c["params"])
        tr = R.hosttest_poa_msa_trace(c["seqs"], p)
        assert np.array_equal(tr["msa"], c["msa"]), c["id"]
        assert tr["read_id_map"] == c["order"], c["id"]
        assert tr["cells"] == c["cells"], c["id"]
        assert np.array_equal(np.concatenate([a["cigar"] for a in tr["alns"]]), c["cigar"]), c["id"]
        assert np.array_equal(np.concatenate([a["dp_beg"] for a in tr["alns"]]), c["beg"]), c["id"]
        assert np.array_equal(np.concatenate([a["dp_end"] for a in tr["alns"]]), c["end"]), c["id"]


def test_hosttest_random_vs_oracle(oracle_built):
    rng = np.random.default_rng(77)
    for it in range(60):
        K = int(rng.integers(2, 14))
        L = int(rng.choice([5, 20, 60, 150, 300, 400, 800]))
        kw = dict(sub=float(rng.choice([0.0, 0.02, 0.08, 0.2])), ins=float(rng.choice([0, 0.005, 0.03])),
                  dele=float(rng.choice([0, 0.005, 0.03])), nfrac=float(rng.choice([0, 0, 0.01])))
        seqs = family(rng, K, L, sort=bool(rng.random() < 0.7), **kw)
        p = R.cactus_params() if rng.random() < 0.5 else R.cactus_params(
            wb=int(rng.choice([0, 5, 10, 30, 100])), wf=float(rng.choice([0.0, 0.01, 0.02, 0.1])), progressive=int(rng.integers(0, 2)))
        assert_same_trace(R.oracle_poa_msa_trace(seqs, p), R.hosttest_poa_msa_trace(seqs, p), (it, K, L, kw))


def test_traceback_rule_without_f_planes_many_gap_models(oracle_built):
    """the warp traceback's rule (insertions whole, from the row's H values; F1 only within the convex crossover distance), stated
    serially, runs in lock step with the reference's rule inside the host build's traceback (poa_graph.cuh: dp_backtrack) and fails the
    job on any disagreement: a few hundred alignments with block indels under random convex gap penalties of every ordering, each
    equal to the oracle's. Extensions of 0 and 1 are drawn often: with both at most 1 the reference's minus infinity lies within a few
    hundred of INT32_MIN"""
    rng = np.random.default_rng(2024)
    fixed = [(400, 30, 1200, 1), (4, 2, 24, 1), (10, 3, 10, 3), (50, 1, 3, 9), (7, 5, 100, 5), (300, 2, 20, 40), (1, 1, 1, 1),
             (4, 1, 24, 1), (2, 1, 30, 0), (400, 0, 1200, 1)]

    def ext():
        return int(rng.choice([0, 1, int(rng.integers(2, 40))]))

    for it in range(60):
        if it < len(fixed):
            o1, e1, o2, e2 = fixed[it]
        else:
            o1, e1, o2, e2 = int(rng.integers(1, 600)), ext(), int(rng.integers(1, 1500)), ext()
            if e1 == 0 and e2 == 0:             # barb200_create requires one extension > 0
                e2 = 1
        p = R.cactus_params(o1=o1, e1=e1, o2=o2, e2=e2, wb=int(rng.choice([20, 100, 1000])), wf=0.05)
        seqs = gapped_family(rng, int(rng.integers(2, 7)), int(rng.choice([40, 150, 400])), [1, 2, 3, 5, 9, 20, 27, 28, 33, 64, 90])
        tr = R.hosttest_poa_msa_trace(seqs, p)           # asserts job status 0
        assert_same_trace(R.oracle_poa_msa_trace(seqs, p), tr, (it, (o1, e1, o2, e2), p.wb))


def test_hosttest_unrelated_ragged(oracle_built):
    rng = np.random.default_rng(78)
    for it in range(40):
        K = int(rng.integers(2, 70))
        seqs = [rng.integers(0, 5 if rng.random() < 0.2 else 4, int(rng.integers(1, 300))).astype(np.uint8) for _ in range(K)]
        p = R.cactus_params(wb=int(rng.choice([0, 1, 5, 10, 1000])), wf=float(rng.choice([0.0, 0.01, 0.1])), progressive=int(rng.integers(0, 2)))
        assert_same_trace(R.oracle_poa_msa_trace(seqs, p), R.hosttest_poa_msa_trace(seqs, p), (it, K))


def test_incremental_topological_order_gives_identical_alignments(oracle_built, monkeypatch):
    """The device does not re-run abPOA's BFS after every fused sequence: it keeps the previous topological order and
    splices the new nodes in (poa_cta.cuh). The DP, the traceback and the MSA do not depend on WHICH topological order
    the rows are swept in (bands, scores and tie-breaks are per node / per in-edge order), so read order, every
    cigar, the banded cell count and the MSA must equal the reference's; only the per-row band lists are permuted."""
    monkeypatch.setenv("HOSTTEST_INCREMENTAL_ORDER", "1")
    rng = np.random.default_rng(79)
    for it in range(120):
        K = int(rng.integers(2, 16))
        L = int(rng.choice([5, 20, 60, 150, 300, 400, 800]))
        kw = dict(sub=float(rng.choice([0.0, 0.02, 0.08, 0.2, 0.4])), ins=float(rng.choice([0, 0.005, 0.03, 0.1])),
                  dele=float(rng.choice([0, 0.005, 0.03, 0.1])), nfrac=float(rng.choice([0, 0, 0.01])))
        if rng.random() < 0.2:
            seqs = [rng.integers(0, 4, int(rng.integers(1, 200))).astype(np.uint8) for _ in range(K)]
        else:
            seqs = family(rng, K, L, sort=bool(rng.random() < 0.7), **kw)
        p = R.cactus_params() if rng.random() < 0.5 else R.cactus_params(
            wb=int(rng.choice([0, 5, 10, 30, 100])), wf=float(rng.choice([0.0, 0.01, 0.02, 0.1])), progressive=int(rng.integers(0, 2)))
        a, b = R.oracle_poa_msa_trace(seqs, p), R.hosttest_poa_msa_trace(seqs, p)
        assert a["read_id_map"] == b["read_id_map"], it
        assert np.array_equal(a["msa"], b["msa"]), (it, K, L, kw)
        assert a["cells"] == b["cells"], it
        for x, y in zip(a["alns"], b["alns"]):
            assert np.array_equal(x["cigar"], y["cigar"]), it
            assert sorted(zip(x["dp_beg"].tolist(), x["dp_end"].tolist())) == sorted(zip(y["dp_beg"].tolist(), y["dp_end"].tolist())), it


def test_group_commit_and_batch_merge_under_threads():
    """cactus_b200/csrc/group_commit.h + batch_merge.h with stand-in devices: concurrent callers get their own answers, batches
    never overlap, requests pile up into wider batches while one runs, a failing batch does not wedge the queue"""
    import ctypes as C
    lib = R._load(R.build_hosttest())
    f = lib.hosttest_group_commit_stress
    f.restype = C.c_longlong
    f.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    m, b, o = C.c_longlong(), C.c_longlong(), C.c_longlong()
    assert f(1, 40, C.byref(m), C.byref(b), C.byref(o)) == 0 and m.value == 0 and b.value == 40 and o.value == 0     # one caller: its own request, unchanged
    assert f(8, 200, C.byref(m), C.byref(b), C.byref(o)) == 0 and o.value == 0 and m.value > 0 and b.value < 8 * 200
    g = lib.hosttest_batch_merge_stress
    g.restype = C.c_longlong
    g.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_longlong)]
    assert g(1, 20, C.byref(m)) == 0 and m.value == 0
    assert g(8, 150, C.byref(m)) == 0 and m.value > 0
