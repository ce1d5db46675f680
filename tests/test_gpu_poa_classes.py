"""The POA kernel's CTA-size classes against the oracle (H100). poa_kernel.cu has one entry point per class: 32, 64, 128, 256, 640
and 1024 threads, and a class takes queries of up to 16 * threads - 1 bases. A job runs in the smallest class its longest read fits
unless PoaParams(threads_per_block=T) asks for at least T. Here the same jobs run under every class, jobs sit exactly at every class
boundary, and a subset runs in the serial debug mode (BARB200_DEBUG_SERIAL=1), whose traceback recomputes F from the stored H / D
planes by a code path of its own (poa_graph.cuh: dp_backtrack). MSA bytes and banded cell counts must equal the oracle's."""
import collections
import functools

import numpy as np
import pytest

import _reflib as R
from _synth import evolve, family, gapped_family
from test_gpu_parity import engine_for

CLASSES = (32, 64, 128, 256, 640, 1024)
GAP_LENS = [1, 2, 3, 8, 27, 28, 33, 64, 90]


def clip(seqs, n=511):
    return [s[:n] for s in seqs]


def run_stage(e, jobs):
    """(buckets, msas, cells) of one stage: the buckets are the class launches the MSAs came from"""
    st = e.stage(jobs)
    try:
        b = st.buckets()
        st.run()
        msas, cells = st.fetch()
    finally:
        st.close()
    return b, msas, cells


def assert_oracle(msas, cells, trs, tag):
    for j, (m, tr) in enumerate(zip(msas, trs)):
        assert m.shape == tr["msa"].shape and np.array_equal(m, tr["msa"]), (tag, j)
        assert int(cells[j]) == tr["cells"], (tag, j)


@functools.lru_cache(maxsize=None)
def small_cases():
    """about 40 jobs whose reads all fit the one-warp class (<= 511 bases), grouped by parameter set: (name, params, jobs)"""
    rng = np.random.default_rng(9090)
    P = R.cactus_params
    fam = lambda K, L, **kw: clip(family(rng, K, L, **kw))                                   # noqa: E731
    gap = lambda K, L: clip(gapped_family(rng, K, L, GAP_LENS))                             # noqa: E731
    ragged = lambda K, n=4: [rng.integers(0, n, int(rng.integers(1, 300))).astype(np.uint8) for _ in range(K)]   # noqa: E731
    return [
        ("default", P(), [fam(4, 30), fam(8, 200, sub=0.05, ins=0.02, dele=0.02), fam(5, 490, sub=0.03, ins=0.01, dele=0.01),
                          fam(3, 505), fam(6, 300, nfrac=0.15), gap(5, 480), fam(12, 400, sub=0.05, ins=0.02, dele=0.02), ragged(70), ragged(90, 5)]),
        ("wb0", P(wb=0, wf=0.0), [fam(4, 100, sub=0.08, ins=0.03, dele=0.03), fam(6, 480, sub=0.05, ins=0.02, dele=0.02),
                                  fam(3, 511), gap(4, 400), gap(6, 490), fam(5, 250, nfrac=0.1), fam(2, 511, sub=0.1)]),
        ("wb10", P(wb=10, wf=0.01), [fam(5, 480, sub=0.08, ins=0.03, dele=0.03), gap(5, 300), gap(4, 495), gap(7, 450),
                                     fam(6, 150, sub=0.2, ins=0.05, dele=0.05), fam(4, 400, nfrac=0.2)]),
        ("wb60", P(wb=60, wf=0.02, progressive=0), [fam(8, 490, sub=0.1, ins=0.03, dele=0.03), gap(5, 480), fam(4, 60),
                                                    ragged(66), fam(5, 350, sub=0.05, ins=0.05, dele=0.05), gap(3, 511)]),
        ("gaps4,1,24,1", P(o1=4, e1=1, o2=24, e2=1, wb=30, wf=0.02), [gap(5, 480), gap(4, 300), gap(6, 495), fam(5, 200, sub=0.05, ins=0.03, dele=0.03)]),
        ("gaps1,1,1,1", P(o1=1, e1=1, o2=1, e2=1, wb=100, wf=0.02), [gap(5, 480), gap(4, 250), gap(6, 490), fam(4, 400, nfrac=0.05)]),
        ("gaps2,1,30,0", P(o1=2, e1=1, o2=30, e2=0), [gap(5, 480), gap(4, 350), gap(6, 500), fam(5, 120, sub=0.05, ins=0.03, dele=0.03)]),
    ]


@functools.lru_cache(maxsize=None)
def small_want():
    return [[R.oracle_poa_msa_trace(job, p) for job in jobs] for _, p, jobs in small_cases()]


def test_small_cases_reach_the_band_edges(oracle_built):
    """the jobs of test_every_class_on_the_same_jobs do what that test relies on (read off the oracle's dp_beg / dp_end): bands that
    start at even and at odd threads, bands that end at the query's last column, rows whose last thread is 30 (the stored range
    then ends with a padding block at thread 31, the last thread of the one-warp class), and reads that need two read-id words"""
    begs, ends, last = set(), set(), False
    for (_, _, jobs), trs in zip(small_cases(), small_want()):
        assert all(len(s) <= 511 for job in jobs for s in job)
        for tr in trs:
            for a in tr["alns"]:
                begs |= {int(b) >> 4 for b in a["dp_beg"] if b > 0}
                ends |= {int(x) >> 4 for x in a["dp_end"]}
                last |= bool(np.any(a["dp_end"] == a["qlen"]))
    assert any(t % 2 for t in begs) and any(t % 2 == 0 and t > 0 for t in begs)
    assert last and 30 in ends and 31 in ends
    assert max(len(job) for _, _, jobs in small_cases() for job in jobs) > 64


@pytest.mark.gpu
@pytest.mark.parametrize("threads", CLASSES)
def test_every_class_on_the_same_jobs(oracle_built, threads):
    """jobs that fit the one-warp class forced into each class in turn (threads_per_block): one launch of exactly that class, and
    the oracle's MSA and banded cells from every one (one warp, 20 warps, the whole 1024-thread block; padding blocks anywhere)"""
    for (name, p, jobs), trs in zip(small_cases(), small_want()):
        e = engine_for(R.params_dict(p), threads_per_block=threads)
        try:
            b, msas, cells = run_stage(e, jobs)
        finally:
            e.close()
        assert [(x["threads"], x["jobs"]) for x in b] == [(threads, len(jobs))], (name, b)
        assert_oracle(msas, cells, trs, (threads, name))


def longest_exactly(rng, K, n, **kw):
    """K reads of one family whose longest read has exactly n bases"""
    parent = rng.integers(0, 4, n).astype(np.uint8)
    seqs = [parent] + [evolve(parent, rng, **kw)[:n] for _ in range(K - 1)]
    seqs.sort(key=lambda s: -len(s))
    return seqs


DEFAULT, NARROW = R.cactus_params(), R.cactus_params(wb=30, wf=0.002)


@functools.lru_cache(maxsize=None)
def edge_cases():
    """(params, [(class the job must run in, job)]): for every class boundary a job whose longest read is 16 T - 1 bases (the
    last thread's last column is the query's last column) and one of 16 T bases (the next class), under the default band, which
    reaches column L, and under a narrow one; and the largest window the engine takes, 16383 bases. K is small under the default
    band: the oracle keeps 20 bytes per banded cell, about 1.7 GB for one 16 kbp alignment"""
    rng = np.random.default_rng(9191)
    kw = dict(sub=0.03, ins=0.01, dele=0.01)
    out = {"default": [], "narrow": []}
    for T, nxt in zip(CLASSES[:-1], CLASSES[1:]):
        for n, cls in ((16 * T - 1, T), (16 * T, nxt)):
            out["default"].append((cls, longest_exactly(rng, 3 if T <= 256 else 2, n, **kw)))
            out["narrow"].append((cls, longest_exactly(rng, 6, n, **kw)))
    out["default"].append((1024, longest_exactly(rng, 2, 16383, **kw)))
    out["narrow"].append((1024, longest_exactly(rng, 5, 16383, **kw)))
    return [(DEFAULT, out["default"]), (NARROW, out["narrow"])]


@functools.lru_cache(maxsize=None)
def edge_want(i, j):
    p, jobs = edge_cases()[i]
    return R.oracle_poa_msa_trace(jobs[j][1], p)


@pytest.mark.gpu
def test_class_edges(oracle_built):
    """reads of exactly 16 T - 1 and 16 T bases at every class boundary, and of 16383 bases (the 1024-thread class, which nothing
    else runs): each job lands in the class its length calls for and equals the oracle"""
    for i, (p, cases) in enumerate(edge_cases()):
        jobs = [job for _, job in cases]
        e = engine_for(R.params_dict(p))
        try:
            b, msas, cells = run_stage(e, jobs)
        finally:
            e.close()
        assert {x["threads"]: x["jobs"] for x in b} == collections.Counter(cls for cls, _ in cases), b
        assert_oracle(msas, cells, [edge_want(i, j) for j in range(len(jobs))], ("edges", p.wb))


@pytest.mark.gpu
def test_serial_debug_mode(oracle_built, monkeypatch):
    """BARB200_DEBUG_SERIAL=1 (read at every launch) runs the graph phases and the reference's traceback rule on one thread, which
    recomputes F from the stored H / D planes instead of reading them the warp traceback's way: a second opinion on every stored
    cell the traceback can reach. In every class, on the narrow-band and small-extension jobs and the narrow class-edge jobs, it
    must return what the default mode returns, and the oracle's answer"""
    runs = []                                       # (engine params, engine knobs, jobs, oracle traces)
    for (name, p, jobs), trs in zip(small_cases(), small_want()):
        if name in ("wb0", "wb10", "gaps4,1,24,1", "gaps1,1,1,1", "gaps2,1,30,0"):
            runs += [(p, dict(threads_per_block=T), jobs, trs) for T in CLASSES]
    i = 1                                           # the narrow-band class-edge jobs
    cases = edge_cases()[i][1]
    runs.append((NARROW, {}, [job for _, job in cases], [edge_want(i, j) for j in range(len(cases))]))
    for p, knobs, jobs, trs in runs:
        e = engine_for(R.params_dict(p), **knobs)
        try:
            monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
            b0, msas0, cells0 = run_stage(e, jobs)
            monkeypatch.setenv("BARB200_DEBUG_SERIAL", "1")
            b1, msas1, cells1 = run_stage(e, jobs)
        finally:
            monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
            e.close()
        tag = (p.wb, p.gap_ext1, p.gap_ext2, knobs)
        assert b0 == b1, tag
        assert np.array_equal(np.asarray(cells0), np.asarray(cells1)), tag
        for j in range(len(jobs)):
            assert np.array_equal(msas0[j], msas1[j]), (tag, j)
        assert_oracle(msas1, cells1, trs, tag)
