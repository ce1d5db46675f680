"""The trace kernels (Engine.poa_msa_trace_batch, barb200_poa_trace_batch) against the reference and the oracle (H100): not only the
MSA bytes and the sum of the banded cells, but every alignment the device makes -- the guide tree's read order, each alignment's node
count, best score and graph cigar, and the band (dp_beg, dp_end) of every row. A band edge off in two rows in opposite directions, or
a tie-break that picks another cigar with the same MSA, fails here; the first differing alignment and field name the place."""
import collections
import functools

import numpy as np
import pytest

from cactus_b200 import first_trace_difference

import _golden as G
import _repeats as RP
import _reflib as R
from _synth import family, gapped_family
from test_gpu_far_rows import families as far_row_families
from test_gpu_parity import engine_for as _engine_for
from test_gpu_poa_classes import edge_cases, edge_want
from test_poa_trace_cpu import RETRY_SCALE, retry_jobs, unrelated_job

pytestmark = pytest.mark.gpu
CLASSES = (32, 64, 128, 256, 640, 1024)


def engine_for(p=None, **knobs):
    return _engine_for(R.params_dict(p or R.cactus_params()), **knobs)


@pytest.fixture(scope="module")
def engine():
    e = engine_for()
    yield e
    e.close()


def assert_traces(got, want, tag):
    assert len(got) == len(want), tag
    for j, (g, w) in enumerate(zip(got, want)):
        d = first_trace_difference(g, w)
        assert d is None, (tag, j, d)


def run_vs_oracle(jobs, p=None, tag="", **knobs):
    e = engine_for(p, **knobs)
    try:
        got = e.poa_msa_trace_batch(jobs)
    finally:
        e.close()
    assert_traces(got, [R.oracle_poa_msa_trace(job, p) for job in jobs], tag)


# ---- 1. the reference's own values ----
def test_golden_cases_equal_the_reference(engine):
    default = R.params_dict(R.cactus_params())
    for c in G.poa_cases():
        same = all(abs(c["params"][k] - default[k]) < 1e-9 for k in c["params"])
        e = engine if same else _engine_for(c["params"])
        try:
            t = e.poa_msa_trace_batch([c["seqs"]])[0]
        finally:
            if not same:
                e.close()
        tag = c["id"]
        assert t["read_id_map"] == c["order"], tag
        assert t["msa"].shape == c["msa"].shape and np.array_equal(t["msa"], c["msa"]) and t["cells"] == c["cells"], tag
        assert [a["best_score"] for a in t["alns"]] == c["best"].tolist(), tag
        assert [len(a["cigar"]) for a in t["alns"]] == c["ncigar"].tolist(), tag
        assert np.array_equal(np.concatenate([a["cigar"] for a in t["alns"]]), c["cigar"].astype(np.uint64)), tag
        assert np.array_equal(np.concatenate([a["dp_beg"] for a in t["alns"]]), c["beg"]), tag
        assert np.array_equal(np.concatenate([a["dp_end"] for a in t["alns"]]), c["end"]), tag


# ---- 2. the oracle, word for word ----
def test_seeded_families(oracle_built):
    rng = np.random.default_rng(500)
    jobs = []
    for _ in range(48):
        K = int(rng.integers(2, 14))
        L = int(rng.choice([1, 5, 20, 60, 150, 300, 400, 800, 1500]))
        kw = dict(sub=float(rng.choice([0.0, 0.02, 0.08, 0.2])), ins=float(rng.choice([0, 0.005, 0.03])),
                  dele=float(rng.choice([0, 0.005, 0.03])), nfrac=float(rng.choice([0, 0, 0.01])))
        jobs.append(family(rng, K, L, sort=bool(rng.random() < 0.7), **kw))
    run_vs_oracle(jobs, tag="families")


def test_unrelated_ragged_rows(oracle_built):
    """ragged unrelated rows, N-rich, up to 90 reads (two read-id words)"""
    rng = np.random.default_rng(42)
    jobs = []
    for _ in range(16):
        K = int(rng.integers(2, 91))
        jobs.append([rng.integers(0, 5 if rng.random() < 0.2 else 4, int(rng.integers(1, 400))).astype(np.uint8) for _ in range(K)])
    run_vs_oracle(jobs, tag="unrelated")


@pytest.mark.parametrize("wb, wf, prog", [(10, 0.01, 1), (0, 0.0, 0), (30, 0.02, 1), (5, 0.1, 0)])
def test_narrow_bands(oracle_built, wb, wf, prog):
    rng = np.random.default_rng(43 + wb)
    p = R.cactus_params(wb=wb, wf=wf, progressive=prog)
    jobs = [family(rng, int(rng.integers(2, 10)), int(rng.choice([50, 300, 900])), sub=0.08, ins=0.03, dele=0.03) for _ in range(10)]
    run_vs_oracle(jobs, p, tag=(wb, wf))


@pytest.mark.parametrize("gaps", [(400, 30, 1200, 1), (4, 2, 24, 1), (400, 30, 1200, 30), (1200, 1, 400, 30), (400, 30, 300, 1), (6, 2, 6, 2),
                                  (4, 1, 24, 1), (1, 1, 1, 1), (2, 1, 30, 0)])
def test_gap_regimes(oracle_built, gaps):
    o1, e1, o2, e2 = gaps
    rng = np.random.default_rng(4242 + o1 + 7 * e2)
    p = R.cactus_params(o1=o1, e1=e1, o2=o2, e2=e2, wb=300, wf=0.05)
    jobs = [gapped_family(rng, int(rng.integers(3, 9)), int(rng.choice([120, 500, 1100])), [1, 2, 3, 8, 27, 28, 29, 33, 64, 65, 150, 300])
            for _ in range(8)]
    run_vs_oracle(jobs, p, tag=gaps)


@pytest.mark.parametrize("name, p", [("default", R.cactus_params()), ("narrow", R.cactus_params(wb=10, wf=0.01))])
def test_far_row_families(oracle_built, name, p):
    jobs = far_row_families(np.random.default_rng(2024 + 700), 700)
    run_vs_oracle(jobs, p, tag=name)


@pytest.mark.parametrize("param", ["default", "narrow", "abpoa_gaps"])
def test_repeat_rich_windows(oracle_built, param):
    jobs = [c.seqs for f in sorted(RP.FAMILIES) for c in RP.cases(f) if sum(len(s) for s in c.seqs) <= 20000]
    run_vs_oracle(jobs, RP.PARAMS[param], tag=param)


def test_one_10kbp_window(engine, oracle_built):
    rng = np.random.default_rng(44)
    job = [s[:10000] for s in family(rng, 4, 10000, sub=0.03, ins=0.01, dele=0.01)]
    assert_traces(engine.poa_msa_trace_batch([job]), [R.oracle_poa_msa_trace(job)], "10kbp")


# ---- 3. every CTA class, and the serial debug mode ----
@functools.lru_cache(maxsize=None)
def small_jobs():
    """jobs whose reads all fit the one-warp class (<= 511 bases), and their oracle traces under the narrow band"""
    rng = np.random.default_rng(9393)
    p = R.cactus_params(wb=10, wf=0.01)
    jobs = far_row_families(np.random.default_rng(2024 + 400), 400)
    jobs += [family(rng, int(rng.integers(2, 8)), int(rng.choice([30, 200, 500])), sub=0.1, ins=0.03, dele=0.03) for _ in range(6)]
    jobs = [[s[:511] for s in job] for job in jobs]
    return p, jobs, [R.oracle_poa_msa_trace(job, p) for job in jobs]


@pytest.mark.parametrize("threads", CLASSES)
def test_every_class(oracle_built, threads):
    p, jobs, want = small_jobs()
    e = engine_for(p, threads_per_block=threads)
    try:
        assert_traces(e.poa_msa_trace_batch(jobs), want, threads)
    finally:
        e.close()


def test_class_edges(oracle_built):
    """reads of 16 T - 1 and 16 T bases at every class boundary and of 16383 bases, under the narrow band"""
    p, cases = edge_cases()[1]
    jobs = [job for _, job in cases]
    assert collections.Counter(cls for cls, _ in cases).keys() == set(CLASSES)
    e = engine_for(p)
    try:
        got = e.poa_msa_trace_batch(jobs)
    finally:
        e.close()
    assert_traces(got, [edge_want(1, j) for j in range(len(jobs))], "edges")


@pytest.mark.parametrize("threads", (32, 640))
def test_serial_debug_mode(oracle_built, monkeypatch, threads):
    """BARB200_DEBUG_SERIAL=1: the serial traceback (dp_best_cell, dp_backtrack) and graph phases trace what the warp forms trace"""
    p, jobs, want = small_jobs()
    monkeypatch.setenv("BARB200_DEBUG_SERIAL", "1")
    e = engine_for(p, threads_per_block=threads)
    try:
        got = e.poa_msa_trace_batch(jobs)
    finally:
        e.close()
        monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
    assert_traces(got, want, ("serial", threads))


# ---- 4. the trace-capacity retry ----
def test_trace_capacity_retry(oracle_built, monkeypatch):
    """BARB200_TRACE_REGION_SCALE shrinks the regions of the first round and of the x4 retry below one record, while the jobs' planes
    fit (test_poa_trace_cpu.py: test_scaled_regions_overflow_before_anything_else): every job ends those rounds with JOB_ERR_TRACE_CAP,
    writing nothing, and its trace comes from the worst-case round. It must equal the oracle's"""
    jobs = retry_jobs()
    monkeypatch.setenv("BARB200_TRACE_REGION_SCALE", repr(RETRY_SCALE))
    e = engine_for()
    try:
        got = e.poa_msa_trace_batch(jobs)
    finally:
        e.close()
        monkeypatch.delenv("BARB200_TRACE_REGION_SCALE", raising=False)
    assert_traces(got, [R.oracle_poa_msa_trace(job) for job in jobs], "trace-capacity retry")


def test_plane_retry(engine, oracle_built):
    """60 unrelated reads outgrow their first-round and x4 planes before their trace regions (test_poa_trace_cpu.py:
    test_unrelated_reads_outgrow_their_first_planes): traced by the worst-case round, next to a job that the first round completes"""
    job = unrelated_job()
    assert_traces(engine.poa_msa_trace_batch([job, job[:7]]), [R.oracle_poa_msa_trace(job), R.oracle_poa_msa_trace(job[:7])], "plane retry")


# ---- 5. no change in behaviour ----
def test_trace_call_computes_what_the_batch_call_computes(engine):
    rng = np.random.default_rng(61)
    jobs = [family(rng, int(rng.integers(2, 9)), int(rng.choice([60, 300, 900, 1800, 4000])), sub=0.05, ins=0.01, dele=0.01) for _ in range(60)]
    before, cells_before = engine.poa_msa_batch(jobs, return_cells=True)
    traces = engine.poa_msa_trace_batch(jobs)
    engine.poa_msa_trace_batch(jobs[::3])
    after, cells_after = engine.poa_msa_batch(jobs, return_cells=True)
    for j, t in enumerate(traces):
        assert np.array_equal(t["msa"], before[j]) and t["cells"] == int(cells_before[j]), j
        assert np.array_equal(after[j], before[j]), j
    assert np.array_equal(cells_after, cells_before)


# ---- 6. several devices ----
def test_every_device_traces_what_one_device_traces(engine):
    import cactus_b200 as cb
    e = cb.Engine(cb.PoaParams(devices="all"))
    try:
        if e.device_count() < 2:
            pytest.skip("one GPU")
        rng = np.random.default_rng(62)
        jobs = [family(rng, int(rng.integers(2, 9)), int(rng.choice([60, 300, 900])), sub=0.05, ins=0.01, dele=0.01) for _ in range(80)]
        assert_traces(e.poa_msa_trace_batch(jobs), engine.poa_msa_trace_batch(jobs), "devices")
    finally:
        e.close()
