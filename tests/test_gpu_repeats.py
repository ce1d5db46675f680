"""The POA kernel on repeat-rich and low-complexity inputs (tests/_repeats.py) against the oracle (H100): MSA bytes and banded
cell counts, bit for bit. test_repeats_cpu.py pins the oracle to the reference on the same cases and shows that each family
reaches its edge: gap placements with several equal-score answers (the warp traceback's MATCH runs, its predecessor ballot and
the insertion scan's smallest t), rows with many equal maxima (the band's arg-max columns), equal-weight edges (the heaviest-edge
pick folded into the shared-memory edge sort), guide trees whose Jaccard values tie (gt_block_argmax's first maximum), and jobs
at the guide tree's key capacity and at the device sort's tile edges. A wrong tie-break anywhere changes an MSA or a cell count
here."""
import functools

import numpy as np
import pytest

import _repeats as RP
import _reflib as R
from test_gpu_poa_classes import CLASSES, assert_oracle
from test_gpu_poa_params import engine_for, run

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def want(param, family):
    return [R.oracle_poa_msa_trace(c.seqs, RP.PARAMS[param]) for c in RP.cases(family)]


def jobs_of(family):
    return [c.seqs for c in RP.cases(family)]


@pytest.mark.parametrize("param", sorted(RP.PARAMS))
def test_each_family_as_one_batch(oracle_built, param):
    e = engine_for(RP.PARAMS[param])
    try:
        for family in sorted(RP.FAMILIES):
            msas, cells = e.poa_msa_batch(jobs_of(family), return_cells=True)
            assert_oracle(msas, cells, want(param, family), (param, family))
    finally:
        e.close()


def test_each_job_alone(oracle_built):
    """every case as a batch of its own under Cactus' defaults (a stage's slots and key plan then come from that job alone)"""
    e = engine_for(RP.PARAMS["default"])
    try:
        for family in sorted(RP.FAMILIES):
            for c, tr in zip(RP.cases(family), want("default", family)):
                msas, cells = e.poa_msa_batch([c.seqs], return_cells=True)
                assert_oracle(msas, cells, [tr], c.name)
    finally:
        e.close()


def small(param):
    """(names, jobs, oracle traces) of the cases whose reads all fit the one-warp class (<= 511 bases)"""
    out = ([], [], [])
    for family in sorted(RP.FAMILIES):
        for c, tr in zip(RP.cases(family), want(param, family)):
            if max(len(s) for s in c.seqs) <= 511:
                out[0].append(c.name), out[1].append(c.seqs), out[2].append(tr)
    return out


@pytest.mark.parametrize("threads", CLASSES)
def test_every_class(oracle_built, threads):
    """the cases of at most 511 bases forced into each CTA class, under the default band and the narrow one"""
    for param in ("default", "narrow"):
        names, jobs, trs = small(param)
        assert len(jobs) >= 20
        b, msas, cells = run(RP.PARAMS[param], jobs, threads_per_block=threads)
        assert [(x["threads"], x["jobs"]) for x in b] == [(threads, len(jobs))], (param, b)
        assert_oracle(msas, cells, trs, (threads, param))


def test_serial_debug_mode(oracle_built, monkeypatch):
    """BARB200_DEBUG_SERIAL=1: the graph phases and the reference's traceback rule on one thread, on the micro, tandem and ties
    families (the gap placements and guide-tree ties) under the narrow band and abPOA's gaps, and the small cases in the one-warp
    and 640-thread classes: the default mode's answer and the oracle's"""
    runs = [(param, {}, jobs_of(f), want(param, f)) for param in ("narrow", "abpoa_gaps") for f in ("micro", "tandem", "ties")]
    runs += [("default", dict(threads_per_block=T)) + small("default")[1:] for T in (32, 640)]
    for param, knobs, jobs, trs in runs:
        p = RP.PARAMS[param]
        monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
        b0, msas0, cells0 = run(p, jobs, **knobs)
        monkeypatch.setenv("BARB200_DEBUG_SERIAL", "1")
        try:
            b1, msas1, cells1 = run(p, jobs, **knobs)
        finally:
            monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
        assert b0 == b1, (param, knobs)
        assert np.array_equal(np.asarray(cells0), np.asarray(cells1)), (param, knobs)
        for j in range(len(jobs)):
            assert np.array_equal(msas0[j], msas1[j]), (param, knobs, j)
        assert_oracle(msas1, cells1, trs, (param, knobs))


@pytest.mark.parametrize("threads", (None, 32, 1024))
def test_global_memory_graph_phases(oracle_built, monkeypatch, threads):
    """BARB200_SCRATCH_KB=0: every class keeps only its sweep's ring (none in the 1024-thread class), so the order splice, the edge
    sort with its heaviest-edge pick and the row tables take their global-memory forms"""
    monkeypatch.setenv("BARB200_SCRATCH_KB", "0")
    knobs = {} if threads is None else dict(threads_per_block=threads)
    for family in ("micro", "homopolymer", "ties"):
        jobs, trs = jobs_of(family), want("default", family)
        if threads is not None and threads < 1024:
            keep = [j for j, job in enumerate(jobs) if max(len(s) for s in job) < 16 * threads]
            jobs, trs = [jobs[j] for j in keep], [trs[j] for j in keep]
        _, msas, cells = run(RP.PARAMS["default"], jobs, **knobs)
        assert_oracle(msas, cells, trs, (family, threads))


# ---- the guide tree's key capacity and the device sort ----
@functools.lru_cache(maxsize=None)
def gt_want(name):
    c = {c.name: c for c in [c for c, _ in RP.gt_capacity()] + [c for c, _ in RP.gt_sort_edges()] + [RP.gt_big_family()]}[name]
    return c.seqs, R.oracle_poa_msa_trace(c.seqs, RP.PARAMS["default"])


def stage_runs(e, jobs, n_runs):
    """launches after each of n_runs runs, the buckets, and what fetch returns"""
    st = e.stage(jobs)
    try:
        b, launches = st.buckets(), []
        for _ in range(n_runs):
            st.run()
            launches.append(st.launches())
        msas, cells = st.fetch()
    finally:
        st.close()
    return b, launches, msas, cells


def test_jobs_within_the_key_plan_run_once(oracle_built):
    """exactly key_cap keys (2048 and 4096, homopolymer reads), and (AC)n reads of 2 kbp: the guide tree kernel and one launch per
    bucket, no retry"""
    e = engine_for(RP.PARAMS["default"])
    try:
        for name in ("gt/cap/exact2048", "gt/cap/exact4096", "gt/cap/dinucleotide_2k"):
            seqs, tr = gt_want(name)
            b, launches, msas, cells = stage_runs(e, [seqs], 1)
            assert launches == [1 + len(b)], (name, launches, b)
            assert_oracle(msas, cells, [tr], name)
    finally:
        e.close()


def test_key_overflow_is_retried(oracle_built):
    """key_cap + 1 keys (2049 and 4097) and the 2 kbp homopolymer job come back with JOB_ERR_GT_CAP and run again with x4 room:
    through the batch call, and through a stage run twice (each run retries on the stage's uploaded reads) and then fetched"""
    names = ("gt/cap/plus1_2048", "gt/cap/plus1_4096", "gt/cap/homopolymer_2k")
    e = engine_for(RP.PARAMS["default"])
    try:
        jobs, trs = zip(*[gt_want(n) for n in names])
        msas, cells = e.poa_msa_batch(list(jobs), return_cells=True)
        assert_oracle(msas, cells, trs, "batch")
        for name, seqs, tr in zip(names, jobs, trs):
            b, launches, smsas, scells = stage_runs(e, [seqs], 2)
            assert all(n > 1 + len(b) for n in launches), (name, launches, b)
            assert_oracle(smsas, scells, [tr], name)
    finally:
        e.close()


def test_stage_plans_keys_from_its_largest_job(oracle_built):
    """the 2049-key homopolymer job next to a larger family: the stage's key plan comes from the family (4096 keys), so nothing is
    retried, and both equal the oracle"""
    e = engine_for(RP.PARAMS["default"])
    try:
        (s1, t1), (s2, t2) = gt_want("gt/cap/plus1_2048"), gt_want("gt/big_family")
        b, launches, msas, cells = stage_runs(e, [s1, s2], 1)
        assert launches == [1 + len(b)], (launches, b)
        assert_oracle(msas, cells, [t1, t2], "mixed")
    finally:
        e.close()


def test_sort_tile_edges(oracle_built):
    """2047, 2048, 2049, 4096 and 4097 distinct-hash keys: one shared-memory tile, then one and two merge sizes of global-stride
    passes; each job alone and all in one batch"""
    names = [c.name for c, _ in RP.gt_sort_edges()]
    e = engine_for(RP.PARAMS["default"])
    try:
        jobs, trs = zip(*[gt_want(n) for n in names])
        for name, seqs, tr in zip(names, jobs, trs):
            msas, cells = e.poa_msa_batch([seqs], return_cells=True)
            assert_oracle(msas, cells, [tr], name)
        msas, cells = e.poa_msa_batch(list(jobs), return_cells=True)
        assert_oracle(msas, cells, trs, "batch")
    finally:
        e.close()


# ---- windows and two-end problems ----
@pytest.mark.parametrize("param", RP.LONG_WINDOW_PARAMS)
def test_long_window_in_the_640_thread_class(oracle_built, param):
    c, p = RP.long_window(), RP.PARAMS[param]
    tr = R.oracle_poa_msa_trace(c.seqs, p)
    b, msas, cells = run(p, [c.seqs])
    assert [(x["threads"], x["jobs"]) for x in b] == [(640, 1)], b
    assert_oracle(msas, cells, [tr], (param, c.name))


@pytest.mark.parametrize("param", ("default", "narrow"))
def test_windows_and_two_ends(oracle_built, param):
    """ends whose windows are cut inside a microsatellite (msa_make_partial_order_alignment), and two-end problems on repeat parents
    through make_consistent_partial_order_alignments and flower_submit / flower_wait"""
    p = RP.PARAMS[param]
    e = engine_for(p)
    try:
        for name, strs, win in RP.window_ends():
            m = e.msa_make_partial_order_alignment(strs, window_size=win)
            o = R.oracle_msa_make_partial_order_alignment(strs, window_size=win, p=p)
            assert m.msa_seq.shape == o.shape and np.array_equal(m.msa_seq, o), (param, name)
        probs = RP.two_end_cases()
        tickets = [e.flower_submit(*prob, window_size=win) for _, prob, win in probs]
        for (name, prob, win), t in zip(probs, tickets):
            o = R.oracle_make_consistent_partial_order_alignments(*prob, window_size=win, p=p)
            for got in (e.make_consistent_partial_order_alignments(*prob, window_size=win), e.flower_wait(t)):
                assert len(got) == len(o), (param, name)
                for a, b in zip(got, o):
                    assert a.msa_seq.shape == b.shape and np.array_equal(a.msa_seq, b), (param, name)
    finally:
        e.close()
