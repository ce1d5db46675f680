"""The POA kernel under substitution matrices and minimizer parameters other than Cactus' defaults, against the oracle (H100). The
parameter sets are those of test_poa_params_cpu.py, where the oracle is pinned to the reference on them. MSA bytes and banded cell
counts must equal the oracle's.

The kernel reads the score as [graph base][query code] from its own table in three places: the sweep's row (poa_kernel.cu:
S.smat), and the warp traceback's step and MATCH-run check (poa_cta.cuh: smat8). The asymmetric matrix and its transpose catch a
transposed table or lookup; abPOA's small scores under very narrow bands make the reference take int16 lanes at 2 kbp and 10 kbp,
where the band snap to 16-column groups (pn_shift) decides dp_beg; the largest accepted scores take the sweep's values close to
INT32_MAX in the 1024-thread class; and the minimizer sets run the guide-tree kernel with windows wider than its 64-position scan
chunks, with k = 20 and with reads that hold no minimizer."""
import functools

import numpy as np
import pytest

import _reflib as R
import test_poa_params_cpu as PP
from test_gpu_poa_classes import CLASSES, assert_oracle, run_stage

pytestmark = pytest.mark.gpu


def engine_for(p, **knobs):
    """an Engine with every POA parameter of the oracle's RefParams p (matrix, gaps, band, minimizer k / w / min_w, progressive
    mode) and optional engine knobs"""
    import cactus_b200 as cb
    return cb.Engine(cb.PoaParams(
        partialOrderAlignmentSubMatrix=list(p.mat),
        partialOrderAlignmentBandConstant=p.wb, partialOrderAlignmentBandFraction=p.wf,
        partialOrderAlignmentGapOpenPenalty1=p.gap_open1, partialOrderAlignmentGapExtensionPenalty1=p.gap_ext1,
        partialOrderAlignmentGapOpenPenalty2=p.gap_open2, partialOrderAlignmentGapExtensionPenalty2=p.gap_ext2,
        partialOrderAlignmentMinimizerK=p.k, partialOrderAlignmentMinimizerW=p.w, partialOrderAlignmentMinimizerMinW=p.min_w,
        partialOrderAlignmentProgressiveMode=p.progressive_poa, partialOrderAlignmentDisableSeeding=p.disable_seeding, **knobs))


def run(p, jobs, **knobs):
    e = engine_for(p, **knobs)
    try:
        return run_stage(e, jobs)
    finally:
        e.close()


def oracle(p, jobs):
    return [R.oracle_poa_msa_trace(job, p) for job in jobs]


@functools.lru_cache(maxsize=None)
def batch(name):
    """24 mixed jobs of 2..13 reads of 1..1500 bases for one matrix set (a matrix and its transpose share them) and their oracle traces"""
    jobs = PP.mixed_jobs(np.random.default_rng(6500 + PP.MATRIX_SETS[name][1]), 24, 1500)
    return jobs, oracle(PP.params(name), jobs)


@pytest.mark.parametrize("name", sorted(PP.MATRIX_SETS))
def test_substitution_matrices(oracle_built, name):
    jobs, trs = batch(name)
    _, msas, cells = run(PP.params(name), jobs)
    assert_oracle(msas, cells, trs, name)


@pytest.mark.parametrize("k,w", PP.MINIMIZERS)
def test_minimizer_parameters(oracle_built, k, w):
    """the ragged, unsorted families of the CPU test (one 70 reads deep) and a mixed batch"""
    p = PP.minimizer_params(k, w)
    jobs = PP.minimizer_jobs(k, w) + PP.mixed_jobs(np.random.default_rng(6600 + 256 * k + w), 10, 1500)
    _, msas, cells = run(p, jobs)
    assert_oracle(msas, cells, oracle(p, jobs), (k, w))


@functools.lru_cache(maxsize=None)
def small(name):
    """16 mixed jobs whose reads all fit the one-warp class (<= 511 bases) and their oracle traces"""
    jobs = [[s[:511] for s in job] for job in PP.mixed_jobs(np.random.default_rng(6700 + PP.MATRIX_SETS[name][1]), 16, 500)]
    return jobs, oracle(PP.params(name), jobs)


@pytest.mark.parametrize("threads", CLASSES)
def test_asymmetric_matrix_in_every_class(oracle_built, threads):
    """the same one-warp jobs under the asymmetric matrix (default and narrow band) forced into each CTA class: one launch of exactly
    that class, and the oracle's answers"""
    for name in ("asymmetric", "asymmetric_narrow"):
        jobs, trs = small(name)
        b, msas, cells = run(PP.params(name), jobs, threads_per_block=threads)
        assert [(x["threads"], x["jobs"]) for x in b] == [(threads, len(jobs))], (name, b)
        assert_oracle(msas, cells, trs, (threads, name))


@functools.lru_cache(maxsize=None)
def narrow_abpoa():
    """the abPOA-scored narrow-band jobs grouped by band: [(params, jobs, oracle traces)]"""
    groups = {}
    for p, job in PP.narrow_abpoa_cases():
        groups.setdefault(p.wb, (p, []))[1].append(job)
    return [(p, jobs, oracle(p, jobs)) for p, jobs in groups.values()]


def test_abpoa_scores_under_narrow_bands(oracle_built):
    """int16-lane jobs of 300 to 10000 bases (test_poa_params_cpu.py asserts the lane count) with bands of 0 to 10 columns, where the
    16-column snap of band starts decides dp_beg and with it the banded cells"""
    for p, jobs, trs in narrow_abpoa():
        _, msas, cells = run(p, jobs)
        assert_oracle(msas, cells, trs, ("abpoa_narrow", p.wb))


@functools.lru_cache(maxsize=None)
def extremes():
    return [(name, p, job, R.oracle_poa_msa_trace(job, p)) for name, p, job in PP.extreme_cases()]


def test_largest_accepted_scores_on_16383_base_reads(oracle_built):
    """Cactus' matrix x 524 and +-65535 with gap open + extension at 65534, on three 16383-base reads: the 1024-thread class with its
    DP values close to INT32_MAX"""
    for name, p, job, tr in extremes():
        b, msas, cells = run(p, [job])
        assert [(x["threads"], x["jobs"]) for x in b] == [(1024, 1)], (name, b)
        assert_oracle(msas, cells, [tr], name)


def test_serial_debug_mode(oracle_built, monkeypatch):
    """BARB200_DEBUG_SERIAL=1 runs the traceback on one thread, which scores from the parameters' matrix (P.mat) instead of the warp
    traceback's table: under the asymmetric matrix, its transpose and the narrow abPOA bands it must return what the default mode
    returns, and the oracle's answer"""
    runs = [(PP.params("asymmetric"), dict(threads_per_block=T)) + small("asymmetric") for T in (32, 256, 1024)]
    runs += [(PP.params("transposed_narrow"), dict(threads_per_block=64)) + small("transposed_narrow")]
    runs += [(p, {}, jobs, trs) for p, jobs, trs in narrow_abpoa()]
    for p, knobs, jobs, trs in runs:
        monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
        b0, msas0, cells0 = run(p, jobs, **knobs)
        monkeypatch.setenv("BARB200_DEBUG_SERIAL", "1")
        try:
            b1, msas1, cells1 = run(p, jobs, **knobs)
        finally:
            monkeypatch.delenv("BARB200_DEBUG_SERIAL", raising=False)
        tag = (list(p.mat)[:2], p.wb, knobs)
        assert b0 == b1, tag
        assert np.array_equal(np.asarray(cells0), np.asarray(cells1)), tag
        for j in range(len(jobs)):
            assert np.array_equal(msas0[j], msas1[j]), (tag, j)
        assert_oracle(msas1, cells1, trs, tag)


def test_matrix_that_overflows_int32_is_rejected():
    import cactus_b200 as cb
    for mat in ([65536 if v == 100 else v for v in R.CACTUS_MAT], [-65536 if v == -125 else v for v in R.CACTUS_MAT],
                [20000 * v for v in R.CACTUS_MAT]):
        with pytest.raises(cb.BarB200Error, match="partialOrderAlignmentSubMatrix"):
            cb.Engine(cb.PoaParams(partialOrderAlignmentSubMatrix=mat))
    cb.Engine(cb.PoaParams(partialOrderAlignmentSubMatrix=PP.PM65535, partialOrderAlignmentGapOpenPenalty1=1,
                           partialOrderAlignmentGapExtensionPenalty1=65533)).close()
