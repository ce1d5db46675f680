"""The POA path under substitution matrices and minimizer parameters other than Cactus' defaults (the config's
partialOrderAlignmentSubMatrix, ...MinimizerK and ...MinimizerW). CPU only; test_gpu_poa_params.py runs the same parameter sets on
the device.

Cactus' matrix is symmetric and its N row equals its N column, so a score looked up as [query][graph base] instead of
[graph base][query] would pass every test that uses it. Here the oracle runs an asymmetric matrix and its transpose, abPOA's small
scores (2 / -4, N = 0) under very narrow bands (the reference then runs int16 lanes and snaps band starts to 16-column groups), a
matrix with no positive entry, one with positive N scores, and the largest scores barb200_create accepts on 16383-base reads; and
the guide tree under minimizer windows that span several 64-position scan chunks, k = 20 (the hash fills the top of the key) and
reads too short to hold a minimizer. Every trace is compared with the reference's (digests, tests/_refgold.py) and with the host
build of the product's graph code (tests/hosttest)."""
import ctypes as C
import functools

import numpy as np
import pytest

import _reflib as R
from _synth import family, gapped_family
from test_gpu_poa_classes import longest_exactly
from test_oracle_vs_ref import assert_same_trace, same_trace


def transpose(mat):
    return [mat[5 * (i % 5) + i // 5] for i in range(25)]


def simple_mat(match, mismatch, n):
    return [n if i == 4 or j == 4 else (match if i == j else mismatch) for i in range(5) for j in range(5)]


# [graph base][query base] over A C G T N. Every off-diagonal pair differs, and so do the N row and the N column
ASYM = [95, -60, -20, -110, -80,
        -130, 100, -120, -30, -70,
        -140, -45, 100, -85, -90,
        -115, -135, -50, 90, -25,
        -40, -65, -100, -110, 70]
ABPOA = simple_mat(2, -4, 0)                                   # abPOA's default scores, N scoring 0 against everything
NO_POSITIVE = [0, -11, -7, -12, -5,
               -11, 0, -12, -7, -5,
               -7, -12, 0, -11, -5,
               -12, -7, -11, 0, -5,
               -6, -6, -6, -6, 0]
POSITIVE_N = [v if i % 5 < 4 and i // 5 < 4 else (100 if i == 24 else (30 if i // 5 == 4 else 15)) for i, v in enumerate(R.CACTUS_MAT)]
CACTUS_X524 = [524 * v for v in R.CACTUS_MAT]                  # Cactus' matrix scaled as far as |mat| <= 65535 allows (-125 * 524)
PM65535 = simple_mat(65535, -65535, -65535)
PM65535[24] = 65535
ABPOA_GAPS = dict(o1=4, e1=2, o2=24, e2=1)

# name: (parameters, seed of the jobs). A matrix and its transpose share their jobs
MATRIX_SETS = {
    "asymmetric": (dict(mat=ASYM), 1),
    "asymmetric_narrow": (dict(mat=ASYM, wb=20, wf=0.01), 2),
    "transposed": (dict(mat=transpose(ASYM)), 1),
    "transposed_narrow": (dict(mat=transpose(ASYM), wb=20, wf=0.01), 2),
    "abpoa": (dict(mat=ABPOA, **ABPOA_GAPS), 3),
    "no_positive": (dict(mat=NO_POSITIVE, o1=8, e1=3, o2=30, e2=1, wb=40, wf=0.02), 4),
    "positive_n": (dict(mat=POSITIVE_N), 5),
    "cactus_x524": (dict(mat=CACTUS_X524, o1=30000, e1=35000, o2=60000, e2=5000), 6),
    "pm65535": (dict(mat=PM65535, o1=1, e1=65533, o2=2, e2=65532), 7),
}
MINIMIZERS = [(1, 1), (20, 1), (5, 63), (5, 64), (5, 65), (11, 255), (20, 255)]


def params(name):
    return R.cactus_params(**MATRIX_SETS[name][0])


def mixed_jobs(rng, n, max_len):
    """n jobs of 2..13 reads of 1..max_len bases: related families (sorted or not, some N-rich), families with block indels, and
    unrelated ragged reads"""
    jobs = []
    lens = [v for v in (1, 5, 20, 60, 150, 300, 500, 800, 1100, 1500) if v <= max_len]
    for it in range(n):
        K, L = int(rng.integers(2, 14)), int(rng.choice(lens))
        kind = it % 4
        if kind == 3:
            jobs.append([rng.integers(0, 5 if rng.random() < 0.3 else 4, int(rng.integers(1, L + 1))).astype(np.uint8) for _ in range(K)])
        elif kind == 2 and L >= 60:
            jobs.append(gapped_family(rng, K, L, [1, 2, 3, 8, 27, 33, 64]))
        else:
            jobs.append(family(rng, K, L, sort=bool(rng.random() < 0.5), sub=float(rng.choice([0.02, 0.08, 0.2])),
                               ins=float(rng.choice([0.005, 0.03])), dele=float(rng.choice([0.005, 0.03])),
                               nfrac=float(rng.choice([0.0, 0.01, 0.15]))))
    return jobs


@functools.lru_cache(maxsize=None)
def _seeded_jobs(seed):
    return mixed_jobs(np.random.default_rng(6100 + seed), 14, 800)


def matrix_jobs(name):
    return _seeded_jobs(MATRIX_SETS[name][1])


@functools.lru_cache(maxsize=None)
def minimizer_jobs(k, w):
    """unsorted families with ragged lengths: reads cut short at random, some below k + w - 1 bases (no minimizer, so their
    similarity to every read is 0), N-rich ones; the first job is 70 reads deep"""
    rng = np.random.default_rng(6200 + 256 * k + w)
    jobs = []
    for it in range(6):
        K = 70 if it == 0 else int(rng.integers(3, 20))
        seqs = family(rng, K, int(rng.choice([150, 300, 500])), sort=False, sub=float(rng.choice([0.02, 0.1])), ins=0.01, dele=0.01,
                      nfrac=0.05 if it == 3 else 0.0)
        for i in range(K):
            u = rng.random()
            if u < 0.3:
                seqs[i] = seqs[i][int(rng.integers(0, len(seqs[i]))):]
            elif u < 0.45 and k + w - 1 > 1:
                seqs[i] = seqs[i][: int(rng.integers(1, k + w - 1))]
        jobs.append(seqs)
    return jobs


def minimizer_params(k, w):
    return R.cactus_params(k=k, w=w)


def reference_lane_count(p, qlen, node_n):
    """the lanes the reference's SIMD sweep takes (abpoa_align_simd.c:1293-1302; poa_graph.cuh: reference_lane_count): 16 (int16)
    when the largest possible score fits, else 8 (int32)"""
    mat = list(p.mat)
    max_mat, min_mis = max([0] + mat), max([0] + [-v for v in mat])
    max_score = max(qlen * max_mat, max(qlen, node_n) * p.gap_ext1 + p.gap_open1)
    return 16 if max_score <= 32767 - min_mis - (p.gap_open1 + p.gap_ext1) - (p.gap_open2 + p.gap_ext2) else 8


NARROW_ABPOA_BANDS = (0, 1, 3, 5, 10)


@functools.lru_cache(maxsize=None)
def narrow_abpoa_cases():
    """(params, job) pairs under abPOA's scores and gaps with very narrow bands (wf = 0): gapped and substituted families of 300 to
    2000 bases, and one 10 kbp window. The reference takes int16 lanes for all of them, so a band that starts left of its
    predecessors' inside one 16-column group snaps to theirs (abpoa_align_simd.c:957-959)"""
    rng = np.random.default_rng(6300)
    out = []
    for wb in NARROW_ABPOA_BANDS:
        p = R.cactus_params(mat=ABPOA, wb=wb, wf=0.0, **ABPOA_GAPS)
        for L in (300, 900, 2000):
            out.append((p, gapped_family(rng, int(rng.integers(3, 7)), L, [1, 2, 3, 5, 8, 13, 20])))
            out.append((p, family(rng, int(rng.integers(3, 7)), L, sort=bool(rng.random() < 0.5), sub=0.06, ins=0.01, dele=0.01)))
    p = R.cactus_params(mat=ABPOA, wb=10, wf=0.0, **ABPOA_GAPS)
    out.append((p, [s[:10000] for s in family(rng, 4, 10000, sub=0.03, ins=0.003, dele=0.003)]))
    return out


@functools.lru_cache(maxsize=None)
def extreme_cases():
    """(name, params, job): three 16383-base reads under the largest scores barb200_create accepts, where the sweep's largest value
    H' + (j + 1) e comes close to INT32_MAX (best score + 16384 e is 99.5 % of it under +-65535). A narrow band keeps the oracle's
    run short; the band still reaches column L"""
    rng = np.random.default_rng(6400)
    out = []
    for name, gaps in (("cactus_x524", dict(o1=30000, e1=35000, o2=60000, e2=5000)), ("pm65535", dict(o1=1, e1=65533, o2=2, e2=65532)),
                       ("pm65535_b", dict(o1=1, e1=65533, o2=65000, e2=1))):
        mat = CACTUS_X524 if name == "cactus_x524" else PM65535
        p = R.cactus_params(mat=mat, wb=50, wf=0.005, **gaps)
        out.append((name, p, longest_exactly(rng, 3, 16383, sub=0.005, ins=0.0005, dele=0.0005)))
    return out


def check_cases(tag, cases):
    for it, (p, seqs) in enumerate(cases):
        tr = R.oracle_poa_msa_trace(seqs, p)
        same_trace("%s/%d" % (tag, it), tr, seqs, p)
        assert_same_trace(tr, R.hosttest_poa_msa_trace(seqs, p), (tag, it))


@pytest.mark.parametrize("name", sorted(MATRIX_SETS))
def test_substitution_matrices(oracle_built, name):
    p = params(name)
    check_cases("params/mat/%s" % name, [(p, seqs) for seqs in matrix_jobs(name)])


def test_asymmetric_matrix_and_its_transpose_align_differently(oracle_built):
    """the matrix tests can only catch a transposed score lookup if the transpose changes the answer: it must change the MSA of at
    least a third of the jobs"""
    assert all(ASYM[5 * i + j] != ASYM[5 * j + i] for i in range(5) for j in range(i))
    for a, b in (("asymmetric", "transposed"), ("asymmetric_narrow", "transposed_narrow")):
        assert matrix_jobs(a) is matrix_jobs(b)
        differ = 0
        for seqs in matrix_jobs(a):
            ma, mb = R.oracle_poa_msa(seqs, params(a)), R.oracle_poa_msa(seqs, params(b))
            differ += ma.shape != mb.shape or not np.array_equal(ma, mb)
        assert 3 * differ >= len(matrix_jobs(a)), (a, differ)


@pytest.mark.parametrize("k,w", MINIMIZERS)
def test_minimizer_parameters(oracle_built, k, w):
    jobs = minimizer_jobs(k, w)
    assert any(len(s) < k + w - 1 for seqs in jobs for s in seqs) or k + w - 1 == 1
    check_cases("params/minimizer/%d,%d" % (k, w), [(minimizer_params(k, w), seqs) for seqs in jobs])


def test_abpoa_scores_under_narrow_bands(oracle_built):
    cases = narrow_abpoa_cases()
    for p, seqs in cases:
        for a in R.oracle_poa_msa_trace(seqs, p)["alns"]:
            assert reference_lane_count(p, a["qlen"], a["node_n"]) == 16, (p.wb, a["qlen"], a["node_n"])
    assert max(len(s) for _, seqs in cases for s in seqs) == 10000
    check_cases("params/abpoa_narrow", cases)


@pytest.mark.parametrize("i", range(3))
def test_largest_accepted_scores_on_16383_base_reads(oracle_built, i):
    name, p, seqs = extreme_cases()[i]
    assert max(len(s) for s in seqs) == 16383 and max(abs(v) for v in p.mat) <= 65535
    tr = R.oracle_poa_msa_trace(seqs, p)
    assert max(a["best_score"] for a in tr["alns"]) > 0.9 * 16383 * max(p.mat)
    same_trace("params/extreme/%s" % name, tr, seqs, p)
    assert_same_trace(tr, R.hosttest_poa_msa_trace(seqs, p), name)


@pytest.fixture(scope="module")
def lib():
    from cactus_b200 import build as b
    b.build()
    import cactus_b200 as cb
    return cb.load_library()


def create_error(lib, mat):
    """barb200_create's error for PoaParams with this matrix, or None if it created a context (on a machine with a GPU)"""
    import cactus_b200 as cb
    err = C.create_string_buffer(512)
    ctx = lib.barb200_create(C.byref(cb.PoaParams(partialOrderAlignmentSubMatrix=mat).c), err, 512)
    if ctx:
        lib.barb200_destroy(ctx)
        return None
    return err.value.decode()


def test_matrix_scores_that_overflow_int32_are_rejected(lib):
    """|mat| > 65535 can overflow the int32 DP scores at 16383 bases (in the reference too), so barb200_create refuses it before it
    looks for a device; 65535 passes that check"""
    for v in (65536, -65536, 20000 * 100):
        mat = list(R.CACTUS_MAT)
        mat[7] = v
        err = create_error(lib, mat)
        assert err is not None and "partialOrderAlignmentSubMatrix" in err and "int32" in err, err
    for mat in (PM65535, CACTUS_X524):
        err = create_error(lib, mat)
        assert err is None or err.startswith("no CUDA device"), err


def test_matrix_entries_outside_int32_are_refused_before_they_reach_the_library():
    """PoaParams stores the matrix as C ints: an entry of 2^31 or more would wrap into [-65535, 65535] and pass barb200_create's
    check, so PoaParams refuses it"""
    import cactus_b200 as cb
    for v in (2 ** 31, 2 ** 32 + 100, -2 ** 31 - 1):
        mat = list(R.CACTUS_MAT)
        mat[0] = v
        with pytest.raises(ValueError, match="partialOrderAlignmentSubMatrix"):
            cb.PoaParams(partialOrderAlignmentSubMatrix=mat)
