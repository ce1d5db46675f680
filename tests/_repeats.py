"""Seeded repeat-rich and low-complexity POA inputs for the tests (test-only, like _mumlib.py's families).

Random parents almost never force a choice between equal candidates; the sequence of real Cactus ends does, all the time. Each
family below makes such choices the common case:
  * micro: flank + (unit x copies) + flank, units of 1..6, 10, 15 and 40 bases, tracts of 20..600 bases, copy numbers that
    differ between reads by 1..3 units, point mutations in the flanks and, in every other case, inside the tract: a missing unit
    can go at any of n equal-score positions (the traceback's MATCH runs, its predecessor ballot and the insertion scan's
    "smallest t" decide which);
  * homopolymer: several runs per read whose lengths differ between reads, runs longer than 16 columns (one thread's block), 31
    (one MATCH-run probe) and 512 (one warp's columns): rows with many equal maxima (the band's arg-max columns);
  * tandem: a 20..400-base segment in 1..5 copies, the copy number varying per read, evolved with _synth.evolve: long ambiguous
    indels and far predecessors;
  * lowcomplexity: two- and three-letter alphabets, and AT-rich reads with N runs, some of at least k + w bases (the minimizer
    scan restarts after them);
  * ties: identical reads (K = 3 .. 90, one and two read-id words), identical reads plus one that differs, reads shorter than
    k + w - 1 (no minimizer) among longer ones, all-N reads, and groups of duplicated reads whose minimizer multisets are equal
    (Jaccard values tie, so the guide tree's first-maximum rule picks the order);
  * window: 10 kbp reads full of tracts (the 640-thread class), ends cut by window_size inside a microsatellite, and two-end
    problems on repeat parents.
A case is (name, reads); every abpoa_msa family runs under every parameter set of PARAMS."""
import collections
import functools

import numpy as np

import _reflib as R
from _synth import evolve, revcomp, to_ascii

Case = collections.namedtuple("Case", "name seqs")

PARAMS = {
    "default": R.cactus_params(),
    "narrow": R.cactus_params(wb=10, wf=0.01),
    "abpoa_gaps": R.cactus_params(o1=4, e1=2, o2=24, e2=1),
    "prog0": R.cactus_params(progressive=0),
}

MICRO_UNITS = (1, 2, 3, 4, 5, 6, 10, 15, 40)
MICRO_TRACTS = (20, 60, 150, 300, 600)
TANDEM_SEGMENTS = (20, 60, 150, 400)
HOMOPOLYMER_RUNS = ((17, 33), (20, 40, 70), (32, 520), (600,), (5, 16, 31, 12, 48))
IDENTICAL_K = (3, 8, 64, 65, 90)


def _rand(rng, n, p=None):
    return rng.choice(4, int(n), p=p).astype(np.uint8) if p is not None else rng.integers(0, 4, int(n)).astype(np.uint8)


def _point(rng, s, rate):
    """s with a fraction `rate` of its bases substituted (N stays N)"""
    s = s.copy()
    m = (rng.random(len(s)) < rate) & (s < 4)
    s[m] = (s[m] + rng.integers(1, 4, int(m.sum()))) % 4
    return s


def _unit(rng, u):
    """a unit of u bases that is not itself a repeat of a shorter unit"""
    while True:
        x = _rand(rng, u)
        if not any(np.array_equal(x, np.roll(x, d)) for d in range(1, u)):
            return x


def _cat(*parts):
    return np.concatenate([np.asarray(p, np.uint8) for p in parts])


def _copy_numbers(rng, K, base):
    """per read a copy number around `base`: the first two reads differ by 1..3 units, the others by up to 3"""
    d = int(rng.integers(1, 4))
    cn = [base, base + d] + [base + int(rng.integers(-3, 4)) for _ in range(K - 2)]
    return [max(1, c) for c in cn]


@functools.lru_cache(maxsize=None)
def micro():
    rng = np.random.default_rng(7100)
    out = []
    for i, u in enumerate(MICRO_UNITS):
        for j, tract in enumerate((MICRO_TRACTS[i % 5], MICRO_TRACTS[(i + 2) % 5])):
            unit, copies = _unit(rng, u), max(2, tract // u)
            lf, rf = _rand(rng, rng.integers(30, 80)), _rand(rng, rng.integers(30, 80))
            inside = (i + j) % 2 == 1
            seqs = []
            for c in _copy_numbers(rng, int(rng.integers(3, 9)), copies):
                t = np.tile(unit, c)
                seqs.append(_cat(_point(rng, lf, 0.02), _point(rng, t, 0.01) if inside else t, _point(rng, rf, 0.02)))
            out.append(Case("micro/u%d/t%d%s" % (u, tract, "/mut" if inside else ""), seqs))
    return out


@functools.lru_cache(maxsize=None)
def homopolymer():
    rng = np.random.default_rng(7200)
    out = []
    for runs in HOMOPOLYMER_RUNS:
        K = int(rng.integers(3, 7))
        spacers = [_rand(rng, rng.integers(20, 50)) for _ in range(len(runs) + 1)]
        bases = [int(rng.integers(0, 4)) for _ in runs]
        lens = [_copy_numbers(rng, K, n) for n in runs]
        seqs = []
        for r in range(K):
            parts = [_point(rng, spacers[0], 0.02)]
            for q, (b, n) in enumerate(zip(bases, lens)):
                parts += [np.full(n[r], b, np.uint8), _point(rng, spacers[q + 1], 0.02)]
            seqs.append(_cat(*parts))
        out.append(Case("homopolymer/%s" % "-".join(map(str, runs)), seqs))
    return out


@functools.lru_cache(maxsize=None)
def tandem():
    rng = np.random.default_rng(7300)
    out = []
    for seg in TANDEM_SEGMENTS:
        for cn in ((1, 2, 3), (2, 3, 5)):
            s = _rand(rng, seg)
            lf, rf = _rand(rng, rng.integers(30, 60)), _rand(rng, rng.integers(30, 60))
            K = int(rng.integers(3, 7))
            seqs = [evolve(_cat(lf, np.tile(s, int(cn[r % len(cn)])), rf), rng, sub=0.01, ins=0.003, dele=0.003) for r in range(K)]
            out.append(Case("tandem/s%d/c%s" % (seg, "".join(map(str, cn))), seqs))
    return out


def _with_n_runs(rng, s, runs):
    s = s.copy()
    for n in runs:
        at = int(rng.integers(10, len(s) - n - 10))
        s[at:at + n] = 4
    return s


@functools.lru_cache(maxsize=None)
def lowcomplexity():
    rng = np.random.default_rng(7400)
    out = []
    for name, alphabet, L in (("two_letter_at", (0, 3), 300), ("two_letter_cg", (1, 2), 180), ("three_letter", (0, 1, 3), 400)):
        p = np.array(alphabet, np.uint8)[rng.integers(0, len(alphabet), L)]
        seqs = [_point(rng, evolve(p, rng, sub=0.0, ins=0.01, dele=0.01), 0.01) for _ in range(int(rng.integers(3, 8)))]
        out.append(Case("lowcomplexity/%s" % name, seqs))
    at_rich = [0.4, 0.1, 0.1, 0.4]
    for L, runs in ((250, (3, 25)), (500, (12, 40, 20)), (700, (60, 5, 19))):
        p = _with_n_runs(rng, _rand(rng, L, at_rich), runs)
        seqs = [evolve(p, rng, sub=0.01, ins=0.005, dele=0.005) for _ in range(int(rng.integers(3, 7)))]
        # N runs whose length differs between reads
        seqs[1] = _cat(seqs[1][:40], np.full(int(rng.integers(20, 30)), 4, np.uint8), seqs[1][40:])
        out.append(Case("lowcomplexity/at_rich_n/%d" % L, seqs))
    return out


def _micro_parent(rng, u, copies, flank=40):
    return _rand(rng, flank), _unit(rng, u), copies, _rand(rng, flank)


def _micro_read(rng, parent, c, sub=0.0):
    lf, unit, _, rf = parent
    return _cat(_point(rng, lf, sub), np.tile(unit, c), _point(rng, rf, sub))


@functools.lru_cache(maxsize=None)
def ties():
    rng = np.random.default_rng(7500)
    out = []
    for K in IDENTICAL_K:
        p = _micro_read(rng, _micro_parent(rng, 3, 20), 20)
        out.append(Case("ties/identical/K%d" % K, [p.copy() for _ in range(K)]))
    for K in (5, 66):
        par = _micro_parent(rng, 2, 30)
        p = _micro_read(rng, par, 30)
        out.append(Case("ties/identical_plus_one/K%d" % K, [p.copy() for _ in range(K - 1)] + [_micro_read(rng, par, 28, 0.03)]))
    for u in (1, 4):
        par = _micro_parent(rng, u, 60 // u)
        long_reads = [_micro_read(rng, par, 60 // u + d, 0.02) for d in (0, 1, -2, 2)]
        short = [long_reads[0][40:40 + n] for n in (6, 12, 18)] + [_rand(rng, 9)]
        seqs = [long_reads[0], short[0], long_reads[1], short[1], short[2], long_reads[2], short[3], long_reads[3]]
        out.append(Case("ties/short_reads/u%d" % u, seqs))
    out.append(Case("ties/all_n", [np.full(n, 4, np.uint8) for n in (50, 64, 57, 3)]))
    par = _micro_parent(rng, 2, 25)
    out.append(Case("ties/all_n_mixed", [np.full(60, 4, np.uint8), _micro_read(rng, par, 25), np.full(45, 4, np.uint8),
                                         evolve(_micro_read(rng, par, 27), rng, sub=0.04, ins=0.02, dele=0.02),
                                         evolve(_micro_read(rng, par, 23), rng, sub=0.04, ins=0.02, dele=0.02)]))
    # groups of duplicated reads: every duplicate pair has Jaccard 1, so the most similar pair and the greedy order are ties
    for g, (u, copies, deltas) in enumerate(((2, 30, (0, 2, -2)), (3, 25, (0, 1, 3, -1)), (1, 40, (0, 3, -3)), (6, 12, (0, 1, -1, 2)),
                                             (15, 8, (0, 1, 2)), (4, 20, (0, -1, 2)))):
        par = _micro_parent(rng, u, copies)
        variants = [evolve(_micro_read(rng, par, copies + d), rng, sub=0.04, ins=0.02, dele=0.02) for d in deltas]
        seqs = [v.copy() for v in variants for _ in range(2)]
        if g % 2:
            seqs = [seqs[i] for i in range(0, len(seqs), 2)] + [seqs[i] for i in range(1, len(seqs), 2)]
        out.append(Case("ties/duplicate_groups/%d" % g, seqs))
    return out


FAMILIES = {"micro": micro, "homopolymer": homopolymer, "tandem": tandem, "lowcomplexity": lowcomplexity, "ties": ties}


def cases(family):
    return FAMILIES[family]()


def all_cases():
    return [c for f in FAMILIES for c in cases(f)]


# ---- window: 10 kbp reads, windows cut inside a tract, two-end problems on repeat parents ----
@functools.lru_cache(maxsize=None)
def long_window():
    """three reads of 9990..10239 bases (the 640-thread class): random stretches between tracts of units 1..40, each read with its
    own copy numbers"""
    rng = np.random.default_rng(7600)
    blocks = []
    while sum(len(b[0]) + b[1] * len(b[2]) for b in blocks) < 9800:
        u = int(rng.choice(MICRO_UNITS))
        blocks.append((_rand(rng, rng.integers(40, 200)), max(2, int(rng.integers(20, 300)) // u), _unit(rng, u)))
    seqs = []
    for r in range(3):
        parts = []
        for spacer, c, unit in blocks:
            parts += [_point(rng, spacer, 0.01), np.tile(unit, max(1, c + int(rng.integers(-3, 4))))]
        seqs.append(_cat(*parts)[:10239 - 3 * r])
    assert all(4096 <= len(s) <= 10239 for s in seqs)
    return Case("window/10k", seqs)


LONG_WINDOW_PARAMS = ("default", "narrow")


@functools.lru_cache(maxsize=None)
def window_ends():
    """(name, ASCII strings, window_size): ends whose windows are cut inside a microsatellite"""
    rng = np.random.default_rng(7700)
    out = []
    for i, (u, copies, win) in enumerate(((1, 150, 100), (2, 90, 120), (3, 70, 150), (6, 40, 110), (15, 14, 160), (40, 6, 200))):
        par = _micro_parent(rng, u, copies, flank=60)
        K = int(rng.integers(2, 7))
        reads = [_micro_read(rng, par, c, 0.02) for c in _copy_numbers(rng, K, copies)]
        assert 60 < win < 60 + copies * u                    # the first cut lies inside the tract
        out.append(("windows/u%d/w%d" % (u, win), [to_ascii(s) for s in reads], win))
    return out


@functools.lru_cache(maxsize=None)
def two_end_cases():
    """(name, (ends, right_end_indexes, right_end_row_indexes, overlaps), window_size) on microsatellite and tandem parents"""
    rng = np.random.default_rng(7800)
    out = []
    for i, (u, copies, K, win) in enumerate(((1, 60, 4, 10000), (2, 40, 3, 50), (3, 30, 5, 10000), (10, 10, 4, 60), (40, 4, 3, 10000))):
        lf, unit, _, rf = _micro_parent(rng, u, copies)
        parent = _cat(lf, np.tile(unit, copies), rf)
        out.append(("two_ends/u%d/w%d" % (u, win), _two_end_problem(rng, parent, K, sub=0.02, ins=0.02, dele=0.02), win))
    return out


def _two_end_problem(rng, parent, K, **kw):
    """_synth.two_end_problem's construction (bar/tests/poaBarTest.c:93-179) on descendants of a given parent: two ends whose
    strings are reverse complements of each other with full-length overlap"""
    s1 = [to_ascii(evolve(parent, rng, **kw)) for _ in range(K)]
    perm = [int(x) for x in rng.permutation(K)]
    s2 = [None] * K
    for i, pi in enumerate(perm):
        s2[pi] = revcomp(s1[i])
    inv = [0] * K
    for i, pi in enumerate(perm):
        inv[pi] = i
    return [s1, s2], [[1] * K, [0] * K], [perm, inv], [[len(s) for s in s1], [len(s) for s in s2]]


# ---- the guide tree's key capacity (slot_plan.h: GtNeeds plans sum / 2 + 64 keys per job, rounded up to a power of two; a job
# with more keys comes back with JOB_ERR_GT_CAP and runs again with x4 room, then at the worst case) and the device sort's
# 2048-key shared-memory tile (poa_kernel.cuh: kGuideTreeTileKeys). Minimizers at k = 15, w = 5 (Cactus' defaults) ----
GT_K, GT_W = 15, 5
SORT_TILE = 2048

# (name, base, read lengths, rung): homopolymer reads of L >= k + w bases make exactly L - k keys each. Rung 0: the job's keys
# fit its optimistic plan (the exact cases hold exactly key_cap keys); 1: they take the x4 retry
HOMOPOLYMER_CAP_CASES = (
    ("gt/cap/exact2048", 1, (715, 705, 673), 0),
    ("gt/cap/plus1_2048", 1, (716, 705, 673), 1),
    ("gt/cap/exact4096", 2, (1040, 1030, 1050, 1036), 0),
    ("gt/cap/plus1_4096", 2, (1041, 1030, 1050, 1036), 1),
    ("gt/cap/homopolymer_2k", 3, tuple(2000 - 3 * r for r in range(8)), 1),
)
# (name, seed, K, L, length the last read is cut to, keys): related families (sub 0.08, indels 0.02) whose minimizers are
# distinct hashes, at the edges of the sort's tile: 2047 and 2048 keys sort in one tile, 2049 and 4096 / 4097 need the
# global-stride passes (one merge size above the tile, two)
SORT_EDGE_CASES = (
    ("gt/sort/2047", 9007, 8, 760, 753, 2047),
    ("gt/sort/2048", 9008, 8, 760, 733, 2048),
    ("gt/sort/2049", 9008, 8, 760, 734, 2049),
    ("gt/sort/4096", 9000, 12, 1100, 90, 4096),
    ("gt/sort/4097", 9000, 12, 1100, 95, 4097),
)


@functools.lru_cache(maxsize=None)
def gt_capacity():
    """(case, rung): the homopolymer capacity cases and (AC)n reads of 2 kbp, whose period-2 minimizer makes one key every
    second base: below sum / 2, so a dinucleotide job never outgrows its plan (rung 0)"""
    out = [(Case(name, [np.full(n, b, np.uint8) for n in lens]), rung) for name, b, lens, rung in HOMOPOLYMER_CAP_CASES]
    ac = np.tile(np.array([0, 1], np.uint8), 1000)
    out.append((Case("gt/cap/dinucleotide_2k", [ac[:2000 - 2 * r] for r in range(8)]), 0))
    return out


@functools.lru_cache(maxsize=None)
def gt_sort_edges():
    """(case, keys)"""
    from _synth import family
    out = []
    for name, seed, K, L, cut, keys in SORT_EDGE_CASES:
        seqs = family(np.random.default_rng(seed), K, L, sort=False, sub=0.08, ins=0.02, dele=0.02)
        seqs[-1] = seqs[-1][:cut]
        out.append((Case(name, seqs), keys))
    return out


@functools.lru_cache(maxsize=None)
def gt_big_family():
    """a related family of 6 x 900 bases: its optimistic key plan (4096) holds the 2049 keys of gt/cap/plus1_2048"""
    from _synth import family
    return Case("gt/big_family", family(np.random.default_rng(9100), 6, 900, sub=0.03, ins=0.01, dele=0.01))
