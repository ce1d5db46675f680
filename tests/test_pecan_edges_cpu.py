"""Edge cases of cPecan's pair-HMM launch plan (cactus_b200/csrc/pecan.cu: stage_build) for the block program
(cactus_b200/csrc/pecan_cta.cuh), with the premise of every case pinned here on the product's own split and plan
(pecan_plan.cpp, behind a C symbol in tests/hosttest/pecan_plan_view.cpp, compiled here into a temporary directory).

A stage groups its sub-jobs by their widest diagonal into two classes and gives every class one launch. group_plan() restates
that rule; edge_batches() names the cases of four families:
  class  unanchored pairs (their band is the whole matrix: max_w = min(lx, ly) + 1) at the class boundary (widths 96 / 97), at the
         general class's shared ring width (320 / 321), long pairs whose every middle diagonal fills the ring (95 x 3000) or spills
         one position into the overflow block (320 x 3000), 0 x 5000 and 1 x 5000, and a 2500 x 2500 pair whose ring is mostly
         overflow;
  group  jobs that run with a ring wider than their own widest diagonal: the ring width of a launch is set by its widest job,
         and the band drift of a long or one-sidedly gapped job carries cells into the overflow block and round from below zero;
  room   threshold 0 with one traceback, so that every interior cell is a candidate: exactly the output room a stage reserves,
         one under it, one over it (the case that re-runs the job with room for every cell);
  fm     several tracebacks with the longest span between two of them exactly the FM ring's size (a full ring that wraps
         between segments), at 1024 doubles and at a larger power of two.
Here every case's premise is asserted, and every case runs through the host emulation of the block program in the
configuration its launch has on the device (threads, shared ring width, ring modulus), bit for bit against the
plain-C oracle. tests/test_gpu_pecan_edges.py runs the same cases on the device and checks that each launch is the
one planned here."""
import atexit
import collections
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import _reflib as R

# stage_build's block classes (kClass): (widest diagonal up to, threads, blocks per SM, ring positions in shared memory)
NARROW, GENERAL = (96, 32, 24, 96), (None, 128, 6, 320)
DEFAULT = (0.01, 1000, 40, 20)             # threshold, minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion
SPLIT = 3000                               # splitMatrixBiggerThanThis as the side length (bar.c squares it)
FAMILIES = ("class", "group", "room", "fm")

Case = collections.namedtuple("Case", "family name sx sy anchors params split")

_ACGT = np.frombuffer(b"ACGT", np.uint8)


def _bases(codes):
    return _ACGT[np.asarray(codes, np.int64)].tobytes()


def _mutated(rng, codes, sub):
    out = np.array(codes, np.int64)
    flip = rng.random(len(out)) < sub
    out[flip] = (out[flip] + rng.integers(1, 4, int(flip.sum()))) % 4
    return out


def _pair(seed, lx, ly, sub=0.1):
    """X of lx random bases; Y of ly bases holding a mutated copy of X in its middle (or of X's middle when ly < lx)"""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 4, lx)
    core = _mutated(rng, x, sub)
    if ly >= lx:
        pad = ly - lx
        y = np.concatenate([rng.integers(0, 4, pad // 2), core, rng.integers(0, 4, pad - pad // 2)])
    else:
        y = core[(lx - ly) // 2:(lx - ly) // 2 + ly]
    return _bases(x), _bases(y)


def _drift(seed, flank, mid, ins, in_y=True):
    """identical anchored flanks around an unanchored stretch of `mid` bases, against its mutated copy with `ins` extra bases
    in Y (or X): the band widens to about `mid` cells there and its centre moves by ins / 2 ring positions"""
    rng = np.random.default_rng(seed)
    a, m, b = rng.integers(0, 4, flank), rng.integers(0, 4, mid), rng.integers(0, 4, flank)
    mm = _mutated(rng, m, 0.1)
    long_mid = np.concatenate([mm[:mid // 2], rng.integers(0, 4, ins), mm[mid // 2:]])
    x, y = np.concatenate([a, m, b]), np.concatenate([a, long_mid, b])
    anchors = [(i, i) for i in range(flank)] + [(flank + mid + i, flank + mid + ins + i) for i in range(flank)]
    if not in_y:
        x, y, anchors = y, x, [(j, i) for i, j in anchors]
    return _bases(x), _bases(y), np.asarray(anchors, np.int64)


def _near_identical(seed, L, every):
    """X of L random bases and Y = X with a substitution every `every` bases; anchors on every other position of the diagonal"""
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 4, L)
    y = x.copy()
    y[every // 2::every] = (y[every // 2::every] + 1) % 4
    at = np.arange(0, L, 2)
    at = at[x[at] == y[at]]
    return _bases(x), _bases(y), np.stack([at, at], 1).astype(np.int64)


def _unanchored(family, name, seed, lx, ly, params=DEFAULT):
    sx, sy = _pair(seed, lx, ly)
    return Case(family, name, sx, sy, np.zeros((0, 2), np.int64), params, SPLIT)


# ---- the cases ----------------------------------------------------------------------------------------------------------------
# widest diagonal of each unanchored case of the class family
CLASS_WIDTHS = dict(sq95=96, sq96=97, sq319=320, sq320=321, long95=96, long320=321, e0=1, e1=2, sq2500=2501)
# output room at threshold 0: lx * ly candidates against min((lx + 1)(ly + 1), lx + ly + 64); (lx - 1)(ly - 1) - 65 = candidates - room
ROOM_SHAPES = dict(full_6x14=(6, 14, 0), full_2x66=(2, 66, 0), under_9x9=(9, 9, -1), under_3x33=(3, 33, -1), over_7x12=(7, 12, 1),
                   over_3x34=(3, 34, 1))
# FM ring exactly full: (seed, L, substitution spacing, minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion) -> capM.
# Found with pecan_plan by a deterministic search (L 1200 and 1600, spacing 40, every expansion 0..20, minDiags 30..200,
# traceBackDiagonals 1..40) for parameters whose longest span between two tracebacks is a power of two, with three or more.
FM_FULL = dict(fm1024=((7, 1200, 40, 83, 5, 10), 1024), fm2048=((7, 1200, 40, 126, 3, 14), 2048))


@functools.lru_cache(maxsize=None)
def edge_cases():
    out = []
    for i, (name, (lx, ly)) in enumerate([("sq95", (95, 95)), ("sq96", (96, 96)), ("sq319", (319, 319)), ("sq320", (320, 320)),
                                          ("long95", (95, 3000)), ("long320", (320, 3000)), ("e0", (0, 5000)), ("e1", (1, 5000)),
                                          ("sq2500", (2500, 2500))]):
        out.append(_unanchored("class", name, 100 + i, lx, ly))
    out.append(_unanchored("group", "long320", 200, 320, 3000))
    out.append(_unanchored("group", "sq700", 201, 700, 700))
    for i, in_y in enumerate((True, False)):
        sx, sy, a = _drift(210 + i, 400, 150, 500, in_y)
        out.append(Case("group", "drift_%s" % ("y" if in_y else "x"), sx, sy, a, DEFAULT, SPLIT))
    for i, (name, (lx, ly, _)) in enumerate(ROOM_SHAPES.items()):
        out.append(_unanchored("room", name, 300 + i, lx, ly, (0.0,) + DEFAULT[1:]))
    for name, ((seed, L, every, md, tb, ex), _) in FM_FULL.items():
        sx, sy, a = _near_identical(seed, L, every)
        out.append(Case("fm", name, sx, sy, a, (DEFAULT[0], md, tb, ex), SPLIT))
    return tuple(out)


QUEUE_SPLIT = 400          # splitMatrixBiggerThanThis of the queue batch: no unanchored pair of it splits, its long pairs do


def queue_batch(sms):
    """(sX, sY, anchors) of one batch with more narrow jobs than 24 blocks per SM (unanchored, 0..90 bases a side, empties
    included), more general jobs than 6 per SM (unanchored, 97..400 a side), and four long pairs whose anchor gaps split them
    into seven sub-jobs each (at QUEUE_SPLIT)"""
    rng = np.random.default_rng(77)
    pairs = []
    for i in range(24 * sms + 200):
        lx, ly = (0, int(rng.integers(0, 91))) if i % 97 == 0 else (int(v) for v in rng.integers(1, 91, 2))
        pairs.append(_pair(1000 + i, lx, ly) + (np.zeros((0, 2), np.int64),))
    for i in range(6 * sms + 100):
        lx, ly = (int(v) for v in rng.integers(97, 401, 2))
        pairs.append(_pair(5000 + i, lx, ly) + (np.zeros((0, 2), np.int64),))
    keep = np.concatenate([np.arange(k, k + 300) for k in range(0, 6000, 900)])      # anchor runs of 300 every 900 bases
    for i in range(4):
        sx, sy, a = _near_identical(9000 + i, 6000, 40)
        pairs.append((sx, sy, a[np.isin(a[:, 0], keep)]))
    order = rng.permutation(len(pairs))
    return [pairs[i] for i in order]


def wide_pairs():
    """eight unanchored pairs of about 1500 x 1500: one general launch whose rings take about 70 MB a block"""
    return [_pair(7000 + i, 1500 - 7 * i, 1500 + 5 * i) + (np.zeros((0, 2), np.int64),) for i in range(8)]


def oversized_pairs():
    """six 1 Mbp near-identical anchored pairs: a stage whose own arrays (about 50 bytes per base) take about 0.6 GB"""
    return [_near_identical(8000 + i, 1000000, 1000) for i in range(6)]


def plan_pairs(pairs, p=DEFAULT, split=SPLIT):
    return [s for sx, sy, a in pairs for s in pecan_plan(len(sx), len(sy), a, R.pecan_params(*p), split * split)]


def edge_batches(family):
    """the cases of `family` as device batches: one batch per parameter set, in case order"""
    batches = collections.OrderedDict()
    for c in edge_cases():
        if c.family == family:
            batches.setdefault((c.params, c.split), []).append(c)
    return list(batches.values())


# ---- the plan -----------------------------------------------------------------------------------------------------------------
PLAN_COLS = ("x1", "y1", "lx", "ly", "ragged", "cells", "max_w", "span_cells", "span_full_cells", "ring_center", "tracebacks", "out_room")
_PLAN_LIB = []


def _plan_lib():
    if not _PLAN_LIB:
        d = tempfile.mkdtemp(prefix="pecan_plan_view_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libpecan_plan_view.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so,
                               os.path.join(R.ROOT, "tests", "hosttest", "pecan_plan_view.cpp"),
                               os.path.join(R.ROOT, "cactus_b200", "csrc", "pecan_plan.cpp")])
        lib = C.CDLL(so)
        lib.hosttest_pecan_plan.restype = C.c_int64
        lib.hosttest_pecan_plan.argtypes = [C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.POINTER(R.PecanParams),
                                            C.c_int64, C.POINTER(C.c_void_p)]
        lib.hosttest_pecan_plan_free.argtypes = [C.c_void_p]
        lib.hosttest_pecan_plan_free.restype = None
        _PLAN_LIB.append(lib)
    return _PLAN_LIB[0]


def pecan_plan(lx, ly, anchors, p, split_bigger):
    """the product's split and plan of one pair (split_pair, plan_subjob in cactus_b200/csrc/pecan_plan.cpp): one dict per
    sub-job with the keys of PLAN_COLS"""
    lib = _plan_lib()
    a = np.ascontiguousarray(np.asarray(anchors, np.int64).reshape(-1, 2))
    out = C.c_void_p()
    n = lib.hosttest_pecan_plan(lx, ly, a.ctypes.data, len(a), 0, 0, C.byref(p), split_bigger, C.byref(out))
    assert n >= 0, "hosttest_pecan_plan failed: %d" % n
    rows = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_int64)), shape=(max(n * len(PLAN_COLS), 1),))[:n * len(PLAN_COLS)].copy()
    lib.hosttest_pecan_plan_free(out)
    return [dict(zip(PLAN_COLS, (int(v) for v in r))) for r in rows.reshape(n, len(PLAN_COLS))]


def params(c):
    return R.pecan_params(*c.params)


_plans, _oracles = {}, {}


def plan(c):
    """the product's sub-jobs of case c (dicts with the keys of PLAN_COLS)"""
    if (c.family, c.name) not in _plans:
        _plans[c.family, c.name] = pecan_plan(len(c.sx), len(c.sy), c.anchors, params(c), c.split * c.split)
    return list(_plans[c.family, c.name])


def oracle(c):
    """(triples, pre-floor posteriors) of the plain-C oracle"""
    if (c.family, c.name) not in _oracles:
        _oracles[c.family, c.name] = R.oracle_pecan_aligned_pairs(c.sx, c.sy, c.anchors, False, False, params(c), c.split * c.split)
    return _oracles[c.family, c.name]


def pow2ceil(v):
    p = 1024
    while p < v:
        p <<= 1
    return p


def class_of(max_w):
    return NARROW if max_w <= NARROW[0] else GENERAL


def group_plan(subs, sms):
    """The launches stage_build plans for sub-jobs `subs` on a device of `sms` SMs, before any cut of the block count for
    memory: per class that has jobs (narrow first) its jobs, threads, blocks, ring width RW (the modulus: the widest diagonal of
    the class, at least its shared part), shared ring positions RWs and FM / FF ring doubles."""
    out = []
    for cls in (NARROW, GENERAL):
        js = [s for s in subs if class_of(s["max_w"]) is cls]
        if not js:
            continue
        out.append(dict(jobs=len(js), threads=cls[1], blocks=min(sms * cls[2], len(js)), RW=max(cls[3], max(s["max_w"] for s in js)),
                        RWs=cls[3], cap_m=pow2ceil(max(1, max(s["span_cells"] for s in js))),
                        cap_f=pow2ceil(5 * max(1, max(s["span_full_cells"] for s in js)))))
    return out


def slot_bytes(g):
    """the ring scratch of one block of launch g (stage_build: slot_doubles): FM ring, FF ring, ring and reduction overflow"""
    return 8 * (g["cap_m"] + g["cap_f"] + 11 * (g["RW"] - g["RWs"]) + 8)


def stage_fixed_bytes(subs):
    """the device memory of a stage besides its rings (stage_build: fixed): symbols, band tables, a Job and an out count per
    sub-job, twice the output room, and 64 MiB"""
    return sum(s["lx"] + s["ly"] + 16 * (s["lx"] + s["ly"] + 2) + 56 + 8 + 32 * s["out_room"] for s in subs) + (64 << 20)


def cut_blocks(groups, budget):
    """stage_build's loop for `budget` bytes of rings: the launch with the most ring bytes loses a quarter of its blocks until
    the rings fit; None when one block each does not"""
    gs = [dict(g) for g in groups]
    while sum(slot_bytes(g) * g["blocks"] for g in gs) > budget:
        big = None
        for g in gs:
            if g["blocks"] > 1 and (big is None or slot_bytes(g) * g["blocks"] > slot_bytes(big) * big["blocks"]):
                big = g
        if big is None:
            return None
        big["blocks"] = max(1, big["blocks"] * 3 // 4)
    return gs


def launch_of(sub, groups):
    """the planned launch (an item of group_plan's list) that runs sub-job `sub`"""
    cls = class_of(sub["max_w"])
    return next(g for g in groups if g["threads"] == cls[1])


def ring_positions(sub, band, RWs):
    """ring positions of every cell of a sub-job before the wrap modulo RW (pecan_cta.cuh: ring_i0): a = (xmyL + parity) / 2 +
    ly - ring_shift + k for cell k of a diagonal, ring_shift = ring_center - RWs / 2 (stage_build); `band` = (xmyL, xmyR) per
    diagonal"""
    L, Rr = band
    d = np.arange(len(L))
    a0 = ((L + (d & 1)) >> 1) + sub["ly"] - (sub["ring_center"] - RWs // 2)
    w = (Rr - L) // 2 + 1
    return a0, a0 + w - 1          # first and last position of every diagonal


@pytest.fixture(scope="module")
def product_band():
    """barb200_pecan_band of the product library (host-only)"""
    import cactus_b200 as cb
    from cactus_b200 import build as b
    b.build()
    return lambda c: cb.pecan_band(len(c.sx), len(c.sy), c.anchors, c.params[3])


def _case(family, name):
    return next(c for c in edge_cases() if (c.family, c.name) == (family, name))


# ---- premises -----------------------------------------------------------------------------------------------------------------
def test_the_group_rule_restates_stage_build():
    subs = [dict(max_w=w, span_cells=s, span_full_cells=f) for w, s, f in ((96, 1, 1), (1, 1024, 205), (97, 1025, 2), (2501, 5, 300))]
    assert group_plan(subs, 132) == [dict(jobs=2, threads=32, blocks=2, RW=96, RWs=96, cap_m=1024, cap_f=2048),
                                     dict(jobs=2, threads=128, blocks=2, RW=2501, RWs=320, cap_m=2048, cap_f=2048)]
    many = [dict(max_w=1 + i % 200, span_cells=1, span_full_cells=1) for i in range(10000)]
    assert [(g["jobs"], g["blocks"]) for g in group_plan(many, 132)] == [(4800, 24 * 132), (5200, 6 * 132)]


def test_class_edges_premise(product_band):
    for c in edge_cases():
        if c.family != "class":
            continue
        (s,) = plan(c)                                  # one sub-job: the whole unanchored matrix
        lx, ly = len(c.sx), len(c.sy)
        assert s["max_w"] == min(lx, ly) + 1 == CLASS_WIDTHS[c.name], c.name
        assert s["cells"] == (lx + 1) * (ly + 1), c.name
        L, Rr = product_band(c)
        w = (Rr - L) // 2 + 1
        assert w.max() == s["max_w"] and w.sum() == s["cells"], c.name
        (g,) = group_plan([s], 132)
        assert g["RW"] == max(g["RWs"], s["max_w"]), c.name
    # alone, the 95 x 3000 job fills its ring (RW = 96) on every middle diagonal; the 320 x 3000 job spills exactly one of its
    # RW = 321 positions into the overflow block there
    for name, rw, rws in (("long95", 96, 96), ("long320", 321, 320)):
        c = _case("class", name)
        (g,) = group_plan(plan(c), 132)
        assert (g["RW"], g["RWs"]) == (rw, rws), name
        L, Rr = product_band(c)
        w = (Rr - L) // 2 + 1
        lx = len(c.sx)
        assert np.all(w[lx:len(c.sy) + 1] == rw), name
    # the class boundary and the general class's shared width sit between the pairs of the two sides
    by = {c.name: group_plan(plan(c), 132)[0] for c in edge_cases() if c.family == "class"}
    assert by["sq95"]["threads"] == 32 and by["sq96"]["threads"] == 128
    assert by["sq319"]["RW"] == by["sq319"]["RWs"] == 320 and by["sq320"]["RW"] == 321
    assert by["sq2500"]["RW"] == 2501 and by["sq2500"]["RW"] > 7 * by["sq2500"]["RWs"]
    (batch,) = edge_batches("class")
    narrow, general = group_plan([s for c in batch for s in plan(c)], 132)
    assert (narrow["jobs"], narrow["RW"], general["jobs"], general["RW"]) == (4, 96, 5, 2501)


def test_group_ring_width_premise(product_band):
    (batch,) = edge_batches("group")
    subs = {c.name: plan(c) for c in batch}
    assert all(len(s) == 1 for s in subs.values())
    (g,) = group_plan([s for c in batch for s in plan(c)], 132)      # all in the general class
    assert (g["RW"], g["RWs"]) == (701, 320) and subs["sq700"][0]["max_w"] == 701
    for c in batch:
        if c.name == "sq700":
            continue
        (s,) = subs[c.name]
        assert NARROW[0] < s["max_w"] < g["RW"], c.name
        lo, hi = ring_positions(s, product_band(c), g["RWs"])
        # cells in the overflow block and cells that wrap round from below zero; no diagonal meets itself modulo RW
        assert hi.max() >= g["RWs"] and lo.min() < 0, (c.name, lo.min(), hi.max())
        assert np.all(hi - lo < g["RW"]), c.name
    lo, hi = ring_positions(subs["long320"][0], product_band(_case("group", "long320")), g["RWs"])
    assert hi.max() >= g["RW"]                      # its drift also wraps round from above the modulus


def test_output_room_premise():
    for c in edge_cases():
        if c.family != "room":
            continue
        lx, ly, delta = ROOM_SHAPES[c.name]
        assert (len(c.sx), len(c.sy)) == (lx, ly) and c.params[0] == 0.0 and c.params[1] > lx + ly
        assert (lx - 1) * (ly - 1) - 65 == delta, c.name
        (s,) = plan(c)
        assert s["tracebacks"] == 1 and s["cells"] == (lx + 1) * (ly + 1), c.name
        assert s["out_room"] == min((lx + 1) * (ly + 1), lx + ly + 64), c.name
        assert lx * ly - s["out_room"] == delta, c.name
        t, po = oracle(c)
        assert len(t) == lx * ly, c.name               # every interior cell is a candidate


def test_fm_ring_full_premise():
    caps = []
    for c in edge_cases():
        if c.family != "fm":
            continue
        (s,) = plan(c)
        (g,) = group_plan([s], 132)
        assert s["tracebacks"] >= 3, c.name
        assert s["span_cells"] == g["cap_m"] == FM_FULL[c.name][1], c.name
        # 5 * span_full is never a power of two >= 1024: the FF ring is never exactly full
        assert g["cap_f"] > 5 * s["span_full_cells"], c.name
        caps.append(g["cap_m"])
    assert 1024 in caps and max(caps) > 1024


# ---- every case through the host emulation, in its launch's configuration ------------------------------------------------------
def _emulate(c, groups):
    (s,) = plan(c)
    g = launch_of(s, groups)
    return R.hosttest_pecan_aligned_pairs(c.sx, c.sy, c.anchors, False, False, params(c), c.split * c.split, threads=g["threads"],
                                          ring_width=g["RWs"], ring_extra=g["RW"] - s["max_w"])


@pytest.mark.parametrize("family", FAMILIES)
def test_family_in_its_launch_configuration_matches_the_oracle(oracle_built, family):
    for batch in edge_batches(family):
        together = group_plan([s for c in batch for s in plan(c)], 132)
        for c in batch:
            to, po = oracle(c)
            configs = [("batch", together)]
            alone = group_plan(plan(c), 132)
            if alone != [launch_of(plan(c)[0], together)]:
                configs.append(("alone", alone))
            for how, groups in configs:
                t, p, cells = _emulate(c, groups)
                assert np.array_equal(t, to) and np.array_equal(p, po), (c.name, how)
                assert cells == sum(s["cells"] for s in plan(c)), (c.name, how)


def test_shared_work_queue_premise():
    pairs = queue_batch(132)
    per_pair = [len(plan_pairs([q], split=QUEUE_SPLIT)) for q in pairs]
    assert sorted(per_pair)[-5:] == [1, 7, 7, 7, 7]
    narrow, general = group_plan(plan_pairs(pairs, split=QUEUE_SPLIT), 132)
    assert narrow["blocks"] == 24 * 132 < narrow["jobs"] and general["blocks"] == 6 * 132 < general["jobs"]
    assert general["RW"] > general["RWs"]              # some sub-jobs of the long pairs and pairs up to 400 wide spill


def test_cut_block_count_premise():
    """the memory share test_gpu_pecan_edges gives the wide jobs (their stage + 3.5 blocks of rings) cuts 8 blocks to 3, and
    still to fewer than 8 when free memory grows by 80 % between two queries; the oversized stage does not fit twice that share"""
    subs = plan_pairs(wide_pairs())
    (g,) = group_plan(subs, 132)
    assert (g["jobs"], g["blocks"], g["threads"], g["RW"]) == (8, 8, 128, 1501) and slot_bytes(g) > 60e6
    share = stage_fixed_bytes(subs) + 3.5 * slot_bytes(g)
    assert stage_fixed_bytes(subs) < (64 << 20) + (2 << 20)
    for free_grows, blocks in ((1.0, 3), (1.2, 4), (1.8, 6)):
        (cut,) = cut_blocks([g], free_grows * share - stage_fixed_bytes(subs))
        assert cut["blocks"] == blocks, free_grows
    assert cut_blocks([g], slot_bytes(g) - 1) is None
    assert stage_fixed_bytes(plan_pairs(oversized_pairs())) > 2 * share
