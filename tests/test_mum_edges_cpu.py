"""Edge cases of cPecan's MUM anchoring (K5, cactus_b200/csrc/mum_anchor.cu), aimed at the parts of the device program the host
build does not share: the k-mer sort (a bitonic sort of kTile = 2048 k-mer starts per tile over keys staged in shared memory,
then merge levels that double the run width) and the batch plumbing around it (second pass, chunks, empty problems).

edge_cases() names (family, case, sX, sY, params) for five families:
  runs       Y of exactly n k-mers, n at the tile and merge-run edges, all in one batch so that one merge level has problems
             below, at and above its width;
  ties       equal keys across tiles and runs: a segment of X twice in Y, tandem repeats, a homopolymer, small k on long pairs;
  widths     symbols of 1 to 7 bits, keys of 1 to 8 words, k = 1, per_word, per_word + 1, 50 and 64 per alphabet;
  recursion  a gap of the chain wider than one tile, holding a segment that is unique only inside the gap;
  degenerate pairs with lX < k, lY < k, lX * lY at the threshold, and empty sequences, between large pairs.
tests/test_gpu_mum_edges.py runs them on the device. The tests here check the generator: the host build of K5 and the plain-C
oracle agree on every case and under any order of equal k-mers, the oracle agrees with the reference where it was built, and every
family still reaches the edge it is named for."""
import collections
import ctypes as C
import functools

import numpy as np
import pytest

import _mumlib as M
import _reflib as R

TILE = 2048                        # mum_anchor.cu: kTile
K, BIGGER = 50, 500 * 500          # cPecan's defaults (bar.c squares anchorMatrixBiggerThanThis)
RUN_COUNTS = (1, 2, 2047, 2048, 2049, 4095, 4096, 4097, 3 * TILE + 1, 5 * TILE + 1, 2 ** 17 + 1)
FAMILIES = ("runs", "ties", "widths", "recursion", "degenerate")

_NOT_UPPER = bytes(c for c in range(1, 128) if not 65 <= c <= 90)    # 101 bytes that stay distinct under tolower()
ALPHABETS = collections.OrderedDict([
    ("bin", b"AC"), ("acgt", b"ACGT"), ("acgtn", b"ACGTN"), ("iupac", b"ACGTNRYKMSWBDHV"), ("mixed", b"ACGTNacgtn"),
    ("ascii17", _NOT_UPPER[::6][:17]), ("ascii33", _NOT_UPPER[::3][:33]), ("ascii127", bytes(range(1, 128)))])
ALPHABET_BITS = dict(bin=1, acgt=2, acgtn=3, iupac=4, mixed=3, ascii17=5, ascii33=6, ascii127=7)

Case = collections.namedtuple("Case", "family name sx sy params")


def _fit(rng, s, n):
    """s cut or padded with random bases to exactly n"""
    return s[:n] if len(s) >= n else s + M.rand_seq(rng, n - len(s))


def _mut(rng, s, alphabet=b"ACGT"):
    return M.mutate(rng, s, 0.02, 0.003, 0.003, alphabet)


def _runs(rng):
    out = []
    for n in RUN_COUNTS:
        ly = n + K - 1
        x = M.rand_seq(rng, max(ly + 300, BIGGER // ly + 1000))
        out.append(("ny%d" % n, x, _fit(rng, _mut(rng, x[150:150 + ly]), ly), {}))
    return out


def _ties(rng):
    out = []
    for gap in (2600, 9000):       # the two copies of s are > 1 and > 4 tiles apart in Y
        a, b, s = M.rand_seq(rng, 3000), M.rand_seq(rng, 3000), M.rand_seq(rng, 1200)
        out.append(("dup_%d" % gap, a + s + b, _mut(rng, a) + s + M.rand_seq(rng, gap) + s + _mut(rng, b), {}))
    for period, copies in ((37, 230), (301, 30)):
        unit = M.rand_seq(rng, period)
        fx, fy = M.related_pair(rng, 2500), M.related_pair(rng, 2500)
        out.append(("tandem_%d" % period, fx[0] + unit * (copies // 2) + fy[0], fx[1] + unit * copies + fy[1], {}))
    a, b = M.related_pair(rng, 3000), M.related_pair(rng, 3000)
    out.append(("homopolymer", a[0] + b"A" * 3000 + b[0], a[1] + b"A" * 5000 + b[1], {}))
    for k, u, L in ((8, 0, 12000), (8, 0, 37000), (12, 3, 15000), (12, 3, 40000)):
        x, y = M.related_pair(rng, L, sub=0.03)
        out.append(("k%d_u%d_%d" % (k, u, L), x, y, dict(k=k, u=u)))
    return out


def _widths(rng):
    out = []
    for name, alpha in ALPHABETS.items():
        per_word = 64 // ALPHABET_BITS[name]
        x = M.rand_seq(rng, 4600, alpha)
        y = _mut(rng, x, alpha)
        if name == "mixed":
            y = y.swapcase()
        for k in sorted({1, per_word, per_word + 1, 50, 64}):
            if k <= 64:
                out.append(("%s_k%d" % (name, k), x, y, dict(k=k)))
    return out


def _recursion(rng):
    a, b = M.related_pair(rng, 3000), M.related_pair(rng, 3000)
    s, d = M.rand_seq(rng, 400), M.rand_seq(rng, 300)
    # the gap between a and b: s once in X's and once in Y's part (unique there), d once in X's and twice, > 1 tile apart, in Y's.
    # The rest of the gap is filler of symbols the other sequence lacks, so that no short chance match splits the gap.
    def fx(n):
        return M.rand_seq(rng, n, b"NR")

    def fy(n):
        return M.rand_seq(rng, n, b"YK")
    gx = fx(1500) + d + fx(1000) + s + fx(2500)
    gy = fy(1000) + d + fy(2500) + s + fy(1200) + d + fy(1800)
    # s once more in Y after b: twice in the whole of Y, so no MUM at the first level
    return [("gap_unique", a[0] + gx + b[0] + M.rand_seq(rng, 2000), a[1] + gy + b[1] + s + M.rand_seq(rng, 2000), {})]


def _degenerate(rng):
    big = iter([M.related_pair(rng, L) for L in (20000, 9000, 15000, 6000, 25000, 11000)])
    y = M.rand_seq(rng, 4717)
    y2 = M.rand_seq(rng, 2809)
    return [("big0",) + next(big) + ({},),
            ("lx_below_k", M.rand_seq(rng, 30), M.rand_seq(rng, 20000), {}),
            ("big1",) + next(big) + ({},),
            ("ly_below_k", M.rand_seq(rng, 9000), M.rand_seq(rng, 40), {}),
            ("area_at_threshold", M.rand_seq(rng, 500), M.rand_seq(rng, 500), {}),
            ("area_above_threshold", y[1000:1053], y, {}),                           # 53 * 4717 = bigger + 1
            ("big2",) + next(big) + ({},),
            ("area_above_threshold_2", y2[300:389], y2, {}),                         # 89 * 2809 = bigger + 1
            ("empty_x", b"", M.rand_seq(rng, 3000), {}),
            ("big3",) + next(big) + ({},),
            ("empty_y", M.rand_seq(rng, 3000), b"", {}),
            ("empty_both", b"", b"", {}),
            ("big4",) + next(big) + ({},),
            ("lx_below_k_2", M.rand_seq(rng, 49), M.rand_seq(rng, 7000), {}),
            ("big5",) + next(big) + ({},)]


@functools.lru_cache(maxsize=None)
def edge_cases():
    """every Case of every family, in batch order; each family from its own seeded generator"""
    gens = dict(runs=_runs, ties=_ties, widths=_widths, recursion=_recursion, degenerate=_degenerate)
    out = []
    for i, fam in enumerate(FAMILIES):
        rng = np.random.default_rng(4100 + i)
        for name, sx, sy, p in gens[fam](rng):
            out.append(Case(fam, name, sx, sy, dict(dict(k=K, u=1, bigger=BIGGER), **p)))
    return tuple(out)


def edge_batches(family):
    """the family's cases grouped into batches of one parameter set, in order: [(params, [Case, ...]), ...]"""
    out = []
    for c in edge_cases():
        if c.family != family:
            continue
        for p, cs in out:
            if p == c.params:
                cs.append(c)
                break
        else:
            out.append((c.params, [c]))
    return out


# ---- what a case takes on the device ------------------------------------------------------------------------------------
def _host_lib():
    lib = R._load(M.MUM_HOST_SO)
    lib.hosttest_mum_key_words.restype = C.c_int
    lib.hosttest_mum_key_words.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int64]
    lib.hosttest_mum_gap_table.restype = C.c_int64
    lib.hosttest_mum_gap_table.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_void_p]
    return lib


def kmers(n, k):
    return max(n - k + 1, 0)


def key_words(c):
    return _host_lib().hosttest_mum_key_words(c.sx, len(c.sx), c.sy, len(c.sy), c.params["k"])


def symbol_bits(c):
    d = len(set(bytes(c.sx + c.sy).lower()))
    return max(1, (d - 1).bit_length())


def is_active(c):
    return len(c.sx) * len(c.sy) > c.params["bigger"]


def top_chain(c):
    """the pair's first-level chain as (x, y, len) MUMs, first to last, read off the oracle's non-recursive anchors: MUMs of a
    chain never touch on one diagonal (a successor starts past its predecessor's end in y), so each run of consecutive bases is
    one MUM"""
    a = M.oracle_mum_anchors(c.sx, c.sy, **dict(c.params, recursive=0))[::-1]
    out = []
    for x, y in a.tolist():
        if out and x == out[-1][0] + out[-1][2] and y == out[-1][1] + out[-1][2]:
            out[-1][2] += 1
        else:
            out.append([x, y, 1])
    return out


def gap_problems(c):
    """the second pass's problems of an active pair: (x0, y0, x1, y1) per gap of its chain (mum_plan.h: gap_table)"""
    ch = np.array(top_chain(c), np.int32).reshape(-1, 3)
    out = np.zeros(4 * (len(ch) + 1), np.int32)
    n = _host_lib().hosttest_mum_gap_table(ch.ctypes.data, len(ch), len(c.sx), len(c.sy), c.params["bigger"], out.ctypes.data)
    return [tuple(g) for g in out[:4 * n].reshape(n, 4).tolist()]


def merge_levels(max_ny):
    """mum_anchor.cu run_pass: run widths kTile, 2 kTile, ... below the longest problem"""
    n, w = 0, TILE
    while w < max_ny:
        n, w = n + 1, 2 * w
    return n


def _pass_launches(probs, k):
    """(nx, ny) per problem -> kernel launches of one pass: tile sort + merge levels when any Y k-mer, search when any X k-mer,
    chain"""
    if not probs:
        return 0
    max_ny = max(ny for _, ny in probs)
    return (1 + merge_levels(max_ny) if max_ny > 0 else 0) + (1 if sum(nx for nx, _ in probs) > 0 else 0) + 1


def planned_launches(cases, recursive):
    """kernel launches of one single-chunk batch of `cases` (one parameter set): the keys kernel when there is any k-mer, then
    the pairs' pass, then with recursiveMums the gaps' pass"""
    act = [c for c in cases if is_active(c)]
    if not act:
        return 0
    k = act[0].params["k"]
    n = 1 if any(kmers(len(c.sx), k) + kmers(len(c.sy), k) for c in act) else 0
    n += _pass_launches([(kmers(len(c.sx), k), kmers(len(c.sy), k)) for c in act], k)
    if recursive:
        n += _pass_launches([(kmers(x1 - x0, k), kmers(y1 - y0, k)) for c in act for x0, y0, x1, y1 in gap_problems(c)], k)
    return n


@functools.lru_cache(maxsize=None)
def _oracle(i, recursive):
    c = edge_cases()[i]
    return M.oracle_mum_anchors(c.sx, c.sy, **dict(c.params, recursive=recursive))


def oracle(c, recursive):
    """the oracle's anchors of a Case (cached: the GPU file compares several runs against it)"""
    return _oracle(edge_cases().index(c), recursive)


def _cases(family):
    return [c for c in edge_cases() if c.family == family]


def _repeated_across_tiles(s, k):
    """a k-mer of s that occurs at two starts in different tiles"""
    first = {}
    for p in range(kmers(len(s), k)):
        q = first.setdefault(s[p:p + k].lower(), p)
        if q // TILE != p // TILE:
            return True
    return False


# ---- the generator reaches its edges -------------------------------------------------------------------------------------
def test_run_count_family_reaches_every_tile_and_merge_edge():
    cs = _cases("runs")
    assert [kmers(len(c.sy), K) for c in cs] == list(RUN_COUNTS)
    assert all(is_active(c) and key_words(c) == 2 for c in cs)
    assert len(edge_batches("runs")) == 1                # one merge level sees problems below, at and above its width
    assert merge_levels(max(RUN_COUNTS)) == 7 and merge_levels(4097) == 2 and merge_levels(2048) == 0
    # keys, then tile sort, merge levels, search and chain
    by_n = {kmers(len(c.sy), K): c for c in cs}
    assert planned_launches([by_n[4097]], 0) == 1 + 1 + 2 + 1 + 1 and planned_launches([by_n[2 ** 17 + 1]], 0) == 1 + 1 + 7 + 1 + 1
    assert planned_launches([by_n[2048]], 0) == 1 + 1 + 0 + 1 + 1 and planned_launches(cs, 0) == planned_launches([by_n[2 ** 17 + 1]], 0)
    # an odd run count at some level: the last run has no partner
    assert any(-(-n // w) % 2 == 1 and n > w for n in RUN_COUNTS for w in (TILE, 2 * TILE, 4 * TILE))
    assert all(len(oracle(c, 1)) > 0 for c in cs if kmers(len(c.sy), K) >= TILE)


def test_tie_family_has_equal_keys_across_tiles():
    cs = {c.name: c for c in _cases("ties")}
    for name in ("dup_2600", "dup_9000"):
        c = cs[name]
        seg = c.sx[3000:4200]
        p, q = c.sy.find(seg), c.sy.rfind(seg)
        assert c.sx.count(seg) == 1 and p >= 0 and q - p > TILE + 1200, name
    assert cs["dup_9000"].sy.rfind(cs["dup_9000"].sx[3000:4200]) - cs["dup_9000"].sy.find(cs["dup_9000"].sx[3000:4200]) > 4 * TILE
    for name, period in (("tandem_37", 37), ("tandem_301", 301)):
        assert TILE % period and kmers(len(cs[name].sy), K) > 3 * TILE, name
    assert b"A" * 5000 in cs["homopolymer"].sy and b"A" * 5010 not in cs["homopolymer"].sy
    for c in cs.values():
        assert _repeated_across_tiles(c.sy, c.params["k"]), c.name
        assert is_active(c) and key_words(c) == (1 if c.params["k"] <= 32 else 2)
    assert {(c.params["k"], c.params["u"]) for c in cs.values()} == {(50, 1), (8, 0), (12, 3)}
    assert all(10000 <= len(c.sx) <= 40000 for c in cs.values() if c.params["k"] < 50)


def test_width_family_covers_every_symbol_and_key_width():
    cs = _cases("widths")
    bits, words = {}, {}
    for c in cs:
        alpha = c.name.rsplit("_k", 1)[0]
        b, w = symbol_bits(c), key_words(c)
        assert b == ALPHABET_BITS[alpha], c.name
        per_word = 64 // b
        assert w == -(-c.params["k"] // per_word), c.name
        assert kmers(len(c.sy), c.params["k"]) > 2 * TILE and is_active(c)
        bits.setdefault(alpha, b)
        words.setdefault(c.params["k"], set()).add(w)
    assert set(bits.values()) == set(range(1, 8))
    assert set().union(*words.values()) == set(range(1, 9))
    assert {1, 8} <= words[64]                           # one batch mixes 1-word and 8-word keys
    for alpha, b in ALPHABET_BITS.items():
        pw = 64 // b
        ks = {c.params["k"] for c in cs if c.name.rsplit("_k", 1)[0] == alpha}
        assert ks == {1, pw, 50, 64} | ({pw + 1} if pw < 64 else set()), alpha
    assert len(set(bytes(ALPHABETS["ascii127"]).lower())) == 101 and ALPHABETS["ascii127"] == bytes(range(1, 128))


def test_recursion_family_has_a_gap_wider_than_a_tile_with_a_segment_unique_only_there():
    (c,) = _cases("recursion")
    s = c.sx[3000 + 1500 + 300 + 1000:][:400]
    assert c.sy.count(s) == 2 and c.sx.count(s) == 1
    gaps = gap_problems(c)
    inner = [g for g in gaps if g[0] <= c.sx.find(s) and c.sx.find(s) + 400 <= g[2]]
    assert len(inner) == 1
    x0, y0, x1, y1 = inner[0]
    assert y0 > 0 and kmers(y1 - y0, K) > TILE and c.sy[y0:y1].count(s) == 1
    # s is anchored by the second pass only. At the first level a MUM reaching into [xs + 60, xs + 350) would have to start
    # on a k-mer inside s, which occurs twice in Y.
    xs, ys = c.sx.find(s), c.sy[y0:y1].find(s) + y0

    def inside(a):
        return int(np.sum((a[:, 0] >= xs + 60) & (a[:, 0] < xs + 350) & (a[:, 0] - xs == a[:, 1] - ys)))
    assert inside(oracle(c, 1)) > 200 and inside(oracle(c, 0)) == 0


def test_degenerate_family_puts_empty_problems_between_large_pairs():
    cs = _cases("degenerate")
    names = [c.name for c in cs]
    assert len(edge_batches("degenerate")) == 1
    for c in cs:
        lx, ly = len(c.sx), len(c.sy)
        if c.name.startswith("lx_below_k"):
            assert lx < K and is_active(c)
        elif c.name == "ly_below_k":
            assert ly < K and is_active(c)
        elif c.name == "area_at_threshold":
            assert lx * ly == BIGGER and not is_active(c)
        elif c.name.startswith("area_above_threshold"):
            assert lx * ly == BIGGER + 1 and is_active(c) and len(oracle(c, 1)) > 0
        elif c.name.startswith("empty"):
            assert (lx == 0 or ly == 0) and not is_active(c)
        else:
            assert c.name.startswith("big") and kmers(ly, K) > TILE
    for i, n in enumerate(names):
        if not n.startswith("big"):
            assert any(m.startswith("big") for m in names[:i]) and any(m.startswith("big") for m in names[i + 1:]), n


# ---- the host build and the oracle on every case ---------------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES)
def test_host_build_matches_the_oracle(family):
    for c in _cases(family):
        for rec in (1, 0):
            want = oracle(c, rec)
            p = dict(c.params, recursive=rec)
            assert np.array_equal(M.hosttest_mum_anchors(c.sx, c.sy, **p), want), (c.name, rec)
            for seed in (1, 2, 3):                  # any order of equal k-mers, as the device's unstable sort leaves them
                assert np.array_equal(M.hosttest_mum_anchors(c.sx, c.sy, tie_seed=seed, **p), want), (c.name, rec, seed)


@pytest.mark.skipif(not M.have_ref(), reason="oracle/_ref/libmum_ref.so not built (needs the reference sources)")
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_the_reference(family):
    checked = 0
    for c in _cases(family):
        for rec in (1, 0):
            p = dict(c.params, recursive=rec)
            want, would_abort = M.oracle_mum_anchors(c.sx, c.sy, with_abort=True, **p)
            if would_abort:                         # the reference is built with asserts on and aborts there (oracle/mum_oracle.c)
                continue
            assert np.array_equal(want, M.ref_mum_anchors(c.sx, c.sy, **p)), (c.name, rec)
            checked += 1
    assert checked >= len(_cases(family))
