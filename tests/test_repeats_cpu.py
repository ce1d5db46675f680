"""The POA path on repeat-rich and low-complexity inputs (tests/_repeats.py), CPU only; test_gpu_repeats.py runs the same cases on
the device.

On such inputs the answer depends on choices between equal candidates that random reads almost never force: where a missing
repeat unit goes, which of a homopolymer row's equal maxima bound the next band, which of many equal-weight edges is heaviest,
and which pair of reads with equal Jaccard similarity starts the guide tree. Here
  * the oracle's full trace (MSA, read order, cigars, every dp_beg / dp_end, cells) equals the reference's (digests in
    tests/golden/ref_digests_repeats.npz, in tests/_refgold.py's format), also for msa_make_partial_order_alignment and make_consistent_partial_order_alignments on windows cut
    inside a microsatellite and on two-end problems built on repeat parents;
  * the host build of the product's graph code (tests/hosttest) equals the oracle, and its shared-memory graph phases equal
    their serial forms (tests/hosttest/graph_phases.cpp) at the one-warp and 128-thread classes' scratch sizes and with none;
  * premises, one per family, show that the inputs reach the edges they are there for: the gap placement is ambiguous, the
    guide tree's tie-break changes the MSA, every key-capacity case holds the number of minimizer keys its name says (counted
    with the product's own sketch, tests/hosttest/gt_keys.cpp), and the worst-case key rung is out of reach."""
import ctypes as C
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

import _refgold as G
import _repeats as RP
import _reflib as R
from test_oracle_vs_ref import assert_same_trace

HOSTTEST = os.path.join(R.ROOT, "tests", "hosttest")
needs_gxx = pytest.mark.skipif(not shutil.which("g++"), reason="needs g++")


@functools.lru_cache(maxsize=None)
def trace(param, family, i):
    return R.oracle_poa_msa_trace(RP.cases(family)[i].seqs, RP.PARAMS[param])


# The reference's answers to this file's checks: digests of their own fixture, checked and recorded the way tests/_refgold.py
# checks and records tests/golden/ref_digests.npz (scripts/make_golden_ref_digests.py records both)
DIGESTS = os.path.join(R.ROOT, "tests", "golden", "ref_digests_repeats.npz")
_recorded, _stored = {}, {}


def check(key, got, ref_fn):
    if G.RECORDING:
        want = ref_fn()
        assert G.digest(want) == G.digest(got), key
        assert key not in _recorded, "duplicate key %s" % key
        _recorded[key] = G.digest(want)
        for name, v in G.parts(want):
            _recorded["%s#%s" % (key, name)] = G.digest(v)[:32]
        return
    if not _stored:
        z = np.load(DIGESTS)
        _stored.update(zip((k.decode() for k in z["keys"]), (v.decode() for v in z["digests"])))
    assert key in _stored, "no stored reference answer for %s (scripts/make_golden_ref_digests.py)" % key
    if G.digest(got) != _stored[key]:
        differ = [name for name, v in G.parts(got) if _stored.get("%s#%s" % (key, name)) != G.digest(v)[:32]]
        raise AssertionError("%s differs from the reference in %s" % (key, ", ".join(differ) or "its shape (number of fields)"))


def save_digests():
    keys = sorted(_recorded)
    np.savez_compressed(DIGESTS, keys=np.array([k.encode() for k in keys]), digests=np.array([_recorded[k].encode() for k in keys]))
    return sum("#" not in k for k in keys)


def same_trace(key, got, seqs, p):
    check(key, G.trace_view(got), lambda: G.trace_view(R.ref_poa_msa_trace(seqs, p)))


def same_msas(key, got, ref_fn):
    check(key, [np.asarray(m, np.uint8) for m in got], lambda: [np.asarray(m, np.uint8) for m in ref_fn()])


def gt_cases():
    return [c for c, _ in RP.gt_capacity()] + [c for c, _ in RP.gt_sort_edges()] + [RP.gt_big_family()]


# ---- the oracle against the reference, the host build against the oracle ----
@pytest.mark.parametrize("family", sorted(RP.FAMILIES))
@pytest.mark.parametrize("param", sorted(RP.PARAMS))
def test_oracle_equals_reference(oracle_built, family, param):
    p = RP.PARAMS[param]
    for i, c in enumerate(RP.cases(family)):
        same_trace("repeats/%s/%s" % (param, c.name), trace(param, family, i), c.seqs, p)


@pytest.mark.parametrize("family", sorted(RP.FAMILIES))
@pytest.mark.parametrize("param", sorted(RP.PARAMS))
def test_host_build_equals_oracle(oracle_built, family, param):
    p = RP.PARAMS[param]
    for i, c in enumerate(RP.cases(family)):
        assert_same_trace(trace(param, family, i), R.hosttest_poa_msa_trace(c.seqs, p), (param, c.name))


def test_key_capacity_cases_equal_reference(oracle_built):
    """the key-capacity and sort-edge jobs (Cactus' defaults: the minimizers they were tuned for)"""
    p = RP.PARAMS["default"]
    for c in gt_cases():
        tr = R.oracle_poa_msa_trace(c.seqs, p)
        same_trace("repeats/default/%s" % c.name, tr, c.seqs, p)
        assert_same_trace(tr, R.hosttest_poa_msa_trace(c.seqs, p), c.name)


@pytest.mark.parametrize("param", RP.LONG_WINDOW_PARAMS)
def test_long_window_equals_reference(oracle_built, param):
    c, p = RP.long_window(), RP.PARAMS[param]
    same_trace("repeats/%s/%s" % (param, c.name), R.oracle_poa_msa_trace(c.seqs, p), c.seqs, p)


@pytest.mark.parametrize("param", ("default", "narrow"))
def test_windows_and_two_ends_equal_reference(oracle_built, param):
    p = RP.PARAMS[param]
    for name, strs, win in RP.window_ends():
        got = R.oracle_msa_make_partial_order_alignment(strs, window_size=win, p=p)
        same_msas("repeats/%s/%s" % (param, name), [got], lambda: [R.ref_msa_make_partial_order_alignment(strs, window_size=win, p=p)])
    for name, (ends, ri, rr, ov), win in RP.two_end_cases():
        got = R.oracle_make_consistent_partial_order_alignments(ends, ri, rr, ov, window_size=win, p=p)
        same_msas("repeats/%s/%s" % (param, name), got,
                  lambda: R.ref_make_consistent_partial_order_alignments(ends, ri, rr, ov, window_size=win, p=p))
        for i in range(len(ends[0])):                  # kept prefix lengths of a shared string add up to its length
            assert int((got[0][i] != 5).sum()) + int((got[1][rr[0][i]] != 5).sum()) == len(ends[0][i]), (param, name, i)


# ---- the shared-memory graph phases ----
@pytest.fixture(scope="module")
def phases_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("graph_phases") / "libgraph_phases.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-pthread", "-fopenmp", "-x", "c++",
                           "-o", so, os.path.join(HOSTTEST, "graph_phases.cpp"), os.path.join(R.ROOT, "cactus_b200", "csrc", "pecan_plan.cpp")])
    lib = C.CDLL(so)
    lib.graph_phases_config.argtypes = [C.c_int, C.c_int]
    lib.graph_phases_stats.restype = C.POINTER(C.c_longlong)
    return so, lib


def phase_jobs():
    """every family under the default and the narrow band, and the key-capacity jobs"""
    return [(c.seqs, RP.PARAMS[param]) for param in ("default", "narrow") for c in RP.all_cases()] + \
        [(c.seqs, RP.PARAMS["default"]) for c in gt_cases()]


def run_phases(lib, so, monkeypatch, scr_bytes, threads):
    monkeypatch.setattr(R, "HOSTTEST_SO", so)
    monkeypatch.setenv("HOSTTEST_INCREMENTAL_ORDER", "1")
    lib.graph_phases_config(scr_bytes, threads)
    before = np.ctypeslib.as_array(lib.graph_phases_stats(), shape=(5,)).copy()
    for seqs, p in phase_jobs():
        R.hosttest_poa_msa_trace(seqs, p)            # asserts job status 0: no difference from the serial forms
    s = np.ctypeslib.as_array(lib.graph_phases_stats(), shape=(5,)).copy() - before
    assert s[4] == 0
    return dict(splice_smem=int(s[0]), splice_global=int(s[1]), topo_smem=int(s[2]), topo_global=int(s[3]))


@needs_gxx
@pytest.mark.parametrize("threads,kb", ((32, 10), (128, 40)))
def test_graph_phases_at_class_scratch(phases_lib, monkeypatch, threads, kb):
    """the one-warp class's 10 KB and the 128-thread class's 40 KB (poa_kernel.cuh: poa_scratch_bytes). In 10 KB the smaller graphs
    take the shared-memory forms and the larger ones (600-base homopolymer runs, 2 kbp tandem arrays) the global-memory forms; in
    40 KB every graph of these families fits"""
    so, lib = phases_lib
    c = run_phases(lib, so, monkeypatch, kb * 1024, threads)
    assert c["splice_smem"] > 0 and c["topo_smem"] > 0, c
    if kb == 10:
        assert c["splice_global"] > 0 and c["topo_global"] > 0, c


@needs_gxx
def test_graph_phases_without_scratch(phases_lib, monkeypatch):
    so, lib = phases_lib
    c = run_phases(lib, so, monkeypatch, 0, 128)
    assert c["splice_smem"] == 0 and c["topo_smem"] == 0 and c["splice_global"] > 0 and c["topo_global"] > 0, c


# ---- premises ----
def test_micro_and_tandem_gap_placement_is_ambiguous(oracle_built):
    """micro / tandem: a missing unit has several equal-score places. Reversing every read and reversing the MSA back gives the same
    MSA only where the reference's traceback rule is symmetric; on a repeat it is not. Both runs align in input order (progressive 0),
    so only the placement differs. At least 3/4 of each family's cases must change"""
    p = R.cactus_params(progressive=0)
    for family in ("micro", "tandem"):
        differ = 0
        for c in RP.cases(family):
            fwd = R.oracle_poa_msa(c.seqs, p)
            rev = R.oracle_poa_msa([s[::-1].copy() for s in c.seqs], p)[:, ::-1]
            differ += fwd.shape != rev.shape or not np.array_equal(fwd, rev)
        assert 4 * differ >= 3 * len(RP.cases(family)), (family, differ, len(RP.cases(family)))


def msa_in_order(seqs, order):
    """the oracle's MSA when the reads are aligned in `order` (progressive 0 on the permuted reads, rows put back)"""
    m = R.oracle_poa_msa([seqs[i] for i in order], R.cactus_params(progressive=0))
    out = np.empty_like(m)
    out[list(order)] = m
    return out


ORDER_SENSITIVE_TIES = ("ties/short_reads", "ties/all_n_mixed", "ties/duplicate_groups")


def test_ties_guide_tree_order_decides_the_msa(oracle_built):
    """ties: the guide tree of the reads listed in reverse picks a different order (its ties are broken by index), and aligning in
    that order changes the MSA, for at least 3/4 of the duplicate-group, short-read and all-N-mixed cases. Aligning in the guide
    tree's own order reproduces its MSA, so the difference is the order's. The identical-read cases have many equal Jaccard values
    but one MSA whatever the order: they are there for the reductions over all-equal values, which the MSA then pins"""
    p = RP.PARAMS["default"]
    sensitive = differ = 0
    for c in RP.ties():
        K = len(c.seqs)
        tr = R.oracle_poa_msa_trace(c.seqs, p)
        order = tr["read_id_map"]
        assert np.array_equal(msa_in_order(c.seqs, order), tr["msa"]), c.name
        rev = [K - 1 - i for i in R.oracle_poa_msa_trace(c.seqs[::-1], p)["read_id_map"]]
        if c.name.startswith("ties/identical/"):
            assert np.array_equal(msa_in_order(c.seqs, rev), tr["msa"]), c.name
        if c.name.startswith(ORDER_SENSITIVE_TIES):
            sensitive += 1
            differ += rev != order and not np.array_equal(msa_in_order(c.seqs, rev), tr["msa"])
    assert sensitive >= 8 and 4 * differ >= 3 * sensitive, (differ, sensitive)
    assert any(len(c.seqs) > 64 for c in RP.ties()) and any(len(c.seqs) <= 64 for c in RP.ties())      # one and two read-id words
    assert any(len(s) < RP.GT_K + RP.GT_W - 1 for c in RP.ties() for s in c.seqs)


def test_homopolymer_runs_reach_block_probe_and_warp_edges():
    """homopolymer: runs longer than one thread's 16 columns, one MATCH-run probe's 31 and one warp's 512, of lengths that differ
    between reads"""
    runs = [n for r in RP.HOMOPOLYMER_RUNS for n in r]
    assert any(16 < n <= 31 for n in runs) and any(31 < n <= 512 for n in runs) and max(runs) > 512
    for c in RP.homopolymer():
        assert len({len(s) for s in c.seqs}) > 1, c.name


def test_lowcomplexity_n_runs_restart_the_minimizer_scan():
    """lowcomplexity: every AT-rich case holds an N run of at least k + w bases"""
    for c in RP.lowcomplexity():
        if "at_rich_n" in c.name:
            longest = max(max((len(r) for r in "".join("N" if b == 4 else "x" for b in s).split("x")), default=0) for s in c.seqs)
            assert longest >= RP.GT_K + RP.GT_W, c.name


def test_window_ends_are_cut_inside_a_tract():
    """window: the first window boundary of every end lies inside its microsatellite, and the long window runs in the 640-thread class"""
    for name, strs, win in RP.window_ends():
        u = int(name.split("/")[1][1:])
        assert 60 < win < min(len(s) for s in strs) - 60, name
        assert all(s[win - u:win] == s[win:win + u] for s in strs[:1]), name        # the window cuts between two equal units
    assert all(4096 <= len(s) < 16 * 640 for s in RP.long_window().seqs)


@pytest.fixture(scope="module")
def key_counter(tmp_path_factory):
    if not shutil.which("g++"):
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("gt_keys") / "libgt_keys.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-x", "c++", "-o", so,
                           os.path.join(HOSTTEST, "gt_keys.cpp")])
    lib = C.CDLL(so)
    lib.gt_keys_count.restype = C.c_longlong
    lib.gt_keys_count.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]

    def count(seqs, k=RP.GT_K, w=RP.GT_W):
        lens = np.array([len(s) for s in seqs], np.int32)
        flat = np.ascontiguousarray(np.concatenate(seqs).astype(np.uint8))
        n = lib.gt_keys_count(k, w, 1, len(seqs), lens.ctypes.data, flat.ctypes.data)
        assert n >= 0
        return n
    return count


def key_cap(seqs, grow, w=RP.GT_W):
    from test_slot_layout_cpu import _lib
    out = (C.c_int64 * 9)()
    _lib().hosttest_gt_layout(1, len(seqs), sum(len(s) for s in seqs), w, grow, 0, out)
    return int(out[1])


def rung(n_keys, seqs, w=RP.GT_W):
    return 0 if n_keys <= key_cap(seqs, 1.0, w) else 1 if n_keys <= key_cap(seqs, 4.0, w) else 2


def test_key_capacity_cases_land_on_their_rungs(key_counter):
    """gt/cap: homopolymer reads of L >= k + w bases make L - k keys each; the exact cases hold exactly the optimistic plan's key_cap
    keys, the plus-one cases one more (the x4 retry), the 2 kbp homopolymer job takes the x4 retry and the (AC)n job none"""
    assert key_counter([np.zeros(RP.GT_K + RP.GT_W, np.uint8)] * 3) == 3 * RP.GT_W
    for c, want in RP.gt_capacity():
        n = key_counter(c.seqs)
        if "homopolymer" in c.name or "exact" in c.name or "plus1" in c.name:
            assert n == sum(len(s) - RP.GT_K for s in c.seqs), c.name
        if "exact" in c.name:
            assert n == key_cap(c.seqs, 1.0), c.name
        if "plus1" in c.name:
            assert n == key_cap(c.seqs, 1.0) + 1, c.name
        assert rung(n, c.seqs) == want, (c.name, n, key_cap(c.seqs, 1.0))
    # a stage plans its keys from its largest job: next to the big family, the plus-one job fits
    plus1 = [c for c, _ in RP.gt_capacity() if c.name == "gt/cap/plus1_2048"][0]
    big = RP.gt_big_family()
    assert key_counter(plus1.seqs) <= key_cap(big.seqs, 1.0) and key_counter(big.seqs) <= key_cap(big.seqs, 1.0)
    assert sum(len(s) for s in big.seqs) > sum(len(s) for s in plus1.seqs)


def test_sort_edge_cases_hold_their_key_counts(key_counter):
    """gt/sort: 2047, 2048 and 2049 keys, and 4096 and 4097, around the device sort's 2048-key shared tile (the sort pads to a power
    of two: up to 2048 keys it runs in one tile, above it the global-stride passes start); all within the optimistic plan"""
    counts = []
    for c, want in RP.gt_sort_edges():
        n = key_counter(c.seqs)
        assert n == want and rung(n, c.seqs) == 0, (c.name, n)
        counts.append(n)
    pad = [1 << (n - 1).bit_length() for n in counts]
    assert pad == [RP.SORT_TILE, RP.SORT_TILE, 2 * RP.SORT_TILE, 2 * RP.SORT_TILE, 4 * RP.SORT_TILE]


def test_worst_case_key_rung_is_out_of_reach(key_counter):
    """Is the worst-case rung (2 w keys per base) reachable? The x4 rung holds 4 (sum / 2 + 64) = 2 sum + 256 keys. A read emits a
    key when a new minimum arrives or the minimum leaves the window, plus the minimum's equal values when the window is rescanned;
    the most keys come from periodic reads, whose minimum recurs. Searching every period up to 2 w (40 random units each, three
    reads of about 2 kbp, w = 5 and 10) the most any job makes is one key per base less k per read (a homopolymer): half of what
    the x4 rung holds. No such input reaches the worst-case rung; it stays as the retry's last resort."""
    rng = np.random.default_rng(7900)
    for w in (5, 10):
        most = 0.0
        for per in range(1, 2 * w + 1):
            for _ in range(40):
                unit = rng.integers(0, 4, per).astype(np.uint8)
                seqs = [np.tile(unit, 2100 // per + 1)[:2000 - 7 * r] for r in range(3)]
                n = key_counter(seqs, w=w)
                assert rung(n, seqs, w) <= 1, (w, unit)
                most = max(most, n / sum(len(s) for s in seqs))
        assert most <= 1.0, (w, most)
