"""barb200_trace_ends on the CPU: the product's window rounds (cactus_b200/csrc/host_end_trace.cpp over bar_windows.h) on the stand-in
device, against the restated chain (oracle_trace_ends) and the unmodified reference's own chain observed through -Wl,--wrap
(libbar_trace_ref.so), window by window: each window's input slice, its POA job's per-alignment trace, its trimmed lengths, and each
end's final MSA."""
import copy

import numpy as np
import pytest

import _end_trace_cases as X
import _endtrace as T
import _reflib as R
import cactus_b200 as cb

needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libbar_trace_ref.so not built (needs the reference sources)")


@pytest.fixture(scope="module")
def built():
    T.build()


def _run(c, which, p=None):
    p = p or R.cactus_params(**c["poa"])
    if which == "standin":
        s = T.Standin(p)
        try:
            return s.trace_ends(*X.args(c))
        finally:
            s.close()
    return (T.oracle_trace_ends if which == "oracle" else T.ref_trace_ends)(*X.args(c), p=p)


def _same(a, b, what):
    for e, (x, y) in enumerate(zip(a, b)):
        d = cb.first_end_trace_difference(cb.parse_end_trace(x), cb.parse_end_trace(y))
        assert d is None and np.array_equal(x, y), "%s: end %d differs at %s" % (what, e, d)
    assert len(a) == len(b)


@pytest.fixture(scope="module")
def flower_cases(built, tmp_path_factory):
    import _flowers as F
    if not F.have("harvest"):
        pytest.skip("oracle/_ref/libflower_harvest.so not built (needs the reference sources)")
    return X.flower_cases(str(tmp_path_factory.mktemp("harvest")))


def _premises(c, words):
    """what each seeded case is there to exercise"""
    ws = [T.read_end_trace(w) for w in words]
    name = c["name"]
    if name == "five_windows":
        assert len(ws[0]["windows"]) == 5
    if name == "odd_overlap":
        from math import floor
        assert (int(floor(0.5 * c["window_size"])) - 1) % 2 == 1
        assert all(len(w["windows"]) >= 3 for w in ws)
    if name in ("n_standin", "one_plus_empty"):
        assert any(win["empty"].any() for w in ws for win in w["windows"])
    if name == "prog_switch":
        assert {win["progressive"] for win in ws[0]["windows"]} == {0, 1}
    if name == "single":
        assert [len(w["windows"]) for w in ws][::2] == [0, 0]
    if name == "one_plus_empty":
        assert len(ws[1]["windows"]) == 0 and ws[1]["msa"].shape == (2, 0)
    if name == "rc_partial":
        assert c["ov"][0][0] < len(c["ends"][0][0])


@needs_ref
@pytest.mark.parametrize("c", X.cases(), ids=lambda c: c["name"])
def test_the_two_oracles_agree_window_by_window(built, c):
    """premise: the restated chain equals the reference's own, word for word"""
    ref = _run(c, "ref")
    _same(_run(c, "oracle"), ref, "restated vs reference")
    _premises(c, ref)


@needs_ref
@pytest.mark.parametrize("c", X.cases()[1:], ids=lambda c: c["name"])
def test_wrapping_changes_nothing(built, c):
    """the wrapped reference library's final MSAs equal libbar_ref.so's, and its recorded MSAs are those"""
    p = R.cactus_params(**c["poa"])
    ends, ri, rr, ov = c["ends"], c["ri"], c["rr"], c["ov"]
    if ri is None:
        ri = [[-1] * len(e) for e in ends]
        rr = [[-1] * len(e) for e in ends]
        ov = [[0] * len(e) for e in ends]
    kw = dict(window_size=c["window_size"], max_prog_rows=c["max_prog_rows"], max_prog_length_diff=c["max_prog_length_diff"], p=p)
    got = T.wrapped_ref_consistent(ends, ri, rr, ov, **kw)
    want = R.ref_make_consistent_partial_order_alignments(ends, ri, rr, ov, **kw)
    rec = [T.read_end_trace(w)["msa"] for w in _run(c, "ref")]
    for a, b, m in zip(got, want, rec):
        assert np.array_equal(a, b) and np.array_equal(a, m)


@pytest.mark.parametrize("c", X.cases(), ids=lambda c: c["name"])
def test_product_rounds_equal_the_oracles(built, c):
    got = _run(c, "standin")
    _same(got, _run(c, "oracle"), "product vs restated")
    if T.have_ref():
        _same(got, _run(c, "ref"), "product vs reference")


@pytest.mark.parametrize("c", X.cases(), ids=lambda c: c["name"])
def test_final_msas_equal_the_end_queue(built, c):
    """the argument that the queue's batching cannot change a window, checked through its result"""
    p = R.cactus_params(**c["poa"])
    s = T.Standin(p)
    try:
        got = [T.read_end_trace(w)["msa"] for w in s.trace_ends(*X.args(c))]
        kw = dict(window_size=c["window_size"], max_prog_rows=c["max_prog_rows"], max_prog_length_diff=c["max_prog_length_diff"])
        want = s.consistent(c["ends"], c["ri"], c["rr"], c["ov"], **kw) if c["ri"] is not None else s.independent(c["ends"], **kw)
    finally:
        s.close()
    for a, b in zip(got, want):
        assert a.shape == b.shape and np.array_equal(a, b)


def test_flowers_of_the_golden_fixture(flower_cases):
    """every top-level alignment call of a reference bar() on the flowers behind tests/golden/flower_golden.npz"""
    assert len(flower_cases) >= 11
    for c in flower_cases:
        got = _run(c, "standin")
        _same(got, _run(c, "oracle"), c["name"] + ": product vs restated")
        _same(got, _run(c, "ref"), c["name"] + ": product vs reference")


def test_first_difference_names_each_planted_field(built):
    c = next(c for c in X.cases() if c["name"] == "n_standin")
    base = cb.parse_end_trace(_run(c, "standin")[0])
    assert len(base["windows"]) >= 3
    assert cb.first_end_trace_difference(base, copy.deepcopy(base)) is None

    def planted(change):
        t = copy.deepcopy(base)
        change(t)
        return cb.first_end_trace_difference(t, base)

    def arr(w, f, i, d=1):
        w[f][i] += d
    assert planted(lambda t: arr(t["windows"][1], "offsets", 2)) == (1, "offsets", 2)
    assert planted(lambda t: arr(t["windows"][2], "lens", 1)) == (2, "lens", 1)
    assert planted(lambda t: arr(t["windows"][0], "empty", 3)) == (0, "empty", 3)
    assert planted(lambda t: t["windows"][2].update(progressive=1 - t["windows"][2]["progressive"])) == (2, "progressive", None)
    assert planted(lambda t: t["windows"][1]["trace"].update(read_id_map=t["windows"][1]["trace"]["read_id_map"][::-1])) == \
        (1, "trace", (None, "read_id_map", None))
    assert planted(lambda t: arr(t["windows"][1]["trace"]["alns"][2], "dp_beg", 4)) == (1, "trace", (2, "dp_beg", 4))
    assert planted(lambda t: arr(t["windows"][0]["trace"]["alns"][1], "dp_end", 0, -1)) == (0, "trace", (1, "dp_end", 0))
    assert planted(lambda t: t["windows"][2]["trace"]["alns"][1].update(best_score=-7)) == (2, "trace", (1, "best_score", None))
    assert planted(lambda t: arr(t["windows"][1]["trace"]["alns"][1], "cigar", 1, np.uint64(1))) == (1, "trace", (1, "cigar", 1))
    assert planted(lambda t: arr(t["windows"][1], "trimmed_lens", 2)) == (1, "trimmed_lens", 2)
    assert planted(lambda t: t["windows"][0].update(column_no=t["windows"][0]["column_no"] + 1)) == (0, "column_no", None)
    n = len(base["windows"])
    assert planted(lambda t: t["windows"].pop()) == (n - 1, "n_windows", "count %d vs %d" % (n - 1, n))
    assert planted(lambda t: t["msa"].__setitem__((0, 0), 5 - t["msa"][0, 0])) == (None, "msa", None)
    # a later window's trace is named before an earlier window's trimmed length (trimming window n depends on window n+1)
    assert planted(lambda t: (arr(t["windows"][0], "trimmed_lens", 0), t["windows"][2]["trace"]["alns"][1].update(best_score=-7))) == \
        (2, "trace", (1, "best_score", None))


def _fails_cleanly(s, c, msg, **kw):
    a = dict(window_size=c["window_size"], max_prog_rows=c["max_prog_rows"], max_prog_length_diff=c["max_prog_length_diff"])
    a.update(kw)
    rc, outs = s.trace_ends_raw(c["ends"], c["ri"], c["rr"], c["ov"], **a)
    assert rc == -3 and s.error() == msg
    assert all(p is None and n == 0 for p, n in outs)
    if c["ri"] is not None and a["window_size"] > 0:
        with pytest.raises(AssertionError, match=msg):           # the end queue's call rejects it with the same message
            s.consistent(c["ends"], c["ri"], c["rr"], c["ov"], **a)


def test_bad_inputs_fail_with_the_queues_messages_and_leave_no_arrays(built):
    base = next(c for c in X.cases() if c["name"] == "rc_full")
    s = T.Standin(R.cactus_params(**base["poa"]))
    try:
        bad = copy.deepcopy(base)
        bad["ri"][0][1] = 7                                      # no such end
        _fails_cleanly(s, bad, "inconsistent end / row indexes or overlaps")
        bad = copy.deepcopy(base)
        bad["rr"][0][0] = 99                                     # no such row
        _fails_cleanly(s, bad, "inconsistent end / row indexes or overlaps")
        bad = copy.deepcopy(base)
        bad["ov"][0][2] = len(bad["ends"][0][2]) + 5             # an overlap longer than the string
        _fails_cleanly(s, bad, "inconsistent end / row indexes or overlaps")
        _fails_cleanly(s, base, "window_size must be positive", window_size=0)
        # one failing end among good ones: a '-' in a string is rejected by the device's job checks; no end keeps an array
        bad = copy.deepcopy(base)
        bad["ends"][1][0] = bad["ends"][1][0][:5] + b"-" + bad["ends"][1][0][6:]
        rc, outs = s.trace_ends_raw(*X.args(bad))
        assert rc != 0 and all(p is None and n == 0 for p, n in outs)
        # an end without strings
        bad = copy.deepcopy(base)
        bad["ends"] = [bad["ends"][0], []]
        bad["ri"], bad["rr"], bad["ov"] = None, None, None
        _fails_cleanly(s, bad, "end without sequences")
        # the context still works afterwards
        _same(s.trace_ends(*X.args(base)), _run(base, "oracle"), "after failures")
    finally:
        s.close()


def test_layout_matches_the_header(built):
    """word counts from the header's description, and the product's parser against the checkers' reader"""
    for c in X.cases():
        for w in _run(c, "standin"):
            r = T.read_end_trace(w)
            K = r["seq_no"]
            n = 2 + sum(1 + 3 * K + 2 + len(win["trace_words"]) + K + 1 for win in r["windows"]) + 2 + (K * r["msa"].shape[1] + 7) // 8
            assert n == len(w) == r["n_words"]
            p = cb.parse_end_trace(w)
            assert p["seq_no"] == K and np.array_equal(p["msa"], r["msa"]) and len(p["windows"]) == len(r["windows"])
            for k, (a, b) in enumerate(zip(p["windows"], r["windows"])):
                assert a["index"] == b["index"] == k
                for f in ("offsets", "lens", "empty", "trimmed_lens"):
                    assert np.array_equal(a[f], b[f])
                assert a["progressive"] == b["progressive"] and a["column_no"] == b["column_no"]
                assert cb.first_trace_difference(a["trace"], b["trace"]) is None
                for x, y in zip(a["trace"]["alns"], b["trace"]["alns"]):
                    assert np.array_equal(x["cigar"], y["cigar"]) and np.array_equal(x["dp_beg"], y["dp_beg"])
            with pytest.raises(ValueError):
                cb.parse_end_trace(np.concatenate([w, [0]]))
