"""barb200_trace_ends on the H100: every window of every end through the device's trace kernels, against the restated chain
(oracle_trace_ends, oracle/_build) and against the reference's own chain frozen in tests/golden/end_trace_golden.npz
(scripts/make_golden_end_trace.py). The final MSAs must equal the production call's. Reads nothing from the reference tree."""
import json

import numpy as np
import pytest

import _end_trace_cases as X
import _endtrace as T
import _reflib as R
import cactus_b200 as cb
from test_gpu_parity import engine_for
from test_poa_trace_cpu import RETRY_SCALE

pytestmark = pytest.mark.gpu


def golden():
    z = np.load(X.GOLDEN)
    return json.loads(bytes(z["digests"]).decode())


def _engine(c, **knobs):
    return engine_for(R.params_dict(R.cactus_params(**c["poa"])), **knobs)


def _words(e, c):
    """the raw words of the C call (what the goldens hash)"""
    import ctypes as C
    a = T._Args(c["ends"], c["ri"], c["rr"], c["ov"])
    outs = (C.c_void_p * max(a.n, 1))()
    nw = np.zeros(max(a.n, 1), np.int64)
    e._check(e.lib.barb200_trace_ends(e.ctx, a.n, a.end_lengths, a.strs, a.lens, a.ri, a.rr, a.ov, c["window_size"], c["max_prog_rows"],
                                      c["max_prog_length_diff"], outs, nw.ctypes.data))
    return T._take(e.lib.barb200_free, outs, nw, a.n)


def _check(c, words, gold):
    want = T.oracle_trace_ends(*X.args(c), p=R.cactus_params(**c["poa"]))
    assert len(words) == len(want)
    for e, (g, w) in enumerate(zip(words, want)):
        d = cb.first_end_trace_difference(cb.parse_end_trace(g), cb.parse_end_trace(w))
        assert d is None and np.array_equal(g, w), "%s end %d: first difference from the oracle at %s" % (c["name"], e, d)
    if gold is not None:
        assert [X.digest(w) for w in words] == gold[c["name"]], c["name"] + ": differs from the reference golden"


def _run(c, **knobs):
    e = _engine(c, **knobs)
    try:
        return _words(e, c)
    finally:
        e.close()


@pytest.fixture(scope="module")
def gold(oracle_built):
    T.build()
    return golden()


@pytest.mark.parametrize("c", X.cases() + X.gpu_cases(), ids=lambda c: c["name"])
def test_device_windows_equal_the_oracle_and_the_golden(gold, c):
    _check(c, _run(c), gold)


@pytest.mark.parametrize("c", X.repeat_cases(), ids=lambda c: c["name"])
def test_repeat_rich_windows(gold, c):
    _check(c, _run(c), gold)


def test_flowers_of_the_golden_fixture(gold, tmp_path):
    import _flowers as F
    if not F.have("harvest"):
        pytest.skip("oracle/_ref/libflower_harvest.so not built")
    cases = X.flower_cases(str(tmp_path))
    assert len(cases) >= 11
    for c in cases:
        _check(c, _run(c), gold)


def test_cta_class_premise():
    """the cta_classes chain holds windows of the smallest and of the 10 kbp classes in the same rounds"""
    c = X.gpu_cases()[0]
    lens = [max(len(s) for s in e) for e in c["ends"]]
    assert min(lens) <= 200 and max(lens) > 2 * c["window_size"]


@pytest.mark.parametrize("c", X.cases() + X.gpu_cases(), ids=lambda c: c["name"])
def test_final_msas_equal_the_production_call(gold, c):
    e = _engine(c)
    try:
        got = [cb.parse_end_trace(w)["msa"] for w in _words(e, c)]
        kw = dict(window_size=c["window_size"], max_prog_rows=c["max_prog_rows"], max_prog_length_diff=c["max_prog_length_diff"])
        if c["ri"] is not None:
            want = [m.msa_seq for m in e.make_consistent_partial_order_alignments(c["ends"], c["ri"], c["rr"], c["ov"], **kw)]
        else:
            want = [m.msa_seq for m in e.msa_make_partial_order_alignment_batch(c["ends"], **kw)]
    finally:
        e.close()
    for a, b in zip(got, want):
        assert a.shape == b.shape and np.array_equal(a, b), c["name"]


def test_every_device_traces_what_one_device_traces(gold):
    cases = [c for c in X.cases() + X.gpu_cases() if c["name"] in ("five_windows", "rc_full", "default_band", "cta_classes")]
    e = _engine(cases[0], devices="all")
    try:
        if e.device_count() < 2:
            pytest.skip("one GPU")
    finally:
        e.close()
    for c in cases:
        got = _run(c, devices="all")
        want = _run(c)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), c["name"]


def test_trace_capacity_retry_inside_a_chain(gold, monkeypatch):
    """BARB200_TRACE_REGION_SCALE shrinks every round's first trace regions below one record: each window's job ends its first rounds
    with the trace-capacity status and is traced by the worst-case retry. The words equal those of a run without the retry"""
    cases = [c for c in X.cases() if c["name"] in ("odd_overlap", "rc_partial", "default_band")]
    want = [_run(c) for c in cases]
    monkeypatch.setenv("BARB200_TRACE_REGION_SCALE", repr(RETRY_SCALE))
    try:
        got = [_run(c) for c in cases]
    finally:
        monkeypatch.delenv("BARB200_TRACE_REGION_SCALE", raising=False)
    for c, g, w in zip(cases, got, want):
        assert all(np.array_equal(a, b) for a, b in zip(g, w)), c["name"]
        _check(c, g, golden())


def test_bad_indexes_leave_no_arrays(gold):
    c = next(c for c in X.cases() if c["name"] == "rc_full")
    e = _engine(c)
    try:
        bad = [list(r) for r in c["ri"]]
        bad[0][1] = 7
        with pytest.raises(cb.BarB200Error, match="inconsistent end / row indexes or overlaps"):
            e.trace_ends(c["ends"], bad, c["rr"], c["ov"], c["window_size"])
        got = _words(e, c)                       # the context still works
    finally:
        e.close()
    _check(c, got, golden())
