"""The seeded end sets of the barb200_trace_ends tests, golden generator and scripts/end_trace_diff.py (test infrastructure).

A case is a dict: name, ends (lists of ASCII strings), ri / rr / ov (None: independent ends), window_size, max_prog_rows,
max_prog_length_diff and poa (RefParams keyword arguments)."""
import functools
import hashlib
import os

import numpy as np

from _synth import family, to_ascii, two_end_problem

NARROW = dict(wb=10, wf=0.01)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "end_trace_golden.npz")


def _case(name, ends, ri=None, rr=None, ov=None, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0, poa=None):
    return dict(name=name, ends=ends, ri=ri, rr=rr, ov=ov, window_size=window_size, max_prog_rows=max_prog_rows,
                max_prog_length_diff=max_prog_length_diff, poa=dict(NARROW if poa is None else poa))


def _fam(rng, K, L, **kw):
    return [to_ascii(s) for s in family(rng, K, L, **kw)]


@functools.lru_cache(maxsize=None)
def cases():
    rng = np.random.default_rng(9100)
    out = []
    # 30 kbp ends at a 10 kbp window: five windows (each starts ~5.1 kbp after the previous one, the trimmed overlap before it)
    out.append(_case("five_windows", [_fam(rng, 3, 30000)], window_size=10000))
    # window 21: overlap int(0.5 * 21) - 1 = 9, odd
    out.append(_case("odd_overlap", [_fam(rng, 4, 90), _fam(rng, 3, 70)], window_size=21))
    # a row that runs out of bases several windows before the others gets the N stand-in
    out.append(_case("n_standin", [_fam(rng, 3, 80) + [to_ascii(rng.integers(0, 4, 12))]], window_size=20))
    # the last row's share shrinks once it runs short: 1 - len[K-1] / len[0] > 0.3 switches progressive mode off
    long_rows = _fam(rng, 2, 64)
    out.append(_case("prog_switch", [long_rows + [long_rows[0][:41]]], window_size=20, max_prog_length_diff=0.3))
    # single-sequence ends are their own alignment: no windows
    out.append(_case("single", [[to_ascii(rng.integers(0, 4, 37))], _fam(rng, 3, 50), [to_ascii(rng.integers(0, 4, 5))]], window_size=30))
    # one string plus empty strings (the empty rows take the N stand-in in every window), and an end of empty strings only
    out.append(_case("one_plus_empty", [[to_ascii(rng.integers(0, 4, 70)), b"", b""], [b"", b""]], window_size=30))
    # reverse-complement pairs (bar/tests/poaBarTest.c:93-179): full overlaps, then half of each string's length
    ends, ri, rr, ov = two_end_problem(rng, 4, 70)
    out.append(_case("rc_full", ends, ri, rr, ov, window_size=30))
    ends, ri, rr, ov = two_end_problem(rng, 3, 90)
    out.append(_case("rc_partial", ends, ri, rr, [[len(s) // 2 for s in e] for e in ends], window_size=25))
    # the default band on 1 kbp windows
    out.append(_case("default_band", [_fam(rng, 4, 2600), _fam(rng, 2, 900)], window_size=1000, poa={}))
    return out


@functools.lru_cache(maxsize=None)
def gpu_cases():
    """device-only sets: a chain whose ends fall into different CTA classes (a short end beside 10 kbp windows)"""
    rng = np.random.default_rng(9200)
    return [_case("cta_classes", [_fam(rng, 4, 150), _fam(rng, 3, 21000), _fam(rng, 5, 700)], window_size=10000)]


@functools.lru_cache(maxsize=None)
def repeat_cases():
    """repeat-rich windows (tests/_repeats.py): ends cut inside microsatellites, and reverse-complement pairs on tandem parents"""
    import _repeats
    out = [_case("repeats/" + name, [strs], window_size=win, poa={}) for name, strs, win in _repeats.window_ends()]
    out += [_case("repeats/" + name, e, ri, rr, ov, window_size=win, poa={}) for name, (e, ri, rr, ov), win in _repeats.two_end_cases()]
    return out


def flower_cases(tmpdir):
    """the top-level alignment calls of a reference bar() on every flower behind tests/golden/flower_golden.npz (needs
    oracle/_ref/libflower_harvest.so)"""
    import _endtrace as T
    import _flower_golden as G
    out = []
    for name, fl, params, _, _ in G.cases():
        recs = T.harvest_flower(fl, params, os.path.join(tmpdir, name + ".harvest"))
        p = T.flower_params(params)
        for i, r in enumerate(recs):
            out.append(_case("flower/%s/%d" % (name, i), r["ends"], r["right_end_indexes"], r["right_end_row_indexes"], r["overlaps"],
                             r["window_size"], r["max_prog_rows"], r["max_prog_length_diff"], poa=dict(wb=p.wb, wf=float(p.wf))))
    return out


def digest(words):
    return hashlib.sha256(np.ascontiguousarray(words, np.int64).tobytes()).hexdigest()


def args(c):
    return (c["ends"], c["ri"], c["rr"], c["ov"], c["window_size"], c["max_prog_rows"], c["max_prog_length_diff"])
