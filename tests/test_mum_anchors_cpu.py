"""cPecan's MUM anchors without a GPU: the plain-C oracle against the reference's recorded answers (tests/golden/mum_golden.npz)
and, where oracle/_ref/libmum_ref.so exists, against the reference itself on fresh inputs; the host build of the product's
K5 (mum_anchor.cuh / mum_plan.h through tests/hosttest/mum_host.cpp) against the oracle; the order of equal k-mers; the planning code; and
one cPecan bar() whose adjacencies reach MUM anchoring, through the pecan shim on the CPU stand-in device."""
import ctypes as C
import os

import numpy as np
import pytest

import _flowers as F
import _mumlib as M
import _reflib as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mum_golden.npz")


def golden_cases():
    g = np.load(GOLDEN)
    lens = g["lens"]
    offs = np.concatenate([[0], np.cumsum(lens)])
    aoffs = np.concatenate([[0], np.cumsum(g["counts"])])
    seqs = g["seqs"].tobytes()
    for i, name in enumerate(g["names"]):
        k, u, bigger, rec = (int(v) for v in g["params"][i])
        sx, sy = seqs[offs[2 * i]:offs[2 * i + 1]], seqs[offs[2 * i + 1]:offs[2 * i + 2]]
        yield str(name), sx, sy, dict(k=k, u=u, bigger=bigger, recursive=rec), g["anchors"][aoffs[i]:aoffs[i + 1]].astype(np.int64)


def test_oracle_matches_the_recorded_reference():
    n = 0
    for name, sx, sy, p, want in golden_cases():
        assert np.array_equal(M.oracle_mum_anchors(sx, sy, **p), want), name
        n += 1
    assert n >= 20


@pytest.mark.skipif(not M.have_ref(), reason="oracle/_ref/libmum_ref.so not built (needs the reference sources)")
def test_oracle_matches_the_reference_on_fresh_inputs():
    rng = np.random.default_rng(77)
    checked = 0
    for seed in range(12):
        L = int(rng.integers(300, 4000))
        sx, sy = M.related_pair(rng, L, sub=float(rng.choice([0.01, 0.05, 0.15])))
        if seed % 3 == 0:
            sy = M.rand_seq(rng, int(rng.integers(600, 2000))) + sy + M.rand_seq(rng, 900)
        p = dict(k=int(rng.choice([12, 20, 50])), u=int(rng.integers(0, 3)), bigger=int(rng.choice([200, 500])) ** 2, recursive=int(seed % 2))
        want, would_abort = M.oracle_mum_anchors(sx, sy, with_abort=True, **p)
        if would_abort:                  # the reference is built with asserts on and aborts there (oracle/mum_oracle.c)
            continue
        assert np.array_equal(want, M.ref_mum_anchors(sx, sy, **p)), seed
        checked += 1
    assert checked >= 8


def test_host_build_matches_the_oracle():
    for name, sx, sy, p, want in golden_cases():
        assert np.array_equal(M.hosttest_mum_anchors(sx, sy, **p), want), name
    for name, sx, sy, kw in M.case_set(np.random.default_rng(5)):
        assert np.array_equal(M.hosttest_mum_anchors(sx, sy, **kw), M.oracle_mum_anchors(sx, sy, **kw)), name


def test_threshold_edges_and_short_sequences():
    rng = np.random.default_rng(8)
    a = M.rand_seq(rng, 501)
    assert len(M.hosttest_mum_anchors(a[:500], a[:500])) == 0                # 500 x 500 is not searched
    got = M.hosttest_mum_anchors(a[:500], a)                                  # 500 x 501 is
    assert len(got) > 0 and np.array_equal(got, M.oracle_mum_anchors(a[:500], a))
    assert len(M.hosttest_mum_anchors(a[:49], a * 20)) == 0                   # lX < k
    assert len(M.hosttest_mum_anchors(a * 20, a[:49])) == 0                   # lY < k


def test_identical_sequences_skip_the_base_after_each_mum():
    """on an exact diagonal a MUM is at most k long and the position at offset k is not a MUM start (pXEnd == x), so the
    anchors miss every (k+1)-th base; a MUM that would end exactly at lX is never added to the sweep line"""
    s = M.rand_seq(np.random.default_rng(9), 1000)
    got = M.hosttest_mum_anchors(s, s)
    assert np.array_equal(got, M.oracle_mum_anchors(s, s))
    xs = set(got[:, 0].tolist())
    assert all(x in xs for x in range(50)) and 50 not in xs and 51 in xs and 101 not in xs
    assert np.array_equal(got[:, 0], got[:, 1])
    s2 = s[:50 + 51 * 12]                                                     # last MUM would end at lX
    got2, would_abort = M.oracle_mum_anchors(s2, s2, with_abort=True)
    assert would_abort and got2[-1, 0] < len(s2) - 50
    assert np.array_equal(M.hosttest_mum_anchors(s2, s2), got2)


def test_repeats_have_no_unique_matches():
    assert len(M.hosttest_mum_anchors(b"A" * 800, b"A" * 700)) == 0
    rep = b"ACGTTGCAT" * 150
    assert len(M.hosttest_mum_anchors(rep, rep[4:])) == 0


def test_equal_kmers_in_any_order():
    """mum_anchor.cuh: runs of equal k-mers may be sorted in any order -- shuffle every run after the sort"""
    rng = np.random.default_rng(10)
    unit = M.rand_seq(rng, 300)
    for name, sx, sy, kw in [("dup", unit * 3 + M.rand_seq(rng, 900), M.rand_seq(rng, 400) + unit * 2, {}),
                             ("tandem_k12", (b"ACGTAC" * 80) + M.rand_seq(rng, 700), M.rand_seq(rng, 300) + b"ACGTAC" * 90, dict(k=12, u=0))] + \
                            [c for c in M.case_set(rng) if c[0] in ("duplication", "mixed_case", "k8_u0", "k12_u3")]:
        base = M.hosttest_mum_anchors(sx, sy, **kw)
        for seed in (1, 2, 3):
            assert np.array_equal(M.hosttest_mum_anchors(sx, sy, tie_seed=seed, **kw), base), (name, seed)
            assert np.array_equal(M.oracle_mum_anchors(sx, sy, tie_seed=seed, **kw), base), (name, seed)


def test_rejects_what_is_not_built():
    s = M.rand_seq(np.random.default_rng(11), 800)
    for kw in (dict(k=0), dict(k=65), dict(u=-1)):
        with pytest.raises(ValueError):
            M.hosttest_mum_anchors(s, s, **kw)
    with pytest.raises(ValueError):
        M.hosttest_mum_anchors(s[:400] + b"\x80" + s[401:], s)
    assert len(M.hosttest_mum_anchors(s, s, k=64)) > 0


def _lib():
    lib = R._load(M.MUM_HOST_SO)
    lib.hosttest_mum_plan_chunks.restype = C.c_int64
    lib.hosttest_mum_plan_chunks.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    lib.hosttest_mum_pair_bytes.restype = C.c_int64
    lib.hosttest_mum_pair_bytes.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int]
    lib.hosttest_mum_key_words.restype = C.c_int
    lib.hosttest_mum_key_words.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int64]
    lib.hosttest_mum_gap_table.restype = C.c_int64
    lib.hosttest_mum_gap_table.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_void_p]
    return lib


def test_plan_chunks_under_a_memory_budget():
    lib = _lib()
    b = np.array([lib.hosttest_mum_pair_bytes(2000, 2000, 50, 3)] * 10 + [lib.hosttest_mum_pair_bytes(1 << 20, 1 << 20, 50, 3)] +
                 [0, 0, lib.hosttest_mum_pair_bytes(700, 900, 50, 3)], np.int64)
    budget = int(b[0] * 4 + 10)
    out = np.zeros(2 * len(b), np.int64)
    n = lib.hosttest_mum_plan_chunks(b.ctypes.data, len(b), budget, out.ctypes.data)
    chunks = out[:2 * n].reshape(n, 2).tolist()
    assert chunks[0] == [0, 4] and chunks[1] == [4, 8] and chunks[2] == [8, 10]
    assert chunks[3] == [10, 11]                         # larger than the budget: a chunk of its own
    assert chunks[4] == [11, 14] and chunks[-1][1] == len(b)
    for c0, c1 in chunks:
        assert c1 - c0 == 1 or b[c0:c1].sum() <= budget
    # key width: 3 bits per symbol for ACGT(N) gives 21 symbols a word, 3 words for k = 50; a wider alphabet takes more
    assert lib.hosttest_mum_key_words(b"ACGTN", 5, b"acgt", 4, 50) == 3
    assert lib.hosttest_mum_key_words(b"ACGTNRYKMSWBDHV", 15, b"", 0, 50) == 4
    assert lib.hosttest_mum_key_words(bytes(range(1, 128)), 127, b"", 0, 64) == 8


def test_gap_table():
    lib = _lib()
    chain = np.array([[100, 200, 50], [900, 950, 40], [1000, 1010, 50]], np.int32)
    out = np.zeros(16, np.int32)
    n = lib.hosttest_mum_gap_table(chain.ctypes.data, 3, 3000, 3000, 500 * 500, out.ctypes.data)
    # before the first MUM: 100 x 200 (too small); 150..900 x 250..950 (750 x 700); 940..1000 x 990..1010 (too small); after: 1050.. x 1060..
    assert out[:4 * n].reshape(n, 4).tolist() == [[150, 250, 900, 950], [1050, 1060, 3000, 3000]]
    assert lib.hosttest_mum_gap_table(chain.ctypes.data, 0, 3000, 3000, 0, out.ctypes.data) == 0      # no chain: no gaps


def long_pecan_flowers():
    """flowers whose adjacencies are 500-1500 bp, so that makeAlignment's pairs exceed anchorMatrixBiggerThanThis (500 x 500)"""
    return [F.random_flower(700 + s, n_threads=4, n_blocks=2, seg_len=900, p_skip=0.0, p_loop=0.0, p_empty=0.0) for s in range(2)]


@pytest.mark.skipif(not M.have_flower_standin(), reason="oracle/_ref/libflower_standin_mum.so not built (needs the reference sources, oracle/mum.mk)")
def test_cpecan_bar_with_mum_anchors_through_the_shim_on_the_standin_device():
    from test_flowers_cpu import PECAN
    fls = long_pecan_flowers()
    want = F.bar("ref", fls, PECAN, threads=1)
    got = F.bar("standin_mum", fls, PECAN, threads=1)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), i
