"""cPecan mode on every device of a context (-m gpu): the pair-HMM batch (barb200_pecan_aligned_pairs_batch) and the MUM-anchor
batch (barb200_pecan_anchor_pairs_batch) on a context over all visible devices equal a single-device context bit for bit -- triples,
pre-floor posteriors and cells on the golden cases and on seeded pairs checked against the oracle, anchors against the single-device
anchors and the recorded reference's --, under concurrent callers, on edge-case batches and invalid input, with work on every device
(barb200_pecan_device_stats). These need 2 or more visible devices and skip otherwise. The cPecan-configuration bar() through the
pecan shim with BARB200_DEVICES=all runs on any number of devices."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import _flowers as F
import _golden as G
import _mumlib as M
import _reflib as R
from _synth import pecan_pair
from test_mum_anchors_cpu import golden_cases as mum_golden_cases

pytestmark = pytest.mark.gpu

EINVAL = -3
TESTS = os.path.dirname(os.path.abspath(__file__))


def _visible_devices():
    import torch
    return torch.cuda.device_count()


@pytest.fixture(scope="module")
def engines():
    import cactus_b200 as cb
    n = _visible_devices()
    if n < 2:
        pytest.skip("needs 2 or more visible GPUs to compare a context over all of them with a single-device one (%d visible)" % n)
    single, multi = cb.Engine(), cb.Engine(cb.PoaParams(devices="all"))
    assert single.device_count() == 1 and multi.device_count() == min(n, 8)
    yield single, multi
    multi.close()
    single.close()


def _cb_params(threshold, min_diags, tb_diags, expansion, split):
    import cactus_b200 as cb
    p = cb.PairwiseAlignmentParameters(threshold, min_diags, tb_diags, expansion, 1)
    p.c.split_matrix_bigger_than_this = split
    return p


def _mum_params(k=50, u=1, bigger=500 * 500, recursive=1):
    import cactus_b200 as cb
    mp = cb.MumParams(k=k, u=u, recursiveMums=recursive)
    mp.c.anchor_matrix_bigger_than_this = bigger
    return mp


def _same_pairs(a, b, where):
    assert len(a) == len(b), where
    for i, (x, y) in enumerate(zip(a, b)):
        assert len(x) == len(y), (where, i)
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and np.array_equal(u, v), (where, i)
            else:
                assert u == v, (where, i)


def _seeded_pairs(seed, n, lengths=(1, 30, 300, 1500, 2000, 4000)):
    rng = np.random.default_rng(seed)
    pairs = []
    for _ in range(n):
        sx, sy, a = pecan_pair(rng, int(rng.choice(lengths)), k_anchor=int(rng.choice([12, 50])), sub=float(rng.choice([0.02, 0.1])))
        pairs.append((sx, sy, a, bool(rng.integers(0, 2)), bool(rng.integers(0, 2))))
    return pairs


def test_golden_cases_equal_a_single_device_context(engines):
    single, multi = engines
    cases = list(G.pecan_cases())
    for c in cases:
        p = _cb_params(c["threshold"], c["min_diags"], c["tb_diags"], c["expansion"], c["split"])
        q = [(c["sx"], c["sy"], c["anchors"], c["rl"], c["rr"])]
        got, want = multi.get_aligned_pairs_using_anchors_batch(q, p, True), single.get_aligned_pairs_using_anchors_batch(q, p, True)
        _same_pairs(got, want, c["id"])
        assert np.array_equal(got[0][0], c["triples"]), c["id"]
    dflt = [c for c in cases if (c["threshold"], c["min_diags"], c["tb_diags"], c["expansion"], c["split"]) == (0.01, 1000, 40, 20, 9000000)]
    q = [(c["sx"], c["sy"], c["anchors"], c["rl"], c["rr"]) for c in dflt] * 7          # enough pairs for every device
    got = multi.get_aligned_pairs_using_anchors_batch(q, None, True)
    _same_pairs(got, single.get_aligned_pairs_using_anchors_batch(q, None, True), "batched")
    for c, (t, _, _) in zip(dflt * 7, got):
        assert np.array_equal(t, c["triples"]), c["id"]


def test_seeded_pairs_equal_a_single_device_context_and_the_oracle(engines, oracle_built):
    single, multi = engines
    for rnd, (thr, sb) in enumerate([(0.01, 9000000), (0.0001, 400 * 400), (0.0, 100 * 100)]):
        pairs = _seeded_pairs(77 + rnd, 160) + [(b"", b"", [], False, False), (b"A", b"", [], False, True), (b"", b"ACGT", [], True, False)]
        p = _cb_params(thr, 1000, 40, 20, sb)
        got = multi.get_aligned_pairs_using_anchors_batch(pairs, p, True)
        _same_pairs(got, single.get_aligned_pairs_using_anchors_batch(pairs, p, True), rnd)
        for i in range(0, len(pairs), 23):
            to, poo = R.oracle_pecan_aligned_pairs(*pairs[i], R.pecan_params(thr), sb)
            assert np.array_equal(got[i][0], to) and np.array_equal(got[i][1], poo), (rnd, i)


def test_triples_without_posteriors(engines):
    single, multi = engines
    pairs = _seeded_pairs(5, 64)
    _same_pairs(multi.get_aligned_pairs_using_anchors_batch(pairs), single.get_aligned_pairs_using_anchors_batch(pairs), "no posteriors")


def test_anchors_equal_a_single_device_context_and_the_goldens(engines):
    single, multi = engines
    for name, sx, sy, p, want in mum_golden_cases():
        got = multi.mum_anchor_pairs_batch([(sx, sy)] * 5, _mum_params(**p))
        for a in got:
            assert np.array_equal(a, want), name
    rng = np.random.default_rng(321)
    pairs = [M.related_pair(rng, int(L), sub=float(rng.choice([0.01, 0.05]))) for L in rng.integers(100, 8000, 90)]
    pairs.insert(40, M.related_pair(rng, 120000))
    for rec in (1, 0):
        got, want = multi.mum_anchor_pairs_batch(pairs, _mum_params(recursive=rec)), single.mum_anchor_pairs_batch(pairs, _mum_params(recursive=rec))
        for i, (a, b) in enumerate(zip(got, want)):
            assert a.dtype == b.dtype and np.array_equal(a, b), (rec, i)
        for i in (0, 40, 89):
            assert np.array_equal(got[i], M.oracle_mum_anchors(*pairs[i], recursive=rec)), (rec, i)
    t = multi.mum_last_timing()
    assert t["kernel_ms"] > 0 and t["launches"] > 0 and t["wall_ms"] >= t["kernel_ms"] * 0.5


def test_concurrent_callers_get_the_single_device_answers(engines):
    single, multi = engines
    pairs = _seeded_pairs(99, 96, lengths=(100, 700, 2000))
    want = single.get_aligned_pairs_using_anchors_batch(pairs, None, True)
    want_a = single.mum_anchor_pairs_batch(pairs)
    slices = [slice(k, k + 12) for k in range(0, 96, 12)]
    got, got_a, errors = [None] * len(slices), [None] * len(slices), []

    def work(j):
        try:
            for _ in range(3):
                got[j] = multi.get_aligned_pairs_using_anchors_batch(pairs[slices[j]], None, True)
                got_a[j] = multi.mum_anchor_pairs_batch(pairs[slices[j]])
        except Exception as e:              # reported below: an assertion in a thread would be lost
            errors.append(repr(e))
    th = [threading.Thread(target=work, args=(j,)) for j in range(len(slices))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    for j, s in enumerate(slices):
        _same_pairs(got[j], want[s], j)
        for a, b in zip(got_a[j], want_a[s]):
            assert np.array_equal(a, b), j


def test_empty_and_one_pair_batches(engines):
    single, multi = engines
    assert multi.get_aligned_pairs_using_anchors_batch([], None, True) == []
    assert multi.mum_anchor_pairs_batch([]) == []
    one = _seeded_pairs(3, 1, lengths=(2000,))
    _same_pairs(multi.get_aligned_pairs_using_anchors_batch(one, None, True), single.get_aligned_pairs_using_anchors_batch(one, None, True), "one")
    rng = np.random.default_rng(4)
    q = [M.related_pair(rng, 3000)]
    assert np.array_equal(multi.mum_anchor_pairs_batch(q)[0], single.mum_anchor_pairs_batch(q)[0])


def test_one_invalid_pair_fails_the_batch_and_leaves_no_outputs(engines):
    import cactus_b200 as cb
    single, multi = engines
    pairs = _seeded_pairs(8, 40, lengths=(300, 2000))
    sx, sy = pairs[25][0], pairs[25][1]
    pairs[25] = (sx, sy, [[5, 5], [3, 9]], False, False)          # anchors not increasing in x
    t = cb.api._PairTable(pairs)
    m = t.n
    trip, post = (C.c_void_p * m)(), (C.c_void_p * m)()
    n_out, cells = np.zeros(m, np.int64), np.zeros(m, np.int64)
    rc = multi.lib.barb200_pecan_aligned_pairs_batch(multi.ctx, C.byref(cb.PairwiseAlignmentParameters().c), m, *t.args(), trip, n_out.ctypes.data,
                                                     post, cells.ctypes.data)
    assert rc == EINVAL
    assert b"anchor pairs must be strictly increasing" in multi.lib.barb200_last_error(multi.ctx)
    assert all(trip[i] is None for i in range(m)) and all(post[i] is None for i in range(m))
    good = pairs[:25] + pairs[26:]                                   # the context still works, and agrees with one device
    _same_pairs(multi.get_aligned_pairs_using_anchors_batch(good, None, True), single.get_aligned_pairs_using_anchors_batch(good, None, True), "after")
    mp = [(q[0], q[1]) for q in good]
    mp[7] = (mp[7][0][:50] + b"\xc3" + mp[7][0][51:], mp[7][1])
    with pytest.raises(cb.BarB200Error, match="not a NUL-free ASCII symbol"):
        multi.mum_anchor_pairs_batch(mp)


def test_a_large_batch_runs_on_every_device(engines):
    single, multi = engines
    n = multi.device_count()
    before = multi.pecan_device_stats()
    assert len(before["hmm_pairs"]) == n and len(before["mum_pairs"]) == n
    pairs = _seeded_pairs(12, 64 * n, lengths=(2000,))
    multi.get_aligned_pairs_using_anchors_batch(pairs)
    multi.mum_anchor_pairs_batch(pairs)
    after = multi.pecan_device_stats()
    hmm = [a - b for a, b in zip(after["hmm_pairs"], before["hmm_pairs"])]
    mum = [a - b for a, b in zip(after["mum_pairs"], before["mum_pairs"])]
    assert sum(hmm) == len(pairs) and all(h > 0 for h in hmm), hmm
    assert sum(mum) == len(pairs) and all(v > 0 for v in mum), mum
    s = single.pecan_device_stats()
    assert len(s["hmm_pairs"]) == 1


_SHIM_BAR = """
import sys
sys.path[:0] = [%r, %r]
import numpy as np
import _flowers as F
from test_flowers_cpu import PECAN, pecan_flowers
from test_mum_anchors_cpu import long_pecan_flowers
fls = pecan_flowers() + long_pecan_flowers()
want = F.bar("ref", fls, PECAN, threads=1)
got = F.bar("shim", fls, PECAN, threads=1)
bad = [i for i, (a, b) in enumerate(zip(got, want)) if not np.array_equal(a, b)]
print("flowers", len(fls), "differ", bad)
sys.exit(1 if bad or len(got) != len(fls) else 0)
"""


def test_cpecan_bar_through_the_shim_with_every_device_equals_the_reference():
    """bar() with partialOrderAlignment="0" over shim/cactus_pecan_shim.c with BARB200_DEVICES=all (the shim's context is made
    once per process, so in a process of its own): every flower as the unmodified reference leaves it, on any number of GPUs"""
    assert F.have("shim") and F.have("ref"), "oracle/_ref/libflower_shim.so / libflower_ref.so are missing"
    env = dict(os.environ, BARB200_DEVICES="all")
    env.pop("BARB200_DEVICE", None)
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(py + ["-c", _SHIM_BAR % (TESTS, os.path.dirname(TESTS))], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "differ []" in r.stdout

