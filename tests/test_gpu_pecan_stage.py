"""The staged pair-HMM path on the GPU (-m gpu): overflow retries run by a stage's fetch, several live stages and batch calls
sharing one context (its streams and its grow-only ring scratch), each checked against the batch call and the plain-C oracle."""
import numpy as np
import pytest

import _reflib as R
from _synth import pecan_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import cactus_b200 as cb
    e = cb.Engine()
    yield e
    e.close()


def _params(threshold):
    import cactus_b200 as cb
    return cb.PairwiseAlignmentParameters(threshold)


def _anchored(seed, n, L):
    rng = np.random.default_rng(seed)
    return [pecan_pair(rng, L, k_anchor=50) + (False, False) for _ in range(n)]


def _wide():
    """700 x 700 without anchors (test_gpu_pecan.py::test_wide_unanchored_and_overflow): at threshold 0 its candidates
    overflow the optimistic output room, so a fetch re-runs it"""
    sx, sy, _ = pecan_pair(np.random.default_rng(5), 700, k_anchor=9999, sub=0.1, ins=0.02, dele=0.02)
    return (sx, sy, [], False, False)


def _assert_same(got, want):
    assert len(got) == len(want)
    for i, ((t, po, c), (t2, po2, c2)) in enumerate(zip(got, want)):
        assert np.array_equal(t, t2) and np.array_equal(po, po2) and c == c2, i


def test_staged_overflow_retry(eng, oracle_built):
    wide = _wide()
    pairs = [wide] + _anchored(21, 3, 2000) + [(b"ACGTACG", b"ACGAACG", [], False, False), (b"", b"ACGT", [], True, False)]
    p = _params(0.0)
    batch = eng.get_aligned_pairs_using_anchors_batch(pairs, p, True)
    st = eng.pecan_stage(pairs, p)
    st.run()
    st.run()
    run_launches = st.launches()
    res = st.fetch(True)
    launches = st.launches()
    assert launches > run_launches + 1            # the run's launches + compaction, then the retry's launches
    _assert_same(res, batch)
    assert res[0][2] == (len(wide[0]) + 1) * (len(wide[1]) + 1)
    for i, q in enumerate(pairs):
        to, poo = R.oracle_pecan_aligned_pairs(*q, R.pecan_params(0.0), 9000000)
        assert np.array_equal(res[i][0], to) and np.array_equal(res[i][1], poo), i
    _assert_same(st.fetch(True), res)
    st.run()                                      # the count restarts with every run
    _assert_same(st.fetch(True), res)
    assert st.launches() == launches
    st.close()


def test_several_live_stages(eng):
    sets = [(_anchored(31, 24, 2000), _params(0.01)),
            ([_wide()] + _anchored(32, 4, 1500), _params(0.0)),
            (_anchored(33, 6, 5000) + _anchored(34, 40, 300), _params(0.01))]
    stages = [eng.pecan_stage(q, p) for q, p in sets]
    want = [None] * 3
    stages[0].run()
    stages[1].run()
    want[2] = eng.get_aligned_pairs_using_anchors_batch(*sets[2], True)
    stages[2].run()
    _assert_same(stages[1].fetch(True), eng.get_aligned_pairs_using_anchors_batch(*sets[1], True))
    want[0] = eng.get_aligned_pairs_using_anchors_batch(*sets[0], True)
    _assert_same(stages[0].fetch(True), want[0])
    stages[1].run()
    stages[0].run()
    want[1] = eng.get_aligned_pairs_using_anchors_batch(*sets[1], True)
    _assert_same(stages[2].fetch(True), want[2])
    _assert_same(stages[1].fetch(True), want[1])
    _assert_same(stages[0].fetch(True), want[0])
    for st in stages:
        st.close()


def test_ring_scratch_across_paths():
    import cactus_b200 as cb
    e = cb.Engine()
    try:
        small = _anchored(41, 4, 300)
        first = e.get_aligned_pairs_using_anchors_batch(small, None, True)     # before any stage: the rings are sized for this call
        big = _anchored(42, 64, 2000) + [_wide()]
        st = e.pecan_stage(big)
        st.run()                                                                # grows the context's rings
        _assert_same(e.get_aligned_pairs_using_anchors_batch(small, None, True), first)
        _assert_same(st.fetch(True), e.get_aligned_pairs_using_anchors_batch(big, None, True))
        st.close()
    finally:
        e.close()
