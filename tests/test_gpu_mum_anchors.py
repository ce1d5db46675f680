"""K5 on the device: barb200_pecan_anchor_pairs_batch against the reference's recorded answers, the plain-C oracle (mixed
batches, one pair long enough for the global-memory merge path), batch independence, the anchors fed to the pair-HMM batch,
and a cPecan bar() with long adjacencies through the real pecan shim."""
import numpy as np
import pytest

import _flowers as F
import _mumlib as M
import _reflib as R
from test_mum_anchors_cpu import golden_cases, long_pecan_flowers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import cactus_b200 as cb
    e = cb.Engine()
    yield e
    e.close()


def _params(p):
    import cactus_b200 as cb
    mp = cb.MumParams(k=p.get("k", 50), u=p.get("u", 1), recursiveMums=p.get("recursive", 1))
    mp.c.anchor_matrix_bigger_than_this = p.get("bigger", 500 * 500)
    return mp


def test_device_matches_the_goldens(eng):
    for name, sx, sy, p, want in golden_cases():
        got = eng.mum_anchor_pairs_batch([(sx, sy)], _params(p))[0]
        assert np.array_equal(got, want), name


def test_device_matches_the_oracle_on_mixed_batches(eng):
    rng = np.random.default_rng(123)
    pairs = []
    for i in range(60):
        L = int(rng.integers(100, 10000))
        sx, sy = M.related_pair(rng, L, sub=float(rng.choice([0.01, 0.03, 0.1])))
        if i % 4 == 0:
            sx = M.rand_seq(rng, int(rng.integers(500, 3000))) + sx
        if i % 5 == 0:
            sy = sy + M.rand_seq(rng, int(rng.integers(500, 3000)))
        pairs.append((sx, sy))
    big = M.related_pair(rng, 210000)                                  # > kTile * 64 k-mers: several merge levels
    pairs.insert(17, big)
    for rec in (1, 0):
        got = eng.mum_anchor_pairs_batch(pairs, _params(dict(recursive=rec)))
        for i, ((sx, sy), a) in enumerate(zip(pairs, got)):
            assert np.array_equal(a, M.oracle_mum_anchors(sx, sy, recursive=rec)), (rec, i, len(sx), len(sy))
    for k, u in ((12, 0), (20, 3)):
        got = eng.mum_anchor_pairs_batch(pairs[:20], _params(dict(k=k, u=u)))
        for i, ((sx, sy), a) in enumerate(zip(pairs[:20], got)):
            assert np.array_equal(a, M.oracle_mum_anchors(sx, sy, k=k, u=u)), (k, u, i)


def test_a_pair_alone_equals_the_pair_in_a_batch(eng):
    rng = np.random.default_rng(5)
    pairs = [M.related_pair(rng, int(L)) for L in rng.integers(600, 5000, 24)]
    batch = eng.mum_anchor_pairs_batch(pairs)
    for q, a in zip(pairs, batch):
        assert np.array_equal(eng.mum_anchor_pairs_batch([q])[0], a)


def test_rejects_what_is_not_built(eng):
    import cactus_b200 as cb
    s = M.rand_seq(np.random.default_rng(1), 800)
    for kw in (dict(k=0), dict(k=65), dict(u=-1)):
        with pytest.raises(cb.BarB200Error):
            eng.mum_anchor_pairs_batch([(s, s)], _params(kw))
    with pytest.raises(cb.BarB200Error):
        eng.mum_anchor_pairs_batch([(s, s[:100] + b"\xc3" + s[101:])])


def test_device_anchors_give_the_oracles_posteriors(eng):
    rng = np.random.default_rng(9)
    pairs = [M.related_pair(rng, int(L), sub=0.03) for L in (700, 1500, 2500)]
    anchors = eng.mum_anchor_pairs_batch(pairs)
    res = eng.get_aligned_pairs_using_anchors_batch([(sx, sy, a, False, False) for (sx, sy), a in zip(pairs, anchors)], None, True)
    for (sx, sy), a, (t, po, _) in zip(pairs, anchors, res):
        assert len(a) > 0
        to, poo = R.oracle_pecan_aligned_pairs(sx, sy, a, False, False, R.pecan_params())
        assert np.array_equal(t, to) and np.array_equal(po, poo)


def test_cpecan_bar_with_mum_anchors_through_the_shim():
    if not (F.have("shim") and F.have("ref")):
        pytest.fail("oracle/_ref/libflower_shim.so / libflower_ref.so are missing")
    from test_flowers_cpu import PECAN
    fls = long_pecan_flowers()
    want = F.bar("ref", fls, PECAN, threads=1)
    got = F.bar("shim", fls, PECAN, threads=1)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), i
