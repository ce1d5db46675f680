"""K5 on the device at the edges of its k-mer sort (tests/test_mum_edges_cpu.py: edge_cases): every family equals the plain-C
oracle as one batch and pair by pair, with and without recursiveMums; the kernel launches equal the count the batch's plan
implies (so the merge levels and the second pass really ran); a batch cut into many chunks equals the same batch in one chunk;
and the anchors of repeat-heavy and wide-alphabet pairs give the oracle's pair-HMM triples and posteriors."""
import numpy as np
import pytest

import _mumlib as M
import _reflib as R
import test_mum_edges_cpu as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import cactus_b200 as cb
    e = cb.Engine()
    yield e
    e.close()


def _params(p, recursive):
    import cactus_b200 as cb
    mp = cb.MumParams(k=p["k"], u=p["u"], recursiveMums=recursive)
    mp.c.anchor_matrix_bigger_than_this = p["bigger"]
    return mp


def _run(eng, cases, p, recursive):
    """the device's anchors of `cases` as one batch, and the batch's kernel launches"""
    got = eng.mum_anchor_pairs_batch([(c.sx, c.sy) for c in cases], _params(p, recursive))
    return got, eng.mum_last_timing()["launches"]


@pytest.mark.parametrize("family", E.FAMILIES)
def test_family_matches_the_oracle_as_a_batch_and_pair_by_pair(eng, family):
    for p, cases in E.edge_batches(family):
        for rec in (1, 0):
            got, _ = _run(eng, cases, p, rec)
            for c, a in zip(cases, got):
                assert np.array_equal(a, E.oracle(c, rec)), (c.name, rec, "batch")
            for c in cases:
                (a,), _ = _run(eng, [c], p, rec)
                assert np.array_equal(a, E.oracle(c, rec)), (c.name, rec, "alone")


@pytest.mark.parametrize("family", E.FAMILIES)
def test_family_runs_the_planned_launches(eng, family):
    """1 keys launch, then per pass 1 tile sort + one merge per level below the longest problem, 1 search, 1 chain"""
    for p, cases in E.edge_batches(family):
        for rec in (1, 0):
            _, n = _run(eng, cases, p, rec)
            assert n == E.planned_launches(cases, rec), (p, rec)
            for c in cases:
                _, n = _run(eng, [c], p, rec)
                assert n == E.planned_launches([c], rec), (c.name, rec)


def test_a_batch_cut_into_chunks_equals_one_chunk_and_the_oracle(eng):
    """mem_fraction = 1e-6 clamps the chunk budget to its 1 MiB floor: about one pair per chunk, the 200 kbp pair alone"""
    import cactus_b200 as cb
    rng = np.random.default_rng(2026)
    default = dict(k=E.K, u=1, bigger=E.BIGGER)
    cases = [c for c in E.edge_cases() if c.params == default and c.name != "ny131073"]
    for i, L in enumerate([200000] + [int(v) for v in rng.integers(600, 12000, 9)]):
        x, y = M.related_pair(rng, L)
        cases.insert(3 * i, E.Case("chunks", "related_%d" % L, x, y, default))
    assert len(cases) >= 45
    small = cb.Engine(cb.PoaParams(mem_fraction=1e-6))
    try:
        for rec in (1, 0):
            one, n_one = _run(eng, cases, default, rec)
            many, n_many = _run(small, cases, default, rec)
            assert n_one == E.planned_launches(cases, rec) and n_many > n_one + 20, (rec, n_one, n_many)
            for c, a, b in zip(cases, one, many):
                want = M.oracle_mum_anchors(c.sx, c.sy, **dict(c.params, recursive=rec))
                assert np.array_equal(b, a) and np.array_equal(a, want), (c.name, rec)
    finally:
        small.close()


def test_edge_anchors_give_the_oracles_posteriors(eng):
    names = ("dup_2600", "homopolymer", "gap_unique", "ascii127_k64", "iupac_k16", "mixed_k50", "bin_k64")
    cases = [c for c in E.edge_cases() if c.name in names]
    assert len(cases) == len(names)
    anchors = []
    for c in cases:
        (a,), _ = _run(eng, [c], c.params, 1)
        assert len(a) > 0 and np.array_equal(a, E.oracle(c, 1)), c.name
        anchors.append(a)
    res = eng.get_aligned_pairs_using_anchors_batch([(c.sx, c.sy, a, False, False) for c, a in zip(cases, anchors)], None, True)
    for c, a, (t, po, _) in zip(cases, anchors, res):
        to, poo = R.oracle_pecan_aligned_pairs(c.sx, c.sy, a, False, False, R.pecan_params())
        assert len(t) > 0 and np.array_equal(t, to) and np.array_equal(po, poo), c.name
