"""The pair-HMM kernel on the device at the edges of its launch plan (tests/test_pecan_edges_cpu.py: edge_batches, whose
premises are pinned there): every family equals the plain-C oracle bit for bit as one batch and pair by pair, and every launch is
the one the restated plan (group_plan) says, read back from the library's debug lines. Then the output room (a stage's fetch adds
the compaction, and for a job one candidate over its room the retry's launches), a shared work queue with more jobs than resident
blocks in both classes, and the loop that cuts the block count when the rings do not fit the memory the context may use."""
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _reflib as R
import test_pecan_edges_cpu as E

pytestmark = pytest.mark.gpu

_CLASS_LINE = re.compile(r"\[barb200\] pecan class: (\d+) jobs, (\d+) threads x (\d+) blocks, ring (\d+) of which (\d+) shared, "
                         r"FM ring (\d+), FF ring (\d+) doubles")


@pytest.fixture(scope="module")
def eng():
    import cactus_b200 as cb
    e = cb.Engine()
    yield e
    e.close()


@pytest.fixture(scope="module")
def sms(eng):
    return eng.device_info()["sm_count"]


@pytest.fixture
def launches(monkeypatch, capfd):
    """launches() -> the class lines the library printed since the last call, as group_plan dicts"""
    monkeypatch.setenv("BARB200_DEBUG", "1")
    capfd.readouterr()

    def read():
        err = capfd.readouterr().err
        keys = ("jobs", "threads", "blocks", "RW", "RWs", "cap_m", "cap_f")
        return [dict(zip(keys, (int(v) for v in m.groups()))) for m in _CLASS_LINE.finditer(err)]
    return read


def _params(threshold, min_diags, tb_diags, expansion, split):
    import cactus_b200 as cb
    return cb.PairwiseAlignmentParameters(threshold, min_diags, tb_diags, expansion, split)


def _cb_params(c):
    return _params(*c.params, c.split)


def _pairs(cases):
    return [(c.sx, c.sy, c.anchors, False, False) for c in cases]


def _subs(cases):
    return [s for c in cases for s in E.plan(c)]


def _planned(cases, sms):
    """the launches of a batch of cases: its stage, then the retry stage of the jobs whose candidates overflow their room (the
    oracle's triples are the candidates, up to a 1e-9 margin below log(threshold) that these cases do not reach)"""
    over = [s for c in cases for s in E.plan(c) if len(E.oracle(c)[0]) > s["out_room"]]
    assert all(len(E.plan(c)) == 1 for c in cases)
    return E.group_plan(_subs(cases), sms) + E.group_plan(over, sms)


def _check(res, cases):
    for c, (t, po, cells) in zip(cases, res):
        to, poo = E.oracle(c)
        assert np.array_equal(t, to) and np.array_equal(po, poo), c.name
        assert cells == sum(s["cells"] for s in E.plan(c)), c.name


@pytest.mark.parametrize("family", E.FAMILIES)
def test_family_matches_the_oracle_in_its_planned_launches(eng, sms, launches, family):
    for batch in E.edge_batches(family):
        p = _cb_params(batch[0])
        res = eng.get_aligned_pairs_using_anchors_batch(_pairs(batch), p, True)
        assert launches() == _planned(batch, sms), [c.name for c in batch]
        _check(res, batch)
        for c in batch:
            res = eng.get_aligned_pairs_using_anchors_batch(_pairs([c]), p, True)
            assert launches() == _planned([c], sms), c.name
            _check(res, [c])


def test_the_launches_reach_the_named_edges(eng, sms, launches):
    """the class lines themselves show widths 96 / 97 and 320 / 321, and a job run in a ring wider than its own widest diagonal"""
    seen = {}
    for name in ("sq95", "sq96", "sq319", "sq320", "long95", "long320"):
        c = E._case("class", name)
        eng.get_aligned_pairs_using_anchors_batch(_pairs([c]), _cb_params(c), True)
        (g,) = launches()
        seen[name] = (g["threads"], g["RW"], g["RWs"])
    assert seen == dict(sq95=(32, 96, 96), sq96=(128, 320, 320), sq319=(128, 320, 320), sq320=(128, 321, 320), long95=(32, 96, 96),
                        long320=(128, 321, 320))
    (batch,) = E.edge_batches("group")
    eng.get_aligned_pairs_using_anchors_batch(_pairs(batch), _cb_params(batch[0]), True)
    (g,) = launches()
    assert g["jobs"] == 4 and g["RW"] == 701 > E.plan(E._case("group", "long320"))[0]["max_w"] > g["RWs"]


def test_output_room_launches(eng, sms, launches):
    """a stage's fetch launches the compaction; a job one candidate over its room is re-run by a retry stage of its own (its
    launch + its compaction; nothing else is left to compact first)"""
    (batch,) = E.edge_batches("room")
    p = _cb_params(batch[0])
    for c in batch:
        delta = E.ROOM_SHAPES[c.name][2]
        st = eng.pecan_stage(_pairs([c]), p)
        st.run()
        ran = st.launches()
        res = st.fetch(True)
        assert ran == 1 and st.launches() - ran == (2 if delta > 0 else 1), c.name
        _check(res, [c])
        lines = launches()
        assert lines == _planned([c], sms) and len(lines) == (2 if delta > 0 else 1), c.name
        st.close()
    st = eng.pecan_stage(_pairs(batch), p)             # all six: one compaction, then the retry of the two over their room
    st.run()
    res = st.fetch(True)
    assert st.launches() == 1 + 1 + 2
    _check(res, batch)
    assert launches() == _planned(batch, sms) and _planned(batch, sms)[1]["jobs"] == 2
    st.close()


def _oracle_many(pairs, split):
    po = R.pecan_params(*E.DEFAULT)
    with ThreadPoolExecutor(16) as ex:
        return list(ex.map(lambda q: R.oracle_pecan_aligned_pairs(q[0], q[1], q[2], False, False, po, split * split), pairs))


def test_shared_work_queue(eng, sms, launches):
    """more jobs than resident blocks in both classes (tests/test_pecan_edges_cpu.py: queue_batch), so that blocks run further,
    smaller jobs on the rings and output counters of earlier ones: every pair equals the oracle, and equals itself run alone and
    in the reversed batch"""
    pairs = E.queue_batch(sms)
    batch = [(sx, sy, a, False, False) for sx, sy, a in pairs]
    p = _params(*E.DEFAULT, E.QUEUE_SPLIT)
    res = eng.get_aligned_pairs_using_anchors_batch(batch, p, True)
    lines = launches()
    planned = E.group_plan(E.plan_pairs(pairs, split=E.QUEUE_SPLIT), sms)
    assert lines[:2] == planned
    narrow, general = lines[:2]
    assert narrow["threads"] == 32 and narrow["blocks"] == 24 * sms < narrow["jobs"]
    assert general["threads"] == 128 and general["blocks"] == 6 * sms < general["jobs"] and general["RW"] > general["RWs"]
    for i, ((t, po, _), (to, poo)) in enumerate(zip(res, _oracle_many(pairs, E.QUEUE_SPLIT))):
        assert np.array_equal(t, to) and np.array_equal(po, poo), i
    back = eng.get_aligned_pairs_using_anchors_batch(batch[::-1], p, True)
    for i, ((t, po, c), (t2, po2, c2)) in enumerate(zip(res, back[::-1])):
        assert np.array_equal(t, t2) and np.array_equal(po, po2) and c == c2, i
    for i in list(range(0, len(batch), len(batch) // 7)) + [k for k, q in enumerate(pairs) if len(q[0]) == 6000][:1]:
        ((t, po, c),) = eng.get_aligned_pairs_using_anchors_batch(batch[i:i + 1], p, True)
        assert np.array_equal(t, res[i][0]) and np.array_equal(po, res[i][1]) and c == res[i][2], i


def test_rings_cut_to_the_memory_the_context_may_use(eng, sms, launches):
    """eight unanchored jobs of about 1500 x 1500 on a context whose memory share holds their stage and the rings of about three
    blocks (tests/test_pecan_edges_cpu.py: test_cut_block_count_premise): the block count is cut, and the answers are the
    unconstrained engine's and the oracle's. A stage too large for that share is refused, and the engine still works after it."""
    import cactus_b200 as cb
    pairs = E.wide_pairs()
    batch = [(sx, sy, a, False, False) for sx, sy, a in pairs]
    subs = E.plan_pairs(pairs)
    (g,) = E.group_plan(subs, sms)
    share = E.stage_fixed_bytes(subs) + 3.5 * E.slot_bytes(g)
    want = eng.get_aligned_pairs_using_anchors_batch(batch, None, True)
    free = eng.device_info()["mem_free"]
    if free < 4 * share:
        pytest.skip("%.1f GB free on the device: too little for a stage with a cut block count" % (free / 1e9))
    small = cb.Engine(cb.PoaParams(mem_fraction=share / free))
    try:
        launches()
        got = small.get_aligned_pairs_using_anchors_batch(batch, None, True)
        cut = launches()[0]
        assert cut == dict(g, blocks=cut["blocks"]) and 1 <= cut["blocks"] < min(g["jobs"], 6 * sms), cut
        for i, ((t, po, c), (t2, po2, c2), (to, poo)) in enumerate(zip(got, want, _oracle_many(pairs, E.SPLIT))):
            assert np.array_equal(t, t2) and np.array_equal(po, po2) and c == c2, i
            assert np.array_equal(t, to) and np.array_equal(po, poo), i
        with pytest.raises(cb.BarB200Error, match="does not fit"):
            small.get_aligned_pairs_using_anchors_batch([q + (False, False) for q in E.oversized_pairs()], None, True)
        again = small.get_aligned_pairs_using_anchors_batch(batch, None, True)
        for (t, po, c), (t2, po2, c2) in zip(again, want):
            assert np.array_equal(t, t2) and np.array_equal(po, po2) and c == c2
    finally:
        small.close()
