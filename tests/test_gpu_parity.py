"""GPU parity tests (H100): the CUDA path, called through the C ABI, against the committed golden vectors of the
unmodified reference, against the plain-C oracle on seeded inputs, and -- at benchmark scale -- through
size-independent properties. Bit-exact: these are integer/byte results."""
import numpy as np
import pytest

import _golden as G
import _reflib as R
from _synth import family, gapped_family, to_ascii, two_end_problem
import workload  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import cactus_b200 as cb
    e = cb.Engine()
    yield e
    e.close()


def engine_for(params, **engine_knobs):
    """an Engine with the oracle's parameters (R.params_dict) and optional engine knobs (threads_per_block, ...)"""
    import cactus_b200 as cb
    return cb.Engine(cb.PoaParams(
        partialOrderAlignmentBandConstant=params["wb"], partialOrderAlignmentBandFraction=params["wf"],
        partialOrderAlignmentGapOpenPenalty1=params["o1"], partialOrderAlignmentGapExtensionPenalty1=params["e1"],
        partialOrderAlignmentGapOpenPenalty2=params["o2"], partialOrderAlignmentGapExtensionPenalty2=params["e2"],
        partialOrderAlignmentMinimizerK=params["k"], partialOrderAlignmentMinimizerW=params["w"],
        partialOrderAlignmentMinimizerMinW=params["min_w"], partialOrderAlignmentProgressiveMode=params["progressive"], **engine_knobs))


def test_golden_poa(engine):
    """every golden abpoa_msa case: MSA bytes and banded cell count equal to the reference's"""
    default = R.params_dict(R.cactus_params())
    for c in G.poa_cases():
        same = all(abs(c["params"][k] - default[k]) < 1e-9 for k in c["params"])
        e = engine if same else engine_for(c["params"])
        msas, cells = e.poa_msa_batch([c["seqs"]], return_cells=True)
        assert msas[0].shape == c["msa"].shape and np.array_equal(msas[0], c["msa"]), c["id"]
        assert int(cells[0]) == c["cells"], c["id"]
        if not same:
            e.close()


def test_golden_poa_one_batch(engine):
    """all default-parameter golden cases in ONE launch (mixed K and L in a batch)"""
    default = R.params_dict(R.cactus_params())
    cases = [c for c in G.poa_cases() if all(abs(c["params"][k] - default[k]) < 1e-9 for k in c["params"])]
    msas = engine.poa_msa_batch([c["seqs"] for c in cases])
    for m, c in zip(msas, cases):
        assert m.shape == c["msa"].shape and np.array_equal(m, c["msa"]), c["id"]


@pytest.mark.parametrize("seed", range(3))
def test_random_vs_oracle(engine, oracle_built, seed):
    rng = np.random.default_rng(500 + seed)
    jobs = []
    for it in range(48):
        K = int(rng.integers(2, 14))
        L = int(rng.choice([1, 5, 20, 60, 150, 300, 400, 800, 1500]))
        kw = dict(sub=float(rng.choice([0.0, 0.02, 0.08, 0.2])), ins=float(rng.choice([0, 0.005, 0.03])),
                  dele=float(rng.choice([0, 0.005, 0.03])), nfrac=float(rng.choice([0, 0, 0.01])))
        jobs.append(family(rng, K, L, sort=bool(rng.random() < 0.7), **kw))
    msas, cells = engine.poa_msa_batch(jobs, return_cells=True)
    for j, (m, job) in enumerate(zip(msas, jobs)):
        tr = R.oracle_poa_msa_trace(job)
        assert m.shape == tr["msa"].shape and np.array_equal(m, tr["msa"]), (seed, j)
        assert int(cells[j]) == tr["cells"], (seed, j)


def test_unrelated_ragged_and_wide(engine, oracle_built):
    """ragged unrelated rows, N-rich, K > 64 (two read-id words), the int16/int32 lane switch"""
    rng = np.random.default_rng(42)
    jobs = []
    for it in range(24):
        K = int(rng.integers(2, 90))
        jobs.append([rng.integers(0, 5 if rng.random() < 0.2 else 4, int(rng.integers(1, 400))).astype(np.uint8) for _ in range(K)])
    msas = engine.poa_msa_batch(jobs)
    for j, (m, job) in enumerate(zip(msas, jobs)):
        o = R.oracle_poa_msa(job)
        assert m.shape == o.shape and np.array_equal(m, o), j


def test_narrow_band_params(oracle_built):
    """non-default bands force the adaptive band edges into play"""
    rng = np.random.default_rng(43)
    for wb, wf, prog in [(10, 0.01, 1), (0, 0.0, 0), (30, 0.02, 1), (5, 0.1, 0)]:
        p = R.cactus_params(wb=wb, wf=wf, progressive=prog)
        e = engine_for(R.params_dict(p))
        jobs = [family(rng, int(rng.integers(2, 10)), int(rng.choice([50, 300, 900])), sub=0.08, ins=0.03, dele=0.03) for _ in range(12)]
        msas = e.poa_msa_batch(jobs)
        for j, (m, job) in enumerate(zip(msas, jobs)):
            o = R.oracle_poa_msa(job, p)
            assert m.shape == o.shape and np.array_equal(m, o), (wb, wf, j)
        e.close()


@pytest.mark.parametrize("gaps", [(400, 30, 1200, 1), (4, 2, 24, 1), (400, 30, 1200, 30), (1200, 1, 400, 30), (400, 30, 300, 1), (6, 2, 6, 2),
                                  (4, 1, 24, 1), (1, 1, 1, 1), (2, 1, 30, 0)])
def test_long_gaps_and_gap_models(oracle_built, gaps):
    """block indels of 1..300 bases under Cactus' penalties, abPOA's defaults, equal extensions, swapped gap pairs, a second gap
    that is cheaper everywhere, and two identical gaps: the insertion scan's crossover bound in every regime. The models with
    extensions of at most 1 put the reference's minus infinity within a few hundred of INT32_MIN (the row maximum's seed must not
    wrap there), and (2, 1, 30, 0) has a gap that costs nothing to extend"""
    o1, e1, o2, e2 = gaps
    rng = np.random.default_rng(4242 + o1 + 7 * e2)
    p = R.cactus_params(o1=o1, e1=e1, o2=o2, e2=e2, wb=300, wf=0.05)
    e = engine_for(R.params_dict(p))
    jobs = [gapped_family(rng, int(rng.integers(3, 9)), int(rng.choice([120, 500, 1100])), [1, 2, 3, 8, 27, 28, 29, 33, 64, 65, 150, 300]) for _ in range(14)]
    msas, cells = e.poa_msa_batch(jobs, return_cells=True)
    for j, (m, job) in enumerate(zip(msas, jobs)):
        tr = R.oracle_poa_msa_trace(job, p)
        assert m.shape == tr["msa"].shape and np.array_equal(m, tr["msa"]), (gaps, j)
        assert int(cells[j]) == tr["cells"], (gaps, j)
    e.close()


def test_long_window_10k(engine, oracle_built):
    """a full 10 kbp window: rows wider than the shared-memory row cache use the global-memory predecessor path"""
    rng = np.random.default_rng(44)
    job = [s[:10000] for s in family(rng, 4, 10000, sub=0.03, ins=0.01, dele=0.01)]
    m = engine.poa_msa_batch([job])[0]
    o = R.oracle_poa_msa(job)
    assert m.shape == o.shape and np.array_equal(m, o)


def test_bench_shape_properties(engine, oracle_built):
    """BASELINE.json's synthetic shape (8 x 2 kbp, Cactus defaults) in bulk: every row spells its input
    (bar/tests/poaBarTest.c:19-31 validate_msa), no all-gap column, results independent of batch composition,
    and the first ends equal to the oracle bit for bit."""
    import cactus_b200 as cb
    n = 600
    n_seq, lens, flat = workload.synth_ends(0, n, 8, 2000)
    st = engine.stage(packed=(n_seq, lens, flat))
    st.run()
    msas, cells = st.fetch()
    st.close()
    offs = np.concatenate([[0], np.cumsum(lens)])
    for e in range(n):
        m = msas[e]
        for i in range(8):
            s = flat[offs[e * 8 + i]:offs[e * 8 + i + 1]]
            assert np.array_equal(m[i][m[i] != 5], s), (e, i)
        assert not np.any(np.all(m == 5, axis=0)), e
    for e in range(4):
        job = [flat[offs[e * 8 + i]:offs[e * 8 + i + 1]] for i in range(8)]
        tr = R.oracle_poa_msa_trace(job)
        assert np.array_equal(msas[e], tr["msa"]) and int(cells[e]) == tr["cells"], e
    # same ends, different batch (reversed order, different slot assignment): identical output
    jobs_rev = [[flat[offs[e * 8 + i]:offs[e * 8 + i + 1]] for i in range(8)] for e in reversed(range(40))]
    again = engine.poa_msa_batch(jobs_rev)
    for k, e in enumerate(reversed(range(40))):
        assert np.array_equal(again[k], msas[e]), e


def test_golden_windows_and_two_ends(engine):
    """poaBarAligner.h level through the C ABI: sliding windows + trimming, and two-end consistency"""
    for c in G.window_cases():
        m = engine.msa_make_partial_order_alignment(c["strs"], window_size=c["win"])
        assert m.msa_seq.shape == c["msa"].shape and np.array_equal(m.msa_seq, c["msa"]), c["id"]
    for c in G.two_end_cases():
        ms = engine.make_consistent_partial_order_alignments(c["ends"], c["ri"], c["rr"], c["ov"], window_size=c["win"])
        for a, b in zip(ms, c["msas"]):
            assert a.msa_seq.shape == b.shape and np.array_equal(a.msa_seq, b), c["id"]


def test_windows_vs_oracle_and_invariant(engine, oracle_built):
    rng = np.random.default_rng(45)
    ends, wins = [], []
    for it in range(16):
        K = int(rng.integers(1, 8))
        L = int(rng.choice([10, 50, 200, 700]))
        strs = [to_ascii(s) for s in family(rng, K, L, sub=0.05, ins=0.02, dele=0.02, nfrac=0.01)]
        if rng.random() < 0.2 and K > 1:
            strs[-1] = b""
        ends.append(strs)
    for win in (20, 110, 10000):
        ms = engine.msa_make_partial_order_alignment_batch(ends, window_size=win)
        for e, m in zip(ends, ms):
            o = R.oracle_msa_make_partial_order_alignment(e, window_size=win)
            assert m.msa_seq.shape == o.shape and np.array_equal(m.msa_seq, o), win
    # the reference's two-end invariant (poaBarTest.c:160-176)
    for it in range(6):
        K = int(rng.integers(1, 10))
        ends2, ri, rr, ov = two_end_problem(rng, K, int(rng.choice([10, 60, 150])), sub=0.05, ins=0.02, dele=0.02)
        ms = engine.make_consistent_partial_order_alignments(ends2, ri, rr, ov)
        o = R.oracle_make_consistent_partial_order_alignments(ends2, ri, rr, ov)
        for a, b in zip(ms, o):
            assert np.array_equal(a.msa_seq, b)
        for i in range(K):
            assert int((ms[0].msa_seq[i] != 5).sum()) + int((ms[1].msa_seq[rr[0][i]] != 5).sum()) == len(ends2[0][i])


def test_errors_are_loud(engine):
    import cactus_b200 as cb
    with pytest.raises(cb.BarB200Error):
        engine.poa_msa_batch([[np.array([0, 1, 7], np.uint8), np.array([0, 1], np.uint8)]])
    with pytest.raises(cb.BarB200Error):
        engine.poa_msa_batch([[np.array([], np.uint8), np.array([0, 1], np.uint8)]])
    with pytest.raises(cb.BarB200Error):            # one base past the largest CTA class (1024 threads x 16 columns - 1)
        engine.poa_msa_batch([[np.zeros(16384, np.uint8), np.array([0, 1], np.uint8)]])
    with pytest.raises(cb.BarB200Error):
        cb.Engine(cb.PoaParams(partialOrderAlignmentGapOpenPenalty2=0))


def test_pipelined_batch_equals_single_stage(engine, oracle_built):
    """a batch large enough to be cut into pipelined chunks (producer thread, two slot arenas, two streams) returns
    exactly what one single-stage launch returns; spot-checked against the oracle"""
    rng = np.random.default_rng(46)
    jobs = []
    for it in range(2600):
        K = int(rng.integers(2, 6))
        L = int(rng.choice([8, 30, 70, 120]))
        jobs.append(family(rng, K, L, sub=0.05, ins=0.02, dele=0.02))
    msas, cells = engine.poa_msa_batch(jobs, return_cells=True)          # pipelined path (>= 2 * 8 * SMs jobs)
    st = engine.stage(jobs)
    st.run()
    msas1, cells1 = st.fetch()
    st.close()
    assert len(msas) == len(msas1) == len(jobs)
    for j in range(len(jobs)):
        assert msas[j].shape == msas1[j].shape and np.array_equal(msas[j], msas1[j]), j
    assert np.array_equal(np.asarray(cells), np.asarray(cells1))
    for j in range(0, len(jobs), 173):
        tr = R.oracle_poa_msa_trace(jobs[j])
        assert np.array_equal(msas[j], tr["msa"]) and int(cells[j]) == tr["cells"], j


def test_mixed_shapes_are_bucketed(engine, oracle_built):
    """ends bucketed by the CTA class their longest sequence needs (north star: "bucketed by (seq-count x max-length)"): a
    batch of short adjacencies, 2 kbp windows and a long window runs as several class launches with per-class slot sizes and
    returns, job by job in the caller's order, what the oracle computes"""
    rng = np.random.default_rng(47)
    shapes = [(4, 150)] * 12 + [(3, 700)] * 6 + [(5, 1500)] * 3 + [(3, 2500)] * 2 + [(2, 5200)] + [(6, 40)] * 9
    order = rng.permutation(len(shapes))
    jobs = [family(rng, shapes[i][0], shapes[i][1], sub=0.03, ins=0.01, dele=0.01) for i in order]
    msas, cells = engine.poa_msa_batch(jobs, return_cells=True)
    for j, job in enumerate(jobs):
        tr = R.oracle_poa_msa_trace(job)
        assert msas[j].shape == tr["msa"].shape and np.array_equal(msas[j], tr["msa"]) and int(cells[j]) == tr["cells"], (j, shapes[order[j]])
    st = engine.stage(jobs)
    b = st.buckets()
    st.close()
    assert len(b) >= 4 and [x["threads"] for x in b] == sorted([x["threads"] for x in b], reverse=True)
    assert sum(x["jobs"] for x in b) == len(jobs)
    assert b[0]["plane_ints"] > 20 * b[-1]["plane_ints"]          # slots are sized per class, not from the largest job


def test_capacity_misses_grow_geometrically(oracle_built):
    """unrelated sequences outgrow the optimistic plane / MSA sizing: the flagged jobs are re-run with x4 slots, then at worst
    case, and still equal the oracle"""
    rng = np.random.default_rng(48)
    jobs = [[rng.integers(0, 4, size=int(rng.integers(150, 400))).astype(np.uint8) for _ in range(int(rng.integers(6, 12)))] for _ in range(10)]
    jobs += [family(rng, 4, 300) for _ in range(6)]
    import cactus_b200 as cb
    e = cb.Engine()
    msas = e.poa_msa_batch(jobs)
    e.close()
    for j, job in enumerate(jobs):
        o = R.oracle_poa_msa(job)
        assert msas[j].shape == o.shape and np.array_equal(msas[j], o), j


def test_band_wider_than_planned_is_retried(oracle_built):
    """long windows are planned at 2.5 w columns per row; reads whose best columns drift far from the diagonal (block indels of up to
    1 kbp under a narrow band constant) outgrow that, are re-run with more room, and still equal the oracle"""
    rng = np.random.default_rng(77)
    p = R.cactus_params(wb=60, wf=0.01)
    e = engine_for(R.params_dict(p))
    jobs = [gapped_family(rng, int(rng.integers(3, 6)), 3000, [300, 600, 1000, 1000]) for _ in range(6)]
    jobs += [gapped_family(rng, 4, 2600, [5, 10]) for _ in range(3)]
    msas, cells = e.poa_msa_batch(jobs, return_cells=True)
    e.close()
    for j, job in enumerate(jobs):
        tr = R.oracle_poa_msa_trace(job, p)
        assert msas[j].shape == tr["msa"].shape and np.array_equal(msas[j], tr["msa"]), j
        assert int(cells[j]) == tr["cells"], j


def test_flower_submit_wait_equals_the_synchronous_call(engine, oracle_built):
    """barb200_flower_submit / barb200_flower_wait: 30 tickets submitted before the first wait share a few device batches and
    deliver what the synchronous call (and the oracle) delivers"""
    rng = np.random.default_rng(49)
    probs = [two_end_problem(rng, int(rng.integers(1, 7)), int(rng.choice([20, 90, 300])), sub=0.04, ins=0.02, dele=0.02) for _ in range(30)]
    before = engine.queue_stats()
    tickets = [engine.flower_submit(*p) for p in probs]
    res = [engine.flower_wait(t) for t in tickets]
    after = engine.queue_stats()
    assert after["batches"] - before["batches"] < len(probs) // 2
    for k, (p, ms) in enumerate(zip(probs, res)):
        if k % 5 == 0:
            o = R.oracle_make_consistent_partial_order_alignments(*p)
            for a, b in zip(ms, o):
                assert a.msa_seq.shape == b.shape and np.array_equal(a.msa_seq, b), k
        else:
            s = engine.make_consistent_partial_order_alignments(*p)
            for a, b in zip(ms, s):
                assert np.array_equal(a.msa_seq, b.msa_seq), k
    # independent ends (no consistency information), several windows
    ends = [[to_ascii(s) for s in family(rng, 4, 260)] for _ in range(5)]
    t = engine.flower_submit(ends, window_size=100)
    ms = engine.flower_wait(t)
    for e, m in zip(ends, ms):
        o = R.oracle_msa_make_partial_order_alignment(e, window_size=100)
        assert m.msa_seq.shape == o.shape and np.array_equal(m.msa_seq, o)


def test_a_bad_ticket_fails_alone(engine):
    """one caller's invalid input ('-' is code 5, which the device rejects) must not fail the tickets that shared its batch"""
    import cactus_b200 as cb
    rng = np.random.default_rng(50)
    probs = [two_end_problem(rng, 3, 40) for _ in range(8)]
    ends, ri, rr, ov = probs[3]
    ends = [list(e) for e in ends]
    ends[0][0] = ends[0][0][:2] + b"-" + ends[0][0][3:]
    probs[3] = (ends, ri, rr, ov)
    tickets = [engine.flower_submit(*p) for p in probs]
    for k, t in enumerate(tickets):
        if k == 3:
            with pytest.raises(cb.BarB200Error):
                engine.flower_wait(t)
        else:
            assert len(engine.flower_wait(t)) == 2


def test_one_context_over_every_visible_device(engine, oracle_built):
    """barb200_params.devices[]: ONE context drives every GPU of the box (the batch call deals jobs by estimated cost, the end queue's
    lane workers of every device pull ends); results are those of the single-device context, in the caller's order. On a one-GPU
    box this is the same code path with one device."""
    import cactus_b200 as cb
    rng = np.random.default_rng(51)
    jobs = [family(rng, int(rng.integers(2, 9)), int(rng.choice([60, 300, 900, 1800])), sub=0.03, ins=0.01, dele=0.01) for _ in range(300)]
    one = engine.poa_msa_batch(jobs)
    e = cb.Engine(cb.PoaParams(devices="all"))
    assert e.device_count() >= 1
    many, cells = e.poa_msa_batch(jobs, return_cells=True)
    for a, b in zip(one, many):
        assert a.shape == b.shape and np.array_equal(a, b)
    probs = [two_end_problem(rng, int(rng.integers(2, 6)), int(rng.choice([50, 400]))) for _ in range(40)]
    tickets = [e.flower_submit(*p) for p in probs]
    for p, t in zip(probs, tickets):
        got = e.flower_wait(t)
        want = engine.make_consistent_partial_order_alignments(*p)
        for a, b in zip(got, want):
            assert np.array_equal(a.msa_seq, b.msa_seq)
    e.close()


def test_retry_plan_cut_to_a_small_device_budget(oracle_built):
    """a capacity retry whose upper-bound plan exceeds the memory the context may use (here a small share of the device, the
    situation of a deep 10 kbp window on an 80 GB card) is cut to fit instead of failing, and still equals the oracle"""
    import cactus_b200 as cb
    from test_slot_plan_cpu import _lib
    rng = np.random.default_rng(4711)
    job = family(rng, 12, 2000, sub=0.2, ins=0.02, dele=0.02)
    K, S, ML = len(job), sum(len(s) for s in job), max(len(s) for s in job)
    tr = R.oracle_poa_msa_trace(job)
    p = R.cactus_params()
    lib = _lib()
    optimistic = lib.hosttest_plane_ints_for_job(p.wb, p.wf, K, S, ML, 1.0, 0)
    x4 = lib.hosttest_plane_ints_for_job(p.wb, p.wf, K, S, ML, 4.0, 0)
    assert max(a["node_n"] for a in tr["alns"]) > ML + (S - ML) // 8 + 256     # the optimistic plan is outgrown: a retry runs
    # a memory share that leaves the context ~2.5 x the optimistic plan: enough for the job, not for the x4 retry's upper bound
    probe = cb.Engine()
    free = probe.device_info()["mem_free"]
    probe.close()
    budget = 2.5 * 4 * optimistic
    assert 4 * x4 > budget
    e = cb.Engine(cb.PoaParams(mem_fraction=budget / free))
    msas = e.poa_msa_batch([job])
    e.close()
    assert msas[0].shape == tr["msa"].shape and np.array_equal(msas[0], tr["msa"])
