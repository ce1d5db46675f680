"""cPecan-mode recordings, no GPU: shim/cactus_pecan_harvest.c records every pair cPecan's multiple aligner aligns during a REFERENCE
bar() run (oracle/_ref/libflower_pecan_harvest.so, oracle/pecan_harvest.mk), workload.read_pecan_harvest reads the file back, and
workload.pecan_replay runs it through the barb200 C ABI -- here over the test-only CPU stand-in device of tests/hosttest, on the GPU
in test_gpu_pecan_harvest.py. The recorded hashes are recomputed with the unmodified reference's own pair-HMM and MUM anchoring."""
import ctypes as C
import os

import numpy as np
import pytest

import _flowers as F
import _mumlib as M
import _reflib as R
import workload
from workload import pecan_replay as PR

GOLDEN = os.path.join(R.ROOT, "tests", "golden", "pecan_harvest.bin")
STANDIN_SO = os.path.join(R.ROOT, "tests", "hosttest", "_build", "libbarb200_standin_mum.so")
F._PATHS.setdefault("pecan_harvest", os.path.join(R.ROOT, "oracle", "_ref", "libflower_pecan_harvest.so"))
PECAN = {"bar/partialOrderAlignment": "0"}

needs_recorder = pytest.mark.skipif(not F.have("pecan_harvest"),
                                    reason="oracle/_ref/libflower_pecan_harvest.so not built (needs the reference sources, oracle/pecan_harvest.mk)")
needs_ref = pytest.mark.skipif(not (R.have_pecan_ref() and M.have_ref()),
                               reason="oracle/_ref/libpecan_ref.so / libmum_ref.so not built (needs the reference sources)")
needs_standin = pytest.mark.skipif(not os.path.exists(STANDIN_SO), reason="tests/hosttest stand-in not built (make -C tests/hosttest -f mum.mk)")


def recorded_flowers():
    """the cPecan-mode flowers of test_flowers_cpu.py (all-pairs ends and ends of 14+ strings) plus flowers whose pairs exceed
    anchorMatrixBiggerThanThis (test_mum_anchors_cpu.py), so that MUM anchors are recorded"""
    return [F.random_flower(400 + s, n_threads=int(5 + s % 4), n_blocks=3, seg_len=60) for s in range(3)] + \
           [F.random_flower(500 + s, n_threads=14 + s, n_blocks=2, seg_len=70, p_skip=0.0, p_loop=0.0) for s in range(2)] + \
           [F.random_flower(700 + s, n_threads=4, n_blocks=2, seg_len=900, p_skip=0.0, p_loop=0.0, p_empty=0.0) for s in range(2)]


def check_ends(ends):
    """every end id once, its pairs numbered 0, 1, 2, ... in recorded order, and every record's anchors hashing to its anchor hash"""
    ids = [e["end"] for e in ends]
    assert len(ids) == len(set(ids))
    for e in ends:
        assert [q["index"] for q in e["pairs"]] == list(range(len(e["pairs"]))), e["end"]
        for q in e["pairs"]:
            assert q["end"] == e["end"]
            assert workload.fnv1a64(q["anchors"]) == q["anchor_hash"]


def check_against_reference(pairs):
    """each record's anchor hash, triple count and triple hash recomputed by the unmodified reference"""
    for q in pairs:
        pe, mu = q["pecan"], q["mum"]
        if q["use_mum_anchors"]:
            a = M.ref_mum_anchors(q["sx"], q["sy"], mu["k"], mu["u"], mu["anchor_matrix_bigger_than_this"], mu["recursive_mums"])
            assert workload.fnv1a64(a) == q["anchor_hash"], (q["end"], q["index"])
        p = R.pecan_params(pe["threshold"], pe["min_diags_between_traceback"], pe["traceback_diagonals"], pe["diagonal_expansion"])
        t = R.ref_pecan_aligned_pairs(q["sx"], q["sy"], q["anchors"], q["ragged_left"], q["ragged_right"], p,
                                      pe["split_matrix_bigger_than_this"])
        assert len(t) == q["n_triples"] and workload.fnv1a64(t) == q["triple_hash"], (q["end"], q["index"])


def replay_on_standin(ends, ends_per_batch):
    ctx = PR.Context(STANDIN_SO)
    try:
        return PR.replay(ctx, ends, ends_per_batch)
    finally:
        ctx.close()


def test_fnv1a64_is_the_64_bit_fnv1a():
    assert workload.fnv1a64(np.zeros(0, np.int64)) == 0xcbf29ce484222325
    h = 0xcbf29ce484222325
    for b in np.array([[7, -1], [3, 1 << 40]], np.int64).tobytes():
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    assert workload.fnv1a64(np.array([[7, -1], [3, 1 << 40]], np.int64)) == h


def test_fixture_reads_into_whole_ends():
    ends = workload.read_pecan_harvest(GOLDEN)
    pairs = [q for e in ends for q in e["pairs"]]
    assert 200 <= len(pairs) <= 1000
    check_ends(ends)
    # what the fixture is for: MUM-anchored pairs, ragged pairs, all-pairs ends and an end of makeAlignment's incremental selection
    assert any(len(q["anchors"]) > 0 and len(q["sx"]) * len(q["sy"]) > q["mum"]["anchor_matrix_bigger_than_this"] for q in pairs)
    assert any(q["ragged_left"] or q["ragged_right"] for q in pairs)
    assert any(len(e["pairs"]) not in {n * (n - 1) // 2 for n in range(2, 100)} for e in ends)     # not every pair of the end
    assert all(q["use_mum_anchors"] and q["pecan"]["split_matrix_bigger_than_this"] == 3000 * 3000 for q in pairs)


def test_reader_rejects_a_bad_magic_and_a_truncated_record(tmp_path):
    data = open(GOLDEN, "rb").read()
    ends = workload.read_pecan_harvest(GOLDEN)
    first = ends[0]["pairs"][0]
    second_at = 8 * 22 + len(first["sx"]) + len(first["sy"]) + 16 * len(first["anchors"])     # the second record's offset
    cut = tmp_path / "cut.bin"
    for n in (second_at + 7, second_at + 100, second_at + 8 * 22 + 1):
        cut.write_bytes(data[:n])
        with pytest.raises(ValueError, match="at byte %d" % second_at):
            workload.read_pecan_harvest(str(cut))
    cut.write_bytes(data[:len(data) - 1])
    with pytest.raises(ValueError, match="truncated"):
        workload.read_pecan_harvest(str(cut))
    bad = bytearray(data)
    bad[second_at] ^= 1
    cut.write_bytes(bytes(bad))
    with pytest.raises(ValueError, match="bad pecan harvest record at byte %d" % second_at):
        workload.read_pecan_harvest(str(cut))
    cut.write_bytes(data[:second_at])
    assert len(workload.read_pecan_harvest(str(cut))) == 1


@needs_ref
def test_fixture_hashes_are_the_references():
    check_against_reference([q for e in workload.read_pecan_harvest(GOLDEN) for q in e["pairs"]])


@needs_standin
def test_fixture_replays_on_the_standin_device():
    ends = workload.read_pecan_harvest(GOLDEN)
    for n in (1, 0):
        r = replay_on_standin(ends, n)
        assert r["mismatches"] == [] and r["pairs"] == sum(len(e["pairs"]) for e in ends)
        assert r["calls"] == (len(ends) if n == 1 else 1)
        assert r["anchor_calls"] > 0 and r["cells"] > 0


@needs_standin
def test_replay_reports_a_pair_that_differs():
    ends = workload.read_pecan_harvest(GOLDEN)[:3]
    ends[1]["pairs"][0]["triple_hash"] ^= 1
    anchored = next(q for e in workload.read_pecan_harvest(GOLDEN) for q in e["pairs"] if len(q["anchors"]))
    anchored["anchor_hash"] ^= 1
    r = replay_on_standin(ends, 0)
    assert r["mismatches"] == [(ends[1]["end"], 0, "triples")]
    r = replay_on_standin([{"end": anchored["end"], "pairs": [anchored]}], 1)
    assert r["mismatches"] == [(anchored["end"], anchored["index"], "anchors")]


@needs_recorder
@needs_ref
@needs_standin
def test_recording_a_cpecan_bar_run(tmp_path):
    """bar() in the cPecan configuration with the recorder, two OpenMP threads: one record per pair the reference aligned, grouped
    into their ends, hashes equal to the reference's and to a replay over the stand-in device. Recording does not change the
    alignment (compared on one thread: with several, the reference's st_random() draws depend on the thread interleaving)."""
    dump = str(tmp_path / "pecan.harvest")
    lib = F._lib("pecan_harvest")
    lib.pecan_harvest_pair_calls.restype = C.c_int64
    fls = recorded_flowers()
    calls0 = lib.pecan_harvest_pair_calls()
    os.environ["BARB200_PECAN_HARVEST"] = dump
    try:
        F.bar("pecan_harvest", fls, PECAN, threads=2)
    finally:
        del os.environ["BARB200_PECAN_HARVEST"]
    calls = lib.pecan_harvest_pair_calls() - calls0
    ends = workload.read_pecan_harvest(dump)
    pairs = [q for e in ends for q in e["pairs"]]
    assert len(pairs) == calls > 0
    check_ends(ends)
    assert all(e["end"] >= 0 for e in ends)                          # every pair was aligned inside a makeAlignment
    assert any(len(q["anchors"]) > 0 for q in pairs)
    assert any(q["ragged_left"] or q["ragged_right"] for q in pairs)
    check_against_reference(pairs)
    r = replay_on_standin(ends, 0)
    assert r["mismatches"] == [] and r["pairs"] == len(pairs)

    os.environ["BARB200_PECAN_HARVEST"] = str(tmp_path / "one_thread.harvest")
    try:
        got = F.bar("pecan_harvest", fls, PECAN, threads=1)
    finally:
        del os.environ["BARB200_PECAN_HARVEST"]
    want = F.bar("ref", fls, PECAN, threads=1)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), i
    # without the variable the recorder only forwards
    sizes = sorted((f.name, f.stat().st_size) for f in tmp_path.iterdir())
    assert np.array_equal(F.bar("pecan_harvest", fls[:1], PECAN, threads=1)[0], want[0])
    assert sorted((f.name, f.stat().st_size) for f in tmp_path.iterdir()) == sizes
