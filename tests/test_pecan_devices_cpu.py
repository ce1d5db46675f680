"""cPecan mode over several devices, CPU only: the deal of a batch's pairs over the devices (pecan_plan.cpp: deal_pairs, which the
pair-HMM and MUM-anchor batch calls run on a context of several devices; its host build is tests/hosttest/pecan_devices.cpp,
compiled here into a temporary directory), and a batch split by it, computed share by share with the host emulation of the
product's block program (tests/hosttest) and put back in caller order, against the unsplit batch. The device runs are under
-m gpu (test_gpu_pecan_devices.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _reflib as R
from _synth import pecan_pair

HOSTTEST = os.path.join(R.ROOT, "tests", "hosttest")
_DEAL_LIB = []


@pytest.fixture(scope="module", autouse=True)
def _deal_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pecan_devices") / "libpecan_devices.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, os.path.join(HOSTTEST, "pecan_devices.cpp"),
                           os.path.join(R.ROOT, "cactus_b200", "csrc", "pecan_plan.cpp")])
    _DEAL_LIB[:] = [C.CDLL(so)]
    yield
    _DEAL_LIB.clear()


def _deal(cost, ndev):
    lib = _DEAL_LIB[0]
    lib.hosttest_pecan_deal_pairs.restype = None
    lib.hosttest_pecan_deal_pairs.argtypes = [C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    cost = np.ascontiguousarray(np.asarray(cost, np.int64))
    counts, pairs = np.zeros(max(ndev, 1), np.int64), np.zeros(max(len(cost), 1), np.int64)
    lib.hosttest_pecan_deal_pairs(len(cost), cost.ctypes.data, ndev, counts.ctypes.data, pairs.ctypes.data)
    return [s.tolist() for s in np.split(pairs[:len(cost)], np.cumsum(counts)[:-1])]


@pytest.mark.parametrize("ndev", [2, 3, 4, 8])
def test_every_pair_lands_once_in_caller_order(ndev):
    rng = np.random.default_rng(ndev)
    cost = rng.integers(0, 5_000_000, 2000)
    shares = _deal(cost, ndev)
    assert len(shares) == ndev
    assert sorted(i for s in shares for i in s) == list(range(len(cost)))
    for s in shares:
        assert s == sorted(s)
        assert len(s) > 0


@pytest.mark.parametrize("ndev", [2, 3, 4, 8])
def test_largest_share_is_within_the_mean_plus_the_largest_pair(ndev):
    for seed in range(5):
        rng = np.random.default_rng(100 + seed)
        cost = np.concatenate([rng.integers(1, 4_000_000, 500), rng.integers(1, 400_000_000, 3)])     # a few pairs far above the rest
        loads = [int(cost[s].sum()) for s in _deal(cost, ndev)]
        assert max(loads) <= cost.sum() / ndev + cost.max(), (seed, loads)


def test_one_device_is_the_identity():
    cost = np.random.default_rng(1).integers(0, 10 ** 9, 777)
    assert _deal(cost, 1) == [list(range(777))]
    assert _deal([], 1) == [[]]


def test_no_pairs_and_fewer_pairs_than_devices():
    assert _deal([], 4) == [[], [], [], []]
    shares = _deal([5, 90, 7], 8)
    assert sorted(i for s in shares for i in s) == [0, 1, 2]
    assert sum(1 for s in shares if s) == 3 and all(len(s) <= 1 for s in shares)
    assert shares[0] == [1]                           # the largest pair goes first, to the lowest device


def test_ties_and_repeat_calls_give_the_same_split():
    cost = [10] * 9 + [0] * 5 + [30, 30]
    first = _deal(cost, 3)
    assert all(_deal(cost, 3) == first for _ in range(5))
    # equal costs: the earlier pair first, each to the least-loaded device, the lowest one on a tie
    assert 14 in first[0] and 15 in first[1] and first[2][:3] == [0, 1, 2] and 3 in first[0]
    rng = np.random.default_rng(9)
    cost = rng.integers(0, 1000, 5000)                 # many equal costs
    assert _deal(cost, 4) == _deal(cost.copy(), 4)


def test_split_batch_reassembled_equals_the_unsplit_batch(oracle_built):
    """split, compute every share on its own (the host emulation of the block program stands in for a device), put the results
    back at the caller's indices: the same triples, posteriors and cells as the batch in one piece"""
    rng = np.random.default_rng(2024)
    pairs = []
    for it in range(20):
        L = int(rng.choice([1, 30, 100, 300, 700]))
        sx, sy, a = pecan_pair(rng, L, k_anchor=int(rng.choice([8, 20])), sub=0.05)
        pairs.append((sx, sy, a, bool(rng.integers(0, 2)), bool(rng.integers(0, 2))))
    pairs += [(b"", b"", [], False, False), (b"A", b"", [], False, True)]
    p = R.pecan_params()
    whole = [R.hosttest_pecan_aligned_pairs(*q, p) for q in pairs]
    cells = [w[2] for w in whole]
    for ndev in (2, 3, 5):
        out = [None] * len(pairs)
        for share in _deal(cells, ndev):
            for i in share:
                out[i] = R.hosttest_pecan_aligned_pairs(*pairs[i], p)
        for i, (w, o) in enumerate(zip(whole, out)):
            assert np.array_equal(w[0], o[0]) and np.array_equal(w[1], o[1]) and w[2] == o[2], (ndev, i)
