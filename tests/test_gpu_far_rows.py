"""Rows whose predecessors are not the previous row, under every CTA-size class (H100). The DP sweep keeps the previous row in
registers, reads a predecessor two rows back from a ring of the last two rows in shared memory (every class but the 1024-thread
one, whose two rows do not fit its shared memory) and older predecessors from the planes in global memory. Each family below is
one parent with hand-placed edits that give the graph such rows once the reads are fused:
  * a substitution: a bubble X -> {A, B} -> Y, where B's only predecessor is X at r - 2 and Y's are A at r - 2 and B;
  * three and four different bases at one column: 3- and 4-way bubbles, predecessors at r - 2, r - 3 and r - 4;
  * deletions of 1, 2 and 40 bases, alone and next to substitutions: predecessors at r - 2, r - 3 and far back;
  * insertions of 1, 5 and 60 bases: the row after an insertion reaches back past all of it;
  * a first base that differs from the parent's: the node after it has row 0 as a predecessor at row 2.
They run under the default band and under narrow ones, so that bands start and end inside a predecessor's stored padding
block. MSA bytes and banded cell counts must equal the oracle's."""
import functools

import numpy as np
import pytest

import _reflib as R
from test_gpu_parity import engine_for

CLASSES = (32, 64, 128, 256, 640, 1024)


def edit(parent, subs=(), dels=(), ins=()):
    """parent with substitutions {pos: base}, deletions [(pos, n)] and insertions [(pos, seq)], positions in parent coordinates"""
    subs, dels, ins = dict(subs), dict(dels), dict(ins)
    out, i = [], 0
    while i < len(parent):
        if i in ins:
            out.extend(ins[i])
        if i in dels:
            i += dels[i]
            continue
        out.append(subs.get(i, parent[i]))
        i += 1
    return np.array(out, np.uint8)


def other(b, k=1):
    return (int(b) + k) % 4


def families(rng, n):
    """jobs whose reads are at most n bases long"""
    p = rng.integers(0, 4, n - 70).astype(np.uint8)
    m = len(p)
    at = lambda f: int(f * m)                                                                   # noqa: E731
    rnd = lambda k: rng.integers(0, 4, k).astype(np.uint8)                                      # noqa: E731
    jobs = []
    # two-way bubbles, and a read that shares them
    jobs.append([p, edit(p, subs={at(.2): other(p[at(.2)]), at(.6): other(p[at(.6)])}),
                 edit(p, subs={at(.2): other(p[at(.2)])}), edit(p, subs={at(.4): other(p[at(.4)])})])
    # 3- and 4-way bubbles at one column. The last read is fused after the last sweep, so each of the three other bases comes
    # in two reads: whichever read the guide tree puts last, the sweeps before it see the 4-way bubbles
    c, d = at(.3), at(.7)
    jobs.append([p] + [edit(p, subs={c: other(p[c], k), d: other(p[d], k), at(.1 * k + .05 * t): other(p[at(.1 * k + .05 * t)])})
                       for k in (1, 2, 3) for t in (0, 1)])
    jobs.append([p, edit(p, subs={c: other(p[c], 1)}), edit(p, subs={c: other(p[c], 2)}), p, edit(p, dels={c: 1})])
    # deletions of 1, 2 and 40 bases, and deletions next to substitutions
    jobs.append([p, edit(p, dels={at(.25): 1}), edit(p, dels={at(.5): 2}), edit(p, dels={at(.75): 40})])
    e = at(.45)
    jobs.append([p, edit(p, subs={e: other(p[e])}, dels={e + 1: 1}), edit(p, subs={e + 2: other(p[e + 2])}, dels={e: 2}),
                 edit(p, subs={e - 1: other(p[e - 1]), e + 1: other(p[e + 1], 2)}, dels={e: 1})])
    # insertions of 1, 5 and 60 bases (long insertions: predecessors far beyond r - 2)
    jobs.append([p, edit(p, ins={at(.3): rnd(1)}), edit(p, ins={at(.5): rnd(5)}), edit(p, ins={at(.6): rnd(60)}),
                 edit(p, ins={at(.6): rnd(60)}, dels={at(.8): 3})])
    # a first base that differs, and one that is deleted
    jobs.append([p, edit(p, subs={0: other(p[0])}), edit(p, subs={0: other(p[0], 2), 1: other(p[1])}), edit(p, dels={0: 1})])
    # everything at once, several times along the read
    mix = {}
    for f in np.linspace(.05, .9, 12):
        mix[at(f)] = other(p[at(f)], int(rng.integers(1, 4)))
    jobs.append([p, edit(p, subs=mix), edit(p, subs=dict(list(mix.items())[::2]), dels={at(.33): 3, at(.66): 1}, ins={at(.5): rnd(12)}),
                 edit(p, dels={at(.1): 1, at(.4): 2}, ins={at(.2): rnd(3), at(.8): rnd(30)})])
    return jobs


PARAMS = {"default": R.cactus_params(), "narrow": R.cactus_params(wb=10, wf=0.01), "narrow30": R.cactus_params(wb=30, wf=0.002)}


@functools.lru_cache(maxsize=None)
def cases(n):
    rng = np.random.default_rng(2024 + n)
    jobs = families(rng, n)
    assert max(len(s) for job in jobs for s in job) <= n
    return [(name, p, jobs, [R.oracle_poa_msa_trace(job, p) for job in jobs]) for name, p in PARAMS.items()]


def run_and_compare(threads, n):
    for name, p, jobs, trs in cases(n):
        e = engine_for(R.params_dict(p), threads_per_block=threads)
        try:
            st = e.stage(jobs)
            try:
                b = st.buckets()
                st.run()
                msas, cells = st.fetch()
            finally:
                st.close()
        finally:
            e.close()
        assert [x["threads"] for x in b] == [threads], (name, b)
        for j, (m, tr) in enumerate(zip(msas, trs)):
            assert m.shape == tr["msa"].shape and np.array_equal(m, tr["msa"]), (threads, name, j)
            assert int(cells[j]) == tr["cells"], (threads, name, j)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", CLASSES)
def test_far_predecessors_every_class(oracle_built, threads):
    """reads of up to 511 bases (they fit the one-warp class) forced into each class in turn"""
    run_and_compare(threads, 511)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", (128, 256))
def test_far_predecessors_2kbp(oracle_built, threads):
    """the same families at 2 kbp, the length of the benchmark's reads"""
    run_and_compare(threads, 2000)
