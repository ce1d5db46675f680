#!/usr/bin/env python
"""Small run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck / initcheck): every POA CTA class in one mixed
batch (with guide trees), the windowed end aligner, a few pair-HMM jobs. Development aid; results are checked against the oracle so
that a sanitizer-clean run is also a correct one."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cactus_b200 as cb  # noqa: E402
import workload  # noqa: E402
import _reflib as R  # noqa: E402
from _synth import pecan_pair  # noqa: E402

big = len(sys.argv) > 1 and sys.argv[1] == "big"
eng = cb.Engine()
jobs = []
shapes = [(5, 120), (8, 300), (4, 700), (3, 1500), (3, 3000)] + ([(3, 6000), (2, 11000)] if big else [])
for K, L in shapes:
    n_seq, lens, flat = workload.synth_ends(len(jobs), 2, K, L)
    offs = np.concatenate([[0], np.cumsum(lens)])
    for e in range(2):
        jobs.append([flat[offs[e * K + i]:offs[e * K + i + 1]] for i in range(K)])
# divergent families (bubbles, N bases, unsorted reads), ragged unrelated rows with K > 64 (two read-id words)
from _synth import family  # noqa: E402
rng0 = np.random.default_rng(11)
for K, L, sub in [(9, 150, 0.2), (13, 300, 0.08), (6, 60, 0.0), (2, 1, 0.0)]:
    jobs.append(family(rng0, K, L, sort=False, sub=sub, ins=0.03, dele=0.03, nfrac=0.01))
jobs.append([rng0.integers(0, 5, int(rng0.integers(1, 200))).astype(np.uint8) for _ in range(70)])
msas, cells = eng.poa_msa_batch(jobs, return_cells=True)
bad = 0
for e, job in enumerate(jobs):
    if sum(len(s) for s in job) > 9000:
        continue                     # (oracle time)
    tr = R.oracle_poa_msa_trace(job)
    ok = msas[e].shape == tr["msa"].shape and np.array_equal(msas[e], tr["msa"]) and int(cells[e]) == tr["cells"]
    bad += not ok
print("poa: %d jobs, %d cells, mismatches vs oracle: %d" % (len(jobs), int(cells.sum()), bad), flush=True)
# the trace kernels, one launch per CTA class: a job whose longest read needs that class (16 T - 1 bases), two reads each
rng1 = np.random.default_rng(12)
for T in (32, 64, 128, 256, 640, 1024):
    tjob = [s[:16 * T - 1] for s in family(rng1, 2, 16 * T - 1, sub=0.02, ins=0.01, dele=0.01)]
    pn = R.cactus_params(wb=30, wf=0.002)
    te = cb.Engine(cb.PoaParams(partialOrderAlignmentBandConstant=30, partialOrderAlignmentBandFraction=0.002, threads_per_block=T))
    d = cb.first_trace_difference(te.poa_msa_trace_batch([tjob])[0], R.oracle_poa_msa_trace(tjob, pn))
    te.close()
    bad += d is not None
    print("trace t%d: identical to the oracle: %s" % (T, d is None), flush=True)
seqs = [bytes(np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(5).integers(0, 4, 900)]) for _ in range(1)]
base = seqs[0]
fam = [base, base[:400] + base[420:], base[:100] + b"ACGT" + base[100:], base[5:880]]
m = eng.msa_make_partial_order_alignment(fam, window_size=300)
o = R.oracle_msa_make_partial_order_alignment(fam, window_size=300)
print("windowed end: identical to the oracle:", bool(np.array_equal(m.msa_seq, o)), flush=True)
rng = np.random.default_rng(3)
pairs = []
for L in (40, 300, 1200):
    sx, sy, a = pecan_pair(rng, L, k_anchor=12)
    pairs.append((sx, sy, a, False, False))
res = eng.get_aligned_pairs_using_anchors_batch(pairs, None, True)
okp = True
for q, (t, po, pc) in zip(pairs, res):
    to, poo = R.oracle_pecan_aligned_pairs(q[0], q[1], q[2], False, False, R.pecan_params())
    okp = okp and np.array_equal(t, to) and np.array_equal(po, poo)
print("pair-HMM: %d pairs, identical to the oracle: %s" % (len(pairs), okp), flush=True)
eng.close()
sys.exit(1 if (bad or not okp) else 0)
