#!/usr/bin/env python
"""Compare the device's per-alignment POA traces with the oracle's on seeded families, and print for every job that differs the first
alignment, field and index where it does. Start here when a GPU parity check of POA mode fails: the first differing alignment names
the read, and the field says whether the band (dp_beg / dp_end), the best cell (best_score), the traceback (cigar) or the guide tree
(read_id_map) went wrong.

The trace numbers its rows in abPOA's order, the BFS order recomputed after every fusion, so that row r is row r of the reference.
The production kernels splice the new nodes into the previous order instead: an equally valid topological order with the same cells
per node, but one that decides which predecessor rows the sweep reads from its shared-memory ring and which from global memory. A fault
that depends on the splice order, or on those far-row paths as that order lays them out, shows in the production MSAs but not here; the
trace still shows every band, cigar and best score the device computes for abPOA's order.

    python scripts/poa_trace_diff.py [--jobs N] [--K 2:12] [--L 20,150,400,1500] [--sub 0.05] [--indel 0.02] [--seed 0]
                                     [--wb 1000] [--wf 0.1] [--gaps 400,30,1200,1] [--threads 0]
Exit status 1 if any job differs."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cactus_b200 as cb  # noqa: E402
import _reflib as R  # noqa: E402
from _synth import family  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--jobs", type=int, default=64)
    ap.add_argument("--K", default="2:12", help="reads per job, lo:hi (inclusive)")
    ap.add_argument("--L", default="20,150,400,1500", help="read lengths to draw from")
    ap.add_argument("--sub", type=float, default=0.05)
    ap.add_argument("--indel", type=float, default=0.02)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--wb", type=int, default=1000)
    ap.add_argument("--wf", type=float, default=0.1)
    ap.add_argument("--gaps", default="400,30,1200,1", help="o1,e1,o2,e2")
    ap.add_argument("--threads", type=int, default=0, help="threads_per_block (minimum CTA class)")
    a = ap.parse_args()
    klo, khi = (int(x) for x in a.K.split(":"))
    lens = [int(x) for x in a.L.split(",")]
    o1, e1, o2, e2 = (int(x) for x in a.gaps.split(","))
    rng = np.random.default_rng(a.seed)
    jobs = [family(rng, int(rng.integers(klo, khi + 1)), int(rng.choice(lens)), sub=a.sub, ins=a.indel, dele=a.indel) for _ in range(a.jobs)]
    p = R.cactus_params(wb=a.wb, wf=a.wf, o1=o1, e1=e1, o2=o2, e2=e2)
    e = cb.Engine(cb.PoaParams(partialOrderAlignmentBandConstant=a.wb, partialOrderAlignmentBandFraction=a.wf,
                               partialOrderAlignmentGapOpenPenalty1=o1, partialOrderAlignmentGapExtensionPenalty1=e1,
                               partialOrderAlignmentGapOpenPenalty2=o2, partialOrderAlignmentGapExtensionPenalty2=e2,
                               threads_per_block=a.threads))
    try:
        got = e.poa_msa_trace_batch(jobs)
    finally:
        e.close()
    bad = 0
    for j, (job, g) in enumerate(zip(jobs, got)):
        d = cb.first_trace_difference(g, R.oracle_poa_msa_trace(job, p))
        if d is None:
            continue
        bad += 1
        aln, field, idx = d
        where = "job" if aln is None else "alignment %d (read %d, %d nodes before it)" % (aln, g["alns"][aln]["read_id"], g["alns"][aln]["node_n"])
        print("job %d (K=%d, longest %d): %s, field %s%s" % (j, len(job), max(len(s) for s in job), where, field,
                                                              "" if idx is None else ", index %s" % idx))
    print("%d of %d jobs differ from the oracle" % (bad, len(jobs)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
