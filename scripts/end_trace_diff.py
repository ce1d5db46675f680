#!/usr/bin/env python
"""Trace every sliding window of every end on the device (barb200_trace_ends) and through a checker, and print for every end that
differs the first window, and inside it the first alignment and field, where it does. Run this when a harvested replay
(bench.py --workload) fails its parity gate: the gate only says which end's MSA hash differs; this names the window and whether its
input slice (offsets, lens, empty, progressive), its POA job (read_id_map, dp_beg / dp_end, best_score, cigar, ...), the trim against
its neighbours (trimmed_lens, column_no) or the cross-end trim (msa) went wrong.

Inputs: the seeded multi-window end sets of tests/_end_trace_cases.py (default), or a harvest file written by shim/cactus_bar_harvest.c
(--workload FILE, optionally one record --flower i and one end --end j of it). Checker: the unmodified reference's own window chain
(oracle/_ref/libbar_trace_ref.so, built where the reference sources exist; default when present) or the restated chain
(--oracle restated, oracle/_build/libend_trace_oracle.so).

Not covered: the production kernels' node order (the trace kernels number rows in abPOA's BFS order) and the end queue's batching,
which tests/test_gpu_end_trace.py checks through the final MSAs.

    python scripts/end_trace_diff.py [--workload FILE [--flower i] [--end j]] [--oracle reference|restated] [--wb 1000] [--wf 0.1]
Exit status 1 if any end differs."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cactus_b200 as cb  # noqa: E402
import _end_trace_cases as X  # noqa: E402
import _endtrace as T  # noqa: E402
import _reflib as R  # noqa: E402


def harvest_cases(path, flower, end, wb, wf):
    import workload
    out = []
    for i, r in enumerate(workload.read_harvest(path)):
        if flower is not None and i != flower:
            continue
        ends, ri, rr, ov = r["ends"], r["right_end_indexes"], r["right_end_row_indexes"], r["overlaps"]
        if end is not None:                   # one end alone: no cross-end trim
            ends, ri, rr, ov = [ends[end]], None, None, None
        out.append(dict(name="flower %d" % i + ("" if end is None else " end %d" % end), ends=ends, ri=ri, rr=rr, ov=ov,
                        window_size=r["window_size"], max_prog_rows=r["max_prog_rows"], max_prog_length_diff=r["max_prog_length_diff"],
                        poa=dict(wb=wb, wf=wf)))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workload", help="a harvest file (shim/cactus_bar_harvest.c)")
    ap.add_argument("--flower", type=int, help="only this record of the harvest file")
    ap.add_argument("--end", type=int, help="only this end of each record (traced alone)")
    ap.add_argument("--oracle", choices=("reference", "restated"), default=None)
    ap.add_argument("--wb", type=int, default=1000, help="band constant of a harvest file's run")
    ap.add_argument("--wf", type=float, default=0.1, help="band fraction of a harvest file's run")
    a = ap.parse_args()
    T.build()
    which = a.oracle or ("reference" if T.have_ref() else "restated")
    if which == "reference" and not T.have_ref():
        sys.exit("oracle/_ref/libbar_trace_ref.so is not built; use --oracle restated")
    cases = harvest_cases(a.workload, a.flower, a.end, a.wb, a.wf) if a.workload else list(X.cases()) + list(X.gpu_cases())
    checker = T.ref_trace_ends if which == "reference" else T.oracle_trace_ends
    from test_gpu_parity import engine_for
    bad = ends = windows = 0
    for c in cases:
        p = R.cactus_params(**c["poa"])
        e = engine_for(R.params_dict(p))
        try:
            got = e.trace_ends(c["ends"], c["ri"], c["rr"], c["ov"], c["window_size"], c["max_prog_rows"], c["max_prog_length_diff"])
        finally:
            e.close()
        want = [cb.parse_end_trace(w) for w in checker(*X.args(c), p=p)]
        for j, (g, w) in enumerate(zip(got, want)):
            ends += 1
            windows += len(w["windows"])
            d = cb.first_end_trace_difference(g, w)
            if d is None:
                continue
            bad += 1
            k, field, index = d
            if field == "trace":
                aln, f, i = index
                where = "window %d: alignment %s, field %s, index %s" % (k, aln, f, i)
                if aln is not None:
                    where += " (read %d)" % w["windows"][k]["trace"]["alns"][aln]["read_id"]
            elif k is None:
                where = "field %s (after every window agreed)" % field
            else:
                where = "window %d: field %s, index %s" % (k, field, index)
                if field in ("offsets", "lens", "empty") and index is not None:
                    where += " (device %d, %s %d)" % (g["windows"][k][field][index], which, w["windows"][k][field][index])
            print("%s, end %d (%d rows, %d windows): first difference at %s" % (c["name"], j, w["seq_no"], len(w["windows"]), where))
    print("%d ends, %d windows, %d differ from the %s chain" % (ends, windows, bad, which))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
