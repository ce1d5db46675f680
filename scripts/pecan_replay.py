#!/usr/bin/env python
"""Replay a cPecan-mode recording (shim/cactus_pecan_harvest.c; BARB200_PECAN_HARVEST=<file> during a reference bar() run, see
INTEGRATION.md) through libbarb200 on every device of one context, and report the workload's shape and the engine's times.

    python scripts/pecan_replay.py <file> [--ends-per-batch N ...] [--devices all|one] [--json out.json]

--ends-per-batch N: N whole ends per barb200 call (1 = what makeAllPairwiseAlignments / one makeAlignment round issues at most;
0 = the whole file in one call, the upper bound); repeat the flag for several settings (default: 1 and 0). Every pair's anchors
and triples are checked against the recording in every setting; if any differs the script says which and exits 1 without
printing a throughput."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import workload  # noqa: E402
from workload import pecan_replay as PR  # noqa: E402


def _hist_line(name, values):
    h = PR.histogram(values)
    return "  %-22s %s" % (name, "  ".join("[%d,%d):%d" % b for b in h) if h else "(none)")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("file")
    ap.add_argument("--ends-per-batch", type=int, action="append", default=None,
                    help="whole ends per call; 0 = all ends in one call; repeatable (default: 1 and 0)")
    ap.add_argument("--devices", choices=["all", "one"], default="all", help="context over every visible device (default) or one")
    ap.add_argument("--lib", default=None, help="library exporting the barb200 cPecan C ABI (default: the in-tree libbarb200.so)")
    ap.add_argument("--json", default=None, help="also write the report as JSON here")
    args = ap.parse_args()
    settings = args.ends_per_batch or [1, 0]

    ends = workload.read_pecan_harvest(args.file)
    pairs = [q for e in ends for q in e["pairs"]]
    if not pairs:
        print("pecan_replay: %s holds no pairs" % args.file)
        return 1
    import cactus_b200
    ctx = PR.Context(args.lib or cactus_b200.library_path(), all_devices=args.devices == "all")
    try:
        # warm-up, so that module loads and first allocations stay out of the report: the first end and the first end with an anchor call
        PR.replay(ctx, ends[:1] + [e for e in ends if any(PR.needs_anchor_call(q) for q in e["pairs"])][:1], 0)
        stats0 = ctx.device_stats()
        runs = {}
        for n in settings:
            runs[n] = PR.replay(ctx, ends, n)
            if runs[n]["mismatches"]:
                break
        stats1 = ctx.device_stats()
    finally:
        ctx.close()

    bad = {n: r["mismatches"] for n, r in runs.items() if r["mismatches"]}
    first = runs[settings[0]]
    print("pecan_replay: %s -- %d ends, %d pairs (%d with MUM anchors, %d ragged)" % (
        os.path.basename(args.file), len(ends), len(pairs), sum(q["use_mum_anchors"] for q in pairs),
        sum(q["ragged_left"] or q["ragged_right"] for q in pairs)))
    print("workload shape (power-of-two buckets [lo,hi):count)")
    for line in (_hist_line("lX", [len(q["sx"]) for q in pairs]), _hist_line("lY", [len(q["sy"]) for q in pairs]),
                 _hist_line("anchors per pair", first["n_anchors"]), _hist_line("sub-jobs per pair", first["sub_jobs"]),
                 _hist_line("banded cells per pair", first["pair_cells"]), _hist_line("pairs per end", [len(e["pairs"]) for e in ends])):
        print(line)
    if bad:
        for n, mm in bad.items():
            print("PARITY FAILED (ends per batch %d): %d of %d pairs differ from the recording" % (n, len({(e, i) for e, i, _ in mm}), len(pairs)))
            for e, i, what in mm[:20]:
                print("  end %d pair %d: %s differ" % (e, i, what))
        return 1
    print("parity: every pair's anchors and triples equal the recording (%d settings)" % len(runs))
    report = {"file": os.path.basename(args.file), "ends": len(ends), "pairs": len(pairs), "cells": first["cells"], "parity": "passed",
              "settings": []}
    for n, r in runs.items():
        label = "all ends in one call" if n <= 0 else "%d end(s) per call" % n
        row = {"ends_per_batch": n, "calls": r["calls"], "hmm_wall_s": r["hmm_s"], "gcell_per_s": r["cells"] / r["hmm_s"] / 1e9,
               "pairs_per_s": r["pairs"] / r["hmm_s"], "anchor_calls": r["anchor_calls"], "anchor_device_ms": r["anchor_device_ms"],
               "anchor_call_ms": r["anchor_call_ms"]}
        report["settings"].append(row)
        anchors = "n/a" if r["anchor_device_ms"] is None else "%.2f ms device / %.2f ms call" % (r["anchor_device_ms"], r["anchor_call_ms"])
        print("%-22s %5d calls  pair-HMM %.4f s  %.3f Gcell/s  %.0f pairs/s  |  MUM anchors: %d calls, %s" % (
            label, r["calls"], r["hmm_s"], row["gcell_per_s"], row["pairs_per_s"], r["anchor_calls"], anchors))
    if stats0 is not None and stats1 is not None:
        hmm, mum = (stats1[0] - stats0[0]).tolist(), (stats1[1] - stats0[1]).tolist()
        report["device_hmm_pairs"], report["device_mum_pairs"] = hmm, mum
        print("pairs per device: pair-HMM %s, MUM anchors %s" % (hmm, mum))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
