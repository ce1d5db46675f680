"""How cPecan mode's batch calls scale over the devices of one context.

For 1, 2, .. N visible devices (one context over devices 0 .. k-1 each), on the same seeded synthetic 2 kbp pairs with MUM-like
anchors (workload.synth_pairs, default 4224 pairs per visible device):
  * get_aligned_pairs_using_anchors_batch (barb200_pecan_aligned_pairs_batch through the host-buffer call, posteriors included):
    wall time of the C call, which returns with the results on the host, and Gcell/s (cells = sum of band diagonal widths);
  * mum_anchor_pairs_batch (barb200_pecan_anchor_pairs_batch): wall time of the C call (barb200_mum_last_timing) and the slowest
    device's kernel time;
after `--warmup` untimed calls, the best and median of `--reps` timed calls. Prints one JSON line per device count with the pairs each
device ran (barb200_pecan_device_stats), then one with the card's name, power limit and clocks; asserts that the outputs hash the
same for every device count. Writes nothing unless --out is given.

    python scripts/pecan_devices_probe.py [--pairs-per-device 4224] [--max-devices N] [--reps 3] [--warmup 1] [--out FILE]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cactus_b200 as cb  # noqa: E402
import workload  # noqa: E402

L_BP = 2000


def card_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        return [dict(zip(q.split(","), (v.strip() for v in line.split(",")))) for line in out.strip().splitlines()]
    except (OSError, subprocess.SubprocessError) as e:
        return [{"error": repr(e)}]


def digest(res, anchors):
    h = hashlib.sha256()
    for t, po, cells in res:
        h.update(np.ascontiguousarray(t).tobytes()); h.update(np.ascontiguousarray(po).tobytes()); h.update(np.int64(cells).tobytes())
    for a in anchors:
        h.update(np.int64(len(a)).tobytes()); h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def measure(k, pairs, reps, warmup):
    eng = cb.Engine(cb.PoaParams(devices=list(range(k))))
    try:
        assert eng.device_count() == k
        table = eng.pecan_table(pairs)
        for _ in range(warmup):
            eng._take_pairs(*eng.pecan_batch_raw(table, None, True), table.n)
            eng.mum_anchor_pairs_batch(table)
        before = eng.pecan_device_stats()
        hmm_s, mum_s, mum_kms, res, anchors = [], [], [], None, None
        for _ in range(reps):
            t0 = time.perf_counter()
            raw = eng.pecan_batch_raw(table, None, True)          # returns with every result on the host
            hmm_s.append(time.perf_counter() - t0)
            res = eng._take_pairs(*raw, table.n)
            anchors = eng.mum_anchor_pairs_batch(table)
            tm = eng.mum_last_timing()
            mum_s.append(tm["wall_ms"] / 1e3)
            mum_kms.append(tm["kernel_ms"])
        after = eng.pecan_device_stats()
        cells = int(sum(r[2] for r in res))
        return {"devices": k, "pairs": len(pairs), "cells": cells,
                "hmm": {"best_s": min(hmm_s), "median_s": float(np.median(hmm_s)), "gcell_per_s": cells / min(hmm_s) / 1e9,
                        "gcell_per_s_median": cells / float(np.median(hmm_s)) / 1e9,
                        "pairs_per_device": [(a - b) // reps for a, b in zip(after["hmm_pairs"], before["hmm_pairs"])]},
                "mum": {"best_s": min(mum_s), "median_s": float(np.median(mum_s)), "slowest_device_kernel_ms": min(mum_kms),
                        "pairs_per_device": [(a - b) // reps for a, b in zip(after["mum_pairs"], before["mum_pairs"])]},
                "digest": digest(res, anchors)}
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--pairs-per-device", type=int, default=4224)
    ap.add_argument("--max-devices", type=int, default=0, help="0: every visible device")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    probe = cb.Engine(cb.PoaParams(devices="all"))
    n = probe.device_count()
    probe.close()
    if args.max_devices > 0:
        n = min(n, args.max_devices)
    pairs = workload.synth_pairs(0, args.pairs_per_device * n, L_BP, k_anchor=50)
    lines = []
    for k in range(1, n + 1):
        r = measure(k, pairs, args.reps, args.warmup)
        lines.append(r)
        print(json.dumps(r), flush=True)
    lines.append({"cards": card_facts(), "visible_devices": n, "pair_length": L_BP, "reps": args.reps, "warmup": args.warmup})
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))
    digests = {r["digest"] for r in lines[:-1]}
    assert len(digests) == 1, "outputs differ between device counts: %s" % [(r["devices"], r["digest"]) for r in lines[:-1]]
    print("outputs identical for 1..%d devices" % n)


if __name__ == "__main__":
    main()
