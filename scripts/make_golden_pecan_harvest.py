#!/usr/bin/env python
"""Writes tests/golden/pecan_harvest.bin: a small cPecan-mode recording made by shim/cactus_pecan_harvest.c
(oracle/_ref/libflower_pecan_harvest.so, built by oracle/pecan_harvest.mk where the reference sources exist) during one reference
bar() run over seeded flowers of tests/_flowers.py -- short ends aligned all-pairs, one end of 14+ strings (makeAlignment's
incremental pair selection), ends whose pairs are long enough for MUM anchors, and ragged ends. One OpenMP thread, so that the
file is the same on every run. The GPU suite replays it (tests/test_gpu_pecan_harvest.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _flowers as F  # noqa: E402
import workload  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "pecan_harvest.bin")
F._PATHS.setdefault("pecan_harvest", os.path.join(ROOT, "oracle", "_ref", "libflower_pecan_harvest.so"))


def flowers():
    return [F.random_flower(400 + s, n_threads=int(5 + s % 4), n_blocks=3, seg_len=60) for s in range(2)] + \
           [F.random_flower(500, n_threads=14, n_blocks=2, seg_len=70, p_skip=0.0, p_loop=0.0)] + \
           [F.random_flower(700, n_threads=3, n_blocks=2, seg_len=900, p_skip=0.0, p_loop=0.0, p_empty=0.0)]


def main():
    if not F.have("pecan_harvest"):
        sys.exit("oracle/_ref/libflower_pecan_harvest.so is not built (make -C oracle -f pecan_harvest.mk)")
    tmp = OUT + ".tmp"
    if os.path.exists(tmp):
        os.remove(tmp)
    os.environ["BARB200_PECAN_HARVEST"] = tmp
    try:
        F.bar("pecan_harvest", flowers(), {"bar/partialOrderAlignment": "0"}, threads=1)
    finally:
        del os.environ["BARB200_PECAN_HARVEST"]
    ends = workload.read_pecan_harvest(tmp)
    os.replace(tmp, OUT)
    pairs = [q for e in ends for q in e["pairs"]]
    print("%s: %d ends, %d pairs (%d with anchors, %d ragged), %d bytes" % (
        OUT, len(ends), len(pairs), sum(len(q["anchors"]) > 0 for q in pairs), sum(q["ragged_left"] or q["ragged_right"] for q in pairs),
        os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
