"""Time cPecan's MUM anchoring at the bench's pecan shape (workload.synth_pairs, 4224 pairs of 2 kbp): the device batch
(barb200_pecan_anchor_pairs_batch: device time and wall time of the C call), the reference's host code over the machine's usable
cores (oracle/_ref/libmum_ref.so), and the shim's align_pair_list equivalent -- anchors plus the pair-HMM batch -- with host and
with device anchors. Prints one JSON line; --out also writes it to a file.

    python scripts/prof_mums.py [--pairs 4224] [--len 2000] [--reps 5] [--out prof_mums.json]
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cactus_b200 as cb  # noqa: E402
import workload  # noqa: E402
import _mumlib as M  # noqa: E402
import _reflib as R  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4224)
    ap.add_argument("--len", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-sample", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pairs = [(q[0], q[1]) for q in workload.synth_pairs(0, a.pairs, a.len, k_anchor=50)]
    eng = cb.Engine()
    info = eng.device_info()
    res = {"pairs": a.pairs, "len": a.len, "device": info["name"], "cores": len(os.sched_getaffinity(0))}
    table = eng.pecan_table([(x, y) for x, y in pairs])
    anchors = eng.mum_anchor_pairs_batch(table)                          # warm-up (sizes the context's block cache)
    for i in range(0, a.pairs, max(1, a.pairs // 8)):
        assert np.array_equal(anchors[i], M.oracle_mum_anchors(*pairs[i])), i
    walls, kern = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        eng.mum_anchor_pairs_batch(table)
        walls.append(time.perf_counter() - t0)
        kern.append(eng.mum_last_timing())
    res["device_call_ms"] = [round(k["wall_ms"], 2) for k in kern]
    res["device_kernel_ms"] = [round(k["kernel_ms"], 2) for k in kern]
    res["device_python_ms"] = [round(w * 1e3, 2) for w in walls]
    res["device_launches"] = kern[-1]["launches"]
    res["device_us_per_pair"] = round(min(k["wall_ms"] for k in kern) * 1e3 / a.pairs, 2)
    res["anchors_per_pair"] = float(np.mean([len(x) for x in anchors]))
    # the reference's host anchoring, one pair per thread over the usable cores (ctypes releases the GIL)
    if M.have_ref():
        # the reference is built with asserts on: skip the pairs where its closing assert fires (oracle/mum_oracle.c)
        samp = [q for q in pairs[: a.host_sample] if not M.oracle_mum_anchors(*q, with_abort=True)[1]]
        res["host_sample"] = len(samp)
        M.ref_mum_anchors(*samp[0])
        with ThreadPoolExecutor(res["cores"]) as ex:
            t0 = time.perf_counter()
            list(ex.map(lambda q: M.ref_mum_anchors(*q), samp))
            secs = time.perf_counter() - t0
        res["host_ref_us_per_pair"] = round(secs * 1e6 / len(samp), 2)
        t0 = time.perf_counter()
        for q in samp[:64]:
            M.ref_mum_anchors(*q)
        res["host_ref_one_core_ms_per_pair"] = round((time.perf_counter() - t0) * 1e3 / 64, 3)
        # align_pair_list: anchors + the pair-HMM batch
        ptab = eng.pecan_table([(x, y, an, False, False) for (x, y), an in zip(pairs, anchors)])
        eng._take_pairs(*eng.pecan_batch_raw(ptab), ptab.n)
        t0 = time.perf_counter()
        eng._take_pairs(*eng.pecan_batch_raw(ptab), ptab.n)
        hmm = time.perf_counter() - t0
        res["pair_hmm_batch_ms"] = round(hmm * 1e3, 2)
        res["align_pair_list_host_anchors_ms"] = round(hmm * 1e3 + res["host_ref_us_per_pair"] * a.pairs / 1e3, 2)
        res["align_pair_list_device_anchors_ms"] = round(hmm * 1e3 + min(k["wall_ms"] for k in kern), 2)
    eng.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
