#!/usr/bin/env python
"""Development aid: time barb200_poa_msa_batch (host buffers) on the bench shape (argument: number of ends)."""
import os, sys, time
import numpy as np
import ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cactus_b200 as cb
import workload  # noqa: E402
n = int(sys.argv[1]) if len(sys.argv) > 1 else 2368
eng = cb.Engine()
n_seq, lens, flat = workload.synth_ends(0, n, 8, 2000)
def once():
    outs = (C.c_void_p * n)(); ml = np.zeros(n, np.int32); cc = np.zeros(n, np.int64)
    eng._check(eng.lib.barb200_poa_msa_batch(eng.ctx, n, n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data, None, outs, ml.ctypes.data, cc.ctypes.data))
    for i in range(n): eng.lib.barb200_free(outs[i])
    return int(cc.sum())
for it in range(3):
    t = time.time(); cells = once(); dt = time.time() - t
    print("e2e iter", it, "%.1f ms" % (dt * 1e3), "%.1f Gcell/s" % (cells / dt / 1e9), flush=True)
