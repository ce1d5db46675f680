#!/usr/bin/env python
"""Freeze the window-by-window traces of the UNMODIFIED reference's BAR window chain (oracle/_ref/libbar_trace_ref.so, built from the
reference sources by oracle/end_trace.mk) into tests/golden/end_trace_golden.npz: for every seeded end set of tests/_end_trace_cases.py
(and for the top-level alignment calls a reference bar() makes on the flowers behind tests/golden/flower_golden.npz) the SHA-256 of
each end's words in barb200_trace_ends' layout (include/barb200.h). tests/test_gpu_end_trace.py compares the device's words with them.
Run where the reference sources are (they do not travel to the GPU machine; the fixture does)."""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _end_trace_cases as X  # noqa: E402
import _endtrace as T  # noqa: E402
import _reflib as R  # noqa: E402


def main():
    T.build()
    if not T.have_ref():
        sys.exit("oracle/_ref/libbar_trace_ref.so is not built: the reference sources are needed")
    with tempfile.TemporaryDirectory() as tmp:
        cases = list(X.cases()) + list(X.gpu_cases()) + list(X.repeat_cases()) + X.flower_cases(tmp)
    out = {}
    for c in cases:
        words = T.ref_trace_ends(*X.args(c), p=R.cactus_params(**c["poa"]))
        assert all(np.array_equal(a, b) for a, b in zip(words, T.oracle_trace_ends(*X.args(c), p=R.cactus_params(**c["poa"])))), c["name"]
        out[c["name"]] = [X.digest(w) for w in words]
    np.savez_compressed(X.GOLDEN, digests=np.frombuffer(json.dumps(out, sort_keys=True).encode(), np.uint8))
    print("%s: %d cases, %d ends" % (X.GOLDEN, len(out), sum(len(v) for v in out.values())))


if __name__ == "__main__":
    main()
