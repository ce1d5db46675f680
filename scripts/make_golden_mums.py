"""Record the compiled reference's MUM anchors (getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1, through
oracle/_ref/libmum_ref.so) on a fixed input set into tests/golden/mum_golden.npz: the inputs, their parameters and the anchors.

    python scripts/make_golden_mums.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _mumlib as M  # noqa: E402
import _reflib as R  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mum_golden.npz")


def main():
    assert M.have_ref(), "oracle/_ref/libmum_ref.so is needed (oracle/Makefile with the reference sources)"
    rng = np.random.default_rng(20261016)
    names, seqs, lens, params, anchors, counts = [], [], [], [], [], []
    for name, sx, sy, kw in M.case_set(rng):
        p = dict(k=50, u=1, bigger=500 * 500, recursive=1)
        p.update(kw)
        _, would_abort = M.oracle_mum_anchors(sx, sy, with_abort=True, **p)
        if would_abort:                                  # the assert-enabled reference aborts on these (see oracle/mum_oracle.c)
            continue
        a = M.ref_mum_anchors(sx, sy, **p)
        names.append(name)
        seqs += [sx, sy]
        lens += [len(sx), len(sy)]
        params.append([p["k"], p["u"], p["bigger"], p["recursive"]])
        anchors.append(a.astype(np.int32))
        counts.append(len(a))
    np.savez_compressed(OUT, names=np.array(names), seqs=np.frombuffer(b"".join(seqs), np.uint8), lens=np.array(lens, np.int64),
                        params=np.array(params, np.int64), anchors=np.concatenate(anchors).reshape(-1, 2),
                        counts=np.array(counts, np.int64))
    print("%s: %d cases, %d anchors, %d bytes" % (OUT, len(names), sum(counts), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
