"""Replay of a cPecan-mode recording (shim/cactus_pecan_harvest.c, read by workload.read_pecan_harvest) through the public C ABI
of libbarb200 (include/barb200.h): every recorded pair's anchors (barb200_pecan_anchor_pairs_batch for pairs with useMumAnchors,
the recorded anchors for the lastz path) and posteriors (barb200_pecan_aligned_pairs_batch), whole ends per call, each pair's
anchor and triple hash checked against the reference's. scripts/pecan_replay.py is the command line.

The library is any build exporting those entry points: the product's libbarb200.so (the default) or the test-only CPU stand-in
of tests/hosttest. Loading it is up to the caller; importing this module loads nothing."""
import ctypes as C
import time

import numpy as np

import workload


def _bind(lib):
    from cactus_b200.api import _CMumParams, _CParams, _CPecanParams
    vp, i64, ci = C.c_void_p, C.c_int64, C.c_int
    lib.barb200_params_default.argtypes = [C.POINTER(_CParams)]
    lib.barb200_params_default.restype = None
    lib.barb200_create.argtypes = [C.POINTER(_CParams), C.c_char_p, ci]
    lib.barb200_create.restype = vp
    lib.barb200_destroy.argtypes = [vp]
    lib.barb200_destroy.restype = None
    lib.barb200_last_error.argtypes = [vp]
    lib.barb200_last_error.restype = C.c_char_p
    lib.barb200_free.argtypes = [vp]
    lib.barb200_free.restype = None
    lib.barb200_pecan_aligned_pairs_batch.argtypes = [vp, C.POINTER(_CPecanParams), i64] + [vp] * 12
    lib.barb200_pecan_aligned_pairs_batch.restype = ci
    lib.barb200_pecan_anchor_pairs_batch.argtypes = [vp, C.POINTER(_CMumParams), i64] + [vp] * 6
    lib.barb200_pecan_anchor_pairs_batch.restype = ci
    # report-only entry points; a library without them (the CPU stand-in) replays all the same
    optional = {"barb200_mum_last_timing": ([vp], ci), "barb200_pecan_device_stats": ([vp, vp, vp, ci], ci),
                "barb200_pecan_split_points": ([i64, i64, vp, i64, i64, ci, ci, C.POINTER(vp)], i64)}
    have = set()
    for name, (args, res) in optional.items():
        if hasattr(lib, name):
            getattr(lib, name).argtypes, getattr(lib, name).restype = args, res
            have.add(name)
    return have


class Context:
    """One barb200 context of the library at `path`; all_devices: over every visible device (n_devices = -1), else the default
    single device."""

    def __init__(self, path, all_devices=False):
        from cactus_b200.api import _CParams
        self.lib = C.CDLL(path)
        self.have = _bind(self.lib)
        p = _CParams()
        self.lib.barb200_params_default(C.byref(p))
        if all_devices:
            p.n_devices = -1
        err = C.create_string_buffer(512)
        self.ctx = self.lib.barb200_create(C.byref(p), err, len(err))
        if not self.ctx:
            raise RuntimeError("barb200_create failed: %s" % err.value.decode(errors="replace"))

    def close(self):
        if self.ctx:
            self.lib.barb200_destroy(self.ctx)
            self.ctx = None

    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError("%s failed (%d): %s" % (what, rc, self.lib.barb200_last_error(self.ctx).decode(errors="replace")))

    def _take(self, ptr, n, width):
        a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(max(n * width, 1),))[: n * width].reshape(n, width).copy() \
            if n else np.zeros((0, width), np.int64)
        self.lib.barb200_free(ptr)
        return a

    def anchor_pairs(self, mum, pairs):
        """barb200_pecan_anchor_pairs_batch -> list of int64 [n, 2]"""
        from cactus_b200.api import _CMumParams
        n, m = len(pairs), max(len(pairs), 1)
        sx, sy = (C.c_char_p * m)(*[q["sx"] for q in pairs]), (C.c_char_p * m)(*[q["sy"] for q in pairs])
        lx, ly = np.array([len(q["sx"]) for q in pairs] or [0], np.int64), np.array([len(q["sy"]) for q in pairs] or [0], np.int64)
        out, n_out = (C.c_void_p * m)(), np.zeros(m, np.int64)
        mp = _CMumParams(mum["k"], mum["u"], mum["anchor_matrix_bigger_than_this"], mum["recursive_mums"])
        self._check(self.lib.barb200_pecan_anchor_pairs_batch(self.ctx, C.byref(mp), n, sx, lx.ctypes.data, sy, ly.ctypes.data, out,
                                                              n_out.ctypes.data), "barb200_pecan_anchor_pairs_batch")
        return [self._take(out[i], int(n_out[i]), 2) if out[i] else np.zeros((0, 2), np.int64) for i in range(n)]

    def aligned_pairs(self, pecan, pairs, anchors):
        """barb200_pecan_aligned_pairs_batch -> (list of int64 [n, 3] triples, banded cells per pair, seconds of the call)"""
        from cactus_b200.api import _CPecanParams
        n, m = len(pairs), max(len(pairs), 1)
        sx, sy = (C.c_char_p * m)(*[q["sx"] for q in pairs]), (C.c_char_p * m)(*[q["sy"] for q in pairs])
        lx, ly = np.array([len(q["sx"]) for q in pairs] or [0], np.int64), np.array([len(q["sy"]) for q in pairs] or [0], np.int64)
        anch = [np.ascontiguousarray(a, np.int64) for a in anchors]
        ap = (C.c_void_p * m)(*[a.ctypes.data if len(a) else None for a in anch])
        na = np.array([len(a) for a in anch] or [0], np.int64)
        rl = np.array([q["ragged_left"] for q in pairs] or [0], np.uint8)
        rr = np.array([q["ragged_right"] for q in pairs] or [0], np.uint8)
        trip, n_out, cells = (C.c_void_p * m)(), np.zeros(m, np.int64), np.zeros(m, np.int64)
        pp = _CPecanParams(pecan["threshold"], pecan["min_diags_between_traceback"], pecan["traceback_diagonals"],
                           pecan["diagonal_expansion"], pecan["split_matrix_bigger_than_this"], pecan["dynamic_anchor_expansion"])
        t0 = time.perf_counter()
        rc = self.lib.barb200_pecan_aligned_pairs_batch(self.ctx, C.byref(pp), n, sx, lx.ctypes.data, sy, ly.ctypes.data, ap,
                                                        na.ctypes.data, rl.ctypes.data, rr.ctypes.data, trip, n_out.ctypes.data, None,
                                                        cells.ctypes.data)
        secs = time.perf_counter() - t0
        self._check(rc, "barb200_pecan_aligned_pairs_batch")
        return [self._take(trip[i], int(n_out[i]), 3) for i in range(n)], cells[:n].copy(), secs

    def mum_last_timing(self):
        if "barb200_mum_last_timing" not in self.have:
            return None
        out = np.zeros(3, np.float64)
        return out if self.lib.barb200_mum_last_timing(out.ctypes.data) == 0 else None

    def device_stats(self):
        """(hmm_pairs, mum_pairs) per device of the context, or None"""
        if "barb200_pecan_device_stats" not in self.have:
            return None
        hmm, mum = np.zeros(64, np.int64), np.zeros(64, np.int64)
        n = self.lib.barb200_pecan_device_stats(self.ctx, hmm.ctypes.data, mum.ctypes.data, 64)
        return (hmm[:n].copy(), mum[:n].copy()) if n > 0 else None

    def sub_jobs(self, q, anchors):
        """sub-matrices the pair is split into (barb200_pecan_split_points), or None"""
        if "barb200_pecan_split_points" not in self.have:
            return None
        a = np.ascontiguousarray(anchors, np.int64)
        out = C.c_void_p()
        n = self.lib.barb200_pecan_split_points(len(q["sx"]), len(q["sy"]), a.ctypes.data if len(a) else None, len(a),
                                                q["pecan"]["split_matrix_bigger_than_this"], int(q["ragged_left"]), int(q["ragged_right"]),
                                                C.byref(out))
        if out.value:
            self.lib.barb200_free(out)
        return int(n) if n >= 0 else None


def needs_anchor_call(q):
    """a pair the MUM-anchor batch searches (getAnchorPairsForPairwiseAlignmentParameters: lX * lY > anchorMatrixBiggerThanThis)"""
    return q["use_mum_anchors"] and len(q["sx"]) * len(q["sy"]) > q["mum"]["anchor_matrix_bigger_than_this"]


def _key(q):
    return tuple(sorted(q["pecan"].items())), tuple(sorted(q["mum"].items()))


def replay(ctx, ends, ends_per_batch=1):
    """Run the ends through `ctx`, `ends_per_batch` whole ends per call (0: every end in one call); pairs of one call that were
    recorded with different parameters go to separate calls. Returns a dict: "mismatches" (list of (end, index, what) for every
    pair whose anchor hash, triple count or triple hash differs from the recording), "pairs", "calls", "cells", "hmm_s"
    (seconds inside barb200_pecan_aligned_pairs_batch), "anchor_device_ms" / "anchor_call_ms" (barb200_mum_last_timing, summed
    over the anchor calls; None without it), "anchor_calls", and per pair in the order replayed "n_anchors", "pair_cells",
    "sub_jobs" (None where the library has no barb200_pecan_split_points)."""
    step = len(ends) if ends_per_batch <= 0 else ends_per_batch
    res = {"mismatches": [], "pairs": 0, "calls": 0, "cells": 0, "hmm_s": 0.0, "anchor_device_ms": 0.0, "anchor_call_ms": 0.0,
           "anchor_calls": 0, "n_anchors": [], "pair_cells": [], "sub_jobs": []}
    for b in range(0, len(ends), max(step, 1)):
        pairs = [q for e in ends[b:b + step] for q in e["pairs"]]
        groups = {}
        for q in pairs:
            groups.setdefault(_key(q), []).append(q)
        for group in groups.values():
            mum = [q for q in group if q["use_mum_anchors"]]
            got = {}
            # as the pecan shim: no anchor call when no pair of the round is larger than anchorMatrixBiggerThanThis
            if any(needs_anchor_call(q) for q in mum):
                for q, a in zip(mum, ctx.anchor_pairs(mum[0]["mum"], mum)):
                    got[id(q)] = a
                res["anchor_calls"] += 1
                t = ctx.mum_last_timing()
                if t is None:
                    res["anchor_device_ms"] = res["anchor_call_ms"] = None
                elif res["anchor_device_ms"] is not None:
                    res["anchor_device_ms"] += float(t[0])
                    res["anchor_call_ms"] += float(t[1])
            anchors = [got.get(id(q), np.zeros((0, 2), np.int64)) if q["use_mum_anchors"] else q["anchors"] for q in group]
            trips, cells, secs = ctx.aligned_pairs(group[0]["pecan"], group, anchors)
            res["calls"] += 1
            res["hmm_s"] += secs
            res["cells"] += int(cells.sum())
            for q, a, t, c in zip(group, anchors, trips, cells):
                if workload.fnv1a64(a) != q["anchor_hash"]:
                    res["mismatches"].append((q["end"], q["index"], "anchors"))
                if len(t) != q["n_triples"] or workload.fnv1a64(t) != q["triple_hash"]:
                    res["mismatches"].append((q["end"], q["index"], "triples"))
                res["n_anchors"].append(len(a))
                res["pair_cells"].append(int(c))
                res["sub_jobs"].append(ctx.sub_jobs(q, a))
        res["pairs"] += len(pairs)
    return res


def histogram(values):
    """power-of-two buckets: list of (lo, hi, count) with lo <= v < hi (the first bucket is [0, 1))"""
    v = np.asarray([x for x in values if x is not None], np.int64)
    if len(v) == 0:
        return []
    top = int(v.max()).bit_length()
    edges = [0] + [1 << k for k in range(top + 1)]
    counts = np.histogram(v, bins=edges)[0]
    return [(edges[i], edges[i + 1], int(c)) for i, c in enumerate(counts) if c]
