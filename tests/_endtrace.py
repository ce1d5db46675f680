"""ctypes readers for barb200_trace_ends and its checkers (test infrastructure only):

* ``tests/hosttest/_build/libbarb200_trace_standin.so`` -- the product's host code (host_end_trace.cpp, bar_windows.h) over the CPU
  stand-in device, whose trace jobs are computed by the host build of the product's graph code
* ``oracle/_build/libend_trace_oracle.so`` -- oracle_trace_ends, the restated window chain (oracle/end_trace_oracle.c)
* ``oracle/_ref/libbar_trace_ref.so`` -- the unmodified reference window chain, observed through -Wl,--wrap
  (oracle/end_trace_ref_harness.c)

All three emit the word layout of include/barb200.h; :func:`read_end_trace` is the checkers' own reader of it."""
import ctypes as C
import os
import subprocess

import numpy as np

import _reflib as R

ROOT = R.ROOT
STANDIN_SO = os.path.join(ROOT, "tests", "hosttest", "_build", "libbarb200_trace_standin.so")
ORACLE_SO = os.path.join(ROOT, "oracle", "_build", "libend_trace_oracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libbar_trace_ref.so")


def have_ref():
    return os.path.exists(REF_SO)


def build():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "hosttest"), "-f", "end_trace.mk", "end_trace"])
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "end_trace.mk", "end_trace"])


def read_end_trace(w):
    """the checkers' reader of one end's words: dict(seq_no, windows=[dict(index, offsets, lens, empty, progressive, trace,
    trace_words, trimmed_lens, column_no)], msa, n_words)"""
    w = np.asarray(w, np.int64)
    K, n = int(w[0]), int(w[1])
    o, wins = 2, []
    for _ in range(n):
        d = dict(index=int(w[o]))
        o += 1
        for f in ("offsets", "lens", "empty"):
            d[f] = w[o:o + K].copy()
            o += K
        d["progressive"] = int(w[o])
        nt = int(w[o + 1])
        o += 2
        d["trace_words"] = w[o:o + nt].copy()
        d["trace"] = R._parse_trace(d["trace_words"], K)
        o += nt
        d["trimmed_lens"] = w[o:o + K].copy()
        d["column_no"] = int(w[o + K])
        o += K + 1
        wins.append(d)
    assert int(w[o]) == K
    cols = int(w[o + 1])
    o += 2
    nwm = (K * cols + 7) // 8
    assert len(w) == o + nwm, (len(w), o + nwm)
    msa = w[o:].view(np.uint8)[: K * cols].reshape(K, cols).copy()
    return dict(seq_no=K, windows=wins, msa=msa, n_words=len(w))


class _Args:
    """char*** / int** / int64** of a list of ends (lists of byte strings) and of the index tables; keeps the buffers alive"""

    def __init__(self, ends, ri=None, rr=None, ov=None):
        n = len(ends)
        self.keep = []
        self.n = n
        self.end_lengths = (C.c_int64 * max(n, 1))(*[len(e) for e in ends])
        self.strs, self.lens = (C.c_void_p * max(n, 1))(), (C.c_void_p * max(n, 1))()
        for i, e in enumerate(ends):
            bs = [s if isinstance(s, bytes) else bytes(s) for s in e]
            arr = (C.c_char_p * max(len(bs), 1))(*bs)
            ln = (C.c_int * max(len(bs), 1))(*[len(b) for b in bs])
            self.keep += [bs, arr, ln]
            self.strs[i], self.lens[i] = C.cast(arr, C.c_void_p), C.cast(ln, C.c_void_p)
        self.ri, self.rr, self.ov = (self._table(t) for t in (ri, rr, ov))

    def _table(self, rows):
        if rows is None:
            return None
        arr = (C.c_void_p * max(self.n, 1))()
        for i, r in enumerate(rows):
            a = (C.c_int64 * max(len(r), 1))(*[int(v) for v in r])
            self.keep.append(a)
            arr[i] = C.cast(a, C.c_void_p)
        return arr


def _take(lib_free, outs, nw, n):
    res = []
    for i in range(n):
        w = np.ctypeslib.as_array(C.cast(outs[i], C.POINTER(C.c_int64)), shape=(int(nw[i]),)).copy()
        lib_free(outs[i])
        res.append(w)
    return res


def _checker(path, fname, ends, ri, rr, ov, window_size, max_prog_rows, max_prog_length_diff, p):
    lib = R._load(path)
    f = getattr(lib, fname)
    f.restype = C.c_int
    f.argtypes = [C.POINTER(R.RefParams), C.c_int64] + [C.c_void_p] * 6 + [C.c_int64, C.c_int64, C.c_double, C.c_void_p, C.c_void_p]
    a = _Args(ends, ri, rr, ov)
    outs = (C.c_void_p * max(a.n, 1))()
    nw = np.zeros(max(a.n, 1), np.int64)
    rc = f(C.byref(p or R.cactus_params()), a.n, a.end_lengths, a.strs, a.lens, a.ri, a.rr, a.ov, window_size, max_prog_rows,
           max_prog_length_diff, outs, nw.ctypes.data)
    assert rc == 0, "%s failed: %d" % (fname, rc)
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    return _take(libc.free, outs, nw, a.n)


def oracle_trace_ends(ends, ri=None, rr=None, ov=None, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0, p=None):
    """the restated chain's words per end"""
    return _checker(ORACLE_SO, "oracle_trace_ends", ends, ri, rr, ov, window_size, max_prog_rows, max_prog_length_diff, p)


def ref_trace_ends(ends, ri=None, rr=None, ov=None, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0, p=None):
    """the unmodified reference chain's words per end (observed through the wraps)"""
    return _checker(REF_SO, "bar_trace_ref_ends", ends, ri, rr, ov, window_size, max_prog_rows, max_prog_length_diff, p)


def wrapped_ref_consistent(ends, ri, rr, ov, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0, p=None):
    """make_consistent_partial_order_alignments of the WRAPPED reference library (libbar_trace_ref.so), outside any recording"""
    saved = R.BAR_REF_SO
    try:
        R.BAR_REF_SO = REF_SO
        return R._consistent("ref", ends, ri, rr, ov, window_size, max_prog_rows, max_prog_length_diff, p)
    finally:
        R.BAR_REF_SO = saved


# ---- the product's host code over the CPU stand-in device ---------------------------------------------------------------------
def _standin():
    from cactus_b200.api import _CParams as P, _CMsa
    lib = R._load(STANDIN_SO)
    vp, i64 = C.c_void_p, C.c_int64
    lib.barb200_params_default.argtypes = [C.POINTER(P)]
    lib.barb200_create.argtypes = [C.POINTER(P), C.c_char_p, C.c_int]
    lib.barb200_create.restype = vp
    lib.barb200_destroy.argtypes = [vp]
    lib.barb200_last_error.argtypes = [vp]
    lib.barb200_last_error.restype = C.c_char_p
    lib.barb200_trace_ends.argtypes = [vp, i64] + [vp] * 6 + [i64, i64, C.c_double, vp, vp]
    lib.barb200_trace_ends.restype = C.c_int
    lib.barb200_make_consistent_partial_order_alignments.argtypes = [vp, i64] + [vp] * 6 + [i64, i64, C.c_double]
    lib.barb200_make_consistent_partial_order_alignments.restype = C.POINTER(C.POINTER(_CMsa))
    lib.barb200_msa_make_partial_order_alignment_batch.argtypes = [vp, i64, vp, vp, vp, i64, i64, C.c_double, vp]
    lib.barb200_msa_make_partial_order_alignment_batch.restype = C.c_int
    lib.barb200_msa_destruct.argtypes = [vp]
    lib.barb200_free.argtypes = [vp]
    return lib, P, _CMsa


class Standin:
    """a stand-in context with the POA parameters of a RefParams"""

    def __init__(self, p=None):
        self.lib, P, self._CMsa = _standin()
        p = p or R.cactus_params()
        c = P()
        self.lib.barb200_params_default(C.byref(c))
        c.wb, c.wf = p.wb, p.wf
        c.gap_open1, c.gap_ext1, c.gap_open2, c.gap_ext2 = p.gap_open1, p.gap_ext1, p.gap_open2, p.gap_ext2
        for i in range(25):
            c.mat[i] = p.mat[i]
        c.k, c.w, c.min_w, c.progressive_poa = p.k, p.w, p.min_w, p.progressive_poa
        err = C.create_string_buffer(256)
        self.ctx = self.lib.barb200_create(C.byref(c), err, 256)
        assert self.ctx, err.value

    def close(self):
        if self.ctx:
            self.lib.barb200_destroy(self.ctx)
            self.ctx = None

    def error(self):
        return self.lib.barb200_last_error(self.ctx).decode()

    def trace_ends_raw(self, ends, ri=None, rr=None, ov=None, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """(rc, [words per end] or the raw output pointers when rc != 0)"""
        a = _Args(ends, ri, rr, ov)
        outs = (C.c_void_p * max(a.n, 1))()
        nw = np.zeros(max(a.n, 1), np.int64)
        rc = self.lib.barb200_trace_ends(self.ctx, a.n, a.end_lengths, a.strs, a.lens, a.ri, a.rr, a.ov, window_size, max_prog_rows,
                                         max_prog_length_diff, outs, nw.ctypes.data)
        if rc:
            return rc, [(outs[i], int(nw[i])) for i in range(a.n)]
        return 0, _take(self.lib.barb200_free, outs, nw, a.n)

    def trace_ends(self, *args, **kw):
        rc, w = self.trace_ends_raw(*args, **kw)
        assert rc == 0, "barb200_trace_ends: %d %s" % (rc, self.error())
        return w

    def consistent(self, ends, ri, rr, ov, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """barb200_make_consistent_partial_order_alignments (the end queue) on the same context"""
        a = _Args(ends, ri, rr, ov)
        ms = self.lib.barb200_make_consistent_partial_order_alignments(self.ctx, a.n, a.end_lengths, a.strs, a.lens, a.ri, a.rr, a.ov,
                                                                      window_size, max_prog_rows, max_prog_length_diff)
        assert ms, self.error()
        out = []
        for i in range(a.n):
            m = ms[i].contents
            k, c = int(m.seq_no), int(m.column_no)
            out.append(np.ctypeslib.as_array(m.msa, shape=(max(k * c, 1),))[: k * c].reshape(k, c).copy())
            self.lib.barb200_msa_destruct(ms[i])
        self.lib.barb200_free(C.cast(ms, C.c_void_p))
        return out

    def independent(self, ends, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """barb200_msa_make_partial_order_alignment_batch (the end queue, no cross-end trim)"""
        a = _Args(ends)
        out = (C.c_void_p * max(a.n, 1))()
        rc = self.lib.barb200_msa_make_partial_order_alignment_batch(self.ctx, a.n, a.end_lengths, a.strs, a.lens, window_size,
                                                                    max_prog_rows, max_prog_length_diff, out)
        assert rc == 0, self.error()
        res = []
        for i in range(a.n):
            m = C.cast(out[i], C.POINTER(self._CMsa)).contents
            k, c = int(m.seq_no), int(m.column_no)
            res.append(np.ctypeslib.as_array(m.msa, shape=(max(k * c, 1),))[: k * c].reshape(k, c).copy())
            self.lib.barb200_msa_destruct(out[i])
        return res


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def flower_params(params):
    """the POA fields of a flower golden's BAR configuration as RefParams"""
    kw = {}
    if "bar/poa/partialOrderAlignmentBandConstant" in params:
        kw["wb"] = int(params["bar/poa/partialOrderAlignmentBandConstant"])
    if "bar/poa/partialOrderAlignmentBandFraction" in params:
        kw["wf"] = float(params["bar/poa/partialOrderAlignmentBandFraction"])
    return R.cactus_params(**kw)


def harvest_flower(fl, params, path):
    """the top-level make_consistent_partial_order_alignments / msa_make_partial_order_alignment calls a reference bar() makes on
    one flower (recorded by shim/cactus_bar_harvest.c into `path`)"""
    import workload
    import _flowers as F
    os.environ["BARB200_HARVEST"] = path
    try:
        F.bar("harvest", [fl], params)
    finally:
        del os.environ["BARB200_HARVEST"]
    return workload.read_harvest(path)
