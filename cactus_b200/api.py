"""ctypes binding of include/barb200.h plus a thin object layer named after the reference's interface.

Reference names mirrored (bar/inc/poaBarAligner.h):
  Msa                                          -> :class:`Msa`
  abpoaParamaters_constructFromCactusParams    -> :class:`PoaParams` (the <bar><poa> XML attributes as keywords)
  msa_make_partial_order_alignment             -> :meth:`Engine.msa_make_partial_order_alignment` (+ ``_batch``)
  make_consistent_partial_order_alignments     -> :meth:`Engine.make_consistent_partial_order_alignments`
  msa_to_base / msa_to_byte                    -> module functions
and one level below, abPOA's abpoa_msa (submodules/abPOA/include/abpoa.h:160) -> :meth:`Engine.poa_msa_batch`.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

CACTUS_SUBMAT = [91, -114, -61, -123, -100, -114, 100, -125, -61, -100, -61, -125, 100, -114, -100,
                 -123, -61, -114, 91, -100, -100, -100, -100, -100, 100]


class BarB200Error(RuntimeError):
    pass


def library_path():
    # BARB200_LIB: development aid (A/B runs of differently tuned builds); the product loads the in-tree library
    return os.environ.get("BARB200_LIB") or os.path.join(_HERE, "libbarb200.so")


class _CParams(C.Structure):
    _fields_ = [("mat", C.c_int * 25), ("gap_open1", C.c_int), ("gap_ext1", C.c_int), ("gap_open2", C.c_int),
                ("gap_ext2", C.c_int), ("wb", C.c_int), ("wf", C.c_float), ("k", C.c_int), ("w", C.c_int),
                ("min_w", C.c_int), ("progressive_poa", C.c_int), ("disable_seeding", C.c_int), ("device", C.c_int),
                ("threads_per_block", C.c_int), ("ctas_per_sm", C.c_int), ("mem_fraction", C.c_double),
                ("host_threads", C.c_int), ("collect_phase_clocks", C.c_int), ("n_devices", C.c_int), ("devices", C.c_int * 8),
                ("lanes", C.c_int)]


class _CPecanParams(C.Structure):
    _fields_ = [("threshold", C.c_double), ("min_diags_between_traceback", C.c_int64), ("traceback_diagonals", C.c_int64),
                ("diagonal_expansion", C.c_int64), ("split_matrix_bigger_than_this", C.c_int64),
                ("dynamic_anchor_expansion", C.c_int)]


class _CMumParams(C.Structure):
    _fields_ = [("k", C.c_int64), ("u", C.c_int64), ("anchor_matrix_bigger_than_this", C.c_int64), ("recursive_mums", C.c_int)]


class _CMsa(C.Structure):
    _fields_ = [("seq_no", C.c_int64), ("column_no", C.c_int64), ("seq_lens", C.POINTER(C.c_int)),
                ("msa", C.POINTER(C.c_uint8))]


def load_library():
    """dlopen libbarb200.so (built in-tree by ``python -m cactus_b200.build``). Fails loudly if it is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise BarB200Error("libbarb200.so is not built (%s); run `python -m cactus_b200.build`. "
                           "There is no CPU fallback." % path)
    lib = C.CDLL(path)
    vp, i64, ci = C.c_void_p, C.c_int64, C.c_int
    lib.barb200_params_default.argtypes = [C.POINTER(_CParams)]
    lib.barb200_params_default.restype = None
    lib.barb200_create.argtypes = [C.POINTER(_CParams), C.c_char_p, ci]
    lib.barb200_create.restype = vp
    lib.barb200_destroy.argtypes = [vp]
    lib.barb200_destroy.restype = None
    lib.barb200_last_error.argtypes = [vp]
    lib.barb200_last_error.restype = C.c_char_p
    lib.barb200_poa_msa_batch.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, vp]
    lib.barb200_poa_msa_batch.restype = ci
    lib.barb200_poa_trace_batch.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp]
    lib.barb200_poa_trace_batch.restype = ci
    lib.barb200_trace_ends.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, i64, i64, C.c_double, vp, vp]
    lib.barb200_trace_ends.restype = ci
    lib.barb200_stage_create.argtypes = [vp, i64, vp, vp, vp, vp, C.POINTER(vp)]
    lib.barb200_stage_create.restype = ci
    lib.barb200_stage_run.argtypes = [vp, C.POINTER(C.c_float)]
    lib.barb200_stage_run.restype = ci
    lib.barb200_stage_fetch.argtypes = [vp, vp, vp, vp]
    lib.barb200_stage_fetch.restype = ci
    lib.barb200_stage_launches.argtypes = [vp]
    lib.barb200_stage_launches.restype = i64
    lib.barb200_stage_phase_clocks.argtypes = [vp, vp]
    lib.barb200_stage_phase_clocks.restype = ci
    lib.barb200_stage_destroy.argtypes = [vp]
    lib.barb200_stage_destroy.restype = None
    lib.barb200_msa_destruct.argtypes = [vp]
    lib.barb200_msa_destruct.restype = None
    lib.barb200_msa_make_partial_order_alignment_batch.argtypes = [vp, i64, vp, vp, vp, i64, i64, C.c_double, vp]
    lib.barb200_msa_make_partial_order_alignment_batch.restype = ci
    lib.barb200_msa_make_partial_order_alignment.argtypes = [vp, vp, vp, i64, i64, i64, C.c_double]
    lib.barb200_msa_make_partial_order_alignment.restype = C.POINTER(_CMsa)
    lib.barb200_make_consistent_partial_order_alignments.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, i64, i64, C.c_double]
    lib.barb200_make_consistent_partial_order_alignments.restype = C.POINTER(C.POINTER(_CMsa))
    lib.barb200_stage_buckets.argtypes = [vp, vp, ci]
    lib.barb200_stage_buckets.restype = ci
    lib.barb200_flower_submit.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, i64, i64, C.c_double]
    lib.barb200_flower_submit.restype = vp
    lib.barb200_flower_wait.argtypes = [vp, vp]
    lib.barb200_flower_wait.restype = C.POINTER(C.POINTER(_CMsa))
    lib.barb200_queue_stats.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    lib.barb200_queue_stats.restype = ci
    lib.barb200_last_batch_timing.argtypes = [vp, vp]
    lib.barb200_last_batch_timing.restype = ci
    lib.barb200_device_count.argtypes = [vp]
    lib.barb200_device_count.restype = ci
    lib.barb200_device_info.argtypes = [vp, C.POINTER(ci), C.POINTER(i64), C.POINTER(i64), C.c_char_p, ci]
    lib.barb200_device_info.restype = ci
    lib.barb200_free.argtypes = [vp]
    lib.barb200_free.restype = None
    lib.barb200_free_many.argtypes = [vp, C.c_int64]
    lib.barb200_free_many.restype = None
    lib.barb200_pack_rows.argtypes = [vp, vp, C.c_int64, vp]
    lib.barb200_pack_rows.restype = None
    pp = C.POINTER(_CPecanParams)
    lib.barb200_pecan_params_default.argtypes = [pp]
    lib.barb200_pecan_params_default.restype = None
    lib.barb200_pecan_aligned_pairs_batch.argtypes = [vp, pp, i64] + [vp] * 12
    lib.barb200_pecan_aligned_pairs_batch.restype = ci
    lib.barb200_pecan_stage_create.argtypes = [vp, pp, i64] + [vp] * 8 + [C.POINTER(vp)]
    lib.barb200_pecan_stage_create.restype = ci
    lib.barb200_pecan_stage_run.argtypes = [vp, C.POINTER(C.c_float)]
    lib.barb200_pecan_stage_run.restype = ci
    lib.barb200_pecan_stage_fetch.argtypes = [vp, vp, vp, vp, vp]
    lib.barb200_pecan_stage_fetch.restype = ci
    lib.barb200_pecan_stage_cells.argtypes = [vp]
    lib.barb200_pecan_stage_cells.restype = i64
    lib.barb200_pecan_stage_launches.argtypes = [vp]
    lib.barb200_pecan_stage_launches.restype = i64
    lib.barb200_pecan_stage_destroy.argtypes = [vp]
    lib.barb200_pecan_stage_destroy.restype = None
    lib.barb200_pecan_band.argtypes = [i64, i64, vp, i64, i64, vp, vp]
    lib.barb200_pecan_band.restype = ci
    lib.barb200_pecan_split_points.argtypes = [i64, i64, vp, i64, i64, ci, ci, C.POINTER(vp)]
    lib.barb200_pecan_split_points.restype = i64
    mp = C.POINTER(_CMumParams)
    lib.barb200_mum_params_default.argtypes = [mp]
    lib.barb200_mum_params_default.restype = None
    lib.barb200_pecan_anchor_pairs_batch.argtypes = [vp, mp, i64, vp, vp, vp, vp, vp, vp]
    lib.barb200_pecan_anchor_pairs_batch.restype = ci
    lib.barb200_mum_last_timing.argtypes = [vp]
    lib.barb200_mum_last_timing.restype = ci
    lib.barb200_pecan_device_stats.argtypes = [vp, vp, vp, ci]
    lib.barb200_pecan_device_stats.restype = ci
    _LIB = lib
    return lib


_BASES = "ACGTN-"


def msa_to_base(n):
    """bar/impl/poaBarAligner.c:155-157 restricted to the codes the engine emits"""
    return _BASES[n] if 0 <= n < 6 else "N"


def msa_to_byte(c):
    """bar/impl/poaBarAligner.c:159-161"""
    return {"A": 0, "a": 0, "C": 1, "c": 1, "G": 2, "g": 2, "T": 3, "t": 3, "-": 5}.get(c, 4)


def parse_trace(words, n_seq):
    """One job's trace words (barb200_poa_trace_batch, layout in include/barb200.h) as a dict: msa (uint8 [n_seq, msa_len]), msa_len,
    cells, read_id_map, alns = one dict per alignment in read order with read_id, qlen, node_n, best_score, cigar (uint64),
    dp_beg and dp_end (int32 per row). abPOA's per-alignment state has the same layout, so a reference dump parses alike."""
    w = np.asarray(words, np.int64)
    if int(w[0]) != n_seq:
        raise ValueError("trace of %d sequences, expected %d" % (int(w[0]), n_seq))
    msa_len, cells = int(w[1]), int(w[2])
    pos = 3
    read_id_map = [int(x) for x in w[pos:pos + n_seq]]
    pos += n_seq
    alns = []
    for _ in range(n_seq):
        read_id, qlen, node_n, n_cigar, best, n_rows = (int(x) for x in w[pos:pos + 6])
        pos += 6
        cigar = w[pos:pos + n_cigar].astype(np.uint64, copy=True)
        pos += n_cigar
        dp_beg = w[pos:pos + n_rows].astype(np.int32)
        pos += n_rows
        dp_end = w[pos:pos + n_rows].astype(np.int32)
        pos += n_rows
        alns.append(dict(read_id=read_id, qlen=qlen, node_n=node_n, best_score=best, cigar=cigar, dp_beg=dp_beg, dp_end=dp_end))
    msa = w[pos:].view(np.uint8)[: n_seq * msa_len].reshape(n_seq, msa_len).copy()
    return dict(msa=msa, msa_len=msa_len, cells=cells, read_id_map=read_id_map, alns=alns)


def first_trace_difference(got, want):
    """Where two traces of one job (dicts of :func:`parse_trace`) first differ: None, or (alignment, field, index). alignment is None
    for the job's own fields (read order, MSA length, cells, MSA); index is the first differing entry of a cigar or band array, a
    "length a vs b" note when their lengths differ, and None for scalar fields."""
    for k in ("read_id_map", "msa_len", "cells"):
        if got[k] != want[k]:
            return (None, k, None)
    if got["msa"].shape != want["msa"].shape or not np.array_equal(got["msa"], want["msa"]):
        return (None, "msa", None)
    for a, (x, y) in enumerate(zip(got["alns"], want["alns"])):
        for k in ("read_id", "qlen", "node_n", "best_score"):
            if x[k] != y[k]:
                return (a, k, None)
        for k in ("cigar", "dp_beg", "dp_end"):
            if len(x[k]) != len(y[k]):
                return (a, k, "length %d vs %d" % (len(x[k]), len(y[k])))
            bad = np.flatnonzero(np.asarray(x[k]) != np.asarray(y[k]))
            if len(bad):
                return (a, k, int(bad[0]))
    if len(got["alns"]) != len(want["alns"]):
        return (None, "alns", None)
    return None


def parse_end_trace(words):
    """One end's trace words (barb200_trace_ends, layout in include/barb200.h) as a dict: seq_no, windows = one dict per window in
    chain order (index, offsets, lens, empty (int64 per row), progressive, trace = the window's job as :func:`parse_trace` gives
    it, trimmed_lens, column_no) and msa = the end's final MSA (uint8 [seq_no, column_no])."""
    w = np.asarray(words, np.int64)
    K, n_win = int(w[0]), int(w[1])
    pos = 2
    windows = []
    for _ in range(n_win):
        index = int(w[pos])
        pos += 1
        offsets, lens, empty = (w[pos + i * K:pos + (i + 1) * K].copy() for i in range(3))
        pos += 3 * K
        progressive, n_trace = int(w[pos]), int(w[pos + 1])
        pos += 2
        trace = parse_trace(w[pos:pos + n_trace], K)
        pos += n_trace
        trimmed = w[pos:pos + K].copy()
        column_no = int(w[pos + K])
        pos += K + 1
        windows.append(dict(index=index, offsets=offsets, lens=lens, empty=empty, progressive=progressive, trace=trace,
                            trimmed_lens=trimmed, column_no=column_no))
    if int(w[pos]) != K:
        raise ValueError("end trace: MSA of %d rows, expected %d" % (int(w[pos]), K))
    cols = int(w[pos + 1])
    pos += 2
    msa = w[pos:].view(np.uint8)[: K * cols].reshape(K, cols).copy()
    if len(w) != pos + (K * cols + 7) // 8:
        raise ValueError("end trace: %d words, layout gives %d" % (len(w), pos + (K * cols + 7) // 8))
    return dict(seq_no=K, windows=windows, msa=msa)


def first_end_trace_difference(got, want):
    """Where two traces of one end (dicts of :func:`parse_end_trace`) first differ: None, or (window, field, index).
    Windows are compared in chain order, each by its input (offsets, lens, empty: index = the first differing row; progressive) and
    then its job's trace (field "trace", index = the (alignment, field, index) of :func:`first_trace_difference`). A window's
    trimmed_lens and column_no are compared only after every window's input and trace, since trimming window n also depends on
    window n+1. Then the window count ("n_windows"), and last the end's final MSA ("msa", window None)."""
    if got["seq_no"] != want["seq_no"]:
        return (None, "seq_no", None)
    gw, ww = got["windows"], want["windows"]
    for k, (x, y) in enumerate(zip(gw, ww)):
        for f in ("offsets", "lens", "empty"):
            bad = np.flatnonzero(np.asarray(x[f]) != np.asarray(y[f]))
            if len(bad):
                return (k, f, int(bad[0]))
        if x["progressive"] != y["progressive"]:
            return (k, "progressive", None)
        d = first_trace_difference(x["trace"], y["trace"])
        if d is not None:
            return (k, "trace", d)
    if len(gw) != len(ww):
        return (min(len(gw), len(ww)), "n_windows", "count %d vs %d" % (len(gw), len(ww)))
    for k, (x, y) in enumerate(zip(gw, ww)):
        bad = np.flatnonzero(np.asarray(x["trimmed_lens"]) != np.asarray(y["trimmed_lens"]))
        if len(bad):
            return (k, "trimmed_lens", int(bad[0]))
        if x["column_no"] != y["column_no"]:
            return (k, "column_no", None)
    if got["msa"].shape != want["msa"].shape or not np.array_equal(got["msa"], want["msa"]):
        return (None, "msa", None)
    return None


class PoaParams:
    """The <bar><poa> attributes abpoaParamaters_constructFromCactusParams reads (bar/impl/poaBarAligner.c:24-81),
    defaults from src/cactus/cactus_progressive_config.xml:307-325, plus engine knobs."""

    def __init__(self, partialOrderAlignmentBandConstant=1000, partialOrderAlignmentBandFraction=0.1,
                 partialOrderAlignmentGapOpenPenalty1=400, partialOrderAlignmentGapExtensionPenalty1=30,
                 partialOrderAlignmentGapOpenPenalty2=1200, partialOrderAlignmentGapExtensionPenalty2=1,
                 partialOrderAlignmentSubMatrix=None, partialOrderAlignmentDisableSeeding=1,
                 partialOrderAlignmentMinimizerK=15, partialOrderAlignmentMinimizerW=5,
                 partialOrderAlignmentMinimizerMinW=500, partialOrderAlignmentProgressiveMode=1,
                 device=0, threads_per_block=0, ctas_per_sm=0, mem_fraction=0.0, host_threads=0,
                 collect_phase_clocks=0, devices=None, lanes=0):
        mat = partialOrderAlignmentSubMatrix
        if mat is None:
            mat = CACTUS_SUBMAT
        elif isinstance(mat, str):
            mat = [int(v) for v in mat.split()]
        if len(mat) != 25:
            raise ValueError("partialOrderAlignmentSubMatrix needs 25 values")
        if any(not -2 ** 31 <= int(v) < 2 ** 31 for v in mat):
            # a C int would wrap such a value, possibly into the range barb200_create accepts
            raise ValueError("partialOrderAlignmentSubMatrix values must fit a 32-bit int")
        c = _CParams()
        for i, v in enumerate(mat):
            c.mat[i] = int(v)
        c.gap_open1, c.gap_ext1 = partialOrderAlignmentGapOpenPenalty1, partialOrderAlignmentGapExtensionPenalty1
        c.gap_open2, c.gap_ext2 = partialOrderAlignmentGapOpenPenalty2, partialOrderAlignmentGapExtensionPenalty2
        c.wb, c.wf = partialOrderAlignmentBandConstant, partialOrderAlignmentBandFraction
        c.k, c.w, c.min_w = partialOrderAlignmentMinimizerK, partialOrderAlignmentMinimizerW, partialOrderAlignmentMinimizerMinW
        c.progressive_poa, c.disable_seeding = partialOrderAlignmentProgressiveMode, partialOrderAlignmentDisableSeeding
        c.device, c.threads_per_block, c.ctas_per_sm = device, threads_per_block, ctas_per_sm
        c.mem_fraction, c.host_threads, c.collect_phase_clocks = mem_fraction, host_threads, collect_phase_clocks
        c.lanes = lanes
        if devices == "all":
            c.n_devices = -1
        elif devices:
            c.n_devices = len(devices)
            for i, d in enumerate(devices):
                c.devices[i] = int(d)
        self.c = c


class PairwiseAlignmentParameters:
    """The PairwiseAlignmentParameters fields the posterior path reads (submodules/cPecan/impl/pairwiseAligner.c:1369-1391;
    the <bar><pecan> keys of bar/impl/bar.c:20-37: diagonalExpansion, splitMatrixBiggerThanThis -- the XML value is the
    side length, squared here as bar.c:23-24 does)."""

    def __init__(self, threshold=0.01, minDiagsBetweenTraceBack=1000, traceBackDiagonals=40, diagonalExpansion=20,
                 splitMatrixBiggerThanThis=3000, dynamicAnchorExpansion=0):
        self.c = _CPecanParams(threshold, minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion,
                               int(splitMatrixBiggerThanThis) * int(splitMatrixBiggerThanThis), dynamicAnchorExpansion)


class MumParams:
    """The PairwiseAlignmentParameters fields MUM anchoring reads (getAnchorPairsForPairwiseAlignmentParameters,
    submodules/cPecan/impl/pairwiseAligner.c:1222-1231; the <bar><pecan> keys of bar/impl/bar.c:25-33):
    anchorMatrixBiggerThanThis is the XML side length, squared here as bar.c:26 does."""

    def __init__(self, k=50, u=1, anchorMatrixBiggerThanThis=500, recursiveMums=1):
        self.c = _CMumParams(k, u, int(anchorMatrixBiggerThanThis) * int(anchorMatrixBiggerThanThis), recursiveMums)


class _PairTable:
    """argument arrays of the barb200_pecan_* calls for a list of (sX, sY, anchorPairs, raggedLeft, raggedRight)"""

    def __init__(self, pairs):
        n = len(pairs)
        self.n = n
        m = max(n, 1)
        self.sx_b = [_as_bytes(q[0]) for q in pairs]
        self.sy_b = [_as_bytes(q[1]) for q in pairs]
        self.sx = (C.c_char_p * m)(*self.sx_b)
        self.sy = (C.c_char_p * m)(*self.sy_b)
        self.lx = np.array([len(b) for b in self.sx_b] or [0], np.int64)
        self.ly = np.array([len(b) for b in self.sy_b] or [0], np.int64)
        self.anch = [np.ascontiguousarray(np.asarray(q[2] if len(q) > 2 and q[2] is not None else [], np.int64).reshape(-1, 2)) for q in pairs]
        self.ap = (C.c_void_p * m)(*[a.ctypes.data if len(a) else None for a in self.anch])
        self.na = np.array([len(a) for a in self.anch] or [0], np.int64)
        self.rl = np.array([1 if (len(q) > 3 and q[3]) else 0 for q in pairs] or [0], np.uint8)
        self.rr = np.array([1 if (len(q) > 4 and q[4]) else 0 for q in pairs] or [0], np.uint8)

    def args(self):
        return [self.sx, self.lx.ctypes.data, self.sy, self.ly.ctypes.data, self.ap, self.na.ctypes.data,
                self.rl.ctypes.data, self.rr.ctypes.data]


class PecanStage:
    """Pair-HMM inputs resident in HBM: create (split + band + pack + H2D) once, run any number of times, fetch."""

    def __init__(self, engine, handle, table):
        self.engine, self.h, self.table = engine, handle, table

    def run(self):
        ms = C.c_float()
        self.engine._check(self.engine.lib.barb200_pecan_stage_run(self.h, C.byref(ms)))
        return ms.value

    def cells(self):
        return int(self.engine.lib.barb200_pecan_stage_cells(self.h))

    def launches(self):
        return int(self.engine.lib.barb200_pecan_stage_launches(self.h))

    def fetch(self, return_posteriors=False):
        n = self.table.n
        m = max(n, 1)
        trip, post = (C.c_void_p * m)(), (C.c_void_p * m)()
        n_out, cells = np.zeros(m, np.int64), np.zeros(m, np.int64)
        self.engine._check(self.engine.lib.barb200_pecan_stage_fetch(self.h, trip, n_out.ctypes.data,
                                                                     post if return_posteriors else None, cells.ctypes.data))
        return self.engine._take_pairs(trip, post if return_posteriors else None, n_out, cells, n)

    def close(self):
        if self.h:
            self.engine.lib.barb200_pecan_stage_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Msa:
    """bar/inc/poaBarAligner.h:37-43 -- seq_no, seq_lens, column_no, msa_seq (here one uint8 matrix)."""

    def __init__(self, msa_seq, seq_lens):
        self.msa_seq = msa_seq
        self.seq_no, self.column_no = msa_seq.shape
        self.seq_lens = list(seq_lens)

    def row_string(self, i):
        return "".join(_BASES[b] for b in self.msa_seq[i])


def _as_bytes(s):
    return s if isinstance(s, (bytes, bytearray)) else s.encode()


class _StrTable:
    """char*** + int** for a list of ends, each a list of byte strings; keeps the buffers alive."""

    def __init__(self, ends):
        self.keep = []
        n = len(ends)
        self.seq_no = (C.c_int64 * n)(*[len(e) for e in ends])
        self.strs = (C.c_void_p * n)()
        self.lens = (C.c_void_p * n)()
        for i, e in enumerate(ends):
            bs = [_as_bytes(s) for s in e]
            arr = (C.c_char_p * max(len(bs), 1))(*bs)
            ln = (C.c_int * max(len(bs), 1))(*[len(b) for b in bs])
            self.keep += [bs, arr, ln]
            self.strs[i] = C.cast(arr, C.c_void_p)
            self.lens[i] = C.cast(ln, C.c_void_p)


class Stage:
    """Inputs resident in HBM: create (pack + guide trees + H2D) once, run the kernel any number of times, fetch."""

    def __init__(self, engine, handle, n_seq):
        self.engine, self.h, self.n_seq = engine, handle, n_seq

    def run(self):
        ms = C.c_float()
        self.engine._check(self.engine.lib.barb200_stage_run(self.h, C.byref(ms)))
        return ms.value

    def launches(self):
        return int(self.engine.lib.barb200_stage_launches(self.h))

    def buckets(self):
        """the stage's CTA-size buckets, largest class first: dicts with threads, jobs, ctas, plane_ints"""
        out = (C.c_int64 * 32)()
        n = self.engine.lib.barb200_stage_buckets(self.h, out, 8)
        return [dict(threads=int(out[4 * i]), jobs=int(out[4 * i + 1]), ctas=int(out[4 * i + 2]), plane_ints=int(out[4 * i + 3])) for i in range(n)]

    def phase_clocks(self):
        out = (C.c_uint64 * 7)()
        self.engine._check(self.engine.lib.barb200_stage_phase_clocks(self.h, out))
        return dict(zip(["dp", "backtrack", "fuse", "topo", "msa", "total", "guide_tree"], [int(v) for v in out]))

    def fetch(self):
        n = len(self.n_seq)
        outs = (C.c_void_p * n)()
        ml = np.zeros(n, np.int32)
        cells = np.zeros(n, np.int64)
        self.engine._check(self.engine.lib.barb200_stage_fetch(self.h, outs, ml.ctypes.data, cells.ctypes.data))
        return self.engine._take_msas(outs, self.n_seq, ml), cells

    def close(self):
        if self.h:
            self.engine.lib.barb200_stage_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine:
    """One device context (barb200_ctx). Raises BarB200Error when no CUDA device / library is available."""

    def __init__(self, params=None, **kw):
        self.lib = load_library()
        self.params = params or PoaParams(**kw)
        err = C.create_string_buffer(512)
        self.ctx = self.lib.barb200_create(C.byref(self.params.c), err, 512)
        if not self.ctx:
            raise BarB200Error("barb200_create failed: %s" % err.value.decode())

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.barb200_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise BarB200Error("libbarb200 error %d: %s" % (rc, self.lib.barb200_last_error(self.ctx).decode()))

    def device_info(self):
        sm = C.c_int()
        tot, free = C.c_int64(), C.c_int64()
        name = C.create_string_buffer(128)
        self._check(self.lib.barb200_device_info(self.ctx, C.byref(sm), C.byref(tot), C.byref(free), name, 128))
        return dict(sm_count=sm.value, mem_total=tot.value, mem_free=free.value, name=name.value.decode())

    # ---- abpoa_msa level ------------------------------------------------------------------------------------
    @staticmethod
    def _pack(jobs):
        n_seq = np.array([len(j) for j in jobs], np.int32)
        lens = np.array([len(s) for j in jobs for s in j], np.int32)
        flat = np.concatenate([np.asarray(s, np.uint8) for j in jobs for s in j]) if len(lens) else np.zeros(0, np.uint8)
        return n_seq, lens, np.ascontiguousarray(flat)

    def _take_msas(self, outs, n_seq, ml):
        res = []
        for i in range(len(n_seq)):
            k, m = int(n_seq[i]), int(ml[i])
            a = np.ctypeslib.as_array(C.cast(outs[i], C.POINTER(C.c_uint8)), shape=(max(k * m, 1),))[: k * m]
            res.append(a.reshape(k, m).copy())
            self.lib.barb200_free(outs[i])
        return res

    def poa_msa_batch(self, jobs, progressive=None, return_cells=False):
        """jobs: list of jobs, each a list of uint8 code arrays (0..4). Returns a list of uint8 [K, msa_len]."""
        n_seq, lens, flat = self._pack(jobs)
        n = len(jobs)
        outs = (C.c_void_p * max(n, 1))()
        ml = np.zeros(max(n, 1), np.int32)
        cells = np.zeros(max(n, 1), np.int64)
        prog = None if progressive is None else np.asarray(progressive, np.int32)
        self._check(self.lib.barb200_poa_msa_batch(self.ctx, n, n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data,
                                                   None if prog is None else prog.ctypes.data, outs, ml.ctypes.data,
                                                   cells.ctypes.data))
        msas = self._take_msas(outs, n_seq, ml)
        return (msas, cells[:n]) if return_cells else msas

    def poa_msa_trace_batch(self, jobs, progressive=None):
        """poa_msa_batch through the trace kernels: per job the dict of :func:`parse_trace` -- the MSA and cells, the read order,
        and every alignment's read, query length, node count, best score, graph cigar and DP row bands as the device computed them."""
        n_seq, lens, flat = self._pack(jobs)
        n = len(jobs)
        outs = (C.c_void_p * max(n, 1))()
        nw = np.zeros(max(n, 1), np.int64)
        prog = None if progressive is None else np.asarray(progressive, np.int32)
        self._check(self.lib.barb200_poa_trace_batch(self.ctx, n, n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data,
                                                     None if prog is None else prog.ctypes.data, outs, nw.ctypes.data))
        res = []
        for i in range(n):
            k = int(nw[i])
            w = np.ctypeslib.as_array(C.cast(outs[i], C.POINTER(C.c_int64)), shape=(k,)).copy()
            self.lib.barb200_free(outs[i])
            res.append(parse_trace(w, int(n_seq[i])))
        return res

    def stage(self, jobs=None, packed=None, progressive=None):
        n_seq, lens, flat = packed if packed is not None else self._pack(jobs)
        h = C.c_void_p()
        prog = None if progressive is None else np.asarray(progressive, np.int32)
        self._check(self.lib.barb200_stage_create(self.ctx, len(n_seq), n_seq.ctypes.data, lens.ctypes.data,
                                                  flat.ctypes.data, None if prog is None else prog.ctypes.data,
                                                  C.byref(h)))
        return Stage(self, h, n_seq)

    # ---- cPecan mode: pairwiseAligner.h level -----------------------------------------------------------------
    def _take_pairs(self, trip, post, n_out, cells, n):
        res = []
        for i in range(n):
            k = int(n_out[i])
            t = np.ctypeslib.as_array(C.cast(trip[i], C.POINTER(C.c_int64)), shape=(max(3 * k, 1),))[: 3 * k].reshape(k, 3).copy()
            self.lib.barb200_free(trip[i])
            if post is not None:
                p = np.ctypeslib.as_array(C.cast(post[i], C.POINTER(C.c_double)), shape=(max(k, 1),))[:k].copy()
                self.lib.barb200_free(post[i])
                res.append((t, p, int(cells[i])))
            else:
                res.append((t, int(cells[i])))
        return res

    def get_aligned_pairs_using_anchors_batch(self, pairs, params=None, return_posteriors=False):
        """getAlignedPairsUsingAnchors (submodules/cPecan/impl/pairwiseAligner.c:1477-1495) for many sequence pairs.
        pairs: list of (sX, sY, anchorPairs[n, 2], alignmentHasRaggedLeftEnd, alignmentHasRaggedRightEnd).
        Returns per pair (triples int64 [k, 3] = (score, x, y) in the reference's order, [posteriors,] banded cells)."""
        params = params or PairwiseAlignmentParameters()
        t = pairs if isinstance(pairs, _PairTable) else _PairTable(pairs)
        raw = self.pecan_batch_raw(t, params, return_posteriors)
        return self._take_pairs(*raw, t.n)

    def pecan_table(self, pairs):
        """the C argument arrays of a list of pairs, built once (benchmarks time the C call, not this marshalling)"""
        return _PairTable(pairs)

    def pecan_batch_raw(self, table, params=None, return_posteriors=False):
        """barb200_pecan_aligned_pairs_batch on a prepared table; returns the raw output arrays (trip, post, n_out, cells)"""
        params = params or PairwiseAlignmentParameters()
        m = max(table.n, 1)
        trip, post = (C.c_void_p * m)(), (C.c_void_p * m)()
        n_out, cells = np.zeros(m, np.int64), np.zeros(m, np.int64)
        self._check(self.lib.barb200_pecan_aligned_pairs_batch(self.ctx, C.byref(params.c), table.n, *table.args(), trip, n_out.ctypes.data,
                                                               post if return_posteriors else None, cells.ctypes.data))
        return trip, (post if return_posteriors else None), n_out, cells

    def get_aligned_pairs_using_anchors(self, sX, sY, anchorPairs=(), params=None, alignmentHasRaggedLeftEnd=False,
                                        alignmentHasRaggedRightEnd=False):
        """single-pair form with the reference's argument order; returns the (score, x, y) triples"""
        return self.get_aligned_pairs_using_anchors_batch(
            [(sX, sY, anchorPairs, alignmentHasRaggedLeftEnd, alignmentHasRaggedRightEnd)], params)[0][0]

    def mum_anchor_pairs_batch(self, pairs, params=None):
        """getAnchorPairsForPairwiseAlignmentParameters with MUM anchors for many sequence pairs on the device.
        pairs: list of (sX, sY, ...) (further items are ignored). Returns per pair an int64 [n, 2] array of (x, y) anchors in the
        reference's order."""
        params = params or MumParams()
        t = pairs if isinstance(pairs, _PairTable) else _PairTable(pairs)
        m = max(t.n, 1)
        out = (C.c_void_p * m)()
        n_out = np.zeros(m, np.int64)
        self._check(self.lib.barb200_pecan_anchor_pairs_batch(self.ctx, C.byref(params.c), t.n, t.sx, t.lx.ctypes.data, t.sy,
                                                              t.ly.ctypes.data, out, n_out.ctypes.data))
        res = []
        for i in range(t.n):
            k = int(n_out[i])
            res.append(np.ctypeslib.as_array(C.cast(out[i], C.POINTER(C.c_int64)), shape=(max(2 * k, 1),))[: 2 * k].reshape(k, 2).copy())
            self.lib.barb200_free(out[i])
        return res

    def pecan_device_stats(self):
        """per device of the context, the sequence pairs the batch calls have run there since the context was created:
        dict(hmm_pairs=[...] (get_aligned_pairs_using_anchors_batch), mum_pairs=[...] (mum_anchor_pairs_batch, only pairs that
        needed the device)); the staged form is not counted"""
        n = self.device_count()
        hmm, mum = np.zeros(max(n, 1), np.int64), np.zeros(max(n, 1), np.int64)
        rc = self.lib.barb200_pecan_device_stats(self.ctx, hmm.ctypes.data, mum.ctypes.data, n)
        if rc < 0:
            self._check(rc)
        return dict(hmm_pairs=[int(v) for v in hmm[:n]], mum_pairs=[int(v) for v in mum[:n]])

    def mum_last_timing(self):
        """the calling thread's last mum_anchor_pairs_batch: dict(kernel_ms (with several devices: the slowest device's),
        wall_ms, launches (all devices))"""
        out = np.zeros(3)
        self._check(self.lib.barb200_mum_last_timing(out.ctypes.data))
        return dict(kernel_ms=float(out[0]), wall_ms=float(out[1]), launches=int(out[2]))

    def pecan_stage(self, pairs, params=None):
        params = params or PairwiseAlignmentParameters()
        t = _PairTable(pairs)
        h = C.c_void_p()
        self._check(self.lib.barb200_pecan_stage_create(self.ctx, C.byref(params.c), t.n, *t.args(), C.byref(h)))
        return PecanStage(self, h, t)

    # ---- poaBarAligner.h level --------------------------------------------------------------------------------
    def _wrap(self, cm):
        m = cm.contents
        k, c = int(m.seq_no), int(m.column_no)
        a = np.ctypeslib.as_array(m.msa, shape=(max(k * c, 1),))[: k * c].reshape(k, c).copy()
        lens = [m.seq_lens[i] for i in range(k)]
        self.lib.barb200_msa_destruct(cm)
        return Msa(a, lens)

    def msa_make_partial_order_alignment_batch(self, ends, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """ends: list of ends, each a list of ASCII strings. One Msa per end (bar/impl/poaBarAligner.c:463-749)."""
        t = _StrTable(ends)
        out = (C.POINTER(_CMsa) * max(len(ends), 1))()
        self._check(self.lib.barb200_msa_make_partial_order_alignment_batch(
            self.ctx, len(ends), t.seq_no, t.strs, t.lens, window_size, max_prog_rows, max_prog_length_diff, out))
        return [self._wrap(out[i]) for i in range(len(ends))]

    def msa_make_partial_order_alignment(self, seqs, window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        return self.msa_make_partial_order_alignment_batch([seqs], window_size, max_prog_rows, max_prog_length_diff)[0]

    def make_consistent_partial_order_alignments(self, end_strings, right_end_indexes, right_end_row_indexes, overlaps,
                                                 window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """bar/impl/poaBarAligner.c:751-801; arguments as the reference's, lists instead of C arrays."""
        t = _StrTable(end_strings)
        n = len(end_strings)
        keep = []

        def table(rows):
            arr = (C.c_void_p * max(n, 1))()
            for i, r in enumerate(rows):
                a = (C.c_int64 * max(len(r), 1))(*[int(v) for v in r])
                keep.append(a)
                arr[i] = C.cast(a, C.c_void_p)
            return arr
        ri, rr, ov = table(right_end_indexes), table(right_end_row_indexes), table(overlaps)
        ms = self.lib.barb200_make_consistent_partial_order_alignments(
            self.ctx, n, t.seq_no, t.strs, t.lens, ri, rr, ov, window_size, max_prog_rows, max_prog_length_diff)
        if not ms:
            raise BarB200Error("make_consistent_partial_order_alignments: %s" % self.lib.barb200_last_error(self.ctx).decode())
        out = [self._wrap(ms[i]) for i in range(n)]
        self.lib.barb200_free(C.cast(ms, C.c_void_p))
        return out

    def trace_ends(self, ends, right_end_indexes=None, right_end_row_indexes=None, overlaps=None, window_size=10000,
                   max_prog_rows=5000, max_prog_length_diff=1.0):
        """barb200_trace_ends: every sliding window of every end, with the arguments of make_consistent_partial_order_alignments
        (without the index lists the ends are independent). One dict of :func:`parse_end_trace` per end: each window's input slice,
        its POA job's per-alignment trace and its trimmed lengths, and the end's final MSA."""
        t = _StrTable(ends)
        n = len(ends)
        keep = []

        def table(rows):
            if rows is None:
                return None
            arr = (C.c_void_p * max(n, 1))()
            for i, r in enumerate(rows):
                a = (C.c_int64 * max(len(r), 1))(*[int(v) for v in r])
                keep.append(a)
                arr[i] = C.cast(a, C.c_void_p)
            return arr
        outs = (C.c_void_p * max(n, 1))()
        nw = np.zeros(max(n, 1), np.int64)
        self._check(self.lib.barb200_trace_ends(self.ctx, n, t.seq_no, t.strs, t.lens, table(right_end_indexes),
                                                table(right_end_row_indexes), table(overlaps), window_size, max_prog_rows,
                                                max_prog_length_diff, outs, nw.ctypes.data))
        res = []
        for i in range(n):
            w = np.ctypeslib.as_array(C.cast(outs[i], C.POINTER(C.c_int64)), shape=(int(nw[i]),)).copy()
            self.lib.barb200_free(outs[i])
            res.append(parse_end_trace(w))
        return res

    # ---- the end queue, asynchronously (barb200_flower_submit / barb200_flower_wait) ---------------------------------
    def flower_submit(self, end_strings, right_end_indexes=None, right_end_row_indexes=None, overlaps=None,
                      window_size=10000, max_prog_rows=5000, max_prog_length_diff=1.0):
        """Enqueue the ends of one flower; returns a ticket for flower_wait. Without the index lists the ends are independent."""
        t = _StrTable(end_strings)
        n = len(end_strings)
        keep = []

        def table(rows):
            if rows is None:
                return None
            arr = (C.c_void_p * max(n, 1))()
            for i, r in enumerate(rows):
                a = (C.c_int64 * max(len(r), 1))(*[int(v) for v in r])
                keep.append(a)
                arr[i] = C.cast(a, C.c_void_p)
            return arr
        h = self.lib.barb200_flower_submit(self.ctx, n, t.seq_no, t.strs, t.lens, table(right_end_indexes), table(right_end_row_indexes),
                                           table(overlaps), window_size, max_prog_rows, max_prog_length_diff)
        if not h:
            raise BarB200Error("flower_submit: %s" % self.lib.barb200_last_error(self.ctx).decode())
        return (h, n)

    def flower_wait(self, ticket):
        h, n = ticket
        ms = self.lib.barb200_flower_wait(self.ctx, h)
        if not ms:
            raise BarB200Error("flower_wait: %s" % self.lib.barb200_last_error(self.ctx).decode())
        out = [self._wrap(ms[i]) for i in range(n)]
        self.lib.barb200_free(C.cast(ms, C.c_void_p))
        return out

    def queue_stats(self):
        b, j = C.c_int64(), C.c_int64()
        self._check(self.lib.barb200_queue_stats(self.ctx, C.byref(b), C.byref(j)))
        return {"batches": b.value, "jobs": j.value}

    def last_batch_timing(self):
        out = (C.c_double * 6)()
        self._check(self.lib.barb200_last_batch_timing(self.ctx, out))
        return dict(zip(["build_ms", "run_ms", "device_ms", "fetch_ms", "total_ms", "jobs"], [float(v) for v in out]))

    def device_count(self):
        return int(self.lib.barb200_device_count(self.ctx))


def pecan_band(lx, ly, anchors, expansion=20):
    """Host only: (xmyL, xmyR) of the diagonals 0..lx+ly as the engine builds them (band_construct, pairwiseAligner.c:193-244)."""
    lib = load_library()
    a = np.ascontiguousarray(np.asarray(anchors, np.int64).reshape(-1, 2))
    L, R = np.zeros(lx + ly + 1, np.int64), np.zeros(lx + ly + 1, np.int64)
    if lib.barb200_pecan_band(lx, ly, a.ctypes.data if len(a) else None, len(a), expansion, L.ctypes.data, R.ctypes.data) != 0:
        raise BarB200Error("barb200_pecan_band: bad arguments")
    return L, R


def pecan_split_points(lx, ly, anchors, split_matrix_bigger_than_this, ragged_left=False, ragged_right=False):
    """Host only: getSplitPoints (pairwiseAligner.c:1265-1292) as the engine computes it -> int64 [n, 4] (x1, y1, x2, y2)."""
    lib = load_library()
    a = np.ascontiguousarray(np.asarray(anchors, np.int64).reshape(-1, 2))
    o = C.c_void_p()
    n = lib.barb200_pecan_split_points(lx, ly, a.ctypes.data if len(a) else None, len(a), split_matrix_bigger_than_this,
                                       int(ragged_left), int(ragged_right), C.byref(o))
    if n < 0:
        raise BarB200Error("barb200_pecan_split_points: bad arguments")
    out = np.ctypeslib.as_array(C.cast(o, C.POINTER(C.c_int64)), shape=(max(4 * n, 1),))[: 4 * n].reshape(n, 4).copy()
    lib.barb200_free(o)
    return out
