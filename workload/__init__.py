"""Seeded synthetic BAR workloads (SURVEY.md 8d) shared by bench.py's two arms and the tests.

Deliberately NOT part of the engine: `workload/libbarsynth.so` is a plain host library (g++), so that the reference arm
of bench.py, which must not load any product code, can generate the very same inputs as the GPU arm.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBPATH = os.path.join(_HERE, "libbarsynth.so")
_LIB = None


def build(force=False):
    src = os.path.join(_HERE, "synth.cpp")
    if force or not os.path.exists(_LIBPATH) or os.path.getmtime(src) > os.path.getmtime(_LIBPATH):
        subprocess.check_call(["/usr/bin/g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", _LIBPATH, src])
    return _LIBPATH


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_LIBPATH):
            build()
        lib = C.CDLL(_LIBPATH)
        vp, i64, ci = C.c_void_p, C.c_int64, C.c_int
        lib.barsynth_end.argtypes = [C.c_uint64, C.c_uint64, ci, ci, C.c_double, C.c_double, C.c_double, vp, vp]
        lib.barsynth_end.restype = i64
        lib.barsynth_pair.argtypes = [C.c_uint64, C.c_uint64, ci, C.c_double, C.c_double, C.c_double, ci, vp, vp, vp, vp, vp]
        lib.barsynth_pair.restype = i64
        lib.barsynth_msa_hash.argtypes = [vp, i64, ci]
        lib.barsynth_msa_hash.restype = C.c_uint64
        lib.barsynth_fnv1a.argtypes = [vp, i64]
        lib.barsynth_fnv1a.restype = C.c_uint64
        _LIB = lib
    return _LIB


def msa_hash(msa):
    """FNV-1a over (msa_len, bytes) of one uint8 [K, msa_len] matrix (the parity gate's per-end hash)"""
    m = np.ascontiguousarray(msa, np.uint8)
    return int(_lib().barsynth_msa_hash(m.ctypes.data, m.size, m.shape[1]))


_RC = np.array([3, 2, 1, 0, 4], np.uint8)
_ASCII = np.frombuffer(b"ACGTN", np.uint8)


def synth_flowers(first_flower, n_flowers, ends_per_flower, K, L, seed=0xF10E0000):
    """Seeded synthetic flowers for the end-queue legs of bench.py: every flower has `ends_per_flower` ends (even), in pairs:
    the strings of end 2i+1 are the reverse complements of the strings of end 2i (full-length overlap), row order permuted -- the
    structure of bar/tests/poaBarTest.c:93-179. Returns a list of (end_strings, right_end_indexes, right_end_row_indexes,
    overlaps) with ASCII byte strings, the arguments of make_consistent_partial_order_alignments."""
    assert ends_per_flower % 2 == 0
    out = []
    half = ends_per_flower // 2
    n_seq, lens, flat = synth_ends(first_flower * half, n_flowers * half, K, L, seed=seed)
    offs = np.concatenate([[0], np.cumsum(lens)])
    rng = np.random.default_rng(seed & 0xffffffff)
    for f in range(n_flowers):
        ends, ri, rr, ov = [], [], [], []
        for p in range(half):
            e = f * half + p
            rows = [flat[offs[e * K + i]:offs[e * K + i + 1]] for i in range(K)]
            fwd = [_ASCII[r].tobytes() for r in rows]
            perm = [int(x) for x in rng.permutation(K)]
            rev = [None] * K
            inv = [0] * K
            for i, pi in enumerate(perm):
                rev[pi] = _ASCII[_RC[rows[i]][::-1]].tobytes()
                inv[pi] = i
            ends += [fwd, rev]
            ri += [[2 * p + 1] * K, [2 * p] * K]
            rr += [perm, inv]
            ov += [[len(s) for s in fwd], [len(s) for s in rev]]
        out.append((ends, ri, rr, ov))
    return out


def synth_ends(first_end, n_ends, K, L, seed=0xBA5E0000, sub=0.02, ins=0.005, dele=0.005):
    """Seeded synthetic ends -> (n_seq[int32 n], lens[int32 n*K], flat uint8 codes 0..3). Deterministic in (seed, end index)."""
    lib = _lib()
    n_seq = np.full(n_ends, K, np.int32)
    lens = np.zeros(n_ends * K, np.int32)
    flat = np.zeros(n_ends * K * (2 * L + 16), np.uint8)
    o = 0
    for e in range(n_ends):
        n = lib.barsynth_end(seed, first_end + e, K, L, sub, ins, dele, flat.ctypes.data + o, lens.ctypes.data + 4 * e * K)
        if n < 0:
            raise ValueError("barsynth_end failed")
        o += n
    return n_seq, lens, flat[:o].copy()


def synth_pairs(first_pair, n_pairs, L, k_anchor=50, seed=0xBA5E0000, sub=0.02, ins=0.005, dele=0.005):
    """Seeded synthetic sequence pairs with MUM-like anchors -> list of (sX, sY, anchors[n, 2], False, False)."""
    lib = _lib()
    bx, by = C.create_string_buffer(2 * L + 16), C.create_string_buffer(2 * L + 16)
    an = np.zeros((2 * L, 2), np.int64)
    lx, ly = C.c_int64(), C.c_int64()
    out = []
    for i in range(n_pairs):
        na = lib.barsynth_pair(seed, first_pair + i, L, sub, ins, dele, k_anchor, bx, C.byref(lx), by, C.byref(ly), an.ctypes.data)
        if na < 0:
            raise ValueError("barsynth_pair failed")
        out.append((bx.raw[:lx.value], by.raw[:ly.value], an[:na].copy(), False, False))
    return out


def read_harvest(path):
    """Flowers recorded by shim/cactus_bar_harvest.c (BARB200_HARVEST=<path>) during a reference bar() run -> list of dicts
    {"ends": [[bytes, ...], ...], "right_end_indexes", "right_end_row_indexes", "overlaps" (None for a single-end record),
    "window_size", "max_prog_rows", "max_prog_length_diff"} in the order the calls were made."""
    import struct
    out = []
    with open(path, "rb") as f:
        data = f.read()
    o = 0

    def i64():
        nonlocal o
        v = struct.unpack_from("<q", data, o)[0]
        o += 8
        return v
    while o < len(data):
        if i64() != 0x4852414232303042:
            raise ValueError("bad harvest record at byte %d" % (o - 8))
        kind, end_no, window, max_rows = i64(), i64(), i64(), i64()
        diff = struct.unpack_from("<d", data, o)[0]
        o += 8
        ends, ri, rr, ov = [], [], [], []
        for _ in range(end_no):
            n = i64()
            meta = [(i64(), i64(), i64(), i64()) for _ in range(n)]
            strs = []
            for ln, _, _, _ in meta:
                strs.append(data[o:o + ln])
                o += ln
            ends.append(strs)
            ri.append([m[1] for m in meta])
            rr.append([m[2] for m in meta])
            ov.append([m[3] for m in meta])
        single = kind == 2
        out.append({"ends": ends, "right_end_indexes": None if single else ri, "right_end_row_indexes": None if single else rr,
                    "overlaps": None if single else ov, "window_size": window, "max_prog_rows": max_rows, "max_prog_length_diff": diff})
    return out


PECAN_HARVEST_MAGIC = 0x484E435032303042
PECAN_PARAM_FIELDS = ("min_diags_between_traceback", "traceback_diagonals", "diagonal_expansion", "split_matrix_bigger_than_this",
                      "dynamic_anchor_expansion")
MUM_PARAM_FIELDS = ("anchor_matrix_bigger_than_this", "k", "u", "recursive_mums")


def read_pecan_harvest(path):
    """Sequence pairs recorded by shim/cactus_pecan_harvest.c (BARB200_PECAN_HARVEST=<path>) during a reference cPecan-mode bar()
    run -> list of ends in the order their first pair was recorded, each {"end": end id, "pairs": [pair, ...]} with the pairs
    in recorded order. A pair is a dict: "end", "index" (its number within the end), "sx", "sy" (bytes), "ragged_left",
    "ragged_right", "use_mum_anchors" (bool), "pecan" (threshold and the barb200_pecan_params fields), "mum" (the
    barb200_mum_params fields), "anchors" (int64 [n, 2], the reference's), "anchor_hash", "n_triples", "triple_hash".
    Raises ValueError naming the byte offset of a record with a bad magic or one cut short."""
    import struct
    with open(path, "rb") as f:
        data = f.read()
    head = struct.Struct("<qqqd" + "q" * 15 + "QqQ")
    ends, order, o = {}, [], 0
    while o < len(data):
        start = o
        if len(data) - o >= 8 and struct.unpack_from("<q", data, o)[0] != PECAN_HARVEST_MAGIC:
            raise ValueError("bad pecan harvest record at byte %d: no magic number" % start)
        if len(data) - o < head.size:
            raise ValueError("pecan harvest record at byte %d is truncated" % start)
        v = head.unpack_from(data, o)
        o += head.size
        (_, end, index, threshold), ints, (anchor_hash, n_triples, triple_hash) = v[:4], v[4:19], v[19:]
        lx, ly, na = ints[12:15]
        if min(lx, ly, na) < 0 or len(data) - o < lx + ly + 16 * na:
            raise ValueError("pecan harvest record at byte %d is truncated" % start)
        sx, sy = data[o:o + lx], data[o + lx:o + lx + ly]
        o += lx + ly
        anchors = np.frombuffer(data, np.int64, 2 * na, o).reshape(na, 2).copy()
        o += 16 * na
        pair = {"end": end, "index": index, "sx": sx, "sy": sy, "ragged_left": bool(ints[10]), "ragged_right": bool(ints[11]),
                "use_mum_anchors": bool(ints[9]), "pecan": dict(zip(PECAN_PARAM_FIELDS, ints[0:5]), threshold=threshold),
                "mum": dict(zip(MUM_PARAM_FIELDS, ints[5:9])),
                "anchors": anchors, "anchor_hash": anchor_hash, "n_triples": n_triples, "triple_hash": triple_hash}
        if end not in ends:
            ends[end] = {"end": end, "pairs": []}
            order.append(end)
        ends[end]["pairs"].append(pair)
    return [ends[e] for e in order]


def fnv1a64(words):
    """64-bit FNV-1a over the little-endian bytes of an int64 array: the anchor and triple hashes of a pecan harvest record"""
    w = np.ascontiguousarray(words, "<i8")
    return int(_lib().barsynth_fnv1a(w.ctypes.data, w.nbytes))
