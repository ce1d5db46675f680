"""MUM anchor checkers (cPecan's getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1):
the compiled reference (oracle/_ref/libmum_ref.so: mum_ref_harness.c), the plain-C restatement (oracle/_build/libmum_oracle.so:
mum_oracle.c), both built by oracle/mum.mk, and the host build of the product's K5 (tests/hosttest/_build/libmum_host.so,
tests/hosttest/mum.mk); the flower-level stand-in build that runs it under the real pecan shim; plus the sequence generators the
MUM tests share. Everything here is built by __graft_entry__.build()."""
import ctypes as C
import os

import numpy as np

import _flowers as F
import _reflib as R

MUM_ORACLE_SO = os.path.join(R.ROOT, "oracle", "_build", "libmum_oracle.so")
MUM_REF_SO = os.path.join(R.ROOT, "oracle", "_ref", "libmum_ref.so")
MUM_HOST_SO = os.path.join(R.ROOT, "tests", "hosttest", "_build", "libmum_host.so")
FLOWER_STANDIN_MUM_SO = os.path.join(R.ROOT, "oracle", "_ref", "libflower_standin_mum.so")


def have_ref():
    return os.path.exists(MUM_REF_SO)


def have_flower_standin():
    """the flower-level drop-in build over the stand-in device with K5's host build; registered as F.bar(\"standin_mum\", ...)"""
    F._PATHS.setdefault("standin_mum", FLOWER_STANDIN_MUM_SO)
    return os.path.exists(FLOWER_STANDIN_MUM_SO)


class _MumParams(C.Structure):
    _fields_ = [("k", C.c_int64), ("u", C.c_int64), ("bigger", C.c_int64), ("recursive", C.c_int)]


def _b(s):
    return s if isinstance(s, (bytes, bytearray)) else bytes(s, "ascii") if isinstance(s, str) else bytes(np.asarray(s, np.uint8))


def _take(free, ptr, n):
    a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(max(2 * n, 1),))[: 2 * n].reshape(n, 2).copy()
    free(ptr)
    return a


def oracle_mum_anchors(sx, sy, k=50, u=1, bigger=500 * 500, recursive=1, tie_seed=0, with_abort=False):
    """(n, 2) int64 anchors; with_abort: also whether an assert-enabled reference would abort on this input (a MUM ending at lX)"""
    lib = R._load(MUM_ORACLE_SO)
    f = lib.oracle_mum_anchor_pairs
    f.restype = C.c_int64
    f.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.POINTER(_MumParams), C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
    lib.oracle_mum_free.argtypes = [C.c_void_p]
    sx, sy = _b(sx), _b(sy)
    p = _MumParams(k, u, bigger, recursive)
    out, ab = C.c_void_p(), C.c_int()
    n = f(sx, len(sx), sy, len(sy), C.byref(p), tie_seed, C.byref(out), C.byref(ab))
    a = _take(lib.oracle_mum_free, out, n)
    return (a, bool(ab.value)) if with_abort else a


def ref_mum_anchors(sx, sy, k=50, u=1, bigger=500 * 500, recursive=1):
    lib = R._load(MUM_REF_SO)
    f = lib.mum_ref_anchor_pairs
    f.restype = C.c_int64
    f.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.POINTER(C.c_void_p)]
    lib.mum_ref_free.argtypes = [C.c_void_p]
    sx, sy = _b(sx), _b(sy)
    out = C.c_void_p()
    n = f(sx, len(sx), sy, len(sy), k, u, bigger, recursive, C.byref(out))
    return _take(lib.mum_ref_free, out, n)


def hosttest_mum_anchors(sx, sy, k=50, u=1, bigger=500 * 500, recursive=1, tie_seed=0):
    lib = R._load(MUM_HOST_SO)
    f = lib.hosttest_mum_anchor_pairs
    f.restype = C.c_int64
    f.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_uint64, C.POINTER(C.c_void_p)]
    lib.hosttest_mum_free.argtypes = [C.c_void_p]
    sx, sy = _b(sx), _b(sy)
    out = C.c_void_p()
    n = f(sx, len(sx), sy, len(sy), k, u, bigger, recursive, tie_seed, C.byref(out))
    if n < 0:
        raise ValueError("rejected")
    return _take(lib.hosttest_mum_free, out, n)


# ---- sequences ------------------------------------------------------------------------------------------------------------
def rand_seq(rng, n, alphabet=b"ACGT"):
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def mutate(rng, s, sub=0.02, ins=0.005, dele=0.005, alphabet=b"ACGT"):
    out = bytearray()
    for c in s:
        r = rng.random()
        if r < dele:
            continue
        out.append(alphabet[rng.integers(0, len(alphabet))] if r < dele + sub else c)
        if rng.random() < ins:
            out.append(alphabet[rng.integers(0, len(alphabet))])
    return bytes(out)


def related_pair(rng, n, **kw):
    x = rand_seq(rng, n)
    return x, mutate(rng, x, **kw)


def case_set(rng):
    """named (sx, sy, params) cases covering the MUM rules: threshold edges, short sequences, identical sequences, repeats,
    mixed case / N / IUPAC, skewed lengths, unrelated blocks around and between MUMs, duplications and crossing MUMs"""
    cases = []
    a = rand_seq(rng, 500)
    cases.append(("500x500", a, mutate(rng, a, 0.01, 0, 0)[:500].ljust(500, b"A"), {}))
    b = rand_seq(rng, 501)
    cases.append(("500x501", b[:500], b, {}))
    cases.append(("short_x", rand_seq(rng, 30), rand_seq(rng, 9000), {}))
    cases.append(("short_y", rand_seq(rng, 9000), rand_seq(rng, 40), {}))
    for L in (600, 1000, 1022):
        s = rand_seq(rng, L)
        cases.append(("identical_%d" % L, s, s, {}))
    cases.append(("homopolymer", b"A" * 800, b"A" * 900, {}))
    rep = (b"ACGTTGCA" * 200)[:1500]
    cases.append(("tandem", rep, rep[3:], {}))
    mixed = bytearray(rand_seq(rng, 1500, b"ACGTacgtNnR"))
    cases.append(("mixed_case", bytes(mixed), bytes(mutate(rng, bytes(mixed), 0.01, 0.002, 0.002, b"ACGTacgtNnR")).swapcase(), {}))
    x, y = related_pair(rng, 6000)
    cases.append(("lx_much_longer", x + rand_seq(rng, 6000), y[1000:2500], {}))
    cases.append(("ly_much_longer", y[2000:3000], rand_seq(rng, 3000) + x + rand_seq(rng, 2000), {}))
    for rec in (0, 1):
        x, y = related_pair(rng, 1500)
        x2, y2 = related_pair(rng, 1200)
        sx = rand_seq(rng, 1700) + x + rand_seq(rng, 2100) + x2 + rand_seq(rng, 1300)
        sy = rand_seq(rng, 1100) + y + rand_seq(rng, 2900) + y2 + rand_seq(rng, 2500)
        cases.append(("unrelated_blocks_r%d" % rec, sx, sy, dict(recursive=rec)))
    x, y = related_pair(rng, 3000)
    cases.append(("duplication", x + x[500:1500], y[:2000] + y[300:1200] + y[2000:], {}))
    cases.append(("crossing", x[1500:] + x[:1500], y, {}))
    for k in (8, 12, 20, 50):
        for u in (0, 1, 3):
            x, y = related_pair(rng, 1500, sub=0.03)
            cases.append(("k%d_u%d" % (k, u), x, y, dict(k=k, u=u, bigger=300 * 300)))
    return cases
