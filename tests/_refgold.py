"""The unmodified reference's answers for the differential tests (test_oracle_vs_ref.py, test_poa_params_cpu.py,
test_pecan_cpu.py), stored as SHA-256 digests in tests/golden/ref_digests.npz so that those tests compare against the reference
everywhere, also where the reference libraries (oracle/_ref) cannot be built.

Each check has a key (test, case). `check(key, got, ref_fn)` asserts that the digest of `got` equals the stored digest of
the reference's answer; per-field digests are stored beside it, so that a mismatch names the fields that differ (msa, cigar,
dp_beg, ...). With BARB200_RECORD_REF=1 the reference itself is run (ref_fn()), compared with `got` directly and
its digest recorded; scripts/make_golden_ref_digests.py runs the tests that way and writes the file.
"""
import hashlib
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.npz")
RECORDING = os.environ.get("BARB200_RECORD_REF") == "1"
_recorded = {}
_stored = None


def _feed(h, x):
    if isinstance(x, dict):
        for k in sorted(x):
            h.update(k.encode())
            _feed(h, x[k])
    elif isinstance(x, (list, tuple)):
        h.update(b"[%d" % len(x))
        for v in x:
            _feed(h, v)
    elif isinstance(x, np.ndarray):
        a = np.ascontiguousarray(x)
        h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    else:
        h.update(repr(int(x) if isinstance(x, (bool, int, np.integer)) else x).encode())


def digest(x):
    h = hashlib.sha256()
    _feed(h, x)
    return h.hexdigest()


def parts(x):
    """(name, value) of the fields a mismatch report names: a dict's entries, with a list of dicts split per field across the
    list (alns.cigar, alns.dp_beg, ...); a list's elements by index"""
    if isinstance(x, dict):
        out = []
        for k in sorted(x):
            v = x[k]
            if isinstance(v, list) and v and all(isinstance(e, dict) for e in v):
                out += [("%s.%s" % (k, f), [e[f] for e in v]) for f in sorted(v[0])]
            else:
                out.append((k, v))
        return out
    if isinstance(x, (list, tuple)):
        return [(str(i), v) for i, v in enumerate(x)]
    return []


def trace_view(tr):
    """the fields of a POA trace the differential tests compare (MSA, read order, banded cells, and per alignment its read, query
    length, graph size, best score, cigar and every dp_beg / dp_end)"""
    return dict(msa_len=tr["msa_len"], msa=tr["msa"], read_id_map=list(tr["read_id_map"]), cells=tr["cells"],
                alns=[dict(read_id=a["read_id"], qlen=a["qlen"], node_n=a["node_n"], best_score=a["best_score"],
                           cigar=np.asarray(a["cigar"], np.uint64), dp_beg=np.asarray(a["dp_beg"], np.int32),
                           dp_end=np.asarray(a["dp_end"], np.int32)) for a in tr["alns"]])


def _stored_digests():
    global _stored
    if _stored is None:
        z = np.load(PATH)
        _stored = dict(zip((k.decode() for k in z["keys"]), (v.decode() for v in z["digests"])))
    return _stored


def check(key, got, ref_fn, equal=None):
    """got: the checked implementation's answer; ref_fn(): the reference's answer (called only when recording); equal(a, b):
    the direct comparison used while recording (default: equal digests)"""
    if RECORDING:
        want = ref_fn()
        assert (equal(want, got) if equal else digest(want) == digest(got)), key
        assert key not in _recorded, "duplicate key %s" % key
        _recorded[key] = digest(want)
        for name, v in parts(want):
            _recorded["%s#%s" % (key, name)] = digest(v)[:32]
        return
    stored = _stored_digests()
    assert key in stored, "no stored reference answer for %s (scripts/make_golden_ref_digests.py)" % key
    if digest(got) != stored[key]:
        differ = [name for name, v in parts(got) if stored.get("%s#%s" % (key, name)) != digest(v)[:32]]
        raise AssertionError("%s differs from the reference in %s" % (key, ", ".join(differ) or "its shape (number of fields)"))


def save():
    keys = sorted(_recorded)
    np.savez_compressed(PATH, keys=np.array([k.encode() for k in keys]), digests=np.array([_recorded[k].encode() for k in keys]))
    return sum("#" not in k for k in keys)
