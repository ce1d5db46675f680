"""The POA trace call (barb200_poa_trace_batch, Engine.poa_msa_trace_batch) without a GPU: the production kernels compile as they did
before the trace kernels existed, the trace regions' capacity plan and its retries, the cut of a large trace call into device batches,
and the product's reader of the trace words. test_gpu_poa_trace.py runs the trace kernels against the reference and the oracle."""
import ctypes as C
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import _repeats as RP
import _reflib as R
from _synth import family
from cactus_b200 import build as B
from test_gpu_far_rows import families as far_row_families
from test_stage_plan_cpu import retry_round

JOB_OK, JOB_ERR_PLANE_CAP, JOB_ERR_TRACE_CAP = 0, 3, 11
EJOB = -5
CLASSES = (32, 64, 128, 256, 640, 1024)
HELPER = os.path.join(R.ROOT, "tests", "hosttest", "trace_plan.cpp")
# ptxas -v of the production kernels (registers, stack frame, spill store / load bytes, static shared memory) when the trace kernels
# were added, the same as the commit before them: the trace kernels must not move them
PRODUCTION_RESOURCES = {32: (128, 64, 0, 0, 2816), 64: (127, 64, 0, 0, 3328), 128: (127, 64, 0, 0, 4352), 256: (127, 64, 0, 0, 6400),
                        640: (96, 112, 104, 100, 12544), 1024: (64, 192, 532, 432, 18688)}


def unrelated_job(seed=60):
    """60 unrelated reads of 300 bases: every read adds most of its bases as new nodes, far past the optimistic row estimate"""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 4, 300).astype(np.uint8) for _ in range(60)]


# BARB200_TRACE_REGION_SCALE of the trace-capacity retry test, and its jobs
RETRY_SCALE = 1e-6


def retry_jobs():
    rng = np.random.default_rng(71)
    return [family(rng, K, L, sub=0.05, ins=0.02, dele=0.02) for K, L in ((3, 40), (6, 300), (9, 700), (4, 2500))]


def row_ints(beg, end):
    """ints of the DP planes one row of band [beg, end] takes (poa_types.h: row_ints)"""
    t0 = (beg // 16) & ~1
    return 32 * (((end // 16 - t0) | 1) + 1)


def first_overflows(job, p, grow, worst, plan_lib):
    """(alignment whose DP planes first outgrow the planned planes, alignment whose record first outgrows the planned trace region),
    None where nothing does: the host build's trace of the job replayed against a single-job stage's plan at (grow, worst)"""
    lib = R._load(R.build_hosttest())
    lib.hosttest_plane_ints_for_job.restype = C.c_int64
    lib.hosttest_plane_ints_for_job.argtypes = [C.c_int, C.c_double, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int]
    K, S, ML = len(job), sum(len(s) for s in job), max(len(s) for s in job)
    planes = (lib.hosttest_plane_ints_for_job(p.wb, p.wf, K, S, ML, grow, int(worst)) + 7) // 8 * 8
    region = words_for(plan_lib, job, grow, worst)
    used, plane_at, trace_at = 0, None, None
    for a, x in enumerate(R.hosttest_poa_msa_trace(job, p)["alns"]):
        if plane_at is None and sum(row_ints(b, e) for b, e in zip(x["dp_beg"], x["dp_end"])) > planes:
            plane_at = a
        used += 6 + len(x["cigar"]) + 2 * len(x["dp_beg"])
        if trace_at is None and used > region:
            trace_at = a
    return plane_at, trace_at


def record_words(tr):
    return sum(6 + len(a["cigar"]) + 2 * len(a["dp_beg"]) for a in tr["alns"])


@pytest.fixture(scope="module")
def plan_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("trace_plan") / "libtrace_plan.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-fopenmp", "-x", "c++", "-o", so, HELPER])
    lib = C.CDLL(so)
    i64, vp = C.c_int64, C.c_void_p
    lib.trace_words.restype, lib.trace_words.argtypes = i64, [i64, i64, i64, C.c_double, C.c_int]
    lib.trace_stage.restype, lib.trace_stage.argtypes = i64, [i64, vp, vp, vp, C.c_double, C.c_int, C.c_double, vp, vp, vp, vp]
    lib.trace_retry_batches.restype, lib.trace_retry_batches.argtypes = i64, [i64, vp, vp, vp, C.c_int, C.c_double, C.c_int, vp]
    lib.trace_chunk_ends.restype, lib.trace_chunk_ends.argtypes = i64, [i64, vp, vp, vp, i64, vp]
    lib.trace_batch_limit.restype, lib.trace_batch_limit.argtypes = i64, []
    return lib


def words_for(lib, job, grow=1.0, worst=False):
    return lib.trace_words(len(job), sum(len(s) for s in job), max(len(s) for s in job), grow, int(worst))


# ---- the production kernels ----
@pytest.fixture(scope="module")
def modules(tmp_path_factory):
    """ptxas -v logs of the production module poa_kernel.cu and of the trace module poa_trace_kernel.cu"""
    if not shutil.which(B.NVCC):
        pytest.skip("needs nvcc")
    d = tmp_path_factory.mktemp("trace_modules")

    def compile_one(src):
        cubin = str(d / (os.path.basename(src) + ".cubin"))
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-cubin", "-x", "cu", os.path.join(B.CSRC, src), "-o", cubin], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout + r.stderr
    with ThreadPoolExecutor(2) as ex:
        return dict(zip(("production", "trace"), ex.map(compile_one, ["poa_kernel.cu", "poa_trace_kernel.cu"])))


def entries(log):
    return sorted(set(re.findall(r"Compiling entry function '(\w+)'", log)))


def test_production_and_trace_kernels_are_separate_modules(modules):
    """the production module holds the six production kernels and no trace code; the trace module the six trace kernels"""
    assert entries(modules["production"]) == sorted("poa_msa_kernel_t%d" % T for T in CLASSES)
    assert entries(modules["trace"]) == sorted("poa_trace_kernel_t%d" % T for T in CLASSES)
    assert "trace_record" not in modules["production"]


@pytest.mark.parametrize("T", CLASSES)
def test_production_kernel_resources_are_unchanged(modules, T):
    log = modules["production"]
    m = re.search(r"Function properties for poa_msa_kernel_t%d\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\s*\n[^\n]*Used (\d+) registers, [^\n]*?(\d+) bytes smem" % T, log)
    assert m, log
    regs, stack, st, ld, smem = int(m.group(4)), int(m.group(1)), int(m.group(2)), int(m.group(3)), int(m.group(5))
    assert (regs, stack, st, ld, smem) == PRODUCTION_RESOURCES[T]


# ---- trace capacity ----
def capacity_cases():
    rng = np.random.default_rng(77)
    out = [("random/%d" % i, family(rng, int(rng.integers(2, 12)), int(rng.choice([20, 150, 400, 900])), sub=0.08, ins=0.03, dele=0.03))
           for i in range(8)]
    out += [("far_rows/%d" % i, job) for i, job in enumerate(far_row_families(np.random.default_rng(2024 + 300), 300))]
    out += [(c.name, c.seqs) for f in sorted(RP.FAMILIES) for c in RP.cases(f) if sum(len(s) for s in c.seqs) <= 6000]
    out.append(("unrelated", unrelated_job()))
    return out


def test_worst_case_region_covers_every_host_trace(plan_lib):
    """the worst-case region (6 + cigar_cap + 2 node_cap words per alignment) holds the records of the host build's traces of random,
    far-row, repeat-rich and unrelated jobs"""
    for name, job in capacity_cases():
        tr = R.hosttest_poa_msa_trace(job)
        assert record_words(tr) <= words_for(plan_lib, job, worst=True), name
        assert words_for(plan_lib, job) <= words_for(plan_lib, job, 4.0) <= words_for(plan_lib, job, worst=True), name


def test_unrelated_reads_outgrow_their_first_planes(plan_lib):
    """the premise of test_gpu_poa_trace.py's plane retry test: this job's records outgrow the first-round region, but its DP planes
    overflow earlier, so the first round ends with JOB_ERR_PLANE_CAP, and the x4 round's planes overflow too while its region holds the
    whole trace: the job reaches the worst case through plane retries, its trace through regions planned at x4 and at the worst case"""
    p = R.cactus_params()
    r1, x4 = first_overflows(unrelated_job(), p, 1.0, False, plan_lib), first_overflows(unrelated_job(), p, 4.0, False, plan_lib)
    assert r1[0] is not None and r1[1] is not None and r1[0] < r1[1], r1
    assert x4[0] is not None and x4[1] is None, x4


def test_scaled_regions_overflow_before_anything_else(plan_lib):
    """the premise of test_gpu_poa_trace.py's trace-capacity retry test: with BARB200_TRACE_REGION_SCALE at RETRY_SCALE its jobs' planes
    hold every alignment in the first round while their regions, in the first round and at x4, cannot hold even the first record; the
    worst case is not scaled. So every job ends the first two rounds with JOB_ERR_TRACE_CAP and is traced by the worst-case round"""
    jobs = retry_jobs()
    n_seq, lens, flat = _pack(jobs)
    for grow, worst in ((1.0, False), (4.0, False), (1.0, True)):
        perm, off, cap, blk = np.zeros(len(jobs), np.int64), np.zeros(len(jobs), np.int64), np.zeros(len(jobs), np.int64), np.zeros(2, np.int64)
        plan_lib.trace_stage(len(jobs), n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data, grow, int(worst), RETRY_SCALE, perm.ctypes.data,
                             off.ctypes.data, cap.ctypes.data, blk.ctypes.data)
        for c, k in zip(perm, cap):
            if worst:
                assert k == words_for(plan_lib, jobs[c], worst=True) >= record_words(R.hosttest_poa_msa_trace(jobs[c])), c
            else:
                assert k < 6, (grow, c, k)
    for job in jobs:
        assert first_overflows(job, R.cactus_params(), 1.0, False, plan_lib)[0] is None


def test_related_reads_fit_the_optimistic_region(plan_lib):
    rng = np.random.default_rng(5)
    for K, L in ((4, 300), (8, 2000), (3, 5000)):
        job = family(rng, K, L, sub=0.03, ins=0.01, dele=0.01)
        assert record_words(R.hosttest_poa_msa_trace(job)) <= words_for(plan_lib, job), (K, L)


def test_trace_capacity_misses_are_retried_x4_then_at_the_worst_case():
    perm = [4, 9, 2]
    miss = [JOB_ERR_TRACE_CAP, JOB_OK, JOB_ERR_PLANE_CAP]
    assert retry_round(miss, perm, 1.0, False) == ([4, 2], (4.0, False))
    assert retry_round(miss, perm, 4.0, False) == ([4, 2], (1.0, True))
    rc, err = retry_round([JOB_OK, JOB_ERR_TRACE_CAP, JOB_OK], perm, 1.0, True)
    assert rc == EJOB and err == "job 9 failed on the device with status %d" % JOB_ERR_TRACE_CAP, err


def _pack(jobs):
    n_seq = np.array([len(j) for j in jobs], np.int32)
    lens = np.array([len(s) for j in jobs for s in j], np.int32)
    flat = np.concatenate([np.asarray(s, np.uint8) for j in jobs for s in j])
    return n_seq, lens, flat


@pytest.mark.parametrize("grow, worst", [(1.0, False), (4.0, False), (1.0, True)])
def test_trace_regions_are_planned_in_the_stage_block(plan_lib, grow, worst):
    """every job gets its region back to back in the stage's internal order, sized by trace_words_for_job, and the regions are part of
    the stage's one device block, which counts against the lane's budget"""
    rng = np.random.default_rng(8)
    jobs = [family(rng, int(rng.integers(2, 9)), int(rng.choice([40, 300, 1200, 3000])), sub=0.05) for _ in range(17)]
    n_seq, lens, flat = _pack(jobs)
    n = len(jobs)
    perm, off, cap, blk = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(2, np.int64)
    total = plan_lib.trace_stage(n, n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data, grow, int(worst), 1.0, perm.ctypes.data,
                                 off.ctypes.data, cap.ctypes.data, blk.ctypes.data)
    assert sorted(perm.tolist()) == list(range(n))
    assert [words_for(plan_lib, jobs[c], grow, worst) for c in perm] == cap.tolist()
    assert off.tolist() == np.concatenate([[0], np.cumsum(cap)[:-1]]).tolist() and total == cap.sum()
    assert blk[1] - blk[0] >= 8 * total + 3 * 8 * n


def test_a_large_trace_call_is_cut_into_device_batches(plan_lib):
    """jobs whose first-round regions add up to more than one device batch's trace limit run in several batches, each within the limit
    (a single job larger than the limit runs alone); the same jobs without a trace are one batch"""
    limit = plan_lib.trace_batch_limit()
    K, ML = 100, 10000
    n_seq = np.full(20, K, np.int32)
    sum_len, max_len = np.full(20, K * ML, np.int64), np.full(20, ML, np.int32)
    per_job = plan_lib.trace_words(K, K * ML, ML, 1.0, 0)
    assert 2 * per_job <= limit < 20 * per_job
    ends = np.zeros(20, np.int64)
    n = plan_lib.trace_chunk_ends(20, n_seq.ctypes.data, sum_len.ctypes.data, max_len.ctypes.data, limit, ends.ctypes.data)
    cuts = [0] + ends[:n].tolist()
    assert n > 1 and cuts[-1] == 20
    assert all(0 < (b - a) * per_job <= limit for a, b in zip(cuts, cuts[1:]))
    assert plan_lib.trace_chunk_ends(20, n_seq.ctypes.data, sum_len.ctypes.data, max_len.ctypes.data, 0, ends.ctypes.data) == 1
    huge = np.full(1, 40 * ML, np.int32)
    big_sum = np.full(1, 40 * ML * 5000, np.int64)
    assert plan_lib.trace_words(40 * ML, 40 * ML * 5000, 5000, 1.0, 0) > limit
    assert plan_lib.trace_chunk_ends(1, huge.ctypes.data, big_sum.ctypes.data, np.full(1, 5000, np.int32).ctypes.data, limit, ends.ctypes.data) == 1


# ---- the reader ----
def oracle_words(seqs, p=None):
    lens, flat = R._flat(seqs)
    lib = R._load(R.build_oracle())
    nw = C.c_int64()
    ptr = R._trace_fn(lib, "oracle_poa_msa_trace")(C.byref(p or R.cactus_params()), len(seqs), lens.ctypes.data, flat.ctypes.data, C.byref(nw))
    words = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int64)), shape=(nw.value,)).copy()
    lib.oracle_free.argtypes = [C.c_void_p]
    lib.oracle_free(ptr)
    return words


def same_trace(a, b):
    if set(a) != set(b) or a["msa_len"] != b["msa_len"] or a["cells"] != b["cells"] or a["read_id_map"] != b["read_id_map"]:
        return False
    if a["msa"].dtype != b["msa"].dtype or not np.array_equal(a["msa"], b["msa"]) or len(a["alns"]) != len(b["alns"]):
        return False
    for x, y in zip(a["alns"], b["alns"]):
        if set(x) != set(y):
            return False
        for k in x:
            if isinstance(x[k], np.ndarray):
                if x[k].dtype != y[k].dtype or not np.array_equal(x[k], y[k]):
                    return False
            elif x[k] != y[k]:
                return False
    return True


def test_product_reader_equals_the_checkers_reader(oracle_built):
    import cactus_b200 as cb
    rng = np.random.default_rng(31)
    jobs = [family(rng, int(rng.integers(1, 9)), int(rng.choice([1, 7, 60, 400])), sub=0.1, ins=0.03, dele=0.03) for _ in range(10)]
    jobs.append([rng.integers(0, 5, int(rng.integers(1, 90))).astype(np.uint8) for _ in range(70)])
    for j, job in enumerate(jobs):
        w = oracle_words(job)
        assert same_trace(cb.parse_trace(w, len(job)), R._parse_trace(w, len(job))), j
    with pytest.raises(ValueError):
        cb.parse_trace(oracle_words(jobs[0]), len(jobs[0]) + 1)


def test_a_large_trace_retry_is_cut_into_stages(plan_lib):
    """a capacity retry of a trace stage runs in as many stages as keep each one's regions (x4, worst case) within the batch limit; a
    plain stage's retry is one stage"""
    limit = plan_lib.trace_batch_limit()
    n, K, ML = 2000, 8, 2000
    n_seq, sum_len, max_len = np.full(n, K, np.int32), np.full(n, K * ML, np.int64), np.full(n, ML, np.int32)
    sizes = np.zeros(n, np.int64)
    for grow, worst in ((4.0, False), (1.0, True)):
        per_job = plan_lib.trace_words(K, K * ML, ML, grow, int(worst))
        assert n * per_job > limit
        m = plan_lib.trace_retry_batches(n, n_seq.ctypes.data, sum_len.ctypes.data, max_len.ctypes.data, 1, grow, int(worst), sizes.ctypes.data)
        assert m > 1 and sizes[:m].sum() == n and all(0 < k * per_job <= limit for k in sizes[:m]), (grow, worst, sizes[:m])
        assert plan_lib.trace_retry_batches(n, n_seq.ctypes.data, sum_len.ctypes.data, max_len.ctypes.data, 0, grow, int(worst), sizes.ctypes.data) == 1
