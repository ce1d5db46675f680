"""The plan of a POA stage (cactus_b200/csrc/stage_plan.h, which barb200.cu runs), CPU only: the parameter and job checks with the
messages the library raises, the internal order and the buckets, the output strides, the fit into device memory, the capacity-retry
schedule, the cut of a batch into device batches and the deal over devices. The CPU stand-in device runs its batches through the
same checks, so it rejects what the product rejects."""
import ctypes as C
import os

import numpy as np
import pytest

import _reflib as R
from _synth import family, to_ascii, two_end_problem

EINVAL, ENOMEM, EJOB = -3, -2, -5
JOB_OK, JOB_ERR_PLANE_CAP, JOB_ERR_MSA_CAP, JOB_ERR_TOPO, JOB_ERR_GT_CAP = 0, 3, 5, 6, 10
CLASSES = (32, 64, 128, 256, 640, 1024)
BUCKET_FIELDS = ("threads", "job_base", "jobs", "slots", "plane_ints", "slot_bytes")
H100_BYTES = 81559 * 2 ** 20            # cudaMemGetInfo total of an H100 80GB HBM3
SHARED_BUDGET = H100_BYTES * 0.85 / 2   # one lane's share once the end queue runs (lane_budget_bytes)
H100_SMS = 132
MIXED_SHAPES = [(4, 150)] * 12 + [(3, 700)] * 6 + [(5, 1500)] * 3 + [(3, 2500)] * 2 + [(2, 5200)] + [(6, 40)] * 9
STANDIN_SO = os.path.join(R.ROOT, "tests", "hosttest", "_build", "libbarb200_standin.so")


def _lib():
    lib = R._load(R.build_hosttest())
    vp, i64 = C.c_void_p, C.c_int64
    lib.hosttest_stage_plan.restype = C.c_int
    lib.hosttest_stage_plan.argtypes = [i64, vp, vp, vp, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, C.c_double, vp, vp, vp, vp, vp,
                                        C.c_char_p, C.c_int]
    lib.hosttest_retry_round.restype = C.c_int
    lib.hosttest_retry_round.argtypes = [i64, vp, vp, C.c_double, C.c_int, i64, vp, C.POINTER(i64), C.POINTER(C.c_double), C.POINTER(C.c_int),
                                         C.c_char_p, C.c_int]
    lib.hosttest_chunk_ends.restype = i64
    lib.hosttest_chunk_ends.argtypes = [i64, vp, vp]
    lib.hosttest_deal_jobs.restype = None
    lib.hosttest_deal_jobs.argtypes = [i64, vp, C.c_int, vp, vp]
    return lib


def plan(jobs, threads_per_block=0, grow=1.0, worst=False, per_sm=0, sms=H100_SMS, budget=0.0):
    """hosttest_stage_plan: (rc, message) of a rejection, else the plan (per_sm > 0: fitted into `budget`)"""
    n, m = len(jobs), max(len(jobs), 1)
    n_seq = np.array([len(j) for j in jobs] or [0], np.int32)
    seqs = [np.asarray(s, np.uint8) for j in jobs for s in j]
    lens = np.array([len(s) for s in seqs] or [0], np.int32)
    flat = np.concatenate(seqs + [np.zeros(1, np.uint8)])
    cost = np.zeros(m)
    perm, msa_off, msa_stride = (np.zeros(m, np.int64) for _ in range(3))
    buckets = np.zeros((len(CLASSES), len(BUCKET_FIELDS)), np.int64)
    err = C.create_string_buffer(512)
    rc = _lib().hosttest_stage_plan(n, n_seq.ctypes.data, lens.ctypes.data, flat.ctypes.data, threads_per_block, grow, int(worst), per_sm, sms,
                                    budget, cost.ctypes.data, perm.ctypes.data, msa_off.ctypes.data, msa_stride.ctypes.data, buckets.ctypes.data,
                                    err, 512)
    if rc < 0:
        return rc, err.value.decode()
    return dict(cost=cost[:n], perm=perm[:n].tolist(), msa_off=msa_off[:n].tolist(), msa_stride=msa_stride[:n].tolist(),
                buckets=[dict(zip(BUCKET_FIELDS, (int(v) for v in b))) for b in buckets[:rc]])


def class_threads(max_len, threads_per_block=0):
    return next(T for T in CLASSES if 16 * T >= max_len + 1 and T >= threads_per_block)


def planned_bytes(buckets):
    return sum(b["slots"] * (b["slot_bytes"] + 4 * b["plane_ints"]) for b in buckets)


def mixed_jobs():
    rng = np.random.default_rng(47)
    order = rng.permutation(len(MIXED_SHAPES))
    jobs = [family(rng, MIXED_SHAPES[i][0], MIXED_SHAPES[i][1], sub=0.03, ins=0.01, dele=0.01) for i in order]
    # jobs of equal cost (same K, same lengths): the order must keep them in the caller's order
    return jobs + [[rng.integers(0, 4, 100).astype(np.uint8) for _ in range(3)] for _ in range(5)]


# ---- checks ----
def test_rejected_jobs_give_the_library_messages():
    """the five rejections test_gpu_parity.py::test_errors_are_loud expects from the library"""
    ok = np.array([0, 1], np.uint8)
    bad = [([[ok], []], "job without sequences"),
           ([[np.array([], np.uint8), ok]], "empty sequence"),
           ([[np.array([0, 1, 7], np.uint8), ok]], "sequence code > 4"),
           ([[np.zeros(16384, np.uint8), ok]], "row limit"),         # one base past the largest CTA class (1024 threads x 16 columns - 1)
           ([[np.zeros(1, np.uint8)] * 65536], "more than 65535 sequences")]
    for jobs, msg in bad:
        rc, err = plan(jobs)
        assert rc == EINVAL and msg in err, (msg, err)
    assert isinstance(plan([[np.zeros(16383, np.uint8), ok]]), dict)


def create_error(**kw):
    """the stand-in's barb200_create (the product's parameter check): its message, or None if it made a context"""
    import cactus_b200 as cb
    R.build_hosttest()
    lib = R._load(STANDIN_SO)
    lib.barb200_create.restype = C.c_void_p
    lib.barb200_create.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    lib.barb200_destroy.argtypes = [C.c_void_p]
    lib.barb200_destroy.restype = None
    err = C.create_string_buffer(512)
    params = cb.PoaParams(**kw).c
    ctx = lib.barb200_create(C.addressof(params), err, 512)
    if ctx:
        lib.barb200_destroy(ctx)
        return None
    return err.value.decode()


@pytest.mark.parametrize("kw, msg", [
    (dict(partialOrderAlignmentGapOpenPenalty2=0), "convex gap model"),
    (dict(partialOrderAlignmentBandConstant=-1), "BandConstant must be >= 0"),
    (dict(partialOrderAlignmentGapOpenPenalty1=65000, partialOrderAlignmentGapExtensionPenalty1=535), "below 65535"),
    (dict(partialOrderAlignmentSubMatrix=[65536] + list(R.CACTUS_MAT[1:])), "SubMatrix entries must lie in"),
    (dict(partialOrderAlignmentDisableSeeding=0), "seeding"),
    (dict(partialOrderAlignmentMinimizerK=21), "minimizer k must be in 1..20"),
    (dict(partialOrderAlignmentMinimizerW=256), "w in 1..255"),
])
def test_parameters_the_engine_cannot_run_are_refused(kw, msg):
    err = create_error(**kw)
    assert err is not None and msg in err, err


def test_default_parameters_are_accepted():
    assert create_error() is None
    assert create_error(partialOrderAlignmentGapOpenPenalty1=65000, partialOrderAlignmentGapExtensionPenalty1=534,
                        partialOrderAlignmentSubMatrix=[65535] + list(R.CACTUS_MAT[1:]), partialOrderAlignmentMinimizerK=20,
                        partialOrderAlignmentMinimizerW=255) is None


# ---- order, buckets, strides ----
def test_mixed_shapes_are_ordered_and_bucketed():
    jobs = mixed_jobs()
    P = plan(jobs, per_sm=2, budget=SHARED_BUDGET)
    b, perm, cost = P["buckets"], P["perm"], P["cost"]
    threads = [x["threads"] for x in b]
    assert len(b) >= 4 and threads == sorted(threads, reverse=True) and len(set(threads)) == len(threads)
    assert sum(x["jobs"] for x in b) == len(jobs)
    assert b[0]["plane_ints"] > 20 * b[-1]["plane_ints"]          # slots are sized per class, not from the largest job
    assert sorted(perm) == list(range(len(jobs)))
    base = 0
    for x in b:
        assert x["job_base"] == base
        part = perm[base:base + x["jobs"]]
        assert all(class_threads(max(len(s) for s in jobs[c])) == x["threads"] for c in part)
        key = [(-cost[c], c) for c in part]                         # cost-descending, the caller's order on ties
        assert key == sorted(key)
        base += x["jobs"]
    ties = list(range(len(jobs) - 5, len(jobs)))
    assert len(set(cost[ties])) == 1 and [c for c in perm if c in ties] == ties


def test_threads_per_block_raises_the_class():
    jobs = mixed_jobs()
    b = plan(jobs, threads_per_block=256)["buckets"]
    assert [x["threads"] for x in b] == [640, 256]
    assert b[0]["jobs"] == 1 and sum(x["jobs"] for x in b) == len(jobs)


@pytest.mark.parametrize("grow, worst", [(1.0, False), (4.0, False), (1.0, True)])
def test_msa_strides(grow, worst):
    """a job's output rows are planned at 1.5 x its longest read + 64 (x grow), at most its bases, 16-byte aligned; at the worst case
    at its bases; the jobs' output blocks follow each other in the internal order"""
    jobs = mixed_jobs()
    P = plan(jobs, grow=grow, worst=worst)
    off = 0
    for j, c in enumerate(P["perm"]):
        K, S, ML = len(jobs[c]), sum(len(s) for s in jobs[c]), max(len(s) for s in jobs[c])
        want = S if worst else min(S, int(grow * (ML + ML // 2 + 64)))
        want = (want + 15) // 16 * 16
        assert P["msa_stride"][j] == want and P["msa_off"][j] == off, j
        off += want * K


# ---- memory fit ----
@pytest.mark.parametrize("per_sm", [1, 3])
def test_slots_fit_occupancy_and_budget(per_sm):
    jobs = mixed_jobs()
    roomy = plan(jobs, per_sm=per_sm, budget=SHARED_BUDGET)["buckets"]
    for b in roomy:
        assert 1 <= b["slots"] <= min(b["jobs"], per_sm * H100_SMS)
    assert planned_bytes(roomy) <= SHARED_BUDGET
    one_each = planned_bytes([dict(b, slots=1) for b in roomy])
    budget = one_each + (planned_bytes(roomy) - one_each) / 3        # the slots shrink to fit
    tight = plan(jobs, per_sm=per_sm, budget=budget)["buckets"]
    assert planned_bytes(tight) <= budget
    assert all(1 <= t["slots"] <= r["slots"] for t, r in zip(tight, roomy)) and tight != roomy


def test_retry_plan_is_cut_to_a_small_budget():
    """the situation of test_gpu_parity.py::test_retry_plan_cut_to_a_small_device_budget: a budget of 2.5 x the job's optimistic
    planes holds its first round as planned, and its x4 retry with the planes cut instead of failing"""
    rng = np.random.default_rng(4711)
    job = family(rng, 12, 2000, sub=0.2, ins=0.02, dele=0.02)
    first = plan([job])["buckets"][0]
    budget = 2.5 * 4 * first["plane_ints"]
    fitted = plan([job], per_sm=4, budget=budget)["buckets"][0]
    assert fitted["slots"] == 1 and fitted["plane_ints"] == first["plane_ints"]
    x4 = plan([job], grow=4.0)["buckets"][0]
    assert 4 * x4["plane_ints"] > budget
    cut = plan([job], grow=4.0, per_sm=4, budget=budget)["buckets"][0]
    assert cut["slots"] == 1 and first["plane_ints"] < cut["plane_ints"] < x4["plane_ints"] and cut["plane_ints"] % 8 == 0
    assert planned_bytes([cut]) <= budget


@pytest.mark.parametrize("grow", [1.0, 4.0])
def test_a_job_whose_slot_alone_exceeds_the_budget_fails(grow):
    job = family(np.random.default_rng(5), 4, 300)
    slot_bytes = plan([job])["buckets"][0]["slot_bytes"]
    rc, err = plan([job], grow=grow, per_sm=4, budget=slot_bytes / 2)
    assert rc == ENOMEM and "a single job needs more device memory than is available" in err, err


# ---- capacity retries ----
def retry_round(status, perm, grow, worst, plane_cap=1 << 28):
    n = len(status)
    st, pm, redo = np.array(status, np.int32), np.array(perm, np.int64), np.zeros(max(n, 1), np.int64)
    n_redo, next_grow, next_worst = C.c_int64(), C.c_double(), C.c_int()
    err = C.create_string_buffer(512)
    rc = _lib().hosttest_retry_round(n, st.ctypes.data, pm.ctypes.data, grow, int(worst), plane_cap, redo.ctypes.data, C.byref(n_redo),
                                     C.byref(next_grow), C.byref(next_worst), err, 512)
    if rc:
        return rc, err.value.decode()
    return redo[:n_redo.value].tolist(), (next_grow.value, bool(next_worst.value))


def test_capacity_misses_grow_x4_then_to_the_worst_case():
    perm = [7, 3, 5, 11]
    miss = [JOB_OK, JOB_ERR_PLANE_CAP, JOB_ERR_MSA_CAP, JOB_ERR_GT_CAP]
    assert retry_round(miss, perm, 1.0, False) == ([3, 5, 11], (4.0, False))
    assert retry_round(miss, perm, 4.0, False) == ([3, 5, 11], (1.0, True))
    rc, err = retry_round(miss, perm, 1.0, True, plane_cap=250_000_000)
    assert rc == EJOB and err.startswith("job 3 needs more DP-plane memory than this lane can plan") and "1.0 GB of planes per slot" in err, err
    assert retry_round([JOB_OK] * 4, perm, 1.0, False)[0] == []


def test_other_statuses_fail_at_once():
    rc, err = retry_round([JOB_OK, JOB_OK, JOB_ERR_TOPO, JOB_ERR_PLANE_CAP], [7, 3, 5, 11], 1.0, False)
    assert rc == EJOB and err == "job 5 failed on the device with status %d" % JOB_ERR_TOPO, err


# ---- device batches and devices ----
def chunk_ends(sum_len):
    s = np.array(sum_len, np.int64)
    ends = np.zeros(len(s), np.int64)
    n = _lib().hosttest_chunk_ends(len(s), s.ctypes.data, ends.ctypes.data)
    return ends[:n].tolist()


def test_batches_are_cut_at_the_job_and_base_limits():
    MiB = 2 ** 20
    assert chunk_ends([300] * 40000) == [32768, 40000]
    assert chunk_ends([100 * MiB] * 10) == [7, 10]                 # 7 x 100 MiB within 768 MiB, 8 x not
    assert chunk_ends([10 * MiB, 1024 * MiB, 10 * MiB, 10 * MiB]) == [1, 2, 4]   # an oversized job forms its own chunk


@pytest.mark.parametrize("ndev", [1, 2, 8])
def test_jobs_are_dealt_over_devices_once(ndev):
    rng = np.random.default_rng(ndev)
    cost = np.ascontiguousarray(rng.uniform(1e3, 1e7, 3001))
    counts, jobs = np.zeros(ndev, np.int64), np.zeros(len(cost), np.int64)
    _lib().hosttest_deal_jobs(len(cost), cost.ctypes.data, ndev, counts.ctypes.data, jobs.ctypes.data)
    assert sorted(jobs.tolist()) == list(range(len(cost)))
    shares = np.split(jobs, np.cumsum(counts)[:-1])
    loads = [cost[s].sum() for s in shares]
    for s in shares:
        assert list(s) == sorted(s)                                 # each device's share in the caller's order
    assert max(loads) - min(loads) <= cost.max()                   # LPT: no device more than one job behind


# ---- the stand-in device ----
def test_the_stand_in_device_rejects_what_the_product_rejects(oracle_built):
    """a window over 16383 bases is past the device engine's row limit: the ticket holding a read that long fails alone with a
    nonzero rc, and the tickets that shared its batches still deliver what the oracle delivers"""
    rng = np.random.default_rng(16)
    p = R.cactus_params(wb=10, wf=0.01)
    flowers = [two_end_problem(rng, int(rng.integers(2, 5)), int(rng.integers(20, 60))) for _ in range(8)]
    bad = 5
    ends, ri, rr, ov = flowers[bad]
    ends = [list(e) for e in ends]
    ends[0][0] = to_ascii(rng.integers(0, 4, 17000))
    flowers[bad] = (ends, ri, rr, ov)
    res, rcs, _ = R.hosttest_flowers(flowers, p=p, n_lanes=2, n_threads=3, window_size=20000)
    assert rcs[bad] != 0 and res[bad] is None
    for i, ((e, a, b, o), got) in enumerate(zip(flowers, res)):
        if i == bad:
            continue
        assert rcs[i] == 0
        want = R.oracle_make_consistent_partial_order_alignments(e, a, b, o, p=p, window_size=20000)
        assert got is not None and len(got) == len(want)
        for x, y in zip(got, want):
            assert x.shape == y.shape and np.array_equal(x, y), i
