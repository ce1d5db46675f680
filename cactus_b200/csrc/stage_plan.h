// stage_plan.h -- the plan of a POA stage (barb200.cu): parameter and job checks, internal order and buckets, the fit into device
// memory, capacity retries, the cut into device batches. CUDA-free: barb200.cu measures occupancy and free memory and runs what
// the plan decides; the CPU suite (tests/hosttest) runs the same plan. The layouts it sizes are slot_plan.h's.
#pragma once
#include <stdio.h>
#include <numeric>
#include "host_api.h"
#include "poa_kernel.cuh"
#include "slot_plan.h"

namespace barb200 {

// CTA-size classes: a CTA of T threads sweeps rows of up to 16 T columns (query length + 1). barb200.cu: kKernels, in this order.
constexpr int kClassThreads[] = {32, 64, 128, 256, 640, 1024};
constexpr int kNumClasses = 6;

// The smallest class whose rows hold a read of max_len bases and that has at least threads_per_block threads; -1 if none does.
inline int class_of_len(int64_t max_len, int threads_per_block) {
    for (int i = 0; i < kNumClasses; ++i) if ((int64_t)kClassThreads[i] * CPT >= max_len + 1 && kClassThreads[i] >= threads_per_block) return i;
    return -1;
}
// banded cells the job will sweep, roughly: (K-1) alignments x ~mean length rows x band width (SURVEY.md 8e's cost)
inline double job_cost(const barb200_params &p, int K, int64_t sum, int64_t ml) {
    const double w = 2.0 * (p.wb + p.wf * (double)ml) + 1.0;
    return (double)(K - 1) * (double)(sum / std::max(1, K) + 1) * std::min<double>((double)ml + 1.0, w) + 2000.0 * K;
}

// barb200_create's checks of parameters the device engine cannot run: "" if they pass, else the message.
inline std::string check_params(const barb200_params &p) {
    if (p.gap_open1 <= 0 || p.gap_open2 <= 0 || p.gap_ext1 < 0 || p.gap_ext2 < 0 || (p.gap_ext1 == 0 && p.gap_ext2 == 0))
        return "only the convex gap model (both gap opens > 0) is supported; that is what Cactus configures";
    if (p.wb < 0) return "partialOrderAlignmentBandConstant must be >= 0 (adaptive band)";
    if ((int64_t)p.gap_open1 + p.gap_ext1 >= 65535 || (int64_t)p.gap_open2 + p.gap_ext2 >= 65535)
        return "gap open + extension must be below 65535 (the traceback planes keep E as a 16-bit distance below H)";
    // The sweep's scores are int32, as the reference's are. With every |mat| <= 65535, e <= 65533 < 65534 (from the check above)
    // and L <= 16383, the largest value it forms, A = H' + (j + 1) e of the F scan, is below 16383 * 65535 + 16384 * 65534 =
    // 2147368961 < INT32_MAX, and inf_min - min_mis stays above INT32_MIN. Larger scores overflow the reference too (its best
    // scores then wrap), so there is no answer to reproduce.
    for (int i = 0; i < 25; ++i)
        if (p.mat[i] > 65535 || p.mat[i] < -65535)
            return "partialOrderAlignmentSubMatrix entries must lie in [-65535, 65535] (larger scores overflow the int32 DP scores, in the reference too)";
    if (!p.disable_seeding) return "minimizer seeding (partialOrderAlignmentDisableSeeding=0) is not supported";
    if (p.k <= 0 || p.k > 20 || p.w <= 0 || p.w >= 256) return "minimizer k must be in 1..20 and w in 1..255 (guide-tree keys are hash << 24 | span << 16 | read)";
    return "";
}

// The jobs of one call in the caller's order, scanned and checked once. Stages (and their capacity retries) are lists of indices
// into it; it keeps its own copy of the lengths because a stage outlives the arguments of barb200_stage_create.
struct TableJob {
    int n_seq = 0, max_len = 0, cls = 0, progressive = 0;
    int64_t len_off = 0, seq_off = 0, sum_len = 0;     // first length in `lens`, first base in the sequence buffer
    double cost = 0;
};
struct JobTable {
    std::vector<TableJob> jobs;
    std::vector<int> lens;
    int64_t n_bases = 0;                                // the sequence buffer: every job's bases back to back
};

// view(j, len_off, seq_off) -> caller job j, whose lengths and bases the table places at those offsets; the bases are scanned on
// `nthreads` threads. Returns "" or the message of the first rejection.
template <class View>
std::string build_table(const barb200_params &p, int nthreads, int64_t n_jobs, View view, JobTable &t) {
    if (n_jobs > 0x7ffffff0) return "too many jobs in one stage";
    t.jobs.resize(n_jobs);
    int64_t lo = 0, bo = 0;
    for (int64_t j = 0; j < n_jobs; ++j) {
        const HostJob v = view(j, lo, bo);
        if (v.n_seq <= 0) return "job without sequences";
        TableJob &J = t.jobs[j];
        J.n_seq = v.n_seq; J.progressive = v.progressive; J.len_off = lo; J.seq_off = bo;
        for (int i = 0; i < v.n_seq; ++i) {
            const int l = v.lens[i];
            if (l <= 0) return "empty sequence in a POA job (the shim substitutes 'N', poaBarAligner.c:551-562)";
            J.sum_len += l; J.max_len = std::max(J.max_len, l);
        }
        J.cls = class_of_len(J.max_len, p.threads_per_block); J.cost = job_cost(p, J.n_seq, J.sum_len, J.max_len);
        if (J.cls < 0) return "a sequence is longer than the device engine's row limit (16383 bases per window)";
        if (J.progressive && J.n_seq > 65535) return "progressive mode with more than 65535 sequences in one window is not supported";
        t.lens.insert(t.lens.end(), v.lens, v.lens + v.n_seq);
        lo += v.n_seq; bo += J.sum_len;
    }
    t.n_bases = bo;
    int bad = 0;
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthreads) reduction(| : bad)
    for (int64_t j = 0; j < n_jobs; ++j) {
        const uint8_t *s = view(j, t.jobs[j].len_off, t.jobs[j].seq_off).seqs;
        uint8_t m = 0;
        for (int64_t b = 0; b < t.jobs[j].sum_len; ++b) m |= s[b] > 4;
        bad |= m;
    }
    return bad ? "sequence code > 4" : "";
}

// the jobs as barb200_stage_create and barb200_poa_msa_batch take them: lengths and bases back to back
inline std::string table_of_arrays(const barb200_params &p, int nthreads, int64_t n_jobs, const int *n_seq, const int *seq_lens, const uint8_t *seqs,
                                   const int *progressive, JobTable &t) {
    if (n_jobs < 0 || (n_jobs > 0 && (!n_seq || !seq_lens || !seqs))) return "bad arguments";
    return build_table(p, nthreads, n_jobs, [&](int64_t j, int64_t lo, int64_t bo) {
        return HostJob{n_seq[j], seq_lens + lo, seqs + bo, progressive ? progressive[j] : p.progressive_poa};
    }, t);
}

inline std::vector<int64_t> all_jobs(int64_t n) { std::vector<int64_t> v(n); std::iota(v.begin(), v.end(), (int64_t)0); return v; }

// one CTA-size class of a stage: jobs [job_base, job_base + n_jobs) in the stage's internal order
struct PlanBucket {
    int cls = 0, T = 0;
    int64_t job_base = 0, n_jobs = 0;
    SlotLayout lay{}; int slots = 0;
    size_t slot_off = 0; int64_t plane_off = 0; size_t clk_off = 0;   // offsets into the lane's arena (bytes / ints / entries)
};

// The host side of a stage. Every array is in the stage's INTERNAL job order: class-major (largest class first), cost-descending
// inside a class (stable); perm[internal] = the caller's job index in the table.
struct StagePlan {
    double grow = 1.0; bool worst_case = false;        // the capacity retry this plan sizes for
    std::vector<int64_t> perm;
    std::vector<int> lens;
    std::vector<int64_t> soff;
    std::vector<JobDesc> desc;
    std::vector<PlanBucket> buckets;
    int64_t n_seqs = 0, msa_bytes = 0;
    GtLayout gt{}; int gt_ctas = 0;                     // K0's scratch: one slot per resident guide-tree CTA
    // byte offsets of the stage's arrays in its one device block (o_seqs: none when the stage reads another stage's bases)
    int64_t o_seqs = 0, o_lens = 0, o_soff = 0, o_desc = 0, o_msa = 0, o_msa_len = 0, o_status = 0, o_cells = 0, o_next = 0, o_order = 0, o_gt_status = 0, o_gt_scratch = 0, block_bytes = 0;
    // set by fit_stage: the lane arena the buckets take
    size_t slots_bytes = 0, plane_ints = 0, clk_entries = 0;
    // a trace stage (barb200_poa_trace_batch): per job its region of the trace buffer (first word, words; trace_words_for_job), and
    // the byte offsets of the buffer, the two tables and the words each job wrote in the stage's block
    bool trace = false;
    std::vector<int64_t> trace_off, trace_cap;
    int64_t trace_words = 0, o_trace = 0, o_trace_off = 0, o_trace_cap = 0, o_trace_used = 0;
};

// The stage over the table's jobs `jobs` (caller indices) sized for (grow, worst_case), on a device of sm_count SMs; own_seqs:
// its block holds the table's bases (a capacity retry reads its first stage's); trace: the stage runs the trace kernels, and its block
// holds every job's trace region; trace_scale scales the regions below the worst case (a test aid that makes them overflow: the
// kernel's capacity check and the trace-capacity retries then run on any input). Slot layouts are planned; slots are fit_stage's.
inline StagePlan plan_stage_order(const JobTable &T, std::vector<int64_t> jobs, const barb200_params &p, double grow, bool worst_case, int sm_count,
                                  bool own_seqs, bool trace = false, double trace_scale = 1.0) {
    StagePlan S;
    S.grow = grow; S.worst_case = worst_case; S.trace = trace;
    const int64_t n_jobs = (int64_t)jobs.size();
    S.perm = std::move(jobs);
    std::stable_sort(S.perm.begin(), S.perm.end(), [&](int64_t a, int64_t b) {
        if (T.jobs[a].cls != T.jobs[b].cls) return T.jobs[a].cls > T.jobs[b].cls;
        return T.jobs[a].cost > T.jobs[b].cost;
    });
    S.desc.resize(n_jobs);
    int64_t lo = 0, msa_off = 0;
    for (int64_t j = 0; j < n_jobs; ++j) {
        const TableJob &J = T.jobs[S.perm[j]];
        const int K = J.n_seq;
        int64_t o = 0;
        for (int i = 0; i < K; ++i) { S.lens.push_back(T.lens[J.len_off + i]); S.soff.push_back(o); o += T.lens[J.len_off + i]; }
        int64_t stride = J.sum_len;
        if (!worst_case) stride = std::min<int64_t>(J.sum_len, (int64_t)(grow * (double)(J.max_len + J.max_len / 2 + 64)));
        stride = align_up(stride, 16);
        JobDesc &d = S.desc[j];
        d.n_seq = K; d.seq_off = J.seq_off; d.len_off = lo; d.msa_off = msa_off; d.msa_stride = (int)stride; d.progressive = J.progressive;
        msa_off += stride * K;
        lo += K;
        if (S.buckets.empty() || S.buckets.back().cls != J.cls) { PlanBucket B; B.cls = J.cls; B.T = kClassThreads[J.cls]; B.job_base = j; S.buckets.push_back(B); }
        S.buckets.back().n_jobs++;
    }
    const int64_t ns = S.n_seqs = lo;
    S.msa_bytes = msa_off;
    if (n_jobs == 0) return S;
    // every class's slot is sized from ITS largest job
    for (PlanBucket &B : S.buckets) {
        SlotNeeds need;
        for (int64_t j = B.job_base; j < B.job_base + B.n_jobs; ++j) {
            const TableJob &J = T.jobs[S.perm[j]];
            need.add_job(J.n_seq, J.sum_len, J.max_len, plane_ints_for_job(p.wb, p.wf, J.n_seq, J.sum_len, J.max_len, grow, worst_case));
        }
        B.lay = plan_slot(need);
    }
    GtNeeds gt_need;
    for (int64_t c : S.perm) gt_need.add_job(T.jobs[c].progressive, T.jobs[c].n_seq, T.jobs[c].sum_len, p.w, grow, worst_case);
    S.gt = plan_gt_scratch(gt_need);
    S.gt_ctas = (int)std::min<int64_t>(std::min<int64_t>(n_jobs, (int64_t)4 * sm_count), std::max<int64_t>(1, ((int64_t)2 << 30) / S.gt.slot_bytes));
    BumpOffsets sub{256};
    S.o_seqs = own_seqs ? sub.take(T.n_bases) : 0; S.o_lens = sub.take(ns * 4); S.o_soff = sub.take(ns * 8); S.o_desc = sub.take(n_jobs * sizeof(JobDesc));
    S.o_msa = sub.take(S.msa_bytes); S.o_msa_len = sub.take(n_jobs * 4); S.o_status = sub.take(n_jobs * 4); S.o_cells = sub.take(n_jobs * 8);
    S.o_next = sub.take(4 * (kNumClasses + 1)); S.o_order = sub.take(ns * 4); S.o_gt_status = sub.take(n_jobs * 4); S.o_gt_scratch = sub.take(S.gt.slot_bytes * S.gt_ctas);
    if (trace) {
        S.trace_off.resize(n_jobs); S.trace_cap.resize(n_jobs);
        for (int64_t j = 0; j < n_jobs; ++j) {
            const TableJob &J = T.jobs[S.perm[j]];
            int64_t cap = trace_words_for_job(J.n_seq, J.sum_len, J.max_len, grow, worst_case);
            if (!worst_case) cap = std::min(cap, (int64_t)(trace_scale * (double)cap));
            S.trace_off[j] = S.trace_words; S.trace_cap[j] = cap;
            S.trace_words += S.trace_cap[j];
        }
        S.o_trace = sub.take(S.trace_words * 8); S.o_trace_off = sub.take(n_jobs * 8); S.o_trace_cap = sub.take(n_jobs * 8); S.o_trace_used = sub.take(n_jobs * 8);
    }
    S.block_bytes = sub.end;
    return S;
}

// Resident CTAs and arena offsets of S's buckets: bucket b may keep per_sm[b] CTAs on each of sm_count SMs, and all slots and
// planes together must fit `budget` bytes (lane_budget_bytes). Over budget, the slots shrink; a capacity retry's planes are then
// cut (retry_plane_scale). Returns "" or the message of a plan that cannot fit even so.
inline std::string fit_stage(StagePlan &S, const std::vector<int> &per_sm, int sm_count, double budget) {
    for (size_t b = 0; b < S.buckets.size(); ++b) S.buckets[b].slots = (int)std::min<int64_t>(S.buckets[b].n_jobs, (int64_t)per_sm[b] * sm_count);
    auto need_of = [&](const PlanBucket &B) { return (double)B.slots * ((double)B.lay.slot_bytes + (double)B.lay.plane_cap * 4.0); };
    double need = 0;
    for (const PlanBucket &B : S.buckets) need += need_of(B);
    for (int pass = 0; pass < 8 && need > budget; ++pass) {
        const double scale = budget / need;
        need = 0;
        for (PlanBucket &B : S.buckets) { B.slots = std::max(1, (int)((double)B.slots * scale)); need += need_of(B); }
    }
    if (need > budget && (S.grow > 1.0 || S.worst_case)) {
        double fixed = 0, planes = 0;
        for (const PlanBucket &B : S.buckets) { fixed += (double)B.slots * (double)B.lay.slot_bytes; planes += (double)B.slots * (double)B.lay.plane_cap * 4.0; }
        const double scale = retry_plane_scale(budget, fixed, planes);
        need = 0;
        for (PlanBucket &B : S.buckets) {
            B.lay.plane_cap = (int64_t)((double)B.lay.plane_cap * scale) / 8 * 8;
            need += need_of(B);
        }
    }
    if (need > budget) {
        char buf[200];
        snprintf(buf, sizeof(buf), "a single job needs more device memory than is available (%.1f GB planned, %.1f GB usable by this lane)", need / 1e9, budget / 1e9);
        return buf;
    }
    S.slots_bytes = 0; S.plane_ints = 0; S.clk_entries = 0;
    for (PlanBucket &B : S.buckets) {
        B.slot_off = S.slots_bytes; B.plane_off = (int64_t)S.plane_ints; B.clk_off = S.clk_entries;
        S.slots_bytes += (size_t)B.lay.slot_bytes * B.slots; S.plane_ints += (size_t)B.lay.plane_cap * B.slots; S.clk_entries += (size_t)B.slots * PH_N;
    }
    return "";
}

// The capacity retry after a round of S whose jobs ended with `status` (internal order): the caller indices to re-run, with x4
// slots after the first round and at the worst case after that. "" (next.jobs empty: nothing to re-run) or the message of a job
// that failed for good.
struct RetryRound { std::vector<int64_t> jobs; double grow = 1.0; bool worst_case = false; };
inline std::string retry_round(const StagePlan &S, const std::vector<int> &status, RetryRound &next) {
    next = RetryRound();
    for (size_t j = 0; j < status.size(); ++j) {
        const int sc = status[j];
        if (sc == JOB_OK) continue;
        if (!S.worst_case && (sc == JOB_ERR_PLANE_CAP || sc == JOB_ERR_MSA_CAP || sc == JOB_ERR_GT_CAP || sc == JOB_ERR_TRACE_CAP)) {
            next.jobs.push_back(S.perm[j]);
            continue;
        }
        char buf[200];
        if (sc == JOB_ERR_PLANE_CAP)
            snprintf(buf, sizeof(buf), "job %lld needs more DP-plane memory than this lane can plan (%.1f GB of planes per slot)", (long long)S.perm[j],
                     S.buckets.empty() ? 0.0 : (double)S.buckets[0].lay.plane_cap * 4.0 / 1e9);
        else
            snprintf(buf, sizeof(buf), "job %lld failed on the device with status %d", (long long)S.perm[j], sc);
        return buf;
    }
    next.worst_case = S.grow >= 4.0;
    next.grow = next.worst_case ? 1.0 : S.grow * 4.0;
    return "";
}

// job-count / byte limits of ONE device batch (larger requests are cut into chunks)
constexpr int64_t kMaxJobsPerBatch = 1 << 15;
constexpr int64_t kMaxBasesPerBatch = (int64_t)768 << 20;
// a trace call's device batch: its jobs' first-round trace regions (trace_words_for_job) take at most 2 GB of its stage's block, which
// counts against the lane's budget (lane_budget_bytes); a larger call is cut into more device batches
constexpr int64_t kMaxTraceWordsPerBatch = (int64_t)256 << 20;

// Where the device batches of `mine` (caller indices into T) end: a chunk takes jobs in order up to kMaxJobsPerBatch jobs and
// kMaxBasesPerBatch bases, and at least one job; trace_words > 0 (a trace call): also up to that many trace words, the regions
// planned for (grow, worst_case).
inline std::vector<size_t> chunk_ends(const JobTable &T, const std::vector<int64_t> &mine, int64_t trace_words = 0, double grow = 1.0,
                                      bool worst_case = false) {
    std::vector<size_t> ends;
    for (size_t at = 0; at < mine.size();) {
        size_t end = at; int64_t bases = 0, words = 0;
        auto job_words = [&](size_t k) { const TableJob &J = T.jobs[mine[k]]; return trace_words_for_job(J.n_seq, J.sum_len, J.max_len, grow, worst_case); };
        while (end < mine.size() && (int64_t)(end - at) < kMaxJobsPerBatch &&
               (end == at || (bases + T.jobs[mine[end]].sum_len <= kMaxBasesPerBatch && (trace_words <= 0 || words + job_words(end) <= trace_words)))) {
            bases += T.jobs[mine[end]].sum_len;
            if (trace_words > 0) words += job_words(end);
            ++end;
        }
        ends.push_back(end);
        at = end;
    }
    return ends;
}

// The stages of a capacity retry `next` after a round of S: one, or for a trace stage as many as keep each one's trace regions (x4 or
// worst case) within kMaxTraceWordsPerBatch, so that a large retry is cut like a large call instead of failing the lane's budget.
inline std::vector<std::vector<int64_t>> retry_batches(const JobTable &T, const StagePlan &S, const RetryRound &next) {
    if (!S.trace) return {next.jobs};
    std::vector<std::vector<int64_t>> out;
    size_t at = 0;
    for (size_t end : chunk_ends(T, next.jobs, kMaxTraceWordsPerBatch, next.grow, next.worst_case)) {
        out.emplace_back(next.jobs.begin() + at, next.jobs.begin() + end);
        at = end;
    }
    return out;
}

// The table's jobs dealt over ndev devices, each device's share in caller order: one device takes everything; several take the
// jobs cost-sorted, each to the device with the least work so far (LPT, SURVEY.md 8e).
inline std::vector<std::vector<int64_t>> deal_jobs(const JobTable &T, int ndev) {
    const int64_t n = (int64_t)T.jobs.size();
    std::vector<std::vector<int64_t>> share(ndev);
    if (ndev == 1) { share[0] = all_jobs(n); return share; }
    std::vector<int64_t> idx = all_jobs(n);
    std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) { return T.jobs[a].cost > T.jobs[b].cost; });
    std::vector<double> load(ndev, 0.0);
    for (int64_t j : idx) { const int d = (int)(std::min_element(load.begin(), load.end()) - load.begin()); share[d].push_back(j); load[d] += T.jobs[j].cost; }
    for (auto &s : share) std::sort(s.begin(), s.end());
    return share;
}

}  // namespace barb200
