// trace_plan.cpp -- TEST-ONLY (tests/test_poa_trace_cpu.py compiles it): the trace call's plan (slot_plan.h: trace_words_for_job,
// stage_plan.h: the trace stage's regions, its block and its cut into device batches) on the CPU.
#include <string.h>
#include "../../cactus_b200/csrc/stage_plan.h"

using namespace barb200;

extern "C" int64_t trace_words(int64_t K, int64_t sum, int64_t ml, double grow, int worst_case) {
    return trace_words_for_job(K, sum, ml, grow, worst_case != 0);
}
// a stage over n jobs (caller order; lengths and bases back to back) with Cactus' defaults, sized for (grow, worst_case) with the
// regions scaled by `scale` (BARB200_TRACE_REGION_SCALE): per job in internal order its trace region's first word and words, and the
// stage's block bytes with trace = 0 / 1. Returns the trace words.
extern "C" int64_t trace_stage(int64_t n, const int *n_seq, const int *lens, const uint8_t *seqs, double grow, int worst_case, double scale,
                               int64_t *perm, int64_t *off, int64_t *cap, int64_t *block_bytes) {
    barb200_params p;
    params_default(&p);
    JobTable T;
    if (!table_of_arrays(p, 1, n, n_seq, lens, seqs, nullptr, T).empty()) return -1;
    const StagePlan plain = plan_stage_order(T, all_jobs(n), p, grow, worst_case != 0, 132, true);
    const StagePlan S = plan_stage_order(T, all_jobs(n), p, grow, worst_case != 0, 132, true, true, scale);
    for (int64_t j = 0; j < n; ++j) { perm[j] = S.perm[j]; off[j] = S.trace_off[j]; cap[j] = S.trace_cap[j]; }
    block_bytes[0] = plain.block_bytes; block_bytes[1] = S.block_bytes;
    return S.trace_words;
}
static JobTable shapes(int64_t n, const int *n_seq, const int64_t *sum_len, const int *max_len) {
    JobTable T;
    T.jobs.resize(n);
    for (int64_t j = 0; j < n; ++j) { T.jobs[j].n_seq = n_seq[j]; T.jobs[j].sum_len = sum_len[j]; T.jobs[j].max_len = max_len[j]; }
    return T;
}
// where the device batches of n jobs (K, bases, longest read each) end, with the trace call's limit on trace words (0: none)
extern "C" int64_t trace_chunk_ends(int64_t n, const int *n_seq, const int64_t *sum_len, const int *max_len, int64_t limit, int64_t *ends) {
    const std::vector<size_t> e = chunk_ends(shapes(n, n_seq, sum_len, max_len), all_jobs(n), limit);
    for (size_t k = 0; k < e.size(); ++k) ends[k] = (int64_t)e[k];
    return (int64_t)e.size();
}
// the stages a capacity retry of all n jobs at (grow, worst_case) runs in, after a round of a trace (or plain) stage: their sizes
extern "C" int64_t trace_retry_batches(int64_t n, const int *n_seq, const int64_t *sum_len, const int *max_len, int trace, double grow, int worst_case,
                                       int64_t *sizes) {
    StagePlan S;
    S.trace = trace != 0;
    RetryRound next;
    next.jobs = all_jobs(n); next.grow = grow; next.worst_case = worst_case != 0;
    const std::vector<std::vector<int64_t>> b = retry_batches(shapes(n, n_seq, sum_len, max_len), S, next);
    for (size_t k = 0; k < b.size(); ++k) sizes[k] = (int64_t)b[k].size();
    return (int64_t)b.size();
}
extern "C" int64_t trace_batch_limit() { return kMaxTraceWordsPerBatch; }
