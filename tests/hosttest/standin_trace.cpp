// standin_trace.cpp -- TEST-ONLY: the CPU stand-in device of standin_device.cpp plus its trace layer (run_trace_jobs), so that the
// no-GPU suite runs the product's real barb200_trace_ends (cactus_b200/csrc/host_end_trace.cpp) on top of it. Each trace job goes
// through the product's job checks (build_table) and is computed with the host build of the product's graph code
// (hosttest_poa_msa_trace), whose words have barb200_poa_trace_batch's layout. end_trace.mk builds it as libbarb200_trace_standin.so.
#include "standin_device.cpp"

extern "C" int64_t *hosttest_poa_msa_trace(const HtParams *hp, int n_seq, const int *lens, const uint8_t *flat, int64_t *n_words, int *status);

namespace barb200 {
int run_trace_jobs(barb200_ctx *ctx, const std::vector<HostJob> &jobs, std::vector<std::vector<int64_t>> &words) {
    words.assign(jobs.size(), std::vector<int64_t>());
    JobTable T;
    const std::string bad = build_table(ctx->p, 4, (int64_t)jobs.size(), [&](int64_t j, int64_t, int64_t) { return jobs[j]; }, T);
    if (!bad.empty()) { set_error(ctx, bad); return BARB200_EINVAL; }
    HtParams q;
    q.wb = ctx->p.wb; q.wf = ctx->p.wf; q.o1 = ctx->p.gap_open1; q.e1 = ctx->p.gap_ext1; q.o2 = ctx->p.gap_open2; q.e2 = ctx->p.gap_ext2;
    memcpy(q.mat, ctx->p.mat, sizeof(q.mat)); q.k = ctx->p.k; q.w = ctx->p.w; q.min_w = ctx->p.min_w; q.disable_seeding = 1;
    for (size_t c = 0; c < jobs.size(); ++c) {
        q.progressive = T.jobs[c].progressive;
        int64_t nw = 0; int status = 0;
        int64_t *w = hosttest_poa_msa_trace(&q, jobs[c].n_seq, jobs[c].lens, jobs[c].seqs, &nw, &status);
        if (status) { free(w); set_error(ctx, "stand-in device: job failed"); return BARB200_EJOB; }
        words[c].assign(w, w + nw);
        free(w);
    }
    return BARB200_OK;
}
}  // namespace barb200
