// host_end_trace.cpp -- barb200_trace_ends (include/barb200.h): every sliding window of every end, as the end queue would align it,
// with each window's input slice, the per-alignment trace of its POA job and what the trimming made of it.
//
// The rounds here are synchronous and do not go through EndQueue: each round prepares the next window of every unfinished end
// (barwin::end_prepare_window), runs those windows as one trace call (run_trace_jobs: barb200_poa_trace_batch's job checks, deal over
// the devices, cut into batches and capacity retries), and hands each MSA back to its end (barwin::end_consume_window). The queue
// runs the same barwin:: steps; what it adds is only which windows share a device batch, on which lane and device. A window's
// result depends on its job alone (every job is aligned on its own in its own CTA, whatever else is in the batch), so tracing the
// window logic and the kernels covers everything that decides an output. The tests check that argument through the result: the
// final MSAs here equal barb200_make_consistent_partial_order_alignments' on the same inputs.
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "host_api.h"
#include "bar_windows.h"

using namespace barb200;

namespace {

struct WindowRecord {
    std::vector<int64_t> offsets, lens, empty;
    int64_t progressive = 0;
    std::vector<int64_t> trace;
};

// the MSA of a trace (header n_seq, msa_len, cells; the MSA packed in its last words) as the end queue's job result
JobResult result_of_trace(const std::vector<int64_t> &w) {
    JobResult r;
    const int64_t K = w[0], ml = w[1], nb = K * ml, nwm = (nb + 7) / 8;
    const uint8_t *m = (const uint8_t *)(w.data() + (w.size() - (size_t)nwm));
    r.msa.assign(m, m + nb);
    r.msa_len = (int)ml; r.cells = w[2];
    return r;
}

}  // namespace

extern "C" int barb200_trace_ends(barb200_ctx *ctx, int64_t end_no, const int64_t *end_lengths, char ***end_strings,
                                  int **end_string_lengths, int64_t **right_end_indexes, int64_t **right_end_row_indexes,
                                  int64_t **overlaps, int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff,
                                  int64_t **trace_out, int64_t *n_words) {
    if (!ctx) return BARB200_EINVAL;
    // the argument checks and messages of barb200_flower_submit
    if (end_no < 0 || (end_no > 0 && (!end_lengths || !end_strings || !end_string_lengths || !trace_out || !n_words))) {
        set_error(ctx, "bad arguments"); return BARB200_EINVAL;
    }
    for (int64_t e = 0; e < end_no; ++e) { trace_out[e] = nullptr; n_words[e] = 0; }
    if (window_size <= 0) { set_error(ctx, "window_size must be positive"); return BARB200_EINVAL; }
    std::vector<barwin::EndState> ends((size_t)end_no);
    for (int64_t e = 0; e < end_no; ++e) {
        const std::string err = barwin::end_init(ends[e], end_lengths[e], end_strings[e], end_string_lengths[e]);
        if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
    }
    const bool consistent = right_end_indexes != nullptr;
    std::vector<std::vector<int64_t>> rei, reri, ov;
    if (consistent) {
        if (!right_end_row_indexes || !overlaps) { set_error(ctx, "bad arguments"); return BARB200_EINVAL; }
        rei.resize(end_no); reri.resize(end_no); ov.resize(end_no);
        for (int64_t e = 0; e < end_no; ++e) {
            rei[e].assign(right_end_indexes[e], right_end_indexes[e] + end_lengths[e]);
            reri[e].assign(right_end_row_indexes[e], right_end_row_indexes[e] + end_lengths[e]);
            ov[e].assign(overlaps[e], overlaps[e] + end_lengths[e]);
        }
    }
    const int def_prog = default_progressive(ctx);
    std::vector<std::vector<WindowRecord>> recs((size_t)end_no);
    for (;;) {
        std::vector<HostJob> jobs; std::vector<int64_t> owner;
        for (int64_t e = 0; e < end_no; ++e) {
            barwin::EndState &E = ends[e];
            if (E.done) continue;
            HostJob job;
            const std::string err = barwin::end_prepare_window(E, window_size, def_prog, max_prog_rows, max_prog_length_diff, job);
            if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
            WindowRecord r;
            r.offsets = E.offsets;
            r.lens.assign(E.cur_lens.begin(), E.cur_lens.end());
            r.empty.assign(E.empty.begin(), E.empty.end());
            r.progressive = E.cur_progressive;
            recs[e].push_back(std::move(r));
            jobs.push_back(job); owner.push_back(e);
        }
        if (jobs.empty()) break;
        std::vector<std::vector<int64_t>> words;
        const int rc = run_trace_jobs(ctx, jobs, words);
        if (rc) return rc;
        for (size_t k = 0; k < jobs.size(); ++k) {
            barwin::EndState &E = ends[owner[k]];
            JobResult res = result_of_trace(words[k]);
            recs[owner[k]].back().trace.swap(words[k]);
            const std::string err = barwin::end_consume_window(E, res);
            if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
        }
    }
    // stitch and trim across ends exactly as barb200_flower_wait does
    std::vector<barb200_msa *> msas((size_t)end_no, nullptr);
    auto release = [&]() { for (barb200_msa *m : msas) barb200_msa_destruct(m); };
    for (int64_t e = 0; e < end_no; ++e)
        if (!(msas[e] = barwin::end_stitch(ends[e]))) { release(); set_error(ctx, "host allocation failed"); return BARB200_ENOMEM; }
    if (consistent && !barwin::consistency_trim(end_no, msas.data(), rei, reri, ov)) {
        release(); set_error(ctx, "inconsistent end / row indexes or overlaps"); return BARB200_EINVAL;
    }
    for (int64_t e = 0; e < end_no; ++e) {
        const barwin::EndState &E = ends[e];
        const int64_t K = E.seq_no, nwin = (int64_t)recs[e].size();
        int64_t n = 2;
        for (const WindowRecord &r : recs[e]) n += 1 + 3 * K + 1 + 1 + (int64_t)r.trace.size() + K + 1;
        const int64_t nb = K * msas[e]->column_no, nwm = (nb + 7) / 8;
        n += 2 + nwm;
        int64_t *w = (int64_t *)malloc((size_t)n * 8);
        if (!w) {
            for (int64_t f = 0; f < e; ++f) { free(trace_out[f]); trace_out[f] = nullptr; n_words[f] = 0; }
            release(); set_error(ctx, "host allocation failed"); return BARB200_ENOMEM;
        }
        int64_t p = 0;
        w[p++] = K; w[p++] = nwin;
        for (int64_t k = 0; k < nwin; ++k) {
            const WindowRecord &r = recs[e][k];
            const barwin::Window &win = *E.windows[k];
            w[p++] = k;
            for (int64_t i = 0; i < K; ++i) w[p++] = r.offsets[i];
            for (int64_t i = 0; i < K; ++i) w[p++] = r.lens[i];
            for (int64_t i = 0; i < K; ++i) w[p++] = r.empty[i];
            w[p++] = r.progressive;
            w[p++] = (int64_t)r.trace.size();
            memcpy(w + p, r.trace.data(), r.trace.size() * 8); p += (int64_t)r.trace.size();
            for (int64_t i = 0; i < K; ++i) w[p++] = win.seq_lens[i];      // after the trims against both neighbours
            w[p++] = win.column_no;
        }
        w[p++] = K; w[p++] = msas[e]->column_no;
        if (nwm) w[n - 1] = 0;
        memcpy(w + p, msas[e]->msa, (size_t)nb);
        trace_out[e] = w; n_words[e] = n;
    }
    release();
    return BARB200_OK;
}
