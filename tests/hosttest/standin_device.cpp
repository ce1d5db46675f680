// standin_device.cpp -- TEST-ONLY stand-in for the device layer of libbarb200 (barb200.cu), so that the no-GPU suite can run the
// product's REAL host code above it -- host_bar.cpp (C ABI of the end queue), end_queue.h, bar_windows.h -- and, through
// oracle/Makefile's libflower_standin.so, the real shims (shim/cactus_bar_shim.c incl. its bar()) under the reference's own
// flower-level code. A "device batch" is computed job by job with the host build of the product's graph code
// (hosttest_poa_msa_trace). Never shipped, never loaded by cactus_b200; the product itself has no CPU path.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <string>
#include <vector>
#include "../../cactus_b200/csrc/host_api.h"

struct HtParams { int wb; float wf; int o1, e1, o2, e2; int mat[25]; int k, w, min_w; int progressive, disable_seeding; };
extern "C" int64_t *hosttest_poa_msa_trace(const HtParams *hp, int n_seq, const int *lens, const uint8_t *flat, int64_t *n_words, int *status);

struct HtPecanParams { double threshold; int64_t minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion; };
extern "C" int64_t hosttest_pecan_aligned_pairs(const char *csx, int64_t lX, const char *csy, int64_t lY, const int64_t *anchors, int64_t n_anchor,
                                                int ragged_left, int ragged_right, const HtPecanParams *pp, int64_t split_bigger,
                                                int64_t **trip, double **post, int64_t *cells_out);

struct barb200_ctx {
    barb200_params p;
    std::mutex err_mu; std::string err;
    void *dispatcher = nullptr;
};

namespace barb200 {
static thread_local std::string tls_err;
void set_error(barb200_ctx *ctx, const std::string &msg) { if (!ctx) return; tls_err = msg; std::lock_guard<std::mutex> lk(ctx->err_mu); ctx->err = msg; }
std::string get_error(barb200_ctx *ctx) { if (!tls_err.empty()) return tls_err; std::lock_guard<std::mutex> lk(ctx->err_mu); return ctx->err; }
int host_threads(barb200_ctx *) { return 4; }
int default_progressive(barb200_ctx *ctx) { return ctx->p.progressive_poa; }
int total_lanes(barb200_ctx *) { return 2; }
void **dispatcher_slot(barb200_ctx *ctx) { return &ctx->dispatcher; }
void mark_lanes_shared(barb200_ctx *) {}
int run_jobs_on_lane(barb200_ctx *ctx, int, const std::vector<HostJob> &jobs, std::vector<JobResult> &results) {
    results.assign(jobs.size(), JobResult());
    for (size_t j = 0; j < jobs.size(); ++j) {
        HtParams q;
        q.wb = ctx->p.wb; q.wf = ctx->p.wf; q.o1 = ctx->p.gap_open1; q.e1 = ctx->p.gap_ext1; q.o2 = ctx->p.gap_open2; q.e2 = ctx->p.gap_ext2;
        memcpy(q.mat, ctx->p.mat, sizeof(q.mat)); q.k = ctx->p.k; q.w = ctx->p.w; q.min_w = ctx->p.min_w; q.progressive = jobs[j].progressive; q.disable_seeding = 1;
        int sum = 0;
        for (int i = 0; i < jobs[j].n_seq; ++i) sum += jobs[j].lens[i];
        for (int b = 0; b < sum; ++b) if (jobs[j].seqs[b] > 4) { set_error(ctx, "sequence code > 4"); return BARB200_EINVAL; }
        int64_t nw = 0; int status = 0;
        int64_t *w = hosttest_poa_msa_trace(&q, jobs[j].n_seq, jobs[j].lens, jobs[j].seqs, &nw, &status);
        if (status) { free(w); set_error(ctx, "stand-in device: job failed"); return BARB200_EJOB; }
        const int ml = (int)w[1];
        const size_t nb = (size_t)jobs[j].n_seq * ml, nwm = (nb + 7) / 8;
        results[j].msa.assign((const uint8_t *)(w + (nw - (int64_t)nwm)), (const uint8_t *)(w + (nw - (int64_t)nwm)) + nb);
        results[j].msa_len = ml; results[j].cells = w[2];
        free(w);
    }
    return BARB200_OK;
}
}  // namespace barb200

extern "C" void barb200_params_default(barb200_params *p) { barb200::params_default(p); }
extern "C" barb200_ctx *barb200_create(const barb200_params *p, char *, int) { barb200_ctx *c = new barb200_ctx(); c->p = *p; return c; }
extern "C" void barb200_destroy(barb200_ctx *ctx) { if (ctx) { barb200::dispatcher_destroy(ctx); delete ctx; } }
extern "C" const char *barb200_last_error(barb200_ctx *ctx) { static thread_local std::string out; out = ctx ? barb200::get_error(ctx) : "null context"; return out.c_str(); }
extern "C" void barb200_free(void *p) { free(p); }

// cPecan mode: every pair through the host emulation of the product's block program (hosttest_pecan_aligned_pairs)
extern "C" void barb200_pecan_params_default(barb200_pecan_params *p) {
    p->threshold = 0.01; p->min_diags_between_traceback = 1000; p->traceback_diagonals = 40; p->diagonal_expansion = 20;
    p->split_matrix_bigger_than_this = (int64_t)3000 * 3000; p->dynamic_anchor_expansion = 0;
}
extern "C" int barb200_pecan_aligned_pairs_batch(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs, const char *const *sx, const int64_t *lx,
                                                 const char *const *sy, const int64_t *ly, const int64_t *const *anchors, const int64_t *n_anchor,
                                                 const uint8_t *ragged_left, const uint8_t *ragged_right, int64_t **triples_out, int64_t *n_out,
                                                 double **posteriors_out, int64_t *cells_out) {
    HtPecanParams q{p->threshold, p->min_diags_between_traceback, p->traceback_diagonals, p->diagonal_expansion};
    for (int64_t i = 0; i < n_pairs; ++i) {
        int64_t *t = nullptr; double *po = nullptr; int64_t cells = 0;
        const int64_t n = hosttest_pecan_aligned_pairs(sx[i], lx[i], sy[i], ly[i], (anchors && n_anchor && n_anchor[i]) ? anchors[i] : nullptr, n_anchor ? n_anchor[i] : 0,
                                                       ragged_left ? ragged_left[i] : 0, ragged_right ? ragged_right[i] : 0, &q, p->split_matrix_bigger_than_this, &t, &po, &cells);
        if (n < 0) { barb200::set_error(ctx, "stand-in device: pair-HMM job failed"); return BARB200_EJOB; }
        triples_out[i] = t; n_out[i] = n;
        if (posteriors_out) posteriors_out[i] = po; else free(po);
        if (cells_out) cells_out[i] = cells;
    }
    return BARB200_OK;
}
