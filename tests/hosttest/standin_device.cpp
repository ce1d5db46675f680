// standin_device.cpp -- TEST-ONLY stand-in for the device layer of libbarb200 (barb200.cu), so that the no-GPU suite can run the
// product's REAL host code above it -- host_bar.cpp (C ABI of the end queue), end_queue.h, bar_windows.h -- and, through
// oracle/Makefile's libflower_standin.so, the real shims (shim/cactus_bar_shim.c incl. its bar()) under the reference's own
// flower-level code. A "device batch" goes through the product's job checks and stage order and is computed job by job with the
// host build of the product's graph code (hosttest.cpp: hosttest_device_batch). Never shipped, never loaded by cactus_b200; the
// product itself has no CPU path.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <string>
#include <vector>
#include "../../cactus_b200/csrc/host_api.h"
#include "../../cactus_b200/csrc/stage_plan.h"

struct HtParams { int wb; float wf; int o1, e1, o2, e2; int mat[25]; int k, w, min_w; int progressive, disable_seeding; };
int hosttest_device_batch(const HtParams &hp, int threads_per_block, const std::vector<barb200::HostJob> &jobs, std::vector<barb200::JobResult> &res,
                          std::string &err);

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
    HtParams q;
    q.wb = ctx->p.wb; q.wf = ctx->p.wf; q.o1 = ctx->p.gap_open1; q.e1 = ctx->p.gap_ext1; q.o2 = ctx->p.gap_open2; q.e2 = ctx->p.gap_ext2;
    memcpy(q.mat, ctx->p.mat, sizeof(q.mat)); q.k = ctx->p.k; q.w = ctx->p.w; q.min_w = ctx->p.min_w; q.progressive = ctx->p.progressive_poa; q.disable_seeding = 1;
    std::string err;
    const int rc = hosttest_device_batch(q, ctx->p.threads_per_block, jobs, results, err);
    if (rc) set_error(ctx, err);
    return rc;
}
}  // namespace barb200

extern "C" void barb200_params_default(barb200_params *p) { barb200::params_default(p); }
extern "C" barb200_ctx *barb200_create(const barb200_params *p, char *errbuf, int errbuf_len) {
    const std::string bad = p ? barb200::check_params(*p) : "null params";
    if (!bad.empty()) { if (errbuf && errbuf_len > 0) snprintf(errbuf, errbuf_len, "%s", bad.c_str()); return nullptr; }
    barb200_ctx *c = new barb200_ctx(); c->p = *p; return c;
}
extern "C" void barb200_destroy(barb200_ctx *ctx) { if (ctx) { barb200::dispatcher_destroy(ctx); delete ctx; } }
extern "C" const char *barb200_last_error(barb200_ctx *ctx) { static thread_local std::string out; out = ctx ? barb200::get_error(ctx) : "null context"; return out.c_str(); }
extern "C" void barb200_free(void *p) { free(p); }

// cPecan mode: every pair through the host emulation of the product's block program (hosttest_pecan_aligned_pairs)
extern "C" void barb200_pecan_params_default(barb200_pecan_params *p) { barb200::pecan_params_default(p); }
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
