// host_api.h -- internal C++ interfaces between the host-side translation units of libbarb200.
#pragma once
#include <stdint.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/barb200.h"

namespace barb200 {

// barb200_params_default: Cactus' defaults, every field not set here 0
inline void params_default(barb200_params *p) {
    static const int mat[25] = {91, -114, -61, -123, -100, -114, 100, -125, -61, -100, -61, -125, 100, -114, -100,
                                -123, -61, -114, 91, -100, -100, -100, -100, -100, 100};
    memset(p, 0, sizeof(*p));
    memcpy(p->mat, mat, sizeof(mat));
    p->gap_open1 = 400; p->gap_ext1 = 30; p->gap_open2 = 1200; p->gap_ext2 = 1;
    p->wb = 1000; p->wf = 0.1f;
    p->k = 15; p->w = 5; p->min_w = 500;
    p->progressive_poa = 1; p->disable_seeding = 1;
}
// barb200_pecan_params_default: pairwiseAlignmentBandingParameters_construct, pairwiseAligner.c:1369-1391
inline void pecan_params_default(barb200_pecan_params *p) {
    memset(p, 0, sizeof(*p));
    p->threshold = 0.01; p->min_diags_between_traceback = 1000; p->traceback_diagonals = 40; p->diagonal_expansion = 20;
    p->split_matrix_bigger_than_this = (int64_t)3000 * 3000; p->dynamic_anchor_expansion = 0;
}

struct HostParams {
    int k, w, min_w, progressive_poa;
};

// One POA job on the host side: views into caller memory (codes 0..4).
struct HostJob {
    int n_seq;
    const int *lens;          // [n_seq]
    const uint8_t *seqs;      // concatenated
    int progressive;
};

struct JobResult {
    std::vector<uint8_t> msa; // n_seq * msa_len
    int msa_len = 0;
    int64_t cells = 0;
};

// barb200.cu: one device batch of host jobs on device lane `lane` (0 .. total_lanes-1; bucketed by CTA class, capacity misses
// retried with larger slots). Returns a BARB200_* code; the message is get_error(ctx).
int run_jobs_on_lane(barb200_ctx *ctx, int lane, const std::vector<HostJob> &jobs, std::vector<JobResult> &results);
// barb200.cu: host jobs as trace jobs, through barb200_poa_trace_batch (its job checks, deal over the context's devices, batches and
// capacity retries); words[j] = job j's trace in that call's layout (include/barb200.h). barb200_trace_ends' device layer.
int run_trace_jobs(barb200_ctx *ctx, const std::vector<HostJob> &jobs, std::vector<std::vector<int64_t>> &words);
int total_lanes(barb200_ctx *ctx);
void **dispatcher_slot(barb200_ctx *ctx);         // where host_bar.cpp keeps the context's end queue
void mark_lanes_shared(barb200_ctx *ctx);
void dispatcher_destroy(barb200_ctx *ctx);
void set_error(barb200_ctx *ctx, const std::string &msg);
std::string get_error(barb200_ctx *ctx);
int host_threads(barb200_ctx *ctx);
int default_progressive(barb200_ctx *ctx);
// context facts for pecan.cu and mum_anchor.cu, which run cPecan mode's work on the context's devices 0 .. ctx_device_count - 1
int ctx_device_count(barb200_ctx *ctx);
int ctx_device(barb200_ctx *ctx, int dev);     // the CUDA ordinal of the context's device `dev`
int ctx_sm_count(barb200_ctx *ctx, int dev);
double ctx_mem_fraction(barb200_ctx *ctx);
// device blocks from device `dev`'s grow-only cache (cudaMalloc / cudaFree per call cost milliseconds); 0 on success
int device_alloc(barb200_ctx *ctx, int dev, void **p, size_t bytes);
void device_free(barb200_ctx *ctx, int dev, void *p, size_t bytes);
// pinned host blocks from device `dev`'s pool (pinned_take: nullptr if cudaMallocHost fails; *got = the block's size)
void *pinned_take(barb200_ctx *ctx, int dev, size_t bytes, size_t *got);
void pinned_give(barb200_ctx *ctx, int dev, void *p, size_t bytes);
// a host thread that runs one device's share of a batch over `n` devices takes 1/n of host_threads() (1: all of them)
void set_host_thread_share(int n);
// pecan.cu: the context's pair-HMM state (per device: streams, ring scratch; one batch group commit), made by barb200_create
void **pecan_slot(barb200_ctx *ctx);
int pecan_create(barb200_ctx *ctx);            // 0 on success; the slot is set either way, so barb200_destroy cleans up
void pecan_destroy(barb200_ctx *ctx);
void pecan_count_mum_pairs(barb200_ctx *ctx, int dev, int64_t n);   // barb200_pecan_device_stats' MUM-anchor count

}  // namespace barb200

// in a .cu function that returns a BARB200_* code: a failed CUDA call sets the context's message and returns BARB200_ECUDA
#define CUDA_TRY(ctx, call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { \
    set_error(ctx, std::string(#call) + ": " + cudaGetErrorString(_e)); return BARB200_ECUDA; } } while (0)
