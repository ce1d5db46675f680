// host_api.h -- internal C++ interfaces between the host-side translation units of libbarb200.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/barb200.h"

namespace barb200 {

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
int total_lanes(barb200_ctx *ctx);
void **dispatcher_slot(barb200_ctx *ctx);         // where host_bar.cpp keeps the context's end queue
void mark_lanes_shared(barb200_ctx *ctx);
void dispatcher_destroy(barb200_ctx *ctx);
void set_error(barb200_ctx *ctx, const std::string &msg);
std::string get_error(barb200_ctx *ctx);
int host_threads(barb200_ctx *ctx);
int default_progressive(barb200_ctx *ctx);
// context facts for pecan.cu, which runs the pair-HMM work on the context's first device
int ctx_device(barb200_ctx *ctx);
int ctx_sm_count(barb200_ctx *ctx);
double ctx_mem_fraction(barb200_ctx *ctx);
// device blocks from the first device's grow-only cache (cudaMalloc / cudaFree per call cost milliseconds); 0 on success
int device_alloc(barb200_ctx *ctx, void **p, size_t bytes);
void device_free(barb200_ctx *ctx, void *p, size_t bytes);
// pinned host blocks from the first device's pool (pinned_take: nullptr if cudaMallocHost fails; *got = the block's size)
void *pinned_take(barb200_ctx *ctx, size_t bytes, size_t *got);
void pinned_give(barb200_ctx *ctx, void *p, size_t bytes);
// pecan.cu: the context's pair-HMM state (streams, ring scratch, batch group commit), made by barb200_create on the first device
void **pecan_slot(barb200_ctx *ctx);
int pecan_create(barb200_ctx *ctx);            // 0 on success; the slot is set either way, so barb200_destroy cleans up
void pecan_destroy(barb200_ctx *ctx);

}  // namespace barb200

// in a .cu function that returns a BARB200_* code: a failed CUDA call sets the context's message and returns BARB200_ECUDA
#define CUDA_TRY(ctx, call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { \
    set_error(ctx, std::string(#call) + ": " + cudaGetErrorString(_e)); return BARB200_ECUDA; } } while (0)
