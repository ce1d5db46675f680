// guide_tree.cu -- K0: the progressive-POA read order of every job of a stage (guide_tree.cuh has the algorithm and why it equals
// abPOA's). A kernel of its own, launched ahead of the fused POA kernels on the same stream: the sketch / sort / ordering code has
// nothing in common with the DP sweep, and kept apart it cannot disturb the sweep's register allocation. Persistent CTAs of
// 256 threads pull jobs from a counter.
#include <cuda_runtime.h>
#include "poa_kernel.cuh"
#include "guide_tree.cuh"

namespace barb200 {

__global__ void __launch_bounds__(kGuideTreeThreads, 4) guide_tree_kernel(const GuideTreeArgs A) {
    __shared__ uint64_t tile[kGuideTreeTileKeys];
    __shared__ int s_job, s_n_keys;
    __shared__ double ws_v[33];
    __shared__ long long ws_i[33];
    GtScratch G = gt_views(A.lay, A.scratch + (int64_t)blockIdx.x * A.lay.slot_bytes);
    G.n_keys = &s_n_keys; G.tile = tile; G.tile_cap = kGuideTreeTileKeys;
    const GuideTreeParams GP{A.k, A.w};
    while (true) {
        if (threadIdx.x == 0) s_job = atomicAdd(A.next_job, 1);
        __syncthreads();
        const int job = s_job;
        if (job >= A.n_jobs) break;
        const JobDesc jd = A.jobs[job];
        const uint8_t *seqs = A.seqs + jd.seq_off;
        const int64_t *soff = A.soff + jd.len_off;
        const int rc = cta_guide_tree(GP, jd.progressive, jd.n_seq, [=](int i) { return seqs + soff[i]; }, A.lens + jd.len_off, A.order + jd.len_off, G, ws_v, ws_i,
                                      (int)blockDim.x);
        if (threadIdx.x == 0) A.gt_status[job] = rc < 0 ? JOB_ERR_GT_CAP : 0;
        __syncthreads();
    }
}

void launch_guide_tree(const GuideTreeArgs &A, int ctas, void *stream) {
    guide_tree_kernel<<<ctas, kGuideTreeThreads, 0, (cudaStream_t)stream>>>(A);
}

}  // namespace barb200
