// poa_kernel.cuh -- device-side arguments of the fused batched POA kernel (see poa_kernel.cu).
#pragma once
#include "poa_types.h"
#include "slot_plan.h"

namespace barb200 {

// dynamic shared memory per CTA of each CTA-size class, sized so that the class's CTAs per SM still fit: the topological sort's
// scratch between sweeps, and during a sweep the ring of its last two rows where two rows fit (poa_kernel.cu: dp_sweep)
HD constexpr int poa_scratch_bytes(int T) {
    return T == 32 ? 10 * 1024 : T == 64 ? 24 * 1024 : T == 128 ? 40 * 1024 : T == 256 ? 96 * 1024 : 200 * 1024;
}
// bytes of the sweep's two-row ring (two rows of T threads x TB ints), 0 for a class whose scratch cannot hold it. The kernel
// decides at compile time whether a class has a ring, so its launches never get less dynamic shared memory than this
HD constexpr int poa_ring_bytes(int T) {
    return 2 * T * TB * (int)sizeof(int) <= poa_scratch_bytes(T) ? 2 * T * TB * (int)sizeof(int) : 0;
}

enum { PH_DP = 0, PH_BACKTRACK = 1, PH_FUSE = 2, PH_TOPO = 3, PH_MSA = 4, PH_TOTAL = 5, PH_N = 8 };

struct BatchArgs {
    const JobDesc *jobs;        // all jobs of the stage (internal order)
    int job_base, n_jobs;       // this launch's class: jobs [job_base, job_base + n_jobs)
    const uint8_t *seqs;        // packed 0..4 codes of all jobs
    const int *lens;            // per sequence
    const int64_t *soff;        // per sequence: offset from the job's seq_off
    const int *order;           // per sequence slot a: which read is aligned a-th (guide tree, guide_tree_kernel)
    const int *gt_status;       // per job: nonzero = the guide tree ran out of key space (the job is retried with more)
    uint8_t *msa; int *msa_len; int *status; long long *cells;
    uint8_t *slots; int *planes;
    int *next_job;              // the class's work counter
    unsigned long long *phase_clk;   // [gridDim.x * PH_N] clock64 per phase, or nullptr
    int serial_phases;          // debugging aid: 1 = run the graph phases in their serial reference form
    int bfs_order;              // debugging aid: 1 = recompute abPOA's BFS order after every fusion instead of splicing
    int scratch_bytes;          // dynamic shared memory per CTA (topological sort scratch)
    SlotLayout lay;
    PoaParams P;
};

// The trace kernels' output (poa_trace_kernel_t*, barb200_poa_trace_batch): per job of the stage (internal order), a region of
// `words` where every alignment appends its record (poa_kernel.cu: trace_record). Capacities: slot_plan.h, trace_words_for_job.
struct TraceArgs {
    int64_t *words;             // the stage's trace buffer
    const int64_t *off;         // per job: first word of its region
    const int64_t *cap;         // per job: words in its region
    int64_t *used;              // out, per job: words written (0 if the job failed)
};

// ---- K0: guide_tree_kernel (guide_tree.cu): the read order of every job of a stage, one persistent CTA per scratch slot ----
struct GuideTreeArgs {
    const JobDesc *jobs; int n_jobs;
    const uint8_t *seqs; const int *lens; const int64_t *soff;
    int *order;                 // out: per sequence slot, indexed like lens
    int *gt_status;             // out: per job, 0 or JOB_ERR_GT_CAP
    int *next_job;              // work counter
    uint8_t *scratch; GtLayout lay;             // per-CTA scratch slots
    int k, w;
};
constexpr int kGuideTreeThreads = 256;
constexpr int kGuideTreeTileKeys = 2048;        // shared-memory tile of the sort (16 KB)
void launch_guide_tree(const GuideTreeArgs &A, int ctas, void *stream);

}  // namespace barb200

