// pecan.cu -- cPecan mode of libbarb200: the batched banded pair-HMM kernel (one thread block per job, pecan_cta.cuh),
// its host orchestration and the C ABI declared in include/barb200.h (barb200_pecan_*).
//
// A *stage* takes n sequence pairs with their anchors, splits each pair at large anchor gaps, builds the anchor band of
// every sub-matrix and the traceback schedule on host threads (pecan_plan.cpp), packs everything, uploads it once and
// launches persistent blocks that pull jobs (largest first) from a device counter. Two block shapes: jobs whose widest
// diagonal has <= 96 cells run in 32-thread blocks (24 per SM), all others in 128-thread blocks (6 per SM) whose diagonal
// ring keeps 320 positions in shared memory and spills the flanks of wider diagonals to an HBM/L2 overflow block (a per-job
// shift centres the band on the shared part, pecan_cta.cuh). The two launches run concurrently on their own streams.
// Each resident block owns a slot of its device's ring scratch in HBM (PecanContext: rings, streams, one run at a time) for
// the forward MATCH ring, the ring of complete forward cells and the overflow. Candidate pairs (x, y, log posterior) are
// appended by the kernel, put into the reference's order of emission on the host, compacted on the device, copied back once
// and finished on the host with libm's exp (the same function the reference calls), threshold and floor. No CPU fallback:
// the DP only exists as the CUDA kernel below.
// Every device of the context has its own PecanContext. The batch call on a context of several devices deals whole pairs to
// the devices by their planned cells and runs each device's share on a host thread of its own (pecan_batch_devices); the
// staged form runs on the context's first device.
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>
#include <omp.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>
#include "host_api.h"
#include "batch_merge.h"
#include "pecan_plan.h"
#include "pecan_cta.cuh"

using namespace barb200;
using namespace barb200::pecan;

namespace barb200 {
namespace pecan {

struct KernelArgs {
    const Job *jobs;
    const int *order;          // job indices of this launch, largest first
    int n_jobs;
    const uint8_t *sym;
    const DiagMeta *meta;
    Pair *out;
    int *out_n;
    unsigned *counter;
    const double *consts;
    double *scratch;           // per block: FM ring (maskM + 1), FF ring (maskF + 1), ring overflow 10 * (RW - RWs), tbuf overflow (RW - RWs)
    size_t slot_doubles;
    unsigned maskM, maskF;
    int RW, RWs;
    Params P;
};

// dynamic shared memory: constants | total | ring 10 * RWs | tbuf RWs
template <int kMinBlocks> __device__ __forceinline__ void pecan_posterior_body(const KernelArgs &A) {
    extern __shared__ double smem[];
    double *K = smem;
    for (int i = threadIdx.x; i < K_TOTAL; i += blockDim.x) K[i] = A.consts[i];
    __shared__ unsigned next_job;
    __shared__ int n_out;
    CtaMem cm;
    cm.total = smem + K_TOTAL;
    cm.n_out = &n_out;
    cm.RW = A.RW; cm.RWs = A.RWs; cm.T = (int)blockDim.x;
    cm.FM = A.scratch + (size_t)blockIdx.x * A.slot_doubles; cm.maskM = A.maskM;
    cm.FF = cm.FM + (size_t)A.maskM + 1; cm.maskF = A.maskF;
    cm.ring = smem + K_TOTAL + 2; cm.tbuf = cm.ring + 10 * (size_t)A.RWs;
    cm.ring_o = cm.FF + (size_t)A.maskF + 1; cm.tbuf_o = cm.ring_o + 10 * (size_t)(A.RW - A.RWs);
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) next_job = atomicAdd(A.counter, 1u);
        __syncthreads();
        const unsigned idx = next_job;
        if (idx >= (unsigned)A.n_jobs) break;
        const int j = A.order[idx];
        const Job J = A.jobs[j];
        const int n = run_job(J, A.sym, A.meta, cm, A.P, K, A.out);
        if (threadIdx.x == 0) A.out_n[j] = n;
    }
}

// two register budgets: 80 registers (up to 3 x 256 threads per SM) and 64 registers (up to 4 x 256)
extern "C" __global__ void __launch_bounds__(256, 3) pecan_posterior_kernel(const KernelArgs A) { pecan_posterior_body<3>(A); }
extern "C" __global__ void __launch_bounds__(256, 4) pecan_posterior_kernel_r64(const KernelArgs A) { pecan_posterior_body<4>(A); }

// one CTA per job: copy its records to their place in the compact array
extern "C" __global__ void pecan_compact_kernel(const Job *jobs, const int *out_n, const long long *dst_off, const Pair *out, Pair *dst, int n_jobs) {
    for (int j = blockIdx.x; j < n_jobs; j += gridDim.x) {
        const long long d0 = dst_off[j], n = dst_off[j + 1] - d0;
        const Pair *src = out + jobs[j].out_off;
        for (long long i = threadIdx.x; i < n; i += blockDim.x) dst[d0 + i] = src[i];
    }
}

}  // namespace pecan
}  // namespace barb200

// Block-shape classes by the widest diagonal (file header), chosen by a sweep of alternatives on the benchmark workload. Shared
// memory per block = 8 * (58 + 11 * rws) bytes: 8.9 KB for the narrow shape, 28.6 KB for the general one; 80 registers.
struct Class { int max_w, threads, ctas_per_sm, rws; };
static const Class kClass[] = {{96, 32, 24, 96}, {INT_MAX, 128, 6, 320}};
static const int kNumClasses = 2;

// The pair-HMM state of one device of a context (pecan_create). `mu` is held by every use of the device below -- a stage's
// upload, run and collect, and a batch chunk from create to collect -- so one run at a time owns the streams, the events and
// the ring scratch.
struct PecanContext {
    std::mutex mu;
    double *scratch = nullptr; size_t scratch_bytes = 0;   // grow-only rings (tens of GB: cudaMalloc of that size costs ~0.2 s)
    cudaStream_t stream = nullptr, cls[kNumClasses] = {};
    cudaEvent_t done[kNumClasses] = {}, ev0 = nullptr, ev1 = nullptr;
    std::atomic<int64_t> hmm_pairs{0}, mum_pairs{0};      // pairs the batch calls ran here (barb200_pecan_device_stats)
};
// The context's cPecan state: one PecanContext per device, and one queue for concurrent barb200_pecan_aligned_pairs_batch
// callers, whose requests merge into one batch that the leader spreads over the devices.
struct PecanState {
    GroupCommit<PecanRequest> group;
    std::vector<std::unique_ptr<PecanContext>> devs;
};
static PecanState &pecan_state(barb200_ctx *ctx) { return *(PecanState *)*pecan_slot(ctx); }
static PecanContext &pecan_of(barb200_ctx *ctx, int dev) { return *pecan_state(ctx).devs[dev]; }

namespace barb200 {
int pecan_create(barb200_ctx *ctx) {
    PecanState *ps = new PecanState();
    *pecan_slot(ctx) = ps;
    bool ok = true;
    for (int d = 0; d < ctx_device_count(ctx) && ok; ++d) {
        PecanContext *pc = new PecanContext();
        ps->devs.emplace_back(pc);
        if (cudaSetDevice(ctx_device(ctx, d)) != cudaSuccess) { ok = false; break; }
        cudaFuncSetAttribute(pecan_posterior_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(pecan_posterior_kernel_r64, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        // wider classes hold longer jobs: they are launched first and at higher priority so that they are resident from the start
        int prio_lo = 0, prio_hi = 0;
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
        ok = cudaStreamCreateWithFlags(&pc->stream, cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreate(&pc->ev0) == cudaSuccess && cudaEventCreate(&pc->ev1) == cudaSuccess;
        for (int c = 0; c < kNumClasses && ok; ++c)
            ok = cudaStreamCreateWithPriority(&pc->cls[c], cudaStreamNonBlocking, kClass[c].threads <= 32 ? prio_lo : prio_hi) == cudaSuccess &&
                 cudaEventCreateWithFlags(&pc->done[c], cudaEventDisableTiming) == cudaSuccess;
    }
    cudaSetDevice(ctx_device(ctx, 0));
    return ok ? 0 : -1;
}

void pecan_destroy(barb200_ctx *ctx) {
    PecanState *ps = (PecanState *)*pecan_slot(ctx);
    if (!ps) return;
    for (size_t d = 0; d < ps->devs.size(); ++d) {
        PecanContext *pc = ps->devs[d].get();
        cudaSetDevice(ctx_device(ctx, (int)d));
        if (pc->scratch) cudaFree(pc->scratch);
        for (int c = 0; c < kNumClasses; ++c) { if (pc->cls[c]) cudaStreamDestroy(pc->cls[c]); if (pc->done[c]) cudaEventDestroy(pc->done[c]); }
        if (pc->ev0) cudaEventDestroy(pc->ev0);
        if (pc->ev1) cudaEventDestroy(pc->ev1);
        if (pc->stream) cudaStreamDestroy(pc->stream);
    }
    cudaSetDevice(ctx_device(ctx, 0));
    delete ps;
}

void pecan_count_mum_pairs(barb200_ctx *ctx, int dev, int64_t n) { pecan_of(ctx, dev).mum_pairs += n; }
}  // namespace barb200

// a host staging buffer from the device's pinned pool, so that the copy runs at link speed; pageable memory if the pool cannot grow
struct Staging {
    barb200_ctx *ctx; int dev; void *pin = nullptr; size_t got = 0; std::vector<uint8_t> own;
    Staging(barb200_ctx *c, int d) : ctx(c), dev(d) {}
    ~Staging() { release(); }
    Staging(const Staging &) = delete; Staging &operator=(const Staging &) = delete;
    void *take(size_t bytes) {
        pin = pinned_take(ctx, dev, bytes, &got);
        if (pin) return pin;
        own.resize(bytes);
        return own.data();
    }
    void release() { pinned_give(ctx, dev, pin, got); pin = nullptr; std::vector<uint8_t>().swap(own); }
};

struct PecanGroup {              // one launch: a class of jobs with one block shape
    std::vector<int> jobs;       // largest first
    int cls = 0;                 // index into kClass
    int ctas = 0;                // resident blocks = slots
    int RW = 32, RWs = 32;       // ring width (the modulus) and its shared-memory part
    unsigned capM = 1024, capF = 1024;   // ring doubles (powers of two)
    size_t slot_doubles = 0, smem_bytes = 0, scratch_off = 0;
    int order_off = 0;           // into d_order
};

struct barb200_pecan_stage {
    barb200_ctx *ctx = nullptr;
    int dev = 0;                                 // the context's device the stage lives on (the staged C ABI: always 0)
    PlanParams P;
    Params devP;
    int64_t n_pairs = 0;
    bool full_cap = false;                       // retry stage: room for every cell
    std::vector<SubJob> subs;                    // in pair order
    std::vector<int64_t> pair_first;             // subs of pair i: [pair_first[i], pair_first[i+1])
    std::vector<Job> jobs;
    std::vector<PecanGroup> groups;
    int64_t cells = 0, launches = 0;
    size_t scratch_bytes = 0;                    // the rings a run takes from the context's scratch
    // device; a retry stage reads its parent's d_sym, d_meta and d_consts
    uint8_t *d_sym = nullptr; DiagMeta *d_meta = nullptr; int *d_order = nullptr, *d_out_n = nullptr;
    Job *d_jobs = nullptr; Pair *d_out = nullptr; unsigned *d_counter = nullptr; double *d_consts = nullptr;
    bool ran = false;
    struct Block { void *p; size_t bytes; };
    std::vector<Block> blocks;                   // the stage's own device arrays, from the context's block cache
};

extern "C" void barb200_pecan_params_default(barb200_pecan_params *p) { pecan_params_default(p); }

static inline int sym_of(char c) {       // symbol_convertCharToSymbol, pairwiseAligner.c:327-344
    switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; }
}

static unsigned pow2ceil(uint64_t v) { uint64_t p = 1024; while (p < v) p <<= 1; return (unsigned)p; }

extern "C" void barb200_pecan_stage_destroy(barb200_pecan_stage *st) {
    if (!st) return;
    cudaSetDevice(ctx_device(st->ctx, st->dev));
    for (auto &b : st->blocks) device_free(st->ctx, st->dev, b.p, b.bytes);
    delete st;
}

static int plan_params(barb200_ctx *ctx, const barb200_pecan_params *p, PlanParams &P) {
    if (!p) { set_error(ctx, "null pecan params"); return BARB200_EINVAL; }
    if (p->dynamic_anchor_expansion) { set_error(ctx, "dynamicAnchorExpansion is not supported (Cactus never sets it)"); return BARB200_EINVAL; }
    P.threshold = p->threshold; P.min_diags = p->min_diags_between_traceback; P.tb_diags = p->traceback_diagonals;
    P.expansion = p->diagonal_expansion; P.split_bigger = p->split_matrix_bigger_than_this;
    const std::string e = check_params(P);
    if (!e.empty()) { set_error(ctx, e); return BARB200_EINVAL; }
    return BARB200_OK;
}

// Build the device side of a stage from st->subs (already split, not yet planned unless bandL is filled). A fresh stage packs
// the caller's strings (sx, sy) and the band tables straight into one staging block and uploads them. A retry stage re-runs
// jobs of `parent` with room for every cell: its jobs are copies of the parent's and still index the parent's symbols and band
// tables on the device, so it uploads only its job table and launch order.
static int stage_build(barb200_pecan_stage *st, const char *const *sx, const char *const *sy, const barb200_pecan_stage *parent) {
    barb200_ctx *ctx = st->ctx;
    const int dev = st->dev;
    PecanContext &pc = pecan_of(ctx, dev);
    const int64_t ns = (int64_t)st->subs.size();
    std::string err;
    const int nthr = host_threads(ctx);
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthr)
    for (int64_t i = 0; i < ns; ++i) {
        if (!st->subs[i].bandL.empty()) continue;
        const std::string e = plan_subjob(st->P, st->subs[i]);
        if (!e.empty()) {
#pragma omp critical
            err = e;
        }
    }
    if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
    // offsets
    st->jobs.resize(ns);
    int64_t sym_off = 0, band_off = 0, out_off = 0, cells = 0;
    for (int64_t i = 0; i < ns; ++i) {
        SubJob &s = st->subs[i];
        Job &J = st->jobs[i];
        if (!parent) { J.sx_off = sym_off; J.sy_off = sym_off + s.lx; J.band_off = band_off; J.lx = s.lx; J.ly = s.ly; J.ragged = s.ragged; }
        sym_off += (int64_t)s.lx + s.ly; band_off += (int64_t)s.lx + s.ly + 2;
        const int64_t cap = st->full_cap ? s.cells : std::min<int64_t>(s.cells, (int64_t)s.lx + s.ly + 64);
        s.out_cap = (int)cap; J.out_cap = (int)cap; J.out_off = out_off; out_off += cap;
        cells += s.cells;
    }
    st->cells = cells;
    // classes by the widest diagonal (kClass)
    cudaSetDevice(ctx_device(ctx, dev));
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(ctx, cudaMemGetInfo(&free_b, &total_b));
    const size_t fixed = (size_t)sym_off + (size_t)band_off * 16 + (size_t)ns * (sizeof(Job) + 8) + (size_t)out_off * sizeof(Pair) * 2 + (64 << 20);
    if ((double)fixed > ctx_mem_fraction(ctx) * (double)free_b) { set_error(ctx, "pecan stage does not fit in device memory; submit fewer pairs per call"); return BARB200_ENOMEM; }
    size_t budget = (size_t)(ctx_mem_fraction(ctx) * (double)free_b) - fixed;
    st->groups.clear();
    for (int c = 0; c < kNumClasses; ++c) {
        PecanGroup g;
        for (int64_t i = 0; i < ns; ++i) if (st->subs[i].max_w <= kClass[c].max_w && (c == 0 || st->subs[i].max_w > kClass[c - 1].max_w)) g.jobs.push_back((int)i);
        if (g.jobs.empty()) continue;
        int64_t spanM = 1, spanF = 1; int rw = 1;
        for (int j : g.jobs) { spanM = std::max(spanM, st->subs[j].span_cells); spanF = std::max(spanF, st->subs[j].span_full_cells); rw = std::max(rw, st->subs[j].max_w); }
        g.cls = c;
        g.RWs = kClass[c].rws; g.RW = std::max(g.RWs, rw);
        for (int j : g.jobs) st->jobs[j].ring_shift = st->subs[j].ring_center - g.RWs / 2;
        g.capM = pow2ceil((uint64_t)spanM); g.capF = pow2ceil((uint64_t)5 * (uint64_t)spanF);
        g.slot_doubles = (size_t)g.capM + g.capF + 11 * (size_t)(g.RW - g.RWs) + 8;
        g.smem_bytes = sizeof(double) * (K_TOTAL + 2 + 11 * (size_t)g.RWs);
        g.ctas = (int)std::min<int64_t>((int64_t)ctx_sm_count(ctx, dev) * kClass[c].ctas_per_sm, (int64_t)g.jobs.size());
        std::sort(g.jobs.begin(), g.jobs.end(), [&](int a, int b) { return st->subs[a].cells != st->subs[b].cells ? st->subs[a].cells > st->subs[b].cells : a < b; });
        st->groups.push_back(std::move(g));
    }
    // the classes run concurrently, so their slots are disjoint; shrink block counts (largest slots first) if memory is short
    for (;;) {
        size_t need = 0;
        for (PecanGroup &g : st->groups) need += g.slot_doubles * 8 * (size_t)g.ctas;
        if (need <= budget) break;
        PecanGroup *big = nullptr;
        for (PecanGroup &g : st->groups) if (g.ctas > 1 && (!big || g.slot_doubles * g.ctas > big->slot_doubles * big->ctas)) big = &g;
        if (!big) { set_error(ctx, "a pair-HMM job needs more device memory than is available"); return BARB200_ENOMEM; }
        big->ctas = std::max(1, big->ctas * 3 / 4);
    }
    size_t scratch_doubles = 0; int order_off = 0;
    std::vector<int> order((size_t)std::max<int64_t>(ns, 1));
    for (PecanGroup &g : st->groups) {
        g.scratch_off = scratch_doubles; scratch_doubles += g.slot_doubles * (size_t)g.ctas;
        g.order_off = order_off;
        for (int j : g.jobs) order[order_off++] = j;
    }
    st->scratch_bytes = std::max<size_t>(scratch_doubles * 8, 8);
    if (getenv("BARB200_DEBUG"))
        for (const PecanGroup &g : st->groups)
            fprintf(stderr, "[barb200] pecan class: %zu jobs, %d threads x %d blocks, ring %d of which %d shared, FM ring %u, FF ring %u doubles, smem %zu B\n",
                    g.jobs.size(), kClass[g.cls].threads, g.ctas, g.RW, g.RWs, g.capM, g.capF, g.smem_bytes);
    // device arrays
    auto dev_alloc = [&](void **p, size_t bytes) -> bool {
        if (device_alloc(ctx, dev, p, bytes) != 0) return false;
        st->blocks.push_back(barb200_pecan_stage::Block{*p, bytes});
        return true;
    };
    const size_t ns1 = (size_t)std::max<int64_t>(ns, 1), meta_bytes = ((size_t)band_off + 1) * sizeof(DiagMeta);
    if (parent) { st->d_sym = parent->d_sym; st->d_meta = parent->d_meta; st->d_consts = parent->d_consts; }
    if ((!parent && (!dev_alloc((void **)&st->d_meta, meta_bytes + (size_t)std::max<int64_t>(sym_off, 1)) || !dev_alloc((void **)&st->d_consts, sizeof(Consts)))) ||
        !dev_alloc((void **)&st->d_order, order.size() * sizeof(int)) || !dev_alloc((void **)&st->d_out_n, ns1 * sizeof(int)) ||
        !dev_alloc((void **)&st->d_jobs, ns1 * sizeof(Job)) || !dev_alloc((void **)&st->d_out, (size_t)std::max<int64_t>(out_off, 1) * sizeof(Pair)) ||
        !dev_alloc((void **)&st->d_counter, sizeof(unsigned) * (st->groups.size() + 1))) {
        set_error(ctx, "device allocation failed (pecan stage)"); return BARB200_ENOMEM;
    }
    if (!parent) st->d_sym = (uint8_t *)st->d_meta + meta_bytes;
    Staging up(ctx, dev);
    Consts C; fill_constants(C);
    DiagMeta *meta = nullptr;                    // band tables, then symbols 0..4: the layout of d_meta / d_sym
    if (!parent) {
        meta = (DiagMeta *)up.take(meta_bytes + (size_t)sym_off);
        uint8_t *const sym = (uint8_t *)meta + meta_bytes;
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthr)
        for (int64_t i = 0; i < ns; ++i) {
            const SubJob &s = st->subs[i];
            const Job &J = st->jobs[i];
            const char *px = sx[s.pair] + s.x1, *py = sy[s.pair] + s.y1;
            for (int k = 0; k < s.lx; ++k) sym[J.sx_off + k] = (uint8_t)sym_of(px[k]);
            for (int k = 0; k < s.ly; ++k) sym[J.sy_off + k] = (uint8_t)sym_of(py[k]);
            const int D = s.lx + s.ly;
            for (int d = 0; d <= D + 1; ++d) meta[J.band_off + d] = DiagMeta{d <= D ? s.bandL[d] : 0, s.coff[d], s.foff[d], 0};
        }
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(st->d_order, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice, pc.stream));
    if (ns) CUDA_TRY(ctx, cudaMemcpyAsync(st->d_jobs, st->jobs.data(), (size_t)ns * sizeof(Job), cudaMemcpyHostToDevice, pc.stream));
    if (!parent) {     // last and in one copy: no copy from the staging block is in flight when an earlier one fails
        CUDA_TRY(ctx, cudaMemcpyAsync(st->d_consts, &C, sizeof(C), cudaMemcpyHostToDevice, pc.stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(st->d_meta, meta, meta_bytes + (size_t)sym_off, cudaMemcpyHostToDevice, pc.stream));
    }
    CUDA_TRY(ctx, cudaStreamSynchronize(pc.stream));
    st->devP.log_thr_lo = st->P.threshold > 0 ? log(st->P.threshold) - 1e-9 : -INFINITY;
    st->devP.min_diags = (int)st->P.min_diags; st->devP.tb_diags = (int)st->P.tb_diags; st->devP.expansion = (int)st->P.expansion;
    return BARB200_OK;
}

// "" or why one input pair cannot be aligned
static std::string pair_error(int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor) {
    if (lx < 0 || ly < 0 || lx > 0x3fffffff || ly > 0x3fffffff || (n_anchor && !anchors)) return "bad sequence length or anchors";
    return check_anchors(anchors, n_anchor, lx, ly);
}

static int stage_create_impl(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                             const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                             const int64_t *const *anchors, const int64_t *n_anchor,
                             const uint8_t *ragged_left, const uint8_t *ragged_right, barb200_pecan_stage **out) {
    if (!ctx || !out || n_pairs < 0 || (n_pairs > 0 && (!sx || !sy || !lx || !ly))) { if (ctx) set_error(ctx, "bad argument"); return BARB200_EINVAL; }
    PlanParams P;
    int rc = plan_params(ctx, p, P);
    if (rc) return rc;
    barb200_pecan_stage *st = new barb200_pecan_stage();
    st->ctx = ctx; st->P = P; st->n_pairs = n_pairs;
    st->pair_first.assign(n_pairs + 1, 0);
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int64_t na = n_anchor ? n_anchor[i] : 0;
        const int64_t *a = (anchors && na) ? anchors[i] : nullptr;
        const std::string e = pair_error(lx[i], ly[i], a, na);
        if (!e.empty()) { set_error(ctx, e); delete st; return BARB200_EINVAL; }
        st->pair_first[i] = (int64_t)st->subs.size();
        split_pair(P, i, lx[i], ly[i], a, na, ragged_left && ragged_left[i], ragged_right && ragged_right[i], st->subs);
    }
    st->pair_first[n_pairs] = (int64_t)st->subs.size();
    rc = stage_build(st, sx, sy, nullptr);
    if (rc) { barb200_pecan_stage_destroy(st); return rc; }
    *out = st;
    return BARB200_OK;
}

extern "C" int barb200_pecan_stage_create(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                                          const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                                          const int64_t *const *anchors, const int64_t *n_anchor,
                                          const uint8_t *ragged_left, const uint8_t *ragged_right, barb200_pecan_stage **out) {
    if (!ctx) return BARB200_EINVAL;
    std::lock_guard<std::mutex> lk(pecan_of(ctx, 0).mu);
    return stage_create_impl(ctx, p, n_pairs, sx, lx, sy, ly, anchors, n_anchor, ragged_left, ragged_right, out);
}

static int stage_run_locked(barb200_pecan_stage *st, float *kernel_ms) {
    barb200_ctx *ctx = st->ctx;
    PecanContext &pc = pecan_of(ctx, st->dev);
    cudaSetDevice(ctx_device(ctx, st->dev));
    if (pc.scratch_bytes < st->scratch_bytes) {      // grow the context's rings
        cudaFree(pc.scratch);
        pc.scratch_bytes = 0;
        if (cudaMalloc((void **)&pc.scratch, st->scratch_bytes) != cudaSuccess) {
            cudaGetLastError(); pc.scratch = nullptr;
            set_error(ctx, "device allocation failed (pecan rings)"); return BARB200_ENOMEM;
        }
        pc.scratch_bytes = st->scratch_bytes;
    }
    CUDA_TRY(ctx, cudaMemsetAsync(st->d_counter, 0, sizeof(unsigned) * (st->groups.size() + 1), pc.stream));
    CUDA_TRY(ctx, cudaEventRecord(pc.ev0, pc.stream));
    st->launches = 0;
    for (size_t gi = st->groups.size(); gi-- > 0;) {          // widest class first
        const PecanGroup &g = st->groups[gi];
        const Class &K = kClass[g.cls];
        cudaStream_t cs = pc.cls[g.cls];
        KernelArgs A;
        A.jobs = st->d_jobs; A.order = st->d_order + g.order_off; A.n_jobs = (int)g.jobs.size();
        A.sym = st->d_sym; A.meta = st->d_meta; A.out = st->d_out; A.out_n = st->d_out_n;
        A.counter = st->d_counter + gi; A.consts = st->d_consts; A.scratch = pc.scratch + g.scratch_off; A.slot_doubles = g.slot_doubles;
        A.maskM = g.capM - 1; A.maskF = g.capF - 1; A.RW = g.RW; A.RWs = g.RWs; A.P = st->devP;
        CUDA_TRY(ctx, cudaStreamWaitEvent(cs, pc.ev0, 0));
        if (K.threads * K.ctas_per_sm > 768) pecan_posterior_kernel_r64<<<g.ctas, K.threads, g.smem_bytes, cs>>>(A);
        else pecan_posterior_kernel<<<g.ctas, K.threads, g.smem_bytes, cs>>>(A);
        CUDA_TRY(ctx, cudaGetLastError());
        CUDA_TRY(ctx, cudaEventRecord(pc.done[g.cls], cs));
        CUDA_TRY(ctx, cudaStreamWaitEvent(pc.stream, pc.done[g.cls], 0));
        ++st->launches;
    }
    CUDA_TRY(ctx, cudaEventRecord(pc.ev1, pc.stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(pc.stream));
    if (kernel_ms) CUDA_TRY(ctx, cudaEventElapsedTime(kernel_ms, pc.ev0, pc.ev1));
    st->ran = true;
    return BARB200_OK;
}

extern "C" int barb200_pecan_stage_run(barb200_pecan_stage *st, float *kernel_ms) {
    if (!st) return BARB200_EINVAL;
    std::lock_guard<std::mutex> lk(pecan_of(st->ctx, st->dev).mu);
    return stage_run_locked(st, kernel_ms);
}

extern "C" int64_t barb200_pecan_stage_cells(barb200_pecan_stage *st) { return st ? st->cells : 0; }
extern "C" int64_t barb200_pecan_stage_launches(barb200_pecan_stage *st) { return st ? st->launches : 0; }

// candidates of every sub-job, in emission order (host copies); overflowed jobs are re-run with room for every cell
static int stage_collect(barb200_pecan_stage *st, std::vector<std::vector<Pair>> &per_sub) {
    barb200_ctx *ctx = st->ctx;
    const int dev = st->dev;
    const int64_t ns = (int64_t)st->subs.size();
    per_sub.assign(ns, std::vector<Pair>());
    if (ns == 0) return BARB200_OK;
    cudaSetDevice(ctx_device(ctx, dev));
    std::vector<int> out_n(ns);
    CUDA_TRY(ctx, cudaMemcpy(out_n.data(), st->d_out_n, sizeof(int) * ns, cudaMemcpyDeviceToHost));
    std::vector<long long> dst_off(ns + 1, 0);
    std::vector<int64_t> retry;
    for (int64_t i = 0; i < ns; ++i) {
        const bool over = out_n[i] > st->subs[i].out_cap;
        if (over) retry.push_back(i);
        dst_off[i + 1] = dst_off[i] + (over ? 0 : out_n[i]);
    }
    const long long total = dst_off[ns];
    Staging down(ctx, dev);
    Pair *const flat = total > 0 ? (Pair *)down.take(sizeof(Pair) * (size_t)total) : nullptr;
    if (total > 0) {
        long long *d_dst_off = nullptr; Pair *d_flat = nullptr;
        if (device_alloc(ctx, dev, (void **)&d_dst_off, sizeof(long long) * (ns + 1)) != 0) { set_error(ctx, "device allocation failed (compact offsets)"); return BARB200_ENOMEM; }
        cudaError_t e = cudaSuccess;
        if (device_alloc(ctx, dev, (void **)&d_flat, sizeof(Pair) * (size_t)total) != 0) {
            device_free(ctx, dev, d_dst_off, sizeof(long long) * (ns + 1)); set_error(ctx, "device allocation failed (compact output)"); return BARB200_ENOMEM; }
        cudaStream_t s = pecan_of(ctx, dev).stream;
        cudaMemcpyAsync(d_dst_off, dst_off.data(), sizeof(long long) * (ns + 1), cudaMemcpyHostToDevice, s);
        const int grid = (int)std::min<int64_t>(ns, (int64_t)ctx_sm_count(ctx, dev) * 16);
        pecan_compact_kernel<<<grid, 128, 0, s>>>(st->d_jobs, st->d_out_n, d_dst_off, st->d_out, d_flat, (int)ns);
        ++st->launches;
        cudaMemcpyAsync(flat, d_flat, sizeof(Pair) * (size_t)total, cudaMemcpyDeviceToHost, s);
        e = cudaStreamSynchronize(s);
        device_free(ctx, dev, d_dst_off, sizeof(long long) * (ns + 1)); device_free(ctx, dev, d_flat, sizeof(Pair) * (size_t)total);
        if (e != cudaSuccess) { set_error(ctx, std::string("pecan compaction: ") + cudaGetErrorString(e)); return BARB200_ECUDA; }
    }
    const int nthr = host_threads(ctx);
#pragma omp parallel for schedule(dynamic, 8) num_threads(nthr)
    for (int64_t i = 0; i < ns; ++i) {
        per_sub[i].assign(flat + dst_off[i], flat + dst_off[i + 1]);
        // the kernel appends the candidates of a diagonal in no particular order: restore the reference's order of emission
        // (keys computed once per record; the input is nearly sorted, so this is cheap)
        const SubJob &sj = st->subs[i];
        std::vector<Pair> &v = per_sub[i];
        struct Keyed { uint64_t k1; uint32_t k2, idx; };
        std::vector<Keyed> keys(v.size());
        bool sorted = true;
        for (size_t q = 0; q < v.size(); ++q) {
            const std::pair<uint64_t, uint32_t> k = emission_key(sj, v[q].x, v[q].y);
            keys[q] = Keyed{k.first, k.second, (uint32_t)q};
            if (q && (keys[q].k1 < keys[q - 1].k1 || (keys[q].k1 == keys[q - 1].k1 && keys[q].k2 < keys[q - 1].k2))) sorted = false;
        }
        if (!sorted) {
            std::sort(keys.begin(), keys.end(), [](const Keyed &a, const Keyed &b) { return a.k1 != b.k1 ? a.k1 < b.k1 : a.k2 < b.k2; });
            std::vector<Pair> w(v.size());
            for (size_t q = 0; q < v.size(); ++q) w[q] = v[keys[q].idx];
            v.swap(w);
        }
    }
    down.release();
    if (!retry.empty()) {
        if (st->full_cap) { set_error(ctx, "pecan: output overflow with full capacity (internal error)"); return BARB200_EJOB; }
        barb200_pecan_stage *rs = new barb200_pecan_stage();   // on the parent's device: it reads the parent's symbols and bands
        rs->ctx = ctx; rs->dev = dev; rs->P = st->P; rs->full_cap = true;
        for (int64_t i : retry) { rs->subs.push_back(st->subs[i]); rs->jobs.push_back(st->jobs[i]); }
        int rc = stage_build(rs, nullptr, nullptr, st);
        if (rc == BARB200_OK) rc = stage_run_locked(rs, nullptr);
        std::vector<std::vector<Pair>> sub2;
        if (rc == BARB200_OK) rc = stage_collect(rs, sub2);
        st->launches += rs->launches;
        barb200_pecan_stage_destroy(rs);
        if (rc) return rc;
        for (size_t k = 0; k < retry.size(); ++k) per_sub[retry[k]] = std::move(sub2[k]);
    }
    return BARB200_OK;
}

// exp / threshold / floor on the host with the reference's own libm (addPosteriorProb, pairwiseAligner.c:665-674) and the
// coordinate shift of convertAlignedPairs (:1294-1306)
static int finish_pairs(barb200_pecan_stage *st, const std::vector<std::vector<Pair>> &per_sub, int64_t **triples_out, int64_t *n_out,
                        double **posteriors_out, int64_t *cells_out) {
    barb200_ctx *ctx = st->ctx;
    const int nthr = host_threads(ctx);
    const double thr = st->P.threshold;
    bool oom = false;
#pragma omp parallel for schedule(dynamic, 8) num_threads(nthr)
    for (int64_t i = 0; i < st->n_pairs; ++i) {
        int64_t cand = 0, cells = 0;
        for (int64_t s = st->pair_first[i]; s < st->pair_first[i + 1]; ++s) { cand += (int64_t)per_sub[s].size(); cells += st->subs[s].cells; }
        int64_t *tr = (int64_t *)malloc(sizeof(int64_t) * 3 * (size_t)std::max<int64_t>(cand, 1));
        double *po = posteriors_out ? (double *)malloc(sizeof(double) * (size_t)std::max<int64_t>(cand, 1)) : nullptr;
        if (!tr || (posteriors_out && !po)) { oom = true; free(tr); free(po); triples_out[i] = nullptr; if (posteriors_out) posteriors_out[i] = nullptr; n_out[i] = 0; continue; }
        int64_t n = 0;
        for (int64_t s = st->pair_first[i]; s < st->pair_first[i + 1]; ++s) {
            const SubJob &sj = st->subs[s];
            // alignedPairCoordinateCorrectionFn moves a region's pairs over with stList_pop: reverse order of emission (:1457-1464)
            for (int64_t q = (int64_t)per_sub[s].size() - 1; q >= 0; --q) {
                const Pair &c = per_sub[s][q];
                double pp = exp(c.lp);
                if (!(pp >= thr)) continue;
                if (po) po[n] = pp;
                if (pp > 1.0) pp = 1.0;
                tr[3 * n] = (int64_t)floor(pp * 10000000.0);       // PAIR_ALIGNMENT_PROB_1
                tr[3 * n + 1] = c.x + sj.x1; tr[3 * n + 2] = c.y + sj.y1;
                ++n;
            }
        }
        triples_out[i] = tr; n_out[i] = n;
        if (posteriors_out) posteriors_out[i] = po;
        if (cells_out) cells_out[i] = cells;
    }
    if (oom) { set_error(ctx, "host allocation failed"); return BARB200_ENOMEM; }
    return BARB200_OK;
}

extern "C" int barb200_pecan_stage_fetch(barb200_pecan_stage *st, int64_t **triples_out, int64_t *n_out, double **posteriors_out, int64_t *cells_out) {
    if (!st || !triples_out || !n_out) return BARB200_EINVAL;
    if (!st->ran) { set_error(st->ctx, "barb200_pecan_stage_fetch before barb200_pecan_stage_run"); return BARB200_EINVAL; }
    std::vector<std::vector<Pair>> per_sub;
    int rc;
    {
        std::lock_guard<std::mutex> lk(pecan_of(st->ctx, st->dev).mu);
        rc = stage_collect(st, per_sub);
    }
    if (rc) return rc;
    return finish_pairs(st, per_sub, triples_out, n_out, posteriors_out, cells_out);
}

// chunks bounded by the output room a stage reserves (16 B per candidate, ~ (lx + ly) candidates per pair)
static const int64_t kChunkRecords = (int64_t)128 << 20;

// The batch on a single-device context: chunks of pairs in caller order, each split, planned, run and finished as one stage.
static int pecan_batch_now(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                           const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                           const int64_t *const *anchors, const int64_t *n_anchor,
                           const uint8_t *ragged_left, const uint8_t *ragged_right,
                           int64_t **triples_out, int64_t *n_out, double **posteriors_out, int64_t *cells_out) {
    if (!ctx || !triples_out || !n_out) { if (ctx) set_error(ctx, "bad argument"); return BARB200_EINVAL; }
    int64_t i0 = 0;
    while (i0 < n_pairs || (n_pairs == 0 && i0 == 0)) {
        int64_t i1 = i0, rec = 0;
        while (i1 < n_pairs && (i1 == i0 || rec + lx[i1] + ly[i1] + 64 <= kChunkRecords)) { rec += lx[i1] + ly[i1] + 64; ++i1; }
        barb200_pecan_stage *st = nullptr;
        const double t0 = omp_get_wtime();
        std::unique_lock<std::mutex> lk(pecan_of(ctx, 0).mu);   // held from create to collect, like a stage's three calls
        int rc = stage_create_impl(ctx, p, i1 - i0, sx + i0, lx + i0, sy + i0, ly + i0, anchors ? anchors + i0 : nullptr,
                                   n_anchor ? n_anchor + i0 : nullptr, ragged_left ? ragged_left + i0 : nullptr,
                                   ragged_right ? ragged_right + i0 : nullptr, &st);
        const double t1 = omp_get_wtime();
        if (rc == BARB200_OK) rc = stage_run_locked(st, nullptr);
        const double t2 = omp_get_wtime();
        std::vector<std::vector<Pair>> per_sub;
        if (rc == BARB200_OK) rc = stage_collect(st, per_sub);
        lk.unlock();
        if (rc == BARB200_OK) rc = finish_pairs(st, per_sub, triples_out + i0, n_out + i0, posteriors_out ? posteriors_out + i0 : nullptr,
                                                cells_out ? cells_out + i0 : nullptr);
        const double t3 = omp_get_wtime();
        barb200_pecan_stage_destroy(st);
        if (getenv("BARB200_DEBUG")) fprintf(stderr, "[barb200] pecan batch of %lld pairs: create %.1f ms, run %.1f ms, fetch %.1f ms, destroy %.1f ms\n",
                                             (long long)(i1 - i0), (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, (omp_get_wtime() - t3) * 1e3);
        if (rc) return rc;
        pecan_of(ctx, 0).hmm_pairs += i1 - i0;
        if (n_pairs == 0) break;
        i0 = i1;
    }
    return BARB200_OK;
}

// One chunk of device `dev`'s share: the caller's pairs pairs[0, n), already split and planned (subs[caller index], moved into the
// stage), run on the device and finished; the outputs land at the caller's indices, also when a step fails (the caller frees them).
static int pecan_chunk_on_device(barb200_ctx *ctx, int dev, const PlanParams &P, const int64_t *pairs, int64_t n, std::vector<std::vector<SubJob>> &subs,
                                 const char *const *sx, const char *const *sy, int64_t **triples_out, int64_t *n_out, double **posteriors_out,
                                 int64_t *cells_out) {
    barb200_pecan_stage *st = new barb200_pecan_stage();
    st->ctx = ctx; st->dev = dev; st->P = P; st->n_pairs = n;
    st->pair_first.assign(n + 1, 0);
    std::vector<const char *> csx(n), csy(n);
    for (int64_t k = 0; k < n; ++k) {
        csx[k] = sx[pairs[k]]; csy[k] = sy[pairs[k]];
        st->pair_first[k] = (int64_t)st->subs.size();
        for (SubJob &s : subs[pairs[k]]) { s.pair = k; st->subs.push_back(std::move(s)); }
    }
    st->pair_first[n] = (int64_t)st->subs.size();
    std::vector<int64_t *> trip(n, nullptr); std::vector<double *> post(n, nullptr); std::vector<int64_t> no(n, 0), cells(n, 0);
    std::vector<std::vector<Pair>> per_sub;
    int rc;
    {
        std::lock_guard<std::mutex> lk(pecan_of(ctx, dev).mu);
        rc = stage_build(st, csx.data(), csy.data(), nullptr);
        if (rc == BARB200_OK) rc = stage_run_locked(st, nullptr);
        if (rc == BARB200_OK) rc = stage_collect(st, per_sub);
    }
    if (rc == BARB200_OK) rc = finish_pairs(st, per_sub, trip.data(), no.data(), posteriors_out ? post.data() : nullptr, cells.data());
    barb200_pecan_stage_destroy(st);
    for (int64_t k = 0; k < n; ++k) {
        const int64_t i = pairs[k];
        triples_out[i] = trip[k]; n_out[i] = no[k];
        if (posteriors_out) posteriors_out[i] = post[k];
        if (cells_out) cells_out[i] = cells[k];
    }
    if (rc == BARB200_OK) pecan_of(ctx, dev).hmm_pairs += n;
    return rc;
}

// The batch on a context of several devices. Every pair is checked, split and planned once here; the pairs are dealt to the
// devices by their planned cells (deal_pairs), and each device runs its share in chunks (as pecan_batch_now) on a host thread
// of its own. Results are the single-device results, bit for bit: a job's posteriors do not depend on the jobs beside it.
// If a device fails, the whole request fails with that device's message and no outputs.
static int pecan_batch_devices(barb200_ctx *ctx, int ndev, const barb200_pecan_params *p, int64_t n_pairs,
                               const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                               const int64_t *const *anchors, const int64_t *n_anchor,
                               const uint8_t *ragged_left, const uint8_t *ragged_right,
                               int64_t **triples_out, int64_t *n_out, double **posteriors_out, int64_t *cells_out) {
    PlanParams P;
    int rc = plan_params(ctx, p, P);
    if (rc) return rc;
    std::vector<std::vector<SubJob>> subs(n_pairs);
    std::vector<int64_t> cost(n_pairs, 0);
    std::string err; int64_t err_at = n_pairs;
#pragma omp parallel for schedule(dynamic, 16) num_threads(host_threads(ctx))
    for (int64_t i = 0; i < n_pairs; ++i) {
        const int64_t na = n_anchor ? n_anchor[i] : 0;
        const int64_t *a = (anchors && na) ? anchors[i] : nullptr;
        std::string e = pair_error(lx[i], ly[i], a, na);
        if (e.empty()) {
            split_pair(P, i, lx[i], ly[i], a, na, ragged_left && ragged_left[i], ragged_right && ragged_right[i], subs[i]);
            for (SubJob &s : subs[i]) { if (!(e = plan_subjob(P, s)).empty()) break; cost[i] += s.cells; }
        }
        if (!e.empty()) {
#pragma omp critical
            if (i < err_at) { err_at = i; err = e; }       // the first bad pair's message, whichever thread finds it
        }
    }
    if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
    for (int64_t i = 0; i < n_pairs; ++i) { triples_out[i] = nullptr; n_out[i] = 0; if (posteriors_out) posteriors_out[i] = nullptr; }
    const std::vector<std::vector<int64_t>> share = deal_pairs(cost, ndev);
    int active = 0;
    for (const auto &s : share) active += !s.empty();
    std::vector<int> rcs(ndev, BARB200_OK);
    std::vector<std::string> errs(ndev);
    auto run_device = [&](int d) {
        set_host_thread_share(active);
        const std::vector<int64_t> &mine = share[d];
        try {
            for (size_t at = 0; at < mine.size();) {
                size_t end = at; int64_t rec = 0;
                while (end < mine.size() && (end == at || rec + lx[mine[end]] + ly[mine[end]] + 64 <= kChunkRecords)) { rec += lx[mine[end]] + ly[mine[end]] + 64; ++end; }
                const int r = pecan_chunk_on_device(ctx, d, P, mine.data() + at, (int64_t)(end - at), subs, sx, sy, triples_out, n_out, posteriors_out, cells_out);
                if (r) { rcs[d] = r; errs[d] = get_error(ctx); break; }
                at = end;
            }
        } catch (const std::bad_alloc &) { rcs[d] = BARB200_ENOMEM; errs[d] = "host allocation failed"; }
        set_host_thread_share(1);
    };
    std::vector<std::thread> th;
    for (int d = 0; d < ndev; ++d) if (!share[d].empty()) th.emplace_back(run_device, d);
    for (auto &t : th) t.join();
    for (int d = 0; d < ndev; ++d) if (rcs[d]) {
        for (int64_t i = 0; i < n_pairs; ++i) {
            free(triples_out[i]); triples_out[i] = nullptr; n_out[i] = 0;
            if (posteriors_out) { free(posteriors_out[i]); posteriors_out[i] = nullptr; }
        }
        set_error(ctx, errs[d]);
        return rcs[d];
    }
    return BARB200_OK;
}

// Concurrent callers (one per OpenMP thread of bar(), bar/impl/bar.c:90-94) share device batches: whatever is waiting when the
// device becomes free runs as ONE batch (group_commit.h, batch_merge.h); a single caller runs its own request unchanged. On a
// context of several devices the leader spreads that batch over them (pecan_batch_devices).
extern "C" int barb200_pecan_aligned_pairs_batch(barb200_ctx *ctx, const barb200_pecan_params *p, int64_t n_pairs,
                                                 const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                                                 const int64_t *const *anchors, const int64_t *n_anchor,
                                                 const uint8_t *ragged_left, const uint8_t *ragged_right,
                                                 int64_t **triples_out, int64_t *n_out, double **posteriors_out, int64_t *cells_out) {
    if (!ctx || !p || !triples_out || !n_out || n_pairs < 0 || (n_pairs > 0 && (!sx || !sy || !lx || !ly))) { if (ctx) set_error(ctx, "bad argument"); return BARB200_EINVAL; }
    PecanRequest r;
    r.p = *p; r.n = n_pairs; r.sx = sx; r.lx = lx; r.sy = sy; r.ly = ly; r.anchors = anchors; r.n_anchor = n_anchor;
    r.ragged_left = ragged_left; r.ragged_right = ragged_right;
    r.triples_out = triples_out; r.n_out = n_out; r.posteriors_out = posteriors_out; r.cells_out = cells_out;
    const int ndev = ctx_device_count(ctx);
    pecan_state(ctx).group.submit(&r, pecan_can_merge, [ctx, ndev](std::vector<PecanRequest *> &batch) {
        run_pecan_group(batch, [ctx, ndev](const barb200_pecan_params *pp, int64_t n, const char *const *a, const int64_t *la, const char *const *b, const int64_t *lb,
                                           const int64_t *const *an, const int64_t *na, const uint8_t *rl, const uint8_t *rr, int64_t **trip, int64_t *no,
                                           double **post, int64_t *cells) {
            return ndev == 1 ? pecan_batch_now(ctx, pp, n, a, la, b, lb, an, na, rl, rr, trip, no, post, cells)
                             : pecan_batch_devices(ctx, ndev, pp, n, a, la, b, lb, an, na, rl, rr, trip, no, post, cells);
        });
    });
    return r.rc;
}

extern "C" int barb200_pecan_device_stats(barb200_ctx *ctx, int64_t *hmm_pairs, int64_t *mum_pairs, int max_devices) {
    if (!ctx) return BARB200_EINVAL;
    const PecanState &ps = pecan_state(ctx);
    const int n = (int)ps.devs.size();
    for (int d = 0; d < n && d < max_devices; ++d) {
        if (hmm_pairs) hmm_pairs[d] = ps.devs[d]->hmm_pairs.load();
        if (mum_pairs) mum_pairs[d] = ps.devs[d]->mum_pairs.load();
    }
    return n;
}

extern "C" int barb200_pecan_band(int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor, int64_t expansion, int64_t *xmy_l, int64_t *xmy_r) {
    if (lx < 0 || ly < 0 || lx > 0x3fffffff || ly > 0x3fffffff || expansion < 0 || expansion % 2 || !xmy_l || !xmy_r) return BARB200_EINVAL;
    if (!check_anchors(anchors, n_anchor, lx, ly).empty()) return BARB200_EINVAL;
    PlanParams P{0.01, 1000, 40, expansion, (int64_t)1 << 60};
    SubJob s; s.lx = (int)lx; s.ly = (int)ly;
    s.anchors.assign(anchors, anchors + 2 * n_anchor);
    if (!plan_subjob(P, s).empty()) return BARB200_EINVAL;
    for (int64_t d = 0; d <= lx + ly; ++d) { xmy_l[d] = s.bandL[d]; xmy_r[d] = s.bandL[d] + 2 * (int64_t)(s.coff[d + 1] - s.coff[d] - 1); }
    return BARB200_OK;
}

extern "C" int64_t barb200_pecan_split_points(int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor, int64_t split_bigger,
                                              int ragged_left, int ragged_right, int64_t **splits_out) {
    if (lx < 0 || ly < 0 || !splits_out || split_bigger < 1) return BARB200_EINVAL;
    if (!check_anchors(anchors, n_anchor, lx, ly).empty()) return BARB200_EINVAL;
    PlanParams P{0.01, 1000, 40, 20, split_bigger};
    std::vector<SubJob> subs;
    split_pair(P, 0, lx, ly, anchors, n_anchor, ragged_left != 0, ragged_right != 0, subs);
    int64_t *o = (int64_t *)malloc(sizeof(int64_t) * 4 * std::max<size_t>(subs.size(), 1));
    if (!o) return BARB200_ENOMEM;
    for (size_t i = 0; i < subs.size(); ++i) { o[4 * i] = subs[i].x1; o[4 * i + 1] = subs[i].y1; o[4 * i + 2] = subs[i].x1 + subs[i].lx; o[4 * i + 3] = subs[i].y1 + subs[i].ly; }
    *splits_out = o;
    return (int64_t)subs.size();
}
