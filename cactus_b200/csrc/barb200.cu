// barb200.cu -- device orchestration + C ABI of libbarb200.so (see include/barb200.h).
//
// A *stage* is one device batch of POA jobs (one job = one abpoa_msa call of the reference), planned by stage_plan.h:
//   * jobs are BUCKETED by the CTA-size class their longest sequence needs (32 .. 1024 threads, 16 columns per thread) and,
//     inside a class, ordered by estimated cost, largest first. Every class gets its own slot layout sized from ITS largest
//     job, its own persistent launch on its own stream (largest class first; the launches run concurrently, the block
//     scheduler fills whatever a class leaves free) and its own work counter -- a batch of thousands of short adjacencies
//     and a few 10 kbp windows no longer runs everything in the CTA shape and the slot size of the largest job;
//   * the host does no per-job work besides packing: the guide-tree read orders are computed by the CTA that owns the job
//     (guide_tree.cuh);
//   * jobs that outgrow the optimistic plane / MSA sizing come back flagged and are re-run with geometrically larger
//     slots (x4, then worst case) on the stage's uploaded inputs.
// A context drives one or more devices; every device has two *lanes* (slot arena + streams + pinned staging) so that one
// batch's upload / download / unpacking overlaps the other's kernels. host_bar.cpp's dispatcher feeds the lanes of all
// devices from one queue of ends. No CPU fallback exists: if CUDA is unavailable, creation fails.
#include <cuda_runtime.h>
#include <omp.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <unordered_map>
#include <vector>
#include "host_api.h"
#include "poa_kernel.cuh"
#include "stage_plan.h"

namespace barb200 {
extern "C" __global__ void poa_msa_kernel_t32(const BatchArgs A);
extern "C" __global__ void poa_msa_kernel_t64(const BatchArgs A);
extern "C" __global__ void poa_msa_kernel_t128(const BatchArgs A);
extern "C" __global__ void poa_msa_kernel_t256(const BatchArgs A);
extern "C" __global__ void poa_msa_kernel_t640(const BatchArgs A);
extern "C" __global__ void poa_msa_kernel_t1024(const BatchArgs A);
extern "C" __global__ void poa_trace_kernel_t32(const BatchArgs A, const TraceArgs T);
extern "C" __global__ void poa_trace_kernel_t64(const BatchArgs A, const TraceArgs T);
extern "C" __global__ void poa_trace_kernel_t128(const BatchArgs A, const TraceArgs T);
extern "C" __global__ void poa_trace_kernel_t256(const BatchArgs A, const TraceArgs T);
extern "C" __global__ void poa_trace_kernel_t640(const BatchArgs A, const TraceArgs T);
extern "C" __global__ void poa_trace_kernel_t1024(const BatchArgs A, const TraceArgs T);
}
typedef void (*poa_kernel_fn)(const barb200::BatchArgs);
typedef void (*poa_trace_kernel_fn)(const barb200::BatchArgs, const barb200::TraceArgs);
// the kernel of every CTA-size class (stage_plan.h: kClassThreads), scratch = its dynamic shared memory per CTA
// (poa_kernel.cuh: poa_scratch_bytes)
static constexpr struct { int T; poa_kernel_fn fn; int scratch; } kKernels[] = {
    {32, barb200::poa_msa_kernel_t32, barb200::poa_scratch_bytes(32)}, {64, barb200::poa_msa_kernel_t64, barb200::poa_scratch_bytes(64)},
    {128, barb200::poa_msa_kernel_t128, barb200::poa_scratch_bytes(128)}, {256, barb200::poa_msa_kernel_t256, barb200::poa_scratch_bytes(256)},
    {640, barb200::poa_msa_kernel_t640, barb200::poa_scratch_bytes(640)}, {1024, barb200::poa_msa_kernel_t1024, barb200::poa_scratch_bytes(1024)}};
// the trace kernels of the same classes (barb200_poa_trace_batch), with the same dynamic shared memory
static constexpr poa_trace_kernel_fn kTraceKernels[] = {barb200::poa_trace_kernel_t32, barb200::poa_trace_kernel_t64, barb200::poa_trace_kernel_t128,
                                                        barb200::poa_trace_kernel_t256, barb200::poa_trace_kernel_t640, barb200::poa_trace_kernel_t1024};
static const int kNumKernels = barb200::kNumClasses;
static constexpr bool kernels_follow_classes(int i = 0) { return i == kNumKernels || (kKernels[i].T == barb200::kClassThreads[i] && kernels_follow_classes(i + 1)); }
static_assert(sizeof(kKernels) / sizeof(kKernels[0]) == kNumKernels && kernels_follow_classes(), "kKernels must follow stage_plan.h's classes");
static_assert(sizeof(kTraceKernels) / sizeof(kTraceKernels[0]) == kNumKernels, "kTraceKernels must follow stage_plan.h's classes");
static const int kMaxDevices = 8;
using namespace barb200;

namespace barb200 {
// one in-flight device batch: slot arena, streams, pinned staging
struct Lane {
    int index = 0;                      // global lane index (device * lanes_per_device + lane)
    std::mutex busy;                    // held while a batch (or a staged run) owns the arena
    uint8_t *d_slots = nullptr; size_t slots_bytes = 0;
    int *d_planes = nullptr; size_t planes_bytes = 0;
    cudaStream_t main = nullptr, copy = nullptr, cls[kNumKernels] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t cls_done[kNumKernels] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned long long *d_clk = nullptr; size_t clk_entries = 0;
};
struct Device {
    int ordinal = 0, sm_count = 0; size_t mem_total = 0;
    std::vector<std::unique_ptr<Lane>> lanes;
    // grow-only cache of device blocks for the per-stage buffers (cudaMalloc / cudaFree per call cost milliseconds
    // and cudaFree synchronises the device, which would stall the upload / kernel overlap)
    std::mutex cache_mu; std::vector<std::pair<void *, size_t>> free_blocks; size_t cached_bytes = 0;
    // pinned staging blocks (packed inputs up, MSA bytes down), shared by the device's lanes: cudaMallocHost of a large block is
    // slow, so a lane that meets its first large batch borrows the block the other lane has grown already
    std::mutex pin_mu; std::vector<std::pair<void *, size_t>> free_pinned;
};
}  // namespace barb200

struct barb200_ctx {
    barb200_params p;
    PoaParams P;
    HostParams hp;
    std::vector<std::unique_ptr<Device>> devs;
    int lanes_per_device = 2;
    bool lanes_shared = false;          // set once the dispatcher runs: every lane plans with its share of the device memory
    std::mutex err_mu;
    std::string err;
    void *pecan = nullptr;              // pecan.cu's pair-HMM state (created and destroyed with the context)
    void *dispatcher = nullptr;         // host_bar.cpp's end queue (created on first use, destroyed with the context)
    double last_timing[6] = {0, 0, 0, 0, 0, 0};   // of the most recent device batch (barb200_last_batch_timing), under err_mu
};

namespace barb200 {
// the message is kept twice: in the context (for callers whose request ran inside another thread's batch) and per
// thread (concurrent callers do not overwrite each other's text)
static thread_local std::string tls_err;
static thread_local const barb200_ctx *tls_err_ctx = nullptr;
void set_error(barb200_ctx *ctx, const std::string &msg) {
    if (!ctx) return;
    tls_err = msg; tls_err_ctx = ctx;
    std::lock_guard<std::mutex> lk(ctx->err_mu); ctx->err = msg;
}
std::string get_error(barb200_ctx *ctx) {
    if (tls_err_ctx == ctx && !tls_err.empty()) return tls_err;
    std::lock_guard<std::mutex> lk(ctx->err_mu); return ctx->err;
}
// threads for host-side work: the OpenMP default capped by the cgroup CPU quota (containers on big hosts often see
// all logical CPUs but may only use a few; oversubscribing them slows the packing / guide-tree loops down)
static int usable_host_threads() {
    int n = omp_get_max_threads();
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
        char q[64]; long long period = 0;
        if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
            const long long quota = atoll(q);
            const int lim = (int)((quota + period / 2) / period);
            if (lim >= 1 && lim < n) n = lim;
        }
        fclose(f);
    }
    return n;
}
// a batch over several devices runs one host thread per device: each takes its share of the host threads for its parallel loops
static thread_local int tl_thread_divisor = 1;
int host_threads(barb200_ctx *ctx) {
    static const int dflt = usable_host_threads();
    const int n = ctx->p.host_threads > 0 ? ctx->p.host_threads : dflt;
    return std::max(1, n / std::max(1, tl_thread_divisor));
}
int default_progressive(barb200_ctx *ctx) { return ctx->p.progressive_poa; }
void set_host_thread_share(int n) { tl_thread_divisor = std::max(1, n); }
int ctx_device_count(barb200_ctx *ctx) { return (int)ctx->devs.size(); }
int ctx_device(barb200_ctx *ctx, int dev) { return ctx->devs[dev]->ordinal; }
int ctx_sm_count(barb200_ctx *ctx, int dev) { return ctx->devs[dev]->sm_count; }
double ctx_mem_fraction(barb200_ctx *ctx) { return ctx->p.mem_fraction > 0 ? ctx->p.mem_fraction : 0.85; }
int total_lanes(barb200_ctx *ctx) { return (int)ctx->devs.size() * ctx->lanes_per_device; }
void **dispatcher_slot(barb200_ctx *ctx) { return &ctx->dispatcher; }
void **pecan_slot(barb200_ctx *ctx) { return &ctx->pecan; }
void mark_lanes_shared(barb200_ctx *ctx) { ctx->lanes_shared = true; }
static Device &dev_of_lane(barb200_ctx *ctx, int lane) { return *ctx->devs[lane / ctx->lanes_per_device]; }
static Lane &lane_of(barb200_ctx *ctx, int lane) { return *ctx->devs[lane / ctx->lanes_per_device]->lanes[lane % ctx->lanes_per_device]; }
}  // namespace barb200

static size_t block_size_of(size_t bytes) { return (std::max<size_t>(bytes, 16) + 255) & ~(size_t)255; }
static cudaError_t dev_alloc(Device &D, void **p, size_t bytes) {
    bytes = block_size_of(bytes);
    {
        std::lock_guard<std::mutex> lk(D.cache_mu);
        int best = -1;
        for (size_t i = 0; i < D.free_blocks.size(); ++i)
            if (D.free_blocks[i].second >= bytes && D.free_blocks[i].second <= 2 * bytes + (1 << 20) &&
                (best < 0 || D.free_blocks[i].second < D.free_blocks[best].second)) best = (int)i;
        if (best >= 0) { *p = D.free_blocks[best].first; D.cached_bytes -= D.free_blocks[best].second; D.free_blocks.erase(D.free_blocks.begin() + best); return cudaSuccess; }
    }
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) {       // give the cache back and retry once
        cudaGetLastError();
        std::lock_guard<std::mutex> lk(D.cache_mu);
        for (auto &b : D.free_blocks) cudaFree(b.first);
        D.free_blocks.clear(); D.cached_bytes = 0;
        e = cudaMalloc(p, bytes);
    }
    return e;
}
static void *pinned_take(Device &D, size_t bytes, size_t *got) {
    {
        std::lock_guard<std::mutex> lk(D.pin_mu);
        int best = -1;
        for (size_t i = 0; i < D.free_pinned.size(); ++i)
            if (D.free_pinned[i].second >= bytes && (best < 0 || D.free_pinned[i].second < D.free_pinned[best].second)) best = (int)i;
        if (best >= 0) { void *p = D.free_pinned[best].first; *got = D.free_pinned[best].second; D.free_pinned.erase(D.free_pinned.begin() + best); return p; }
        // nothing fits: retire the smallest block (the pool stays at a handful of blocks, each grown to the largest batch seen)
        if (D.free_pinned.size() >= 4) {
            size_t m = 0;
            for (size_t i = 1; i < D.free_pinned.size(); ++i) if (D.free_pinned[i].second < D.free_pinned[m].second) m = i;
            cudaFreeHost(D.free_pinned[m].first); D.free_pinned.erase(D.free_pinned.begin() + m);
        }
    }
    void *p = nullptr;
    const size_t want = bytes + (bytes >> 2) + 4096;
    if (cudaMallocHost(&p, want) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    *got = want;
    return p;
}
static void pinned_give(Device &D, void *p, size_t bytes) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(D.pin_mu);
    D.free_pinned.emplace_back(p, bytes);
}
struct PinnedBlock {       // scope guard
    Device &D; void *p = nullptr; size_t bytes = 0;
    PinnedBlock(Device &d, size_t want) : D(d) { p = pinned_take(D, want, &bytes); }
    ~PinnedBlock() { pinned_give(D, p, bytes); }
    PinnedBlock(const PinnedBlock &) = delete; PinnedBlock &operator=(const PinnedBlock &) = delete;
};

static void dev_free(Device &D, void *p, size_t bytes) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(D.cache_mu);
    if (D.cached_bytes + block_size_of(bytes) > ((size_t)4 << 30) || D.free_blocks.size() >= 64) { cudaFree(p); return; }
    D.free_blocks.emplace_back(p, block_size_of(bytes)); D.cached_bytes += block_size_of(bytes);
}

namespace barb200 {
int device_alloc(barb200_ctx *ctx, int dev, void **p, size_t bytes) { return dev_alloc(*ctx->devs[dev], p, bytes) == cudaSuccess ? 0 : -1; }
void device_free(barb200_ctx *ctx, int dev, void *p, size_t bytes) { dev_free(*ctx->devs[dev], p, bytes); }
void *pinned_take(barb200_ctx *ctx, int dev, size_t bytes, size_t *got) { return ::pinned_take(*ctx->devs[dev], bytes, got); }
void pinned_give(barb200_ctx *ctx, int dev, void *p, size_t bytes) { ::pinned_give(*ctx->devs[dev], p, bytes); }
}  // namespace barb200

extern "C" void barb200_params_default(barb200_params *p) { params_default(p); }

static void fail(char *errbuf, int n, const std::string &m) { if (errbuf && n > 0) { snprintf(errbuf, n, "%s", m.c_str()); } }

extern "C" barb200_ctx *barb200_create(const barb200_params *p, char *errbuf, int errbuf_len) {
    if (!p) { fail(errbuf, errbuf_len, "null params"); return nullptr; }
    const std::string bad = check_params(*p);
    if (!bad.empty()) { fail(errbuf, errbuf_len, bad); return nullptr; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) { fail(errbuf, errbuf_len, std::string("no CUDA device: ") + cudaGetErrorString(e)); return nullptr; }
    // device list: params.devices[0 .. n_devices) (n_devices = -1: every visible device), else the single params.device
    std::vector<int> ords;
    if (p->n_devices < 0) for (int d = 0; d < std::min(ndev, kMaxDevices); ++d) ords.push_back(d);
    else if (p->n_devices > 0) { for (int d = 0; d < std::min(p->n_devices, kMaxDevices); ++d) ords.push_back(p->devices[d]); }
    else ords.push_back(p->device);
    for (size_t a = 0; a < ords.size(); ++a) {
        if (ords[a] < 0 || ords[a] >= ndev) { fail(errbuf, errbuf_len, "device ordinal out of range"); return nullptr; }
        for (size_t b = 0; b < a; ++b) if (ords[a] == ords[b]) { fail(errbuf, errbuf_len, "device listed twice"); return nullptr; }
    }
    std::unique_ptr<barb200_ctx> ctx(new barb200_ctx());
    ctx->p = *p;
    ctx->lanes_per_device = p->lanes > 0 ? std::min(p->lanes, 2) : 2;
    if (getenv("BARB200_LANES")) ctx->lanes_per_device = std::max(1, std::min(2, atoi(getenv("BARB200_LANES"))));
    ctx->P = poa_params(p->mat, p->gap_open1, p->gap_ext1, p->gap_open2, p->gap_ext2, p->wb, p->wf);
    ctx->hp = HostParams{p->k, p->w, p->min_w, p->progressive_poa};
    int lane_index = 0;
    for (int ord : ords) {
        if (cudaSetDevice(ord) != cudaSuccess) { fail(errbuf, errbuf_len, "cudaSetDevice failed"); barb200_destroy(ctx.release()); return nullptr; }
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, ord) != cudaSuccess) { fail(errbuf, errbuf_len, "cudaGetDeviceProperties failed"); barb200_destroy(ctx.release()); return nullptr; }
        std::unique_ptr<Device> D(new Device());
        D->ordinal = ord; D->sm_count = prop.multiProcessorCount; D->mem_total = prop.totalGlobalMem;
        for (int i = 0; i < kNumKernels; ++i) {
            cudaFuncSetAttribute(kKernels[i].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kKernels[i].scratch);
            cudaFuncSetAttribute(kTraceKernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, kKernels[i].scratch);
        }
        bool ok = true;
        for (int l = 0; l < ctx->lanes_per_device && ok; ++l) {
            std::unique_ptr<Lane> L(new Lane());
            L->index = lane_index++;
            ok = cudaStreamCreateWithFlags(&L->main, cudaStreamNonBlocking) == cudaSuccess && cudaStreamCreateWithFlags(&L->copy, cudaStreamNonBlocking) == cudaSuccess;
            for (int c = 0; c < kNumKernels && ok; ++c)
                ok = cudaStreamCreateWithFlags(&L->cls[c], cudaStreamNonBlocking) == cudaSuccess && cudaEventCreateWithFlags(&L->cls_done[c], cudaEventDisableTiming) == cudaSuccess;
            D->lanes.push_back(std::move(L));
        }
        ctx->devs.push_back(std::move(D));
        if (!ok) { fail(errbuf, errbuf_len, "creating streams / pinned memory failed"); barb200_destroy(ctx.release()); return nullptr; }
    }
    cudaSetDevice(ords[0]);
    if (pecan_create(ctx.get()) != 0) { fail(errbuf, errbuf_len, "creating streams / pinned memory failed"); barb200_destroy(ctx.release()); return nullptr; }
    return ctx.release();
}

extern "C" void barb200_destroy(barb200_ctx *ctx) {
    if (!ctx) return;
    dispatcher_destroy(ctx);            // joins the lane threads (host_bar.cpp)
    for (auto &D : ctx->devs) {
        cudaSetDevice(D->ordinal);
        for (auto &L : D->lanes) {
            if (L->d_slots) cudaFree(L->d_slots);
            if (L->d_planes) cudaFree(L->d_planes);
            if (L->d_clk) cudaFree(L->d_clk);
            for (int c = 0; c < kNumKernels; ++c) { if (L->cls[c]) cudaStreamDestroy(L->cls[c]); if (L->cls_done[c]) cudaEventDestroy(L->cls_done[c]); }
            if (L->main) cudaStreamDestroy(L->main);
            if (L->copy) cudaStreamDestroy(L->copy);
        }
        for (auto &b : D->free_blocks) cudaFree(b.first);
        for (auto &b : D->free_pinned) cudaFreeHost(b.first);
    }
    if (!ctx->devs.empty()) cudaSetDevice(ctx->devs[0]->ordinal);
    pecan_destroy(ctx);
    delete ctx;
}

// The returned pointer stays valid until the calling thread's next call of this function (thread-local copy).
extern "C" const char *barb200_last_error(barb200_ctx *ctx) {
    if (!ctx) return "null context";
    static thread_local std::string out;
    out = get_error(ctx);
    return out.c_str();
}
extern "C" void barb200_free(void *p) { free(p); }
extern "C" void barb200_free_many(void *const *p, int64_t n) {
    if (!p) return;
    for (int64_t i = 0; i < n; ++i) free(p[i]);
}
// rows[i] (bytes[i] bytes each, e.g. the MSAs of a batch) -> dst back to back; parallel copy
extern "C" void barb200_pack_rows(void *const *rows, const int64_t *bytes, int64_t n, uint8_t *dst) {
    if (!rows || !bytes || !dst || n <= 0) return;
    std::vector<int64_t> off((size_t)n + 1, 0);
    for (int64_t i = 0; i < n; ++i) off[i + 1] = off[i] + bytes[i];
    static const int nt = std::min(usable_host_threads(), 16);
#pragma omp parallel for schedule(static) num_threads(nt)
    for (int64_t i = 0; i < n; ++i) if (rows[i] && bytes[i] > 0) memcpy(dst + off[i], rows[i], (size_t)bytes[i]);
}

extern "C" int barb200_device_count(barb200_ctx *ctx) { return ctx ? (int)ctx->devs.size() : 0; }

extern "C" int barb200_device_info(barb200_ctx *ctx, int *sm_count, int64_t *mem_total, int64_t *mem_free, char *name, int name_len) {
    if (!ctx) return BARB200_EINVAL;
    cudaSetDevice(ctx->devs[0]->ordinal);
    cudaDeviceProp prop; CUDA_TRY(ctx, cudaGetDeviceProperties(&prop, ctx->devs[0]->ordinal));
    size_t f = 0, t = 0; CUDA_TRY(ctx, cudaMemGetInfo(&f, &t));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (mem_total) *mem_total = (int64_t)t;
    if (mem_free) *mem_free = (int64_t)f;
    if (name && name_len > 0) snprintf(name, name_len, "%s", prop.name);
    return BARB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// stage: its plan is stage_plan.h's; here it is measured, allocated, uploaded, launched and fetched
// ---------------------------------------------------------------------------------------------------------
// a rejected job table: the context's message, BARB200_EINVAL
static int table_rc(barb200_ctx *ctx, const std::string &err) {
    if (err.empty()) return BARB200_OK;
    set_error(ctx, err); return BARB200_EINVAL;
}

struct barb200_stage {
    barb200_ctx *ctx = nullptr;
    int lane = 0;
    std::shared_ptr<const JobTable> tab;
    int64_t n_jobs = 0;
    StagePlan plan;
    std::vector<size_t> dyn_smem;                                    // per bucket: dynamic shared memory per CTA
    // device: one block from the device's cache holds all per-stage arrays; a retry's d_seqs are its first stage's
    void *d_block = nullptr;
    uint8_t *d_seqs = nullptr, *d_msa = nullptr; int *d_lens = nullptr; int64_t *d_soff = nullptr;
    JobDesc *d_desc = nullptr; int *d_msa_len = nullptr, *d_status = nullptr, *d_next = nullptr; long long *d_cells = nullptr;
    int *d_order = nullptr, *d_gt_status = nullptr; uint8_t *d_gt_scratch = nullptr;
    GuideTreeArgs gt; cudaEvent_t e_gt = nullptr;                    // K0: the guide trees of the stage (guide_tree.cu)
    TraceArgs trace{};                                               // a trace stage's regions (plan.trace)
    std::vector<int> status;                                         // of the last run
    std::vector<std::unique_ptr<barb200_stage>> retries;             // the last run's capacity retries: x4, then worst case
    int64_t launches = 0; bool ran = false;
    cudaEvent_t e0 = nullptr, e1 = nullptr; bool launched = false;
    uint64_t clk[7] = {0, 0, 0, 0, 0, 0, 0};
    ~barb200_stage() {
        cudaSetDevice(dev_of_lane(ctx, lane).ordinal);
        retries.clear();
        if (e0) { cudaEventDestroy(e0); cudaEventDestroy(e1); }
        if (e_gt) cudaEventDestroy(e_gt);
        dev_free(dev_of_lane(ctx, lane), d_block, (size_t)plan.block_bytes);
    }
};

extern "C" void barb200_stage_destroy(barb200_stage *st) { delete st; }

// Shared memory and resident CTAs of every bucket, and the memory the lane may plan with; fit_stage sizes the slots from them.
static int plan_stage(barb200_stage *st) {
    barb200_ctx *ctx = st->ctx;
    Device &D = dev_of_lane(ctx, st->lane);
    Lane &LN = lane_of(ctx, st->lane);
    std::vector<int> per_sm(st->plan.buckets.size(), 0);
    st->dyn_smem.assign(st->plan.buckets.size(), 0);
    for (size_t b = 0; b < st->plan.buckets.size(); ++b) {
        const PlanBucket &B = st->plan.buckets[b];
        size_t smem = kKernels[B.cls].scratch;
        if (getenv("BARB200_SCRATCH_KB")) smem = (size_t)atoi(getenv("BARB200_SCRATCH_KB")) * 1024;   // tuning aid
        // never below the sweep's ring, which the kernel uses without a run-time check (the topological sort and the MSA ranking
        // fit whatever is left, falling back to global memory)
        smem = std::max(smem, (size_t)poa_ring_bytes(B.T));
        if (st->plan.trace) CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[b], kTraceKernels[B.cls], B.T, smem));
        else CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[b], kKernels[B.cls].fn, B.T, smem));
        if (per_sm[b] < 1) { set_error(ctx, "kernel does not fit on an SM with the requested configuration"); return BARB200_EINVAL; }
        if (ctx->p.ctas_per_sm > 0) per_sm[b] = std::min(per_sm[b], ctx->p.ctas_per_sm);
        st->dyn_smem[b] = smem;
    }
    // memory: what is free now + what this lane's arena already holds, minus the stage's own block; a lane of a context
    // whose dispatcher runs plans with its share so that the other lane of the device can do the same
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(ctx, cudaMemGetInfo(&free_b, &total_b));
    const double budget = lane_budget_bytes((double)free_b, (double)total_b, (double)(LN.slots_bytes + LN.planes_bytes), (double)st->plan.block_bytes,
                                            ctx_mem_fraction(ctx), ctx->lanes_shared, ctx->lanes_per_device);
    const std::string err = fit_stage(st->plan, per_sm, D.sm_count, budget);
    if (!err.empty()) { set_error(ctx, err); return BARB200_ENOMEM; }
    return BARB200_OK;
}

static int ensure_arena(barb200_ctx *ctx, Device &D, Lane &LN, size_t slots_bytes, size_t planes_bytes, size_t clk_entries) {
    // a lane that has to grow goes straight to what its sibling already needed (same workload, same budget: plan_stage): which lane
    // meets the first large batch is a matter of timing, and a re-allocation costs tens of milliseconds plus a device synchronisation.
    // If that much is not free (the sibling was sized while it had the device to itself) the lane takes what the stage needs.
    auto grow = [&](void **p, size_t *have, size_t need, size_t sibling_max, const char *what) {
        if (need <= *have) return BARB200_OK;
        if (*p) cudaFree(*p);
        *p = nullptr; *have = 0;
        size_t want = std::max(need, sibling_max);
        if (cudaMalloc(p, want) != cudaSuccess) {
            cudaGetLastError(); *p = nullptr;
            if (want == need || cudaMalloc(p, need) != cudaSuccess) { cudaGetLastError(); *p = nullptr; set_error(ctx, std::string("cudaMalloc(") + what + ") failed"); return BARB200_ENOMEM; }
            want = need;
        }
        *have = want;
        return BARB200_OK;
    };
    size_t sib_slots = 0, sib_planes = 0;
    for (auto &other : D.lanes) if (other.get() != &LN) { sib_slots = std::max(sib_slots, other->slots_bytes); sib_planes = std::max(sib_planes, other->planes_bytes); }
    int rc = grow((void **)&LN.d_slots, &LN.slots_bytes, slots_bytes, sib_slots, "slots");
    if (!rc) rc = grow((void **)&LN.d_planes, &LN.planes_bytes, planes_bytes, sib_planes, "planes");
    if (rc) return rc;
    if (clk_entries > LN.clk_entries) {
        if (LN.d_clk) cudaFree(LN.d_clk);
        LN.d_clk = nullptr; LN.clk_entries = 0;
        if (cudaMalloc(&LN.d_clk, clk_entries * sizeof(unsigned long long)) != cudaSuccess) { cudaGetLastError(); set_error(ctx, "cudaMalloc(clk) failed"); return BARB200_ENOMEM; }
        LN.clk_entries = clk_entries;
    }
    return BARB200_OK;
}

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static bool timing_on() { static const bool on = getenv("BARB200_TIMING") != nullptr; return on; }

// BARB200_TRACE_REGION_SCALE (test aid, read at every stage): a factor on a trace stage's regions below the worst case, so that a test
// can make them overflow on any input (the kernel's capacity check, JOB_ERR_TRACE_CAP and its retries)
static double trace_region_scale() {
    const char *v = getenv("BARB200_TRACE_REGION_SCALE");
    return v ? std::max(0.0, atof(v)) : 1.0;
}

// A stage over the table's jobs `jobs` (caller indices); grow / worst_case size the slots (capacity-miss retries). A call's first
// stage uploads the table's bases from `seqs`; a retry runs on its first stage's device copy `d_seqs` and uploads none. trace: the
// stage runs the trace kernels (barb200_poa_trace_batch).
static int stage_build(barb200_ctx *ctx, int lane, std::shared_ptr<const JobTable> tab, std::vector<int64_t> jobs, double grow, bool worst_case,
                       const uint8_t *seqs, uint8_t *d_seqs, barb200_stage **out, bool trace = false) {
    Device &D = dev_of_lane(ctx, lane);
    Lane &LN = lane_of(ctx, lane);
    cudaSetDevice(D.ordinal);
    std::unique_ptr<barb200_stage> st(new barb200_stage());
    const int64_t n_jobs = (int64_t)jobs.size();
    st->ctx = ctx; st->lane = lane; st->tab = std::move(tab); st->n_jobs = n_jobs;
    const double tb0 = now_ms();
    const StagePlan &S = st->plan = plan_stage_order(*st->tab, std::move(jobs), ctx->p, grow, worst_case, D.sm_count, d_seqs == nullptr, trace,
                                                     trace ? trace_region_scale() : 1.0);
    if (n_jobs == 0) { *out = st.release(); return BARB200_OK; }
    const double tb2 = now_ms();
    int rc = plan_stage(st.get());
    if (rc) return rc;
    const double tb3 = now_ms();
    // device buffers (one cached block) + upload on the lane's copy stream, so that it overlaps a running kernel
    cudaError_t e = dev_alloc(D, &st->d_block, (size_t)S.block_bytes);
    if (e != cudaSuccess) {
        cudaGetLastError(); set_error(ctx, std::string("cudaMalloc(stage) failed: ") + cudaGetErrorString(e));
        st->d_block = nullptr; return BARB200_ENOMEM;
    }
    uint8_t *blk = (uint8_t *)st->d_block;
    st->d_seqs = d_seqs ? d_seqs : blk + S.o_seqs; st->d_lens = (int *)(blk + S.o_lens); st->d_soff = (int64_t *)(blk + S.o_soff);
    st->d_desc = (JobDesc *)(blk + S.o_desc); st->d_msa = blk + S.o_msa; st->d_msa_len = (int *)(blk + S.o_msa_len); st->d_status = (int *)(blk + S.o_status);
    st->d_cells = (long long *)(blk + S.o_cells); st->d_next = (int *)(blk + S.o_next);
    st->d_order = (int *)(blk + S.o_order); st->d_gt_status = (int *)(blk + S.o_gt_status); st->d_gt_scratch = blk + S.o_gt_scratch;
    if (S.trace) {
        st->trace.words = (int64_t *)(blk + S.o_trace); st->trace.off = (const int64_t *)(blk + S.o_trace_off);
        st->trace.cap = (const int64_t *)(blk + S.o_trace_cap); st->trace.used = (int64_t *)(blk + S.o_trace_used);
    }
    GuideTreeArgs &GA = st->gt;
    memset(&GA, 0, sizeof(GA));
    GA.jobs = st->d_desc; GA.n_jobs = (int)n_jobs; GA.seqs = st->d_seqs; GA.lens = st->d_lens; GA.soff = st->d_soff; GA.order = st->d_order; GA.gt_status = st->d_gt_status;
    GA.next_job = st->d_next + kNumKernels; GA.scratch = st->d_gt_scratch; GA.lay = S.gt; GA.k = ctx->p.k; GA.w = ctx->p.w;
    cudaStream_t s = LN.copy;
    const int64_t ns = S.n_seqs;
    const double tb4 = now_ms();
    if ((!d_seqs && (e = cudaMemcpyAsync(st->d_seqs, seqs, st->tab->n_bases, cudaMemcpyHostToDevice, s)) != cudaSuccess) ||
        (e = cudaMemcpyAsync(st->d_lens, S.lens.data(), ns * 4, cudaMemcpyHostToDevice, s)) != cudaSuccess ||
        (e = cudaMemcpyAsync(st->d_soff, S.soff.data(), ns * 8, cudaMemcpyHostToDevice, s)) != cudaSuccess ||
        (e = cudaMemcpyAsync(st->d_desc, S.desc.data(), n_jobs * sizeof(JobDesc), cudaMemcpyHostToDevice, s)) != cudaSuccess ||
        (S.trace && (e = cudaMemcpyAsync((void *)st->trace.off, S.trace_off.data(), n_jobs * 8, cudaMemcpyHostToDevice, s)) != cudaSuccess) ||
        (S.trace && (e = cudaMemcpyAsync((void *)st->trace.cap, S.trace_cap.data(), n_jobs * 8, cudaMemcpyHostToDevice, s)) != cudaSuccess) ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess) {
        set_error(ctx, std::string("H2D failed: ") + cudaGetErrorString(e)); return BARB200_ECUDA;
    }
    if (timing_on()) fprintf(stderr, "barb200 timing: stage_build: order + descriptors %.2f ms, plan %.2f, alloc %.2f, upload %.2f\n",
                             tb2 - tb0, tb3 - tb2, tb4 - tb3, now_ms() - tb4);
    *out = st.release();
    return BARB200_OK;
}

extern "C" int barb200_stage_create(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens,
                                    const uint8_t *seqs, const int *progressive, barb200_stage **out) {
    if (!ctx || !out) return BARB200_EINVAL;
    auto tab = std::make_shared<JobTable>();
    const int rc = table_rc(ctx, table_of_arrays(ctx->p, host_threads(ctx), n_jobs, n_seq, seq_lens, seqs, progressive, *tab));
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(lane_of(ctx, 0).busy);
    return stage_build(ctx, 0, tab, all_jobs(n_jobs), 1.0, false, seqs, nullptr, out);
}

// queue the stage's kernels on its lane's streams; returns without waiting
static int stage_launch(barb200_stage *st) {
    barb200_ctx *ctx = st->ctx;
    Device &D = dev_of_lane(ctx, st->lane);
    Lane &LN = lane_of(ctx, st->lane);
    cudaSetDevice(D.ordinal);
    st->launches = 0; st->ran = false; st->launched = false;
    if (st->n_jobs == 0) return BARB200_OK;
    st->retries.clear();
    const StagePlan &S = st->plan;
    const size_t clk_n = ctx->p.collect_phase_clocks ? S.clk_entries : 0;
    int rc = ensure_arena(ctx, dev_of_lane(ctx, st->lane), LN, S.slots_bytes, S.plane_ints * 4, clk_n);
    if (rc) return rc;
    cudaStream_t s = LN.main;
    CUDA_TRY(ctx, cudaMemsetAsync(st->d_next, 0, 4 * (kNumKernels + 1), s));
    CUDA_TRY(ctx, cudaMemsetAsync(st->d_msa, 0, S.msa_bytes, s));     // the rows' padding travels back with the MSAs (one D2H copy): defined bytes
    if (clk_n) CUDA_TRY(ctx, cudaMemsetAsync(LN.d_clk, 0, clk_n * sizeof(unsigned long long), s));
    if (!st->e0) { CUDA_TRY(ctx, cudaEventCreate(&st->e0)); CUDA_TRY(ctx, cudaEventCreate(&st->e1)); }
    if (!st->e_gt) CUDA_TRY(ctx, cudaEventCreate(&st->e_gt));
    CUDA_TRY(ctx, cudaEventRecord(st->e0, s));
    // K0: the guide trees of every job (guide_tree.cu); the POA launches below wait for it through the stream / e_gt
    launch_guide_tree(st->gt, S.gt_ctas, (void *)s);
    { cudaError_t le = cudaGetLastError(); if (le != cudaSuccess) { set_error(ctx, std::string("guide tree launch: ") + cudaGetErrorString(le)); return BARB200_ECUDA; } }
    CUDA_TRY(ctx, cudaEventRecord(st->e_gt, s));
    st->launches++;
    const bool single = S.buckets.size() == 1;
    for (size_t b = 0; b < S.buckets.size(); ++b) {          // largest class first
        const PlanBucket &B = S.buckets[b];
        BatchArgs A;
        A.jobs = st->d_desc; A.job_base = (int)B.job_base; A.n_jobs = (int)B.n_jobs; A.seqs = st->d_seqs; A.lens = st->d_lens; A.soff = st->d_soff;
        A.order = st->d_order; A.gt_status = st->d_gt_status;
        A.msa = st->d_msa; A.msa_len = st->d_msa_len; A.status = st->d_status; A.cells = st->d_cells;
        A.slots = LN.d_slots + B.slot_off; A.planes = LN.d_planes + B.plane_off; A.next_job = st->d_next + b;
        A.phase_clk = clk_n ? LN.d_clk + B.clk_off : nullptr;
        A.serial_phases = getenv("BARB200_DEBUG_SERIAL") ? 1 : 0;
        // a trace stage numbers its rows as abPOA does (the BFS order after every fusion): the splice's order is an equally valid
        // topological order with the same DP values per node, but other row indices, and the trace compares bands row by row. So a
        // trace does not run the production kernels' splice order, nor the far-row paths that order gives the sweep
        A.bfs_order = (S.trace || getenv("BARB200_DEBUG_BFS")) ? 1 : 0;
        A.scratch_bytes = (int)st->dyn_smem[b]; A.lay = B.lay; A.P = ctx->P;
        cudaStream_t cs = single ? s : LN.cls[B.cls];
        if (!single) CUDA_TRY(ctx, cudaStreamWaitEvent(cs, st->e_gt, 0));
        if (S.trace) kTraceKernels[B.cls]<<<B.slots, B.T, st->dyn_smem[b], cs>>>(A, st->trace);
        else kKernels[B.cls].fn<<<B.slots, B.T, st->dyn_smem[b], cs>>>(A);
        cudaError_t le = cudaGetLastError();
        if (le != cudaSuccess) { set_error(ctx, std::string("kernel launch: ") + cudaGetErrorString(le)); return BARB200_ECUDA; }
        if (!single) { CUDA_TRY(ctx, cudaEventRecord(LN.cls_done[B.cls], cs)); CUDA_TRY(ctx, cudaStreamWaitEvent(s, LN.cls_done[B.cls], 0)); }
        st->launches++;
    }
    CUDA_TRY(ctx, cudaEventRecord(st->e1, s));
    // (no device-to-host copy here: into pageable memory it would block the host until the kernels are done;
    // stage_finish fetches the statuses after its synchronisation)
    st->launched = true;
    return BARB200_OK;
}

// wait for the stage's kernels and collect their device time; re-run the capacity misses of each round with larger slots (x4,
// then worst case) on the stage's uploaded inputs
static int stage_finish(barb200_stage *st, float *kernel_ms) {
    barb200_ctx *ctx = st->ctx;
    Device &D = dev_of_lane(ctx, st->lane);
    Lane &LN = lane_of(ctx, st->lane);
    if (kernel_ms) *kernel_ms = 0.f;
    if (st->n_jobs == 0) { st->ran = true; return BARB200_OK; }
    if (!st->launched) { set_error(ctx, "stage_finish without stage_launch"); return BARB200_EINVAL; }
    cudaSetDevice(D.ordinal);
    cudaStream_t s = LN.main;
    float ms = 0.f;
    for (int k = 0; k < 7; ++k) st->clk[k] = 0;
    std::deque<RetryRound> pending;                  // retry stages still to run
    for (barb200_stage *r = st;;) {
        cudaError_t se = cudaStreamSynchronize(s);
        if (se != cudaSuccess) { set_error(ctx, std::string("kernel execution: ") + cudaGetErrorString(se)); return BARB200_ECUDA; }
        float rms = 0.f; cudaEventElapsedTime(&rms, r->e0, r->e1);
        float gt_ms = 0.f; cudaEventElapsedTime(&gt_ms, r->e0, r->e_gt);
        ms += rms;
        r->launched = false;
        r->status.resize(r->n_jobs);
        CUDA_TRY(ctx, cudaMemcpyAsync(r->status.data(), r->d_status, r->n_jobs * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        st->clk[6] += (uint64_t)(gt_ms * 1e6f);          // K0 is a kernel of its own: its device time, in nanoseconds
        if (ctx->p.collect_phase_clocks) {
            const size_t clk_n = r->plan.clk_entries;
            std::vector<unsigned long long> h(clk_n);
            CUDA_TRY(ctx, cudaMemcpy(h.data(), LN.d_clk, clk_n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
            for (size_t b = 0; b < clk_n / PH_N; ++b) for (int k = 0; k < 6; ++k) st->clk[k] += h[b * PH_N + k];
        }
        // capacity misses -> retry launch for just those jobs with larger slots (x4 first, then worst case); a trace stage's retry may
        // be cut into several stages (retry_batches), which run one after the other
        RetryRound next;
        const std::string err = retry_round(r->plan, r->status, next);
        if (!err.empty()) { set_error(ctx, err); return BARB200_EJOB; }
        if (!next.jobs.empty())
            for (std::vector<int64_t> &b : retry_batches(*st->tab, r->plan, next)) pending.push_back(RetryRound{std::move(b), next.grow, next.worst_case});
        if (pending.empty()) break;
        RetryRound todo = std::move(pending.front());
        pending.pop_front();
        barb200_stage *rs = nullptr;
        int rc = stage_build(ctx, st->lane, st->tab, std::move(todo.jobs), todo.grow, todo.worst_case, nullptr, st->d_seqs, &rs, st->plan.trace);
        if (rc) return rc;
        st->retries.emplace_back(rs);
        if ((rc = stage_launch(rs))) return rc;
        st->launches += rs->launches;
        r = rs;
    }
    if (kernel_ms) *kernel_ms = ms;
    st->ran = true;
    return BARB200_OK;
}

extern "C" int barb200_stage_run(barb200_stage *st, float *kernel_ms) {
    if (!st) return BARB200_EINVAL;
    std::lock_guard<std::mutex> lk(lane_of(st->ctx, st->lane).busy);
    const int rc = stage_launch(st);
    return rc ? rc : stage_finish(st, kernel_ms);
}

extern "C" int64_t barb200_stage_launches(barb200_stage *st) { return st ? st->launches : 0; }

extern "C" int barb200_stage_phase_clocks(barb200_stage *st, uint64_t out[7]) {
    if (!st || !out) return BARB200_EINVAL;
    for (int k = 0; k < 7; ++k) out[k] = st->clk[k];
    return BARB200_OK;
}

// per-bucket facts of a stage for reports: for bucket b, out[4b..4b+3] = threads per CTA, jobs, resident CTAs, plane ints per slot
extern "C" int barb200_stage_buckets(barb200_stage *st, int64_t *out, int max_buckets) {
    if (!st) return 0;
    int n = 0;
    for (const PlanBucket &B : st->plan.buckets) {
        if (n >= max_buckets) break;
        if (out) { out[4 * n] = B.T; out[4 * n + 1] = B.n_jobs; out[4 * n + 2] = B.slots; out[4 * n + 3] = B.lay.plane_cap; }
        ++n;
    }
    return n;
}

// dest(caller job index, K, msa_len) -> where the K x msa_len bytes go (nullptr: allocation failure)
typedef std::function<uint8_t *(int64_t, int, int)> MsaDest;

// every job's result comes from the round that completed it: the stage itself or one of its retries
static int stage_fetch_locked(barb200_stage *st, const MsaDest &dest, int *msa_len, int64_t *cells) {
    barb200_ctx *ctx = st->ctx;
    Device &D = dev_of_lane(ctx, st->lane);
    Lane &LN = lane_of(ctx, st->lane);
    if (!st->ran) { set_error(ctx, "stage_fetch before stage_run"); return BARB200_EINVAL; }
    if (st->n_jobs == 0) return BARB200_OK;
    cudaSetDevice(D.ordinal);
    std::vector<barb200_stage *> rounds{st};
    for (auto &rs : st->retries) rounds.push_back(rs.get());
    for (barb200_stage *r : rounds) {
        std::vector<int> r_len(r->n_jobs); std::vector<long long> r_cells(r->n_jobs);
        PinnedBlock down(D, (size_t)r->plan.msa_bytes);
        if (!down.p) { set_error(ctx, "cudaMallocHost failed"); return BARB200_ENOMEM; }
        uint8_t *h_msa = (uint8_t *)down.p;
        cudaStream_t s = LN.main;
        CUDA_TRY(ctx, cudaMemcpyAsync(r_len.data(), r->d_msa_len, r->n_jobs * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(r_cells.data(), r->d_cells, r->n_jobs * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(h_msa, r->d_msa, r->plan.msa_bytes, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        int oom = 0;
        const int nthreads = host_threads(ctx);
#pragma omp parallel for schedule(static) num_threads(nthreads) reduction(| : oom)
        for (int64_t j = 0; j < r->n_jobs; ++j) {
            if (r->status[j] != JOB_OK) continue;           // re-run by a later round
            const JobDesc &d = r->plan.desc[j];
            const int64_t c = r->plan.perm[j];
            const int K = d.n_seq, ml = r_len[j];
            if (msa_len) msa_len[c] = ml;
            if (cells) cells[c] = r_cells[j];
            if (dest) {
                uint8_t *o = dest(c, K, ml);
                if (!o) { oom = 1; continue; }
                const uint8_t *src = h_msa + d.msa_off;
                for (int i = 0; i < K; ++i) memcpy(o + (size_t)i * ml, src + (size_t)i * d.msa_stride, ml);
            }
        }
        if (oom) { set_error(ctx, "host allocation failed"); return BARB200_ENOMEM; }
    }
    return BARB200_OK;
}

static MsaDest malloc_dest(uint8_t **msa_out) {
    if (!msa_out) return MsaDest();
    return [msa_out](int64_t c, int K, int ml) { uint8_t *o = (uint8_t *)malloc((size_t)K * (ml > 0 ? ml : 1)); msa_out[c] = o; return o; };
}

extern "C" int barb200_stage_fetch(barb200_stage *st, uint8_t **msa_out, int *msa_len, int64_t *cells) {
    if (!st) return BARB200_EINVAL;
    std::lock_guard<std::mutex> lk(lane_of(st->ctx, st->lane).busy);
    return stage_fetch_locked(st, malloc_dest(msa_out), msa_len, cells);
}


// one device batch of the table's jobs `jobs` on one lane (the caller holds the lane): build + launch + streamed guide trees +
// finish + fetch; results land at the caller's job indices
static int batch_on_lane(barb200_ctx *ctx, int lane, const std::shared_ptr<const JobTable> &tab, std::vector<int64_t> jobs, const uint8_t *seqs,
                         const MsaDest &dest, int *msa_len, int64_t *cells) {
    barb200_stage *st = nullptr;
    const int64_t n_jobs = (int64_t)jobs.size();
    const double t0 = now_ms();
    int rc = stage_build(ctx, lane, tab, std::move(jobs), 1.0, false, seqs, nullptr, &st);
    if (rc) return rc;
    const double t1 = now_ms(); float kms = 0.f;
    rc = stage_launch(st);
    if (!rc) rc = stage_finish(st, &kms);
    const double t2 = now_ms();
    if (!rc) rc = stage_fetch_locked(st, dest, msa_len, cells);
    const double t3 = now_ms();
    barb200_stage_destroy(st);
    {
        std::lock_guard<std::mutex> lk(ctx->err_mu);
        ctx->last_timing[0] = t1 - t0; ctx->last_timing[1] = t2 - t1; ctx->last_timing[2] = kms; ctx->last_timing[3] = t3 - t2;
        ctx->last_timing[4] = now_ms() - t0; ctx->last_timing[5] = (double)n_jobs;
    }
    if (timing_on()) fprintf(stderr, "barb200 timing: lane %d, %lld jobs: build %.1f ms, run %.1f ms (%.1f on the device), fetch %.1f ms, destroy %.1f ms\n",
                             lane, (long long)n_jobs, t1 - t0, t2 - t1, kms, t3 - t2, now_ms() - t3);
    return rc;
}

// The table's jobs dealt over the context's devices (deal_jobs); each device's share is cut into device batches (chunk_ends, with
// trace_words for a trace call) that run(lane, jobs) runs one after the other on the device's first lane, the devices in parallel.
// Returns BARB200_OK or the code of a failed device, with that device's message.
static int run_dealt(barb200_ctx *ctx, const JobTable &tab, int64_t trace_words, const std::function<int(int, std::vector<int64_t>)> &run) {
    const int ndev = (int)ctx->devs.size();
    const std::vector<std::vector<int64_t>> share = deal_jobs(tab, ndev);
    std::vector<int> rcs(ndev, BARB200_OK);
    std::vector<std::string> errs(ndev);
    int active_devs = 0;
    for (int d = 0; d < ndev; ++d) active_devs += !share[d].empty();
    auto run_device = [&](int d) {
        tl_thread_divisor = std::max(1, active_devs);
        const std::vector<int64_t> &mine = share[d];
        const int lane = d * ctx->lanes_per_device;
        std::lock_guard<std::mutex> lk(lane_of(ctx, lane).busy);
        size_t at = 0;
        for (size_t end : chunk_ends(tab, mine, trace_words)) {
            const int rc = run(lane, std::vector<int64_t>(mine.begin() + at, mine.begin() + end));
            if (rc) { rcs[d] = rc; errs[d] = get_error(ctx); break; }
            at = end;
        }
    };
    if (ndev == 1) run_device(0);
    else {
        std::vector<std::thread> th;
        for (int d = 0; d < ndev; ++d) if (!share[d].empty()) th.emplace_back(run_device, d);
        for (auto &t : th) t.join();
    }
    for (int d = 0; d < ndev; ++d) if (rcs[d]) { set_error(ctx, errs[d]); return rcs[d]; }
    return BARB200_OK;
}

extern "C" int barb200_poa_msa_batch(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens,
                                     const uint8_t *seqs, const int *progressive, uint8_t **msa_out, int *msa_len,
                                     int64_t *cells) {
    if (!ctx) return BARB200_EINVAL;
    if (msa_out) for (int64_t j = 0; j < n_jobs; ++j) msa_out[j] = nullptr;
    auto tab = std::make_shared<JobTable>();
    const int trc = table_rc(ctx, table_of_arrays(ctx->p, host_threads(ctx), n_jobs, n_seq, seq_lens, seqs, progressive, *tab));
    if (trc || n_jobs == 0) return trc;
    const int rc = run_dealt(ctx, *tab, 0, [&](int lane, std::vector<int64_t> jobs) {
        return batch_on_lane(ctx, lane, tab, std::move(jobs), seqs, malloc_dest(msa_out), msa_len, cells);
    });
    if (rc && msa_out) for (int64_t j = 0; j < n_jobs; ++j) { free(msa_out[j]); msa_out[j] = nullptr; }
    return rc;
}

// One device batch of a trace call on one lane (the caller holds the lane): the trace kernels' stage and its capacity retries, then
// every job's word array (include/barb200.h) from the round that completed it -- header, read order, the kernel's records, the MSA.
// cells: per caller job, filled on the way.
static int trace_batch_on_lane(barb200_ctx *ctx, int lane, const std::shared_ptr<const JobTable> &tab, std::vector<int64_t> jobs, const uint8_t *seqs,
                               int64_t **trace_out, int64_t *n_words, int64_t *cells) {
    barb200_stage *stp = nullptr;
    int rc = stage_build(ctx, lane, tab, std::move(jobs), 1.0, false, seqs, nullptr, &stp, true);
    if (rc) return rc;
    std::unique_ptr<barb200_stage> st(stp);
    if ((rc = stage_launch(st.get())) || (rc = stage_finish(st.get(), nullptr))) return rc;
    if (st->n_jobs == 0) return BARB200_OK;
    // the records and read orders of every round, and where each caller job's are
    std::vector<barb200_stage *> rounds{st.get()};
    for (auto &r : st->retries) rounds.push_back(r.get());
    std::vector<std::vector<int64_t>> words(rounds.size()), used(rounds.size());
    std::vector<std::vector<int>> order(rounds.size());
    struct Done { const int64_t *rec; int64_t n; const int *order; };
    std::unordered_map<int64_t, Done> done;
    cudaStream_t s = lane_of(ctx, lane).main;
    for (size_t k = 0; k < rounds.size(); ++k) {
        barb200_stage *r = rounds[k];
        words[k].resize(r->plan.trace_words); used[k].resize(r->n_jobs); order[k].resize(r->plan.n_seqs);
        CUDA_TRY(ctx, cudaMemcpyAsync(words[k].data(), r->trace.words, words[k].size() * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(used[k].data(), r->trace.used, used[k].size() * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(order[k].data(), r->d_order, order[k].size() * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        for (int64_t j = 0; j < r->n_jobs; ++j)
            if (r->status[j] == JOB_OK) done[r->plan.perm[j]] = Done{words[k].data() + r->plan.trace_off[j], used[k][j], order[k].data() + r->plan.desc[j].len_off};
    }
    // the MSA lands behind the records: stage_fetch_locked writes its K rows of msa_len bytes back to back where dest points
    const MsaDest dest = [&](int64_t c, int K, int ml) -> uint8_t * {
        const Done &D = done.at(c);
        const int64_t msa_words = ((int64_t)K * ml + 7) / 8, n = 3 + K + D.n + msa_words;
        int64_t *w = (int64_t *)malloc((size_t)n * 8);
        if (!w) return nullptr;
        w[0] = K; w[1] = ml; w[2] = cells[c];
        for (int i = 0; i < K; ++i) w[3 + i] = D.order[i];
        memcpy(w + 3 + K, D.rec, (size_t)D.n * 8);
        if (msa_words) w[n - 1] = 0;
        trace_out[c] = w; n_words[c] = n;
        return (uint8_t *)(w + 3 + K + D.n);
    };
    return stage_fetch_locked(st.get(), dest, nullptr, cells);
}

extern "C" int barb200_poa_trace_batch(barb200_ctx *ctx, int64_t n_jobs, const int *n_seq, const int *seq_lens, const uint8_t *seqs,
                                       const int *progressive, int64_t **trace_out, int64_t *n_words) {
    if (!ctx) return BARB200_EINVAL;
    if (n_jobs > 0 && (!trace_out || !n_words)) { set_error(ctx, "bad arguments"); return BARB200_EINVAL; }
    for (int64_t j = 0; j < n_jobs; ++j) { trace_out[j] = nullptr; n_words[j] = 0; }
    auto tab = std::make_shared<JobTable>();
    const int trc = table_rc(ctx, table_of_arrays(ctx->p, host_threads(ctx), n_jobs, n_seq, seq_lens, seqs, progressive, *tab));
    if (trc || n_jobs == 0) return trc;
    std::vector<int64_t> cells(n_jobs, 0);
    const int rc = run_dealt(ctx, *tab, kMaxTraceWordsPerBatch, [&](int lane, std::vector<int64_t> jobs) {
        return trace_batch_on_lane(ctx, lane, tab, std::move(jobs), seqs, trace_out, n_words, cells.data());
    });
    if (rc) for (int64_t j = 0; j < n_jobs; ++j) { free(trace_out[j]); trace_out[j] = nullptr; n_words[j] = 0; }
    return rc;
}

// host-side phases of the most recent device batch, milliseconds: out[0] build (ordering, planning, H2D), out[1] launch +
// streamed guide trees + wait, out[2] device time of the kernels, out[3] fetch (D2H + unpack), out[4] total, out[5] jobs
extern "C" int barb200_last_batch_timing(barb200_ctx *ctx, double out[6]) {
    if (!ctx || !out) return BARB200_EINVAL;
    std::lock_guard<std::mutex> lk(ctx->err_mu);
    for (int k = 0; k < 6; ++k) out[k] = ctx->last_timing[k];
    return BARB200_OK;
}

namespace barb200 {
// One device batch of host jobs on lane `lane` (host_bar.cpp's dispatcher): the jobs' sequences are packed once into the
// lane's pinned upload buffer, the MSAs unpacked straight into the results.
int run_jobs_on_lane(barb200_ctx *ctx, int lane, const std::vector<HostJob> &jobs, std::vector<JobResult> &results) {
    const int64_t n = (int64_t)jobs.size();
    results.assign(n, JobResult());
    if (n == 0) return BARB200_OK;
    auto tab = std::make_shared<JobTable>();
    int rc = table_rc(ctx, build_table(ctx->p, host_threads(ctx), n, [&](int64_t j, int64_t, int64_t) { return jobs[j]; }, *tab));
    if (rc) return rc;
    const std::vector<TableJob> &J = tab->jobs;
    Lane &LN = lane_of(ctx, lane);
    std::lock_guard<std::mutex> lk(LN.busy);
    cudaSetDevice(dev_of_lane(ctx, lane).ordinal);
    PinnedBlock up(dev_of_lane(ctx, lane), (size_t)tab->n_bases);
    if (!up.p) { set_error(ctx, "cudaMallocHost failed"); return BARB200_ENOMEM; }
    uint8_t *const h_up = (uint8_t *)up.p;
    const int nthreads = host_threads(ctx);
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (int64_t j = 0; j < n; ++j) memcpy(h_up + J[j].seq_off, jobs[j].seqs, (size_t)J[j].sum_len);
    std::vector<int> ml(n, 0); std::vector<int64_t> cells(n, 0);
    JobResult *res = results.data();
    static uint8_t empty_sink[1];
    MsaDest dest = [res](int64_t c, int K, int m) { res[c].msa.resize((size_t)K * m); return res[c].msa.empty() ? empty_sink : res[c].msa.data(); };
    rc = batch_on_lane(ctx, lane, tab, all_jobs(n), h_up, dest, ml.data(), cells.data());
    if (rc) return rc;
    for (int64_t j = 0; j < n; ++j) { results[j].msa_len = ml[j]; results[j].cells = cells[j]; }
    return BARB200_OK;
}

// host jobs as one barb200_poa_trace_batch call (host_end_trace.cpp's rounds)
int run_trace_jobs(barb200_ctx *ctx, const std::vector<HostJob> &jobs, std::vector<std::vector<int64_t>> &words) {
    const int64_t n = (int64_t)jobs.size();
    words.assign(n, std::vector<int64_t>());
    if (n == 0) return BARB200_OK;
    std::vector<int> n_seq(n), prog(n), lens; std::vector<uint8_t> seqs;
    for (int64_t j = 0; j < n; ++j) {
        const HostJob &J = jobs[j];
        n_seq[j] = J.n_seq; prog[j] = J.progressive;
        int64_t sum = 0;
        for (int i = 0; i < J.n_seq; ++i) { lens.push_back(J.lens[i]); sum += J.lens[i]; }
        seqs.insert(seqs.end(), J.seqs, J.seqs + sum);
    }
    std::vector<int64_t *> out(n, nullptr); std::vector<int64_t> nw(n, 0);
    const int rc = barb200_poa_trace_batch(ctx, n, n_seq.data(), lens.data(), seqs.data(), prog.data(), out.data(), nw.data());
    if (rc) return rc;
    for (int64_t j = 0; j < n; ++j) { words[j].assign(out[j], out[j] + nw[j]); free(out[j]); }
    return BARB200_OK;
}
}  // namespace barb200
