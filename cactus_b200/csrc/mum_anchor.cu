// mum_anchor.cu -- K5: cPecan's MUM anchor chains (getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1,
// submodules/cPecan/impl/pairwiseAligner.c:1222-1231, 1849-2121) for many sequence pairs at once, and the C ABI
// barb200_pecan_anchor_pairs_batch (include/barb200.h).
//
// A batch is cut into chunks that fit the device (mum_plan.h). Per chunk, one pass over its problems (first the pairs, then,
// with recursiveMums, every gap of their chains that exceeds anchorMatrixBiggerThanThis) runs:
//   mum_keys_kernel .......... the key of every X and Y k-mer of every pair (mum_anchor.cuh: make_key), one thread per k-mer;
//   mum_tile_sort_kernel ..... Y's k-mer starts of each problem in tiles of kTile, bitonic-sorted by key in shared memory;
//   mum_merge_kernel ......... merges of sorted runs in global memory (each element finds its place by a binary search in the
//                              partner run), doubling the run width until the longest problem is one run -- the path that
//                              serves Y up to Cactus' bandingLimit and beyond;
//   mum_search_kernel ........ getLongestUniqueMatch of every X position, one thread each;
//   mum_chain_kernel ......... the MUM rule, sweep line and traceback of each problem, one thread each (serial in x), with the
//                              chain copied densely for the host.
// The host splices the chains and the gaps' chains into the reference's order (mum_plan.h: splice).
// On a context of several devices the pairs that need a device are dealt to the devices by their bytes, and every device plans
// and runs its chunks on a host thread of its own (run_devices).
#include <cuda_runtime.h>
#include <omp.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <new>
#include <string>
#include <thread>
#include <vector>
#include "host_api.h"
#include "mum_anchor.cuh"
#include "pecan_plan.h"

using namespace barb200;
using namespace barb200::mum;

namespace {

const int kTile = 2048, kTileThreads = 512;

struct PairDev {
    int64_t codes_off;             // X codes, then Y codes
    int64_t key_off;               // in words: X keys, then Y keys
    int32_t lx, ly, nx, bits, per_word, words;
};

__device__ __forceinline__ KeyView key_view(const PairDev &P, const uint64_t *keys, int k) {
    KeyView K; K.keys = keys + P.key_off; K.y_base = P.nx; K.k = k; K.bits = P.bits; K.per_word = P.per_word; K.words = P.words;
    return K;
}

// last index i with off(i) <= v over a non-decreasing table
template <class F> __device__ __forceinline__ int find_owner(int n, int64_t v, F off) {
    int lo = 0, hi = n;
    while (hi - lo > 1) { const int m = (lo + hi) / 2; if (off(m) <= v) lo = m; else hi = m; }
    return lo;
}

__global__ void mum_keys_kernel(const PairDev *pairs, int n_pairs, const int64_t *kmer_off, const uint8_t *codes, uint64_t *keys, int k) {
    const int64_t total = kmer_off[n_pairs];
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int i = find_owner(n_pairs, t, [&](int m) { return kmer_off[m]; });
        const PairDev P = pairs[i];
        const int64_t r = t - kmer_off[i];                // X k-mers first, then Y k-mers
        const uint8_t *c = codes + P.codes_off + (r < P.nx ? r : P.lx + (r - P.nx));
        make_key(c, k, P.bits, P.per_word, P.words, keys + P.key_off + r * P.words);
    }
}

struct Tile { int32_t prob, start, count, pad; };

// bitonic sort of one tile's k-mer starts by key; keys staged in shared memory, a permutation of tile slots sorted
extern "C" __global__ void __launch_bounds__(kTileThreads) mum_tile_sort_kernel(const Tile *tiles, const Problem *probs, const PairDev *pairs,
                                                                                   const uint64_t *keys, int k, int32_t *sorted) {
    extern __shared__ uint64_t sk[];
    const Tile T = tiles[blockIdx.x];
    const Problem Pb = probs[T.prob];
    const PairDev P = pairs[Pb.pair];
    const KeyView K = key_view(P, keys, k);
    const int W = P.words;
    uint16_t *perm = (uint16_t *)(sk + (size_t)kTile * W);
    for (int i = threadIdx.x; i < kTile; i += blockDim.x) {
        perm[i] = (uint16_t)i;
        if (i < T.count) { const uint64_t *src = K.y(Pb.y0 + T.start + i); for (int w = 0; w < W; ++w) sk[(size_t)i * W + w] = src[w]; }
    }
    int size = 2;
    while (size < T.count) size <<= 1;
    __syncthreads();
    for (int s = 2; s <= size; s <<= 1) {
        for (int st = s >> 1; st > 0; st >>= 1) {
            for (int i = threadIdx.x; i < size; i += blockDim.x) {
                const int j = i ^ st;
                if (j > i) {
                    const int a = perm[i], b = perm[j];
                    // slots >= count sort last
                    const bool gt = a >= T.count ? b < T.count || a > b
                                                 : (b < T.count && key_less(sk + (size_t)b * W, sk + (size_t)a * W, W));
                    if (((i & s) == 0) == gt) { perm[i] = (uint16_t)b; perm[j] = (uint16_t)a; }
                }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < T.count; i += blockDim.x) sorted[Pb.ny_off + T.start + i] = Pb.y0 + T.start + perm[i];
}

// one merge level: runs of `width` (sorted) pairwise into runs of 2 * width; problems with fewer k-mers are copied
__global__ void mum_merge_kernel(const Problem *probs, int n_probs, const PairDev *pairs, const uint64_t *keys, int k, int64_t total,
                                 int32_t width, const int32_t *in, int32_t *out) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int pi = find_owner(n_probs, t, [&](int m) { return probs[m].ny_off; });
        const Problem Pb = probs[pi];
        const int32_t n = n_kmers(Pb.y1 - Pb.y0, k), i = (int32_t)(t - Pb.ny_off);
        const int32_t v = in[t];
        if (n <= width) { out[t] = v; continue; }
        const int32_t run = i / width, a0 = run * width;
        const bool left = (run & 1) == 0;
        const int32_t p0 = left ? a0 + width : a0 - width, p1 = left ? min(a0 + 2 * width, n) : a0;
        if (p0 >= n) { out[t] = v; continue; }
        const KeyView K = key_view(pairs[Pb.pair], keys, k);
        const uint64_t *kv = K.y(v);
        const int32_t *base = in + Pb.ny_off;
        int32_t lo = p0, hi = p1;                         // left run: partner elements < v; right run: partner elements <= v
        while (lo < hi) {
            const int32_t m = (lo + hi) / 2;
            const uint64_t *km = K.y(base[m]);
            const bool before = left ? key_less(km, kv, K.words) : !key_less(kv, km, K.words);
            if (before) lo = m + 1; else hi = m;
        }
        const int32_t dst = (left ? a0 : p0) + (i - a0) + (lo - p0);
        out[Pb.ny_off + dst] = v;
    }
}

__global__ void mum_search_kernel(const Problem *probs, int n_probs, const PairDev *pairs, const uint64_t *keys, int k, int64_t u, int64_t total,
                                  const int32_t *sorted, int32_t *match_y, int32_t *match_len) {
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int pi = find_owner(n_probs, t, [&](int m) { return probs[m].nx_off; });
        const Problem Pb = probs[pi];
        const KeyView K = key_view(pairs[Pb.pair], keys, k);
        const int32_t ny = n_kmers(Pb.y1 - Pb.y0, k), x = Pb.x0 + (int32_t)(t - Pb.nx_off);
        int len = 0;
        const int32_t j = longest_unique_match(K, sorted + Pb.ny_off, ny, x, u, &len);
        match_y[t] = j >= 0 ? sorted[Pb.ny_off + j] : -1;
        match_len[t] = len;
    }
}

__global__ void mum_chain_kernel(const Problem *probs, int n_probs, int k, const int32_t *match_y, const int32_t *match_len, MumRec *mums,
                                 int32_t *sweep, ChainMum *chain, ChainMum *dense, unsigned long long *dense_n, int64_t *out_off, int32_t *out_n) {
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_probs) return;
    const Problem Pb = probs[pi];
    const int64_t o = Pb.nx_off;
    const int32_t n = chain_problem(Pb.x0, Pb.x1, Pb.y0, k, match_y + o, match_len + o, mums + o, sweep + o, chain + o);
    const unsigned long long d = atomicAdd(dense_n, (unsigned long long)n);
    for (int32_t i = 0; i < n; ++i) dense[d + i] = chain[o + i];
    out_off[pi] = (int64_t)d; out_n[pi] = n;
}

thread_local double tl_timing[3];  // kernel ms, wall ms, launches of the calling thread's last batch

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// The device work of one chunk: buffers carved from one cached block, one stream.
struct Chunk {
    barb200_ctx *ctx;
    int dev = 0;                   // the context's device the chunk runs on
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    void *blk = nullptr; size_t blk_bytes = 0;
    PairDev *d_pairs = nullptr; int64_t *d_kmer_off = nullptr; uint8_t *d_codes = nullptr; uint64_t *d_keys = nullptr;
    int32_t *d_sa = nullptr, *d_sb = nullptr, *d_my = nullptr, *d_ml = nullptr, *d_sweep = nullptr;
    MumRec *d_mums = nullptr; ChainMum *d_chain = nullptr, *d_dense = nullptr;
    int64_t cap_nx = 0, cap_ny = 0;
    int n_pairs = 0, k = 0;
    int64_t u = 0;
    int max_words = 1;
    float kernel_ms = 0; int launches = 0;
    ~Chunk() {
        if (blk) device_free(ctx, dev, blk, blk_bytes);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
        if (s) cudaStreamDestroy(s);
    }
};

// one pass over `probs` (sum of their k-mer counts within the chunk's capacity): chains[p] = the chain of problem p
int run_pass(Chunk &C, const std::vector<Problem> &probs, std::vector<std::vector<ChainMum>> &chains) {
    barb200_ctx *ctx = C.ctx;
    const int np = (int)probs.size();
    chains.assign(np, std::vector<ChainMum>());
    if (np == 0) return BARB200_OK;
    const int64_t tot_nx = probs.back().nx_off + kmers(probs.back().x1 - probs.back().x0, C.k);
    const int64_t tot_ny = probs.back().ny_off + kmers(probs.back().y1 - probs.back().y0, C.k);
    std::vector<Tile> tiles;
    int32_t max_ny = 0;
    for (int p = 0; p < np; ++p) {
        const int32_t ny = (int32_t)kmers(probs[p].y1 - probs[p].y0, C.k);
        max_ny = std::max(max_ny, ny);
        for (int32_t s = 0; s < ny; s += kTile) tiles.push_back(Tile{p, s, std::min(kTile, ny - s), 0});
    }
    // per-pass tables: problems, tiles, chain offsets / counts, dense counter
    const size_t b_probs = align256(sizeof(Problem) * np), b_tiles = align256(sizeof(Tile) * std::max<size_t>(tiles.size(), 1)),
                 b_off = align256(8 * (size_t)np), b_n = align256(4 * (size_t)np), bytes = b_probs + b_tiles + b_off + b_n + 256;
    void *tb = nullptr;
    if (device_alloc(ctx, C.dev, &tb, bytes) != 0) { set_error(ctx, "device allocation failed (MUM pass tables)"); return BARB200_ENOMEM; }
    struct Free { barb200_ctx *c; int d; void *p; size_t b; ~Free() { device_free(c, d, p, b); } } fr{ctx, C.dev, tb, bytes};
    Problem *d_probs = (Problem *)tb;
    Tile *d_tiles = (Tile *)((char *)tb + b_probs);
    int64_t *d_out_off = (int64_t *)((char *)tb + b_probs + b_tiles);
    int32_t *d_out_n = (int32_t *)((char *)tb + b_probs + b_tiles + b_off);
    unsigned long long *d_cnt = (unsigned long long *)((char *)tb + b_probs + b_tiles + b_off + b_n);
    CUDA_TRY(ctx, cudaMemcpyAsync(d_probs, probs.data(), sizeof(Problem) * np, cudaMemcpyHostToDevice, C.s));
    if (!tiles.empty()) CUDA_TRY(ctx, cudaMemcpyAsync(d_tiles, tiles.data(), sizeof(Tile) * tiles.size(), cudaMemcpyHostToDevice, C.s));
    CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, 8, C.s));
    const int grid = ctx_sm_count(ctx, C.dev) * 8;
    int32_t *cur = C.d_sa, *other = C.d_sb;
    if (!tiles.empty()) {
        const size_t smem = (size_t)kTile * C.max_words * 8 + (size_t)kTile * 2;
        CUDA_TRY(ctx, cudaFuncSetAttribute(mum_tile_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mum_tile_sort_kernel<<<(unsigned)tiles.size(), kTileThreads, smem, C.s>>>(d_tiles, d_probs, C.d_pairs, C.d_keys, C.k, cur);
        ++C.launches;
        for (int32_t w = kTile; w < max_ny; w *= 2) {
            mum_merge_kernel<<<grid, 256, 0, C.s>>>(d_probs, np, C.d_pairs, C.d_keys, C.k, tot_ny, w, cur, other);
            ++C.launches;
            std::swap(cur, other);
        }
    }
    if (tot_nx > 0) {
        mum_search_kernel<<<grid, 256, 0, C.s>>>(d_probs, np, C.d_pairs, C.d_keys, C.k, C.u, tot_nx, cur, C.d_my, C.d_ml);
        ++C.launches;
    }
    mum_chain_kernel<<<(np + 63) / 64, 64, 0, C.s>>>(d_probs, np, C.k, C.d_my, C.d_ml, C.d_mums, C.d_sweep, C.d_chain, C.d_dense, d_cnt,
                                                     d_out_off, d_out_n);
    ++C.launches;
    CUDA_TRY(ctx, cudaGetLastError());
    unsigned long long total = 0;
    std::vector<int64_t> off(np);
    std::vector<int32_t> cnt(np);
    CUDA_TRY(ctx, cudaMemcpyAsync(&total, d_cnt, 8, cudaMemcpyDeviceToHost, C.s));
    CUDA_TRY(ctx, cudaMemcpyAsync(off.data(), d_out_off, 8 * (size_t)np, cudaMemcpyDeviceToHost, C.s));
    CUDA_TRY(ctx, cudaMemcpyAsync(cnt.data(), d_out_n, 4 * (size_t)np, cudaMemcpyDeviceToHost, C.s));
    CUDA_TRY(ctx, cudaStreamSynchronize(C.s));
    std::vector<ChainMum> dense(total);
    if (total) CUDA_TRY(ctx, cudaMemcpy(dense.data(), C.d_dense, sizeof(ChainMum) * total, cudaMemcpyDeviceToHost));
    for (int p = 0; p < np; ++p) chains[p].assign(dense.begin() + off[p], dense.begin() + off[p] + cnt[p]);
    return BARB200_OK;
}

int run_chunk(barb200_ctx *ctx, int dev, const MumParams &P, int64_t n, const char *const *sx, const int64_t *lx, const char *const *sy,
              const int64_t *ly, const Alphabet *alpha, int64_t **out, int64_t *n_out, float *kernel_ms, int *launches) {
    Chunk C; C.ctx = ctx; C.dev = dev; C.k = (int)P.k; C.u = P.u;
    // active pairs: lX * lY > anchorMatrixBiggerThanThis (the early return of :1224-1226)
    std::vector<int64_t> act;
    for (int64_t i = 0; i < n; ++i) if (lx[i] * ly[i] > P.bigger) act.push_back(i);
    for (int64_t i = 0; i < n; ++i) { out[i] = nullptr; n_out[i] = 0; }
    std::vector<PairDev> pd(act.size());
    std::vector<int64_t> kmer_off(act.size() + 1, 0);
    int64_t codes = 0, words = 0, nx_sum = 0, ny_sum = 0;
    for (size_t a = 0; a < act.size(); ++a) {
        const int64_t i = act[a];
        const Alphabet &A = alpha[i];
        PairDev &d = pd[a];
        d.codes_off = codes; d.key_off = words; d.lx = (int32_t)lx[i]; d.ly = (int32_t)ly[i];
        d.nx = (int32_t)kmers(lx[i], P.k); d.bits = A.bits; d.per_word = A.per_word; d.words = A.words;
        const int64_t ny = kmers(ly[i], P.k);
        codes += lx[i] + ly[i]; words += (d.nx + ny) * A.words; nx_sum += d.nx; ny_sum += ny;
        kmer_off[a + 1] = kmer_off[a] + d.nx + ny;
        C.max_words = std::max(C.max_words, A.words);
    }
    if (act.empty()) { for (int64_t i = 0; i < n; ++i) out[i] = (int64_t *)malloc(16); return BARB200_OK; }
    C.n_pairs = (int)act.size(); C.cap_nx = nx_sum; C.cap_ny = ny_sum;
    const size_t b_pairs = align256(sizeof(PairDev) * act.size()), b_koff = align256(8 * kmer_off.size()), b_codes = align256((size_t)codes),
                 b_keys = align256(8 * (size_t)words), b_ny = align256(4 * (size_t)std::max<int64_t>(ny_sum, 1)),
                 b_nx = align256(4 * (size_t)std::max<int64_t>(nx_sum, 1)), b_mums = align256(sizeof(MumRec) * (size_t)std::max<int64_t>(nx_sum, 1)),
                 b_chain = align256(sizeof(ChainMum) * (size_t)std::max<int64_t>(nx_sum, 1));
    C.blk_bytes = b_pairs + b_koff + b_codes + b_keys + 2 * b_ny + 3 * b_nx + b_mums + 2 * b_chain;
    cudaSetDevice(ctx_device(ctx, dev));
    if (device_alloc(ctx, dev, &C.blk, C.blk_bytes) != 0) { C.blk = nullptr; set_error(ctx, "device allocation failed (MUM anchors); submit fewer or shorter pairs"); return BARB200_ENOMEM; }
    char *p = (char *)C.blk;
    C.d_pairs = (PairDev *)p; p += b_pairs;
    C.d_kmer_off = (int64_t *)p; p += b_koff;
    C.d_codes = (uint8_t *)p; p += b_codes;
    C.d_keys = (uint64_t *)p; p += b_keys;
    C.d_sa = (int32_t *)p; p += b_ny; C.d_sb = (int32_t *)p; p += b_ny;
    C.d_my = (int32_t *)p; p += b_nx; C.d_ml = (int32_t *)p; p += b_nx; C.d_sweep = (int32_t *)p; p += b_nx;
    C.d_mums = (MumRec *)p; p += b_mums;
    C.d_chain = (ChainMum *)p; p += b_chain; C.d_dense = (ChainMum *)p;
    CUDA_TRY(ctx, cudaStreamCreateWithFlags(&C.s, cudaStreamNonBlocking));
    CUDA_TRY(ctx, cudaEventCreate(&C.e0));
    CUDA_TRY(ctx, cudaEventCreate(&C.e1));
    // codes: each byte's rank in its pair's alphabet
    std::vector<uint8_t> hc((size_t)codes);
    const int nthr = host_threads(ctx);
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthr)
    for (int64_t a = 0; a < (int64_t)act.size(); ++a) {
        const int64_t i = act[a];
        const uint8_t *tab = alpha[i].code;
        uint8_t *d = hc.data() + pd[a].codes_off;
        for (int64_t q = 0; q < lx[i]; ++q) d[q] = tab[(unsigned char)sx[i][q]];
        for (int64_t q = 0; q < ly[i]; ++q) d[lx[i] + q] = tab[(unsigned char)sy[i][q]];
    }
    CUDA_TRY(ctx, cudaEventRecord(C.e0, C.s));
    CUDA_TRY(ctx, cudaMemcpyAsync(C.d_pairs, pd.data(), sizeof(PairDev) * pd.size(), cudaMemcpyHostToDevice, C.s));
    CUDA_TRY(ctx, cudaMemcpyAsync(C.d_kmer_off, kmer_off.data(), 8 * kmer_off.size(), cudaMemcpyHostToDevice, C.s));
    CUDA_TRY(ctx, cudaMemcpyAsync(C.d_codes, hc.data(), (size_t)codes, cudaMemcpyHostToDevice, C.s));
    if (kmer_off.back() > 0) {
        mum_keys_kernel<<<ctx_sm_count(ctx, dev) * 8, 256, 0, C.s>>>(C.d_pairs, C.n_pairs, C.d_kmer_off, C.d_codes, C.d_keys, C.k);
        ++C.launches;
    }
    // pass 1: the pairs
    std::vector<Problem> probs(act.size());
    int64_t ox = 0, oy = 0;
    for (size_t a = 0; a < act.size(); ++a) {
        probs[a] = Problem{(int32_t)a, 0, pd[a].lx, 0, pd[a].ly, 0, oy, ox};
        ox += kmers(pd[a].lx, P.k); oy += kmers(pd[a].ly, P.k);
    }
    std::vector<std::vector<ChainMum>> top, sub;
    int rc = run_pass(C, probs, top);
    if (rc) return rc;
    // pass 2: the gaps, one non-recursive level (tracebackMums :2039-2060)
    std::vector<std::vector<int32_t>> gaps(act.size());
    std::vector<int64_t> first_sub(act.size() + 1, 0);
    if (P.recursive) {
        std::vector<Problem> gp;
        ox = oy = 0;
        for (size_t a = 0; a < act.size(); ++a) {
            gap_table(top[a].data(), (int64_t)top[a].size(), pd[a].lx, pd[a].ly, P.bigger, gaps[a]);
            first_sub[a] = (int64_t)gp.size();
            for (size_t g = 0; g < gaps[a].size(); g += 4) {
                gp.push_back(Problem{(int32_t)a, gaps[a][g], gaps[a][g + 2], gaps[a][g + 1], gaps[a][g + 3], 0, oy, ox});
                ox += kmers(gaps[a][g + 2] - gaps[a][g], P.k); oy += kmers(gaps[a][g + 3] - gaps[a][g + 1], P.k);
            }
        }
        first_sub[act.size()] = (int64_t)gp.size();
        rc = run_pass(C, gp, sub);
        if (rc) return rc;
    }
    CUDA_TRY(ctx, cudaEventRecord(C.e1, C.s));
    CUDA_TRY(ctx, cudaEventSynchronize(C.e1));
    float ms = 0;
    CUDA_TRY(ctx, cudaEventElapsedTime(&ms, C.e0, C.e1));
    *kernel_ms += ms; *launches += C.launches;
    // splice
    bool oom = false;
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthr)
    for (int64_t a = 0; a < (int64_t)act.size(); ++a) {
        const int64_t i = act[a];
        std::vector<std::vector<ChainMum>> s(sub.begin() + first_sub[a], P.recursive ? sub.begin() + first_sub[a + 1] : sub.begin() + first_sub[a]);
        int64_t m = chain_bases(top[a]);
        for (const auto &c : s) m += chain_bases(c);
        int64_t *o = (int64_t *)malloc(16 * (size_t)std::max<int64_t>(m, 1));
        if (!o) { oom = true; continue; }
        n_out[i] = splice(top[a].data(), (int64_t)top[a].size(), gaps[a], s, P.recursive != 0, o);
        out[i] = o;
    }
    for (int64_t i = 0; i < n; ++i) if (!out[i]) { out[i] = (int64_t *)malloc(16); if (!out[i]) oom = true; }
    if (oom) { set_error(ctx, "host allocation failed (MUM anchors)"); return BARB200_ENOMEM; }
    pecan_count_mum_pairs(ctx, dev, (int64_t)act.size());
    return BARB200_OK;
}

// The pairs [0, n) on device `dev`: chunks (plan_chunks) under the device's free memory, one after the other. kernel_ms and
// launches accumulate; out / n_out are filled for every pair, also those below anchorMatrixBiggerThanThis.
int run_share(barb200_ctx *ctx, int dev, const MumParams &P, int64_t n, const char *const *sx, const int64_t *lx, const char *const *sy,
              const int64_t *ly, const Alphabet *alpha, const std::vector<int64_t> &bytes, int64_t **out, int64_t *n_out, float *kernel_ms, int *launches) {
    cudaSetDevice(ctx_device(ctx, dev));
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(ctx, cudaMemGetInfo(&free_b, &total_b));
    const int64_t budget = std::max<int64_t>((int64_t)(0.5 * ctx_mem_fraction(ctx) * (double)free_b), 1 << 20);
    for (const auto &c : plan_chunks(bytes, budget)) {
        const int rc = run_chunk(ctx, dev, P, c.second - c.first, sx + c.first, lx + c.first, sy + c.first, ly + c.first, alpha + c.first, out + c.first,
                                 n_out + c.first, kernel_ms, launches);
        if (rc) return rc;
    }
    return BARB200_OK;
}

// The pairs that need a device (bytes > 0) dealt over the context's devices by their bytes (deal_pairs), each device's share
// gathered and run by run_share on a host thread of its own, its anchors put back at the caller's indices; the other pairs get
// an empty list here. kernel_ms = the longest device's kernel time, launches = all devices' launches.
int run_devices(barb200_ctx *ctx, int ndev, const MumParams &P, int64_t n, const char *const *sx, const int64_t *lx, const char *const *sy,
                const int64_t *ly, const Alphabet *alpha, const std::vector<int64_t> &bytes, int64_t **out, int64_t *n_out, float *kernel_ms, int *launches) {
    std::vector<int64_t> act, act_bytes;
    for (int64_t i = 0; i < n; ++i) {
        if (bytes[i] > 0) { act.push_back(i); act_bytes.push_back(bytes[i]); continue; }
        out[i] = (int64_t *)malloc(16);
        if (!out[i]) { set_error(ctx, "host allocation failed (MUM anchors)"); return BARB200_ENOMEM; }
    }
    const std::vector<std::vector<int64_t>> share = barb200::pecan::deal_pairs(act_bytes, ndev);
    int active = 0;
    for (const auto &s : share) active += !s.empty();
    std::vector<int> rcs(ndev, BARB200_OK), dev_launches(ndev, 0);
    std::vector<float> dev_ms(ndev, 0.f);
    std::vector<std::string> errs(ndev);
    auto run_device = [&](int d) {
        set_host_thread_share(active);
        try {
            const std::vector<int64_t> &mine = share[d];
            const size_t m = mine.size();
            std::vector<const char *> dsx(m), dsy(m);
            std::vector<int64_t> dlx(m), dly(m), db(m), dn(m, 0);
            std::vector<Alphabet> da(m);
            std::vector<int64_t *> dout(m, nullptr);
            for (size_t k = 0; k < m; ++k) {
                const int64_t i = act[mine[k]];
                dsx[k] = sx[i]; dsy[k] = sy[i]; dlx[k] = lx[i]; dly[k] = ly[i]; db[k] = bytes[i]; da[k] = alpha[i];
            }
            rcs[d] = run_share(ctx, d, P, (int64_t)m, dsx.data(), dlx.data(), dsy.data(), dly.data(), da.data(), db, dout.data(), dn.data(), &dev_ms[d], &dev_launches[d]);
            if (rcs[d]) errs[d] = get_error(ctx);
            for (size_t k = 0; k < m; ++k) { out[act[mine[k]]] = dout[k]; n_out[act[mine[k]]] = dn[k]; }
        } catch (const std::bad_alloc &) { rcs[d] = BARB200_ENOMEM; errs[d] = "host allocation failed (MUM anchors)"; }
        set_host_thread_share(1);
    };
    std::vector<std::thread> th;
    for (int d = 0; d < ndev; ++d) if (!share[d].empty()) th.emplace_back(run_device, d);
    for (auto &t : th) t.join();
    for (int d = 0; d < ndev; ++d) {
        *kernel_ms = std::max(*kernel_ms, dev_ms[d]); *launches += dev_launches[d];
    }
    for (int d = 0; d < ndev; ++d) if (rcs[d]) { set_error(ctx, errs[d]); return rcs[d]; }
    return BARB200_OK;
}

}  // namespace

extern "C" void barb200_mum_params_default(barb200_mum_params *p) {
    p->k = 50; p->u = 1; p->anchor_matrix_bigger_than_this = (int64_t)500 * 500; p->recursive_mums = 1;
}

extern "C" int barb200_pecan_anchor_pairs_batch(barb200_ctx *ctx, const barb200_mum_params *p, int64_t n_pairs,
                                                const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                                                int64_t **anchors_out, int64_t *n_anchor_out) {
    if (!ctx) return BARB200_EINVAL;
    const double t0 = omp_get_wtime();
    tl_timing[0] = tl_timing[1] = tl_timing[2] = 0;
    if (!p || n_pairs < 0 || (n_pairs > 0 && (!sx || !sy || !lx || !ly || !anchors_out || !n_anchor_out))) { set_error(ctx, "bad argument"); return BARB200_EINVAL; }
    const MumParams P{p->k, p->u, p->anchor_matrix_bigger_than_this, p->recursive_mums};
    std::string err = check_params(P);
    if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
    std::vector<Alphabet> alpha(n_pairs);
    std::vector<int64_t> bytes(n_pairs);
    const int nthr = host_threads(ctx);
#pragma omp parallel for schedule(dynamic, 16) num_threads(nthr)
    for (int64_t i = 0; i < n_pairs; ++i) {
        std::string e;
        if (lx[i] < 0 || ly[i] < 0 || lx[i] > 0x3fffffff || ly[i] > 0x3fffffff || (lx[i] && !sx[i]) || (ly[i] && !sy[i])) e = "MUM anchors: bad sequence length or pointer";
        if (e.empty()) e = check_bytes(sx[i], lx[i], "sX");
        if (e.empty()) e = check_bytes(sy[i], ly[i], "sY");
        if (!e.empty()) {
#pragma omp critical
            if (err.empty()) err = "pair " + std::to_string((long long)i) + ": " + e;
            continue;
        }
        make_alphabet(sx[i], lx[i], sy[i], ly[i], P.k, alpha[i]);
        bytes[i] = lx[i] * ly[i] > P.bigger ? pair_bytes(lx[i], ly[i], P.k, alpha[i].words) : 0;
    }
    if (!err.empty()) { set_error(ctx, err); return BARB200_EINVAL; }
    for (int64_t i = 0; i < n_pairs; ++i) { anchors_out[i] = nullptr; n_anchor_out[i] = 0; }
    float kms = 0; int launches = 0;
    const int ndev = ctx_device_count(ctx);
    const int rc = ndev == 1 ? run_share(ctx, 0, P, n_pairs, sx, lx, sy, ly, alpha.data(), bytes, anchors_out, n_anchor_out, &kms, &launches)
                             : run_devices(ctx, ndev, P, n_pairs, sx, lx, sy, ly, alpha.data(), bytes, anchors_out, n_anchor_out, &kms, &launches);
    if (rc) {
        for (int64_t i = 0; i < n_pairs; ++i) { free(anchors_out[i]); anchors_out[i] = nullptr; n_anchor_out[i] = 0; }
        return rc;
    }
    tl_timing[0] = kms; tl_timing[1] = (omp_get_wtime() - t0) * 1e3; tl_timing[2] = launches;
    return BARB200_OK;
}

extern "C" int barb200_mum_last_timing(double out[3]) {
    if (!out) return BARB200_EINVAL;
    for (int i = 0; i < 3; ++i) out[i] = tl_timing[i];
    return BARB200_OK;
}
