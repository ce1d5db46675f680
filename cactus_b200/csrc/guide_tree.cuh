// guide_tree.cuh -- the progressive-POA read order (which sequence is aligned when) computed by the CTA that owns the job.
//
// With seeding disabled Cactus still lets abPOA pick the alignment order from a guide tree
// (abpoa_build_guide_tree_partition, abPOA src/abpoa_seed.c:705-722): (w,k)-minimizers of every sequence (mm_sketch,
// :85-156; forward strand only, no homopolymer compression), pairwise min-count Jaccard similarity of the minimizer
// multisets and a greedy order (abpoa_build_guide_tree, :232-325). Round 1 computed this on host threads and streamed the
// orders in behind the running kernel; here it is the first phase of the job on the device (SURVEY.md 8(f)-3), so the host does
// no per-job work at all and K in the hundreds costs no host time:
//   1. sketch: the reference's serial window scan (ties and duplicates exactly as mm_sketch reports them -- the multiset
//      matters), cut into 64-position chunks that all threads work on (see gt_scan_chunk for why that is exact); keys
//      (hash << 8 | span) << 16 | read are appended to one array;
//   2. the keys are sorted by the CTA (bitonic network in global memory; only the grouping by hash matters);
//   3. every group of equal hashes adds min(count_a, count_b) to the pair counters (integer atomics: order free);
//   4. Jaccard = shared / total in double (one IEEE division of two integers, the same value as the reference's), first
//      maximum in the reference's loop order; then the greedy order: a read's score is the sum of its similarities to the
//      reads placed so far, accumulated in placement order exactly like the reference's inner loop, first maximum wins.
// The same source compiles for the host (tests/hosttest), where the T threads of every phase run one after the other.
#pragma once
#include <math.h>
#include <stdint.h>
#include "poa_types.h"

namespace barb200 {

struct GuideTreeParams { int k, w; };        // partialOrderAlignmentMinimizerK / W

// per-slot scratch of the guide tree (carved from the slot by the kernel)
struct GtScratch {
    uint64_t *keys; int key_cap;             // minimizer keys, capacity a power of two
    uint64_t *gx;                            // [bases of the job] per-position k-mer values (phase A of the sketch)
    int *hit;                                // [K (K + 1) / 2] pair counters, tri(i, j) = i (i + 1) / 2 + j, i >= j
    double *jac;                             // [K (K - 1) / 2] similarities, jidx(i, j) = i (i - 1) / 2 + j, i > j
    double *score;                           // [K] running greedy scores (-1 once placed)
    int *n_keys;                             // 1 int: keys appended (shared or global)
    int *red_i; double *red_v;               // [T / 32 + 1] block reductions
    uint64_t *tile; int tile_cap;            // shared-memory tile of the sort (a power of two, >= 64 keys)
};

HD uint64_t gt_hash64(uint64_t key, uint64_t mask) {   // minimap2's hash64, abpoa_seed.c:36-46
    key = (~key + (key << 21)) & mask;
    key = key ^ key >> 24;
    key = ((key + (key << 3)) + (key << 8)) & mask;
    key = key ^ key >> 14;
    key = ((key + (key << 2)) + (key << 4)) & mask;
    key = key ^ key >> 28;
    key = (key + (key << 31)) & mask;
    return key;
}

HD void gt_push(const GtScratch &G, uint64_t x, uint32_t rid) {
#if defined(__CUDA_ARCH__)
    const int pos = atomicAdd(G.n_keys, 1);
#else
    const int pos = (*G.n_keys)++;
#endif
    if (pos < G.key_cap) G.keys[pos] = x << 16 | (uint64_t)rid;
}

// ---- minimizer sketch (mm_sketch, abpoa_seed.c:85-156; forward strand only, no homopolymer compression) ------------------------
// The reference scans a sequence serially with a ring of the last w k-mers and a running minimum. Two facts make the scan
// parallel WITHOUT changing a single emission (ties, duplicates and the first-window quirk included):
//   * the ring always equals the last w entries of the per-position array X[i] = (hash << 8 | span) of the k-mer ending at i
//     (NONE where fewer than k unambiguous bases end at i), and "bases since the last ambiguous one" (run) is a function of the
//     position alone -- so X can be computed for all positions independently (phase A);
//   * the scan's state before step i -- the running minimum `best` and its slot -- is always the RIGHTMOST minimum of
//     X[i-w .. i-1] (NONE included as the largest value; checked case by case against the update rule below) -- so any chunk of
//     positions can start from that state and replay the reference's step rule, emitting exactly what the serial scan emits in
//     that chunk (phase B). The emission order differs, which is irrelevant: the keys are sorted next.
constexpr uint64_t GT_NONE = ~0ULL;

// phase A for positions [s, e) of one sequence: X[i] into gx[i]
HD void gt_hash_chunk(const uint8_t *q, int s, int e, int k, uint64_t *gx) {
    const uint64_t mask = (1ULL << 2 * k) - 1;
    int run = 0;                                   // unambiguous bases ending at s-1, capped at k (all that matters here)
    uint64_t kmer = 0;
    for (int i = s - 1; i >= 0 && run < k && q[i] < 4; --i) ++run;
    for (int i = s - run; i < s; ++i) kmer = (kmer << 2 | (uint64_t)q[i]) & mask;
    for (int i = s; i < e; ++i) {
        const int c = q[i];
        uint64_t x = GT_NONE;
        if (c < 4) {
            kmer = (kmer << 2 | (uint64_t)c) & mask;
            if (run < k) ++run;
            if (run >= k) x = gt_hash64(kmer, mask) << 8 | (uint64_t)k;        // span = k once k bases are there (abpoa_seed.c:117)
        } else { run = 0; kmer = 0; }
        gx[i] = x;
    }
}

// phase B for positions [s, e) of one sequence of length len (read id rid): the reference's step rule on X = gx
HD void gt_scan_chunk(const GtScratch &G, const uint8_t *q, const uint64_t *gx, int len, int s, int e, int w, int k, uint32_t rid) {
    auto X = [&](int i) { return i >= 0 ? gx[i] : GT_NONE; };
    // run before the chunk, capped at w + k (the rule only compares it with w + k - 1 and w + k)
    int run = 0;
    for (int i = s - 1; i >= 0 && run < w + k && q[i] < 4; --i) ++run;
    // state before step s: rightmost minimum of X[s-w .. s-1]
    uint64_t bx = GT_NONE; int bi = s - w;         // (bi only matters through bi % w == slot; any slot is fine while bx is NONE ... see below)
    for (int j = s - w; j < s; ++j) { const uint64_t v = X(j); if (bx >= v) { bx = v; bi = j; } }
    for (int i = s; i < e; ++i) {
        const uint64_t cx = gx[i];
        if (q[i] < 4) { if (run < w + k) ++run; } else run = 0;
        if (run == w + k - 1 && bx != GT_NONE) {                              // the first full window: ties of the minimum so far
            for (int j = i - w + 1; j < i; ++j) if (bx == X(j) && j != bi) gt_push(G, bx, rid);
        }
        if (cx <= bx) {
            if (run >= w + k && bx != GT_NONE) gt_push(G, bx, rid);
            bx = cx; bi = i;
        } else if (bi == i - w) {                                             // the minimum slides out of the window
            if (run >= w + k - 1 && bx != GT_NONE) gt_push(G, bx, rid);
            bx = GT_NONE;
            for (int j = i - w + 1; j <= i; ++j) { const uint64_t v = X(j); if (bx >= v) { bx = v; bi = j; } }
            if (run >= w + k - 1 && bx != GT_NONE) {
                for (int j = i - w + 1; j <= i; ++j) if (bx == X(j) && j != bi) gt_push(G, bx, rid);
            }
        }
    }
    if (e == len && bx != GT_NONE) gt_push(G, bx, rid);                        // the last minimum of the sequence
}

HD int64_t gt_tri(int64_t i, int64_t j) { return i * (i + 1) / 2 + j; }     // i >= j
HD int64_t gt_jidx(int64_t i, int64_t j) { return i * (i - 1) / 2 + j; }    // i > j

// first maximum of (value, index): larger value wins, equal values -> smaller index (the reference's `if (v > best)` scans)
HD bool gt_better(double v, int64_t i, double bv, int64_t bi) { return v > bv || (v == bv && i < bi); }

// Block-wide first-maximum of per-thread candidates. All threads; result in red_v[0] / red_i64 (returned to every thread).
// T must be a multiple of 32 on the device. ws_v / ws_i: >= 33 entries.
HD void gt_block_argmax(double &v, int64_t &i, double *ws_v, long long *ws_i, int T) {
#if defined(__CUDA_ARCH__)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = T >> 5;
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        const double ov = __shfl_down_sync(0xffffffffu, v, off); const long long oi = __shfl_down_sync(0xffffffffu, (long long)i, off);
        if (gt_better(ov, oi, v, i)) { v = ov; i = oi; }
    }
    __syncthreads();
    if (lane == 0) { ws_v[warp] = v; ws_i[warp] = i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double bv = ws_v[0]; long long bi = ws_i[0];
        for (int q = 1; q < nw; ++q) if (gt_better(ws_v[q], ws_i[q], bv, bi)) { bv = ws_v[q]; bi = ws_i[q]; }
        ws_v[32] = bv; ws_i[32] = bi;
    }
    __syncthreads();
    v = ws_v[32]; i = ws_i[32];
#else
    (void)ws_v; (void)ws_i; (void)T; (void)v; (void)i;      // the host emulation reduces in the caller (threads run one after the other)
#endif
}

// The read order of one job into order[0 .. n). seq(i) / len(i) give sequence i. Returns 0, or -1 if the key array was too small.
// All threads of the CTA (T of them); ws_v / ws_i: shared scratch of >= 33 doubles / long longs.
template <class SeqFn>
HD int cta_guide_tree(const GuideTreeParams &P, int progressive, int n, SeqFn seq, const int *lens, int *order, const GtScratch &G,
                      double *ws_v, long long *ws_i, int T) {
    GT_THREADS(tid, T) { for (int i = tid; i < n; i += T) order[i] = i; if (tid == 0) *G.n_keys = 0; }
    GT_SYNC();
    if (!(progressive && n > 2)) return 0;
    // ---- 1. sketches: every thread takes chunks of GT_CHUNK positions (offsets of the sequences in gx = prefix sums of lens) ----
    constexpr int GT_CHUNK = 64;
    int64_t total_chunks = 0;
    for (int i = 0; i < n; ++i) total_chunks += (lens[i] + GT_CHUNK - 1) / GT_CHUNK;
    for (int phase = 0; phase < 2; ++phase) {
        GT_THREADS(tid, T) {
            int64_t c0 = 0, off = 0;                  // chunks / bases of the sequences before sequence i
            int i = 0;
            for (int64_t c = tid; c < total_chunks; c += T) {
                while (c >= c0 + (lens[i] + GT_CHUNK - 1) / GT_CHUNK) { c0 += (lens[i] + GT_CHUNK - 1) / GT_CHUNK; off += lens[i]; ++i; }
                const int s0 = (int)(c - c0) * GT_CHUNK, e0 = s0 + GT_CHUNK < lens[i] ? s0 + GT_CHUNK : lens[i];
                if (phase == 0) gt_hash_chunk(seq(i), s0, e0, P.k, G.gx + off);
                else gt_scan_chunk(G, seq(i), G.gx + off, lens[i], s0, e0, P.w, P.k, (uint32_t)i);
            }
        }
        GT_SYNC();
    }
    const int nk = *G.n_keys;
    if (nk > G.key_cap) return -1;
    if (nk == 0) return 0;
    // ---- 2. sort (bitonic network, padded to a power of two with the maximal key). Exchanges whose partners lie within one
    // tile run in shared memory (load the tile once, all strides below the tile size, store it back); only the few passes with a
    // stride >= the tile size touch global memory, and there every thread loads a batch of pairs before it stores any ----
    int n2 = 1;
    while (n2 < nk) n2 <<= 1;
    GT_THREADS(tid, T) { for (int i = nk + tid; i < n2; i += T) G.keys[i] = ~0ULL; }
    GT_SYNC();
    int tile = 64;
    while (tile * 2 <= G.tile_cap && tile < n2) tile <<= 1;
    if (tile > n2) tile = n2;
    // stage 1: every merge size up to the tile size, tile by tile, entirely in shared memory
    for (int base = 0; base < n2; base += tile) {
        GT_THREADS(tid, T) { for (int i = tid; i < tile; i += T) G.tile[i] = G.keys[base + i]; }
        GT_SYNC();
        for (int size = 2; size <= tile; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                GT_THREADS(tid, T) {
                    for (int t = tid; t < (tile >> 1); t += T) {
                        const int lo = ((t / stride) * (stride << 1)) + (t % stride), hi = lo + stride;
                        const bool up = ((base + lo) & size) == 0;
                        const uint64_t a = G.tile[lo], b = G.tile[hi];
                        if ((a > b) == up) { G.tile[lo] = b; G.tile[hi] = a; }
                    }
                }
                GT_SYNC();
            }
        }
        GT_THREADS(tid, T) { for (int i = tid; i < tile; i += T) G.keys[base + i] = G.tile[i]; }
        GT_SYNC();
    }
    // stage 2: the larger merge sizes: strides >= tile in global memory, the rest of the step tile by tile in shared memory
    for (int size = tile << 1; size <= n2; size <<= 1) {
        for (int stride = size >> 1; stride >= tile; stride >>= 1) {
            GT_THREADS(tid, T) {
                for (int t0 = tid; t0 < (n2 >> 1); t0 += 4 * T) {
                    uint64_t a[4], b[4]; int lo[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
                    for (int u = 0; u < 4; ++u) {
                        const int t = t0 + u * T;
                        lo[u] = t < (n2 >> 1) ? ((t / stride) * (stride << 1)) + (t % stride) : -1;
                        if (lo[u] >= 0) { a[u] = G.keys[lo[u]]; b[u] = G.keys[lo[u] + stride]; }
                    }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
                    for (int u = 0; u < 4; ++u) if (lo[u] >= 0) {
                        const bool up = (lo[u] & size) == 0;
                        if ((a[u] > b[u]) == up) { G.keys[lo[u]] = b[u]; G.keys[lo[u] + stride] = a[u]; }
                    }
                }
            }
            GT_SYNC();
        }
        for (int base = 0; base < n2; base += tile) {
            GT_THREADS(tid, T) { for (int i = tid; i < tile; i += T) G.tile[i] = G.keys[base + i]; }
            GT_SYNC();
            for (int stride = tile >> 1; stride > 0; stride >>= 1) {
                GT_THREADS(tid, T) {
                    for (int t = tid; t < (tile >> 1); t += T) {
                        const int lo = ((t / stride) * (stride << 1)) + (t % stride), hi = lo + stride;
                        const bool up = ((base + lo) & size) == 0;
                        const uint64_t a = G.tile[lo], b = G.tile[hi];
                        if ((a > b) == up) { G.tile[lo] = b; G.tile[hi] = a; }
                    }
                }
                GT_SYNC();
            }
            GT_THREADS(tid, T) { for (int i = tid; i < tile; i += T) G.keys[base + i] = G.tile[i]; }
            GT_SYNC();
        }
    }
    // ---- 3. pair counters: every group of equal hashes (abpoa_seed.c:232-284) ----
    const int64_t n_tri = (int64_t)n * (n + 1) / 2;
    GT_THREADS(tid, T) { for (int64_t i = tid; i < n_tri; i += T) G.hit[i] = 0; }
    GT_SYNC();
    GT_THREADS(tid, T) {
        for (int s = tid; s < nk; s += T) {
            const uint64_t x = G.keys[s] >> 16;
            if (s > 0 && (G.keys[s - 1] >> 16) == x) continue;             // not the first entry of its group
            // the group is sorted by read: runs of equal reads are the per-read counts
            int e = s;
            while (e < nk && (G.keys[e] >> 16) == x) ++e;
            for (int a = s; a < e;) {
                const int ra = (int)(G.keys[a] & 0xffff);
                int ae = a; while (ae < e && (int)(G.keys[ae] & 0xffff) == ra) ++ae;
                const int ca = ae - a;
#if defined(__CUDA_ARCH__)
                atomicAdd(&G.hit[gt_tri(ra, ra)], ca);
#else
                G.hit[gt_tri(ra, ra)] += ca;
#endif
                for (int b = ae; b < e;) {
                    const int rb = (int)(G.keys[b] & 0xffff);
                    int be = b; while (be < e && (int)(G.keys[be] & 0xffff) == rb) ++be;
                    const int cb = be - b, m = ca < cb ? ca : cb;           // rb > ra (sorted)
#if defined(__CUDA_ARCH__)
                    atomicAdd(&G.hit[gt_tri(rb, ra)], m);
#else
                    G.hit[gt_tri(rb, ra)] += m;
#endif
                    b = be;
                }
                a = ae;
            }
        }
    }
    GT_SYNC();
    // ---- 4. similarities + the most similar pair (first maximum in the order i ascending, j ascending) ----
    const int64_t n_pairs = (int64_t)n * (n - 1) / 2;
    double bv = -1.0; int64_t bi = INT64_MAX;
    GT_THREADS(tid, T) {
        double tv = -1.0; int64_t ti = INT64_MAX;
        for (int64_t q = tid; q < n_pairs; q += T) {
            // q = jidx(i, j): i = the row with i (i - 1) / 2 <= q
            int64_t i = (int64_t)((1.0 + sqrt(1.0 + 8.0 * (double)q)) / 2.0);
            while (i * (i - 1) / 2 > q) --i;
            while ((i + 1) * i / 2 <= q) ++i;
            const int64_t j = q - i * (i - 1) / 2;
            const int shared = G.hit[gt_tri(i, j)], tot = G.hit[gt_tri(i, i)] + G.hit[gt_tri(j, j)] - shared;
            const double v = tot == 0 ? 0.0 : (0.0 + shared) / tot;
            G.jac[q] = v;
            if (gt_better(v, q, tv, ti)) { tv = v; ti = q; }
        }
#if defined(__CUDA_ARCH__)
        gt_block_argmax(tv, ti, ws_v, ws_i, T);
        bv = tv; bi = ti;
#else
        if (gt_better(tv, ti, bv, bi)) { bv = tv; bi = ti; }
#endif
    }
    GT_SYNC();
    int64_t pi = (int64_t)((1.0 + sqrt(1.0 + 8.0 * (double)bi)) / 2.0);
    while (pi * (pi - 1) / 2 > bi) --pi;
    while ((pi + 1) * pi / 2 <= bi) ++pi;
    const int64_t pj = bi - pi * (pi - 1) / 2;
    // ---- 5. greedy order (abpoa_seed.c:286-325): score(r) = sum over the placed reads, in placement order ----
    GT_THREADS(tid, T) {
        for (int r = tid; r < n; r += T) G.score[r] = (r == pi || r == pj) ? -1.0 : 0.0;
        if (tid == 0) { order[0] = (int)pj; order[1] = (int)pi; }
    }
    GT_SYNC();
    int last[2] = {(int)pj, (int)pi}, n_last = 2;
    for (int placed = 2; placed < n; ++placed) {
        double sv = -1.0; int64_t si = INT64_MAX;
        GT_THREADS(tid, T) {
            double tv = -2.0; int64_t ti = INT64_MAX;
            for (int r = tid; r < n; r += T) {
                double v = G.score[r];
                if (v >= 0.0) {
                    for (int q = 0; q < n_last; ++q) { const int o = last[q]; v += r > o ? G.jac[gt_jidx(r, o)] : G.jac[gt_jidx(o, r)]; }
                    G.score[r] = v;
                    if (gt_better(v, r, tv, ti)) { tv = v; ti = r; }
                }
            }
#if defined(__CUDA_ARCH__)
            gt_block_argmax(tv, ti, ws_v, ws_i, T);
            sv = tv; si = ti;
#else
            if (gt_better(tv, ti, sv, si)) { sv = tv; si = ti; }
#endif
        }
        GT_SYNC();
        GT_THREADS(tid, T) { if (tid == 0) { order[placed] = (int)si; G.score[si] = -1.0; } }
        GT_SYNC();
        last[0] = (int)si; n_last = 1;
    }
    return 0;
}

}  // namespace barb200
