// mum_anchor.cuh -- K5, the MUM anchor chains of cPecan (getAlignedMums2, submodules/cPecan/impl/pairwiseAligner.c:1849-2121),
// written __host__ __device__ so that the kernels of mum_anchor.cu and the host build in tests/hosttest run the same source.
//
// A k-mer is a key of `words` 64-bit words: the pair's symbol codes (mum_plan.h: make_alphabet, the rank of the tolower() byte),
// `bits` bits each, first symbol in the top bits. Comparing keys word by word is cmpKmers (:1848-1861); the number of equal
// leading symbols (its matchLength) is the first differing word's index times per_word plus clz(xor) / bits.
//
// Equal k-mers in any order. The reference sorts Y's k-mers with an unstable sort, and so do the kernels; the result does not
// depend on the order inside a run of equal k-mers: the binary search of getLongestUniqueMatch (:1910-1937) compares the query
// with the CONTENT at each probed index, and the sorted sequence of contents is unique, so the probed indices, p and the match
// lengths are the same for every order. A result j >= 0 needs matchLength(j) > u + matchLength(j +- 1) with u >= 0, which an
// equal neighbour (same match length) fails, so j is alone in its run and y = sorted[j] is unique too.
#pragma once
#include <stdint.h>
#include "mum_plan.h"

#if defined(__CUDACC__)
#define MUM_HD __host__ __device__ __forceinline__
#else
#define MUM_HD inline
#endif

namespace barb200 {
namespace mum {

MUM_HD int clz64(uint64_t v) {
#if defined(__CUDA_ARCH__)
    return __clzll((long long)v);
#else
    return v ? __builtin_clzll(v) : 64;
#endif
}

MUM_HD int32_t n_kmers(int32_t len, int k) { return len - k + 1 > 0 ? len - k + 1 : 0; }

// key of the k-mer starting at codes[0]
MUM_HD void make_key(const uint8_t *codes, int k, int bits, int per_word, int words, uint64_t *key) {
    for (int w = 0; w < words; ++w) {
        uint64_t v = 0;
        const int i0 = w * per_word, i1 = i0 + per_word < k ? i0 + per_word : k;
        for (int i = i0; i < i1; ++i) v |= (uint64_t)codes[i] << (64 - bits * (i - i0 + 1));
        key[w] = v;
    }
}

// cmpKmers: -1 / 0 / 1 and the match length (equal leading symbols, k when equal)
MUM_HD int cmp_keys(const uint64_t *a, const uint64_t *b, int words, int bits, int per_word, int k, int *match) {
    for (int w = 0; w < words; ++w) {
        const uint64_t x = a[w] ^ b[w];
        if (x) {
            const int n = w * per_word + clz64(x) / bits;
            *match = n < k ? n : k;
            return a[w] < b[w] ? -1 : 1;
        }
    }
    *match = k;
    return 0;
}

// the key compare the sorts use (no match length)
MUM_HD bool key_less(const uint64_t *a, const uint64_t *b, int words) {
    for (int w = 0; w < words; ++w) if (a[w] != b[w]) return a[w] < b[w];
    return false;
}

struct KeyView {                   // the keys of one pair: X k-mers at x * words, Y k-mers at (y_base + y) * words
    const uint64_t *keys;
    int64_t y_base;
    int k, bits, per_word, words;
    MUM_HD const uint64_t *x(int32_t p) const { return keys + (int64_t)p * words; }
    MUM_HD const uint64_t *y(int32_t p) const { return keys + (y_base + p) * words; }
};

// getLongestUniqueMatch (:1910-1937) for the X k-mer at x against sorted Y k-mer starts sorted[0, n): returns the index j or -1,
// *len = matchLength
MUM_HD int32_t longest_unique_match(const KeyView &K, const int32_t *sorted, int32_t n, int32_t x, int64_t u, int *len) {
    const uint64_t *q = K.x(x);
    int32_t l = 0, h = n, p = -2;
    int best = 0;
    while (l < h) {
        const int32_t m = (l + h) / 2;
        int mn;
        const int c = cmp_keys(q, K.y(sorted[m]), K.words, K.bits, K.per_word, K.k, &mn);
        if (mn > best) { best = mn; p = m; }
        if (c < 0) h = m;
        else if (c > 0) l = m + 1;
        else break;
    }
    *len = best;
    int lo = 0, hi = 0;                                  // getMatchLength (:1900-1906): 0 outside [0, n)
    if (p - 1 >= 0 && p - 1 < n) cmp_keys(q, K.y(sorted[p - 1]), K.words, K.bits, K.per_word, K.k, &lo);
    if (p + 1 >= 0 && p + 1 < n) cmp_keys(q, K.y(sorted[p + 1]), K.words, K.bits, K.per_word, K.k, &hi);
    return ((int64_t)best > u + lo && (int64_t)best > u + hi) ? p : -1;
}

struct MumRec { int32_t x, y, len, score, pred, next; };

// The chain of one problem: getAlignedMums2's sweep over x (:2063-2109) with updateSweepLine / chainMum (:1972-2032) and the
// traceback's walk (:2039-2056). match_y[i] / match_len[i]: the longest unique match of x = x0 + i (-1: none). mums / sweep:
// scratch of n_x entries. Writes the chain first to last into chain_out (room for n_x) and returns its length.
//
// The sweep line is an array ordered by end y (y + len). Its scores strictly increase along it: an inserted MUM is dropped if
// the entry at or before its end has a score >= its own, and entries at or after its end with a score <= its own are removed
// first -- a contiguous run, replaced by the new entry. So every search is a binary search. MUMs wait for their end x in
// buckets end % (k + 1) (a MUM ends 1..k after its start), each bucket in creation order, which is the order updateSweepLine
// takes them in. A MUM ending at x = lX is never added: the reference's last updateSweepLine is at lX - 1 (its closing
// assert(stList_length(mumsToAdd) == 0) aborts there when asserts are on; the kernels keep the NDEBUG behaviour).
MUM_HD int32_t chain_problem(int32_t x0, int32_t x1, int32_t y0, int k, const int32_t *match_y, const int32_t *match_len,
                             MumRec *mums, int32_t *sweep, ChainMum *chain_out) {
    (void)y0;
    int32_t head[kMaxK + 1], tail[kMaxK + 1];
    for (int b = 0; b <= k; ++b) head[b] = tail[b] = -1;
    int32_t n_mum = 0, n_sw = 0;
    int64_t p_diag = -1;
    int32_t p_x_end = x0 - 1;
    const int32_t lx = x1 - x0;
    for (int32_t xi = 0; xi < lx; ++xi) {
        const int32_t x = x0 + xi;
        // updateSweepLine(x)
        const int b = (int)(x % (k + 1));
        for (int32_t i = head[b]; i >= 0; i = mums[i].next) {
            MumRec &m = mums[i];
            const int32_t e = m.y + m.len;
            int32_t lo = 0, hi = n_sw;                   // first entry with end > e
            while (lo < hi) { const int32_t md = (lo + hi) / 2; if (mums[sweep[md]].y + mums[sweep[md]].len <= e) lo = md + 1; else hi = md; }
            if (lo > 0 && mums[sweep[lo - 1]].score >= m.score) continue;
            int32_t r0 = lo;                             // first entry with end >= e
            if (r0 > 0 && mums[sweep[r0 - 1]].y + mums[sweep[r0 - 1]].len == e) --r0;
            int32_t r1 = r0;
            while (r1 < n_sw && mums[sweep[r1]].score <= m.score) ++r1;
            const int32_t shift = 1 - (r1 - r0);
            if (shift > 0) for (int32_t t = n_sw - 1; t >= r1; --t) sweep[t + shift] = sweep[t];
            else if (shift < 0) for (int32_t t = r1; t < n_sw; ++t) sweep[t + shift] = sweep[t];
            n_sw += shift;
            sweep[r0] = i;
        }
        head[b] = tail[b] = -1;
        if (xi > lx - k) continue;
        const int32_t y = match_y[xi];
        if (y < 0) continue;
        if (p_x_end < x || p_diag != (int64_t)x - y) {
            MumRec &m = mums[n_mum];
            m.x = x; m.y = y; m.len = match_len[xi]; m.next = -1;
            // chainMum: the last entry with end y < y
            int32_t lo = 0, hi = n_sw;
            while (lo < hi) { const int32_t md = (lo + hi) / 2; if (mums[sweep[md]].y + mums[sweep[md]].len < y) lo = md + 1; else hi = md; }
            m.pred = lo > 0 ? sweep[lo - 1] : -1;
            m.score = m.pred >= 0 ? mums[m.pred].score + m.len : m.len;
            const int32_t end = x + m.len;
            if (end < x1) {                              // queued for updateSweepLine(end)
                const int eb = (int)(end % (k + 1));
                if (tail[eb] >= 0) mums[tail[eb]].next = n_mum; else head[eb] = n_mum;
                tail[eb] = n_mum;
            }
            ++n_mum;
            p_diag = (int64_t)x - y;
            p_x_end = end;
        }
    }
    int32_t n = 0;
    for (int32_t i = n_sw > 0 ? sweep[n_sw - 1] : -1; i >= 0; i = mums[i].pred) ++n;
    int32_t w = n;
    for (int32_t i = n_sw > 0 ? sweep[n_sw - 1] : -1; i >= 0; i = mums[i].pred) { --w; chain_out[w].x = mums[i].x; chain_out[w].y = mums[i].y; chain_out[w].len = mums[i].len; }
    return n;
}

}  // namespace mum
}  // namespace barb200
