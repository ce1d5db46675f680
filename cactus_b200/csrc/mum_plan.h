// mum_plan.h -- host-side planning of a MUM-anchor batch (K5, mum_anchor.cu), CUDA-free so that the no-GPU suite checks it:
// parameter and byte checks, each pair's order-preserving symbol codes and key width, the device memory a pair takes and the
// chunking of a batch under a memory budget, the table of gap sub-problems the recursion runs, and the splice of the chains
// into the reference's output order.
//
// Restates getAnchorPairsForPairwiseAlignmentParameters with useMumAnchors = 1 (submodules/cPecan/impl/pairwiseAligner.c:
// 1222-1231) and the recursion of tracebackMums (:2034-2061): a pair whose lX * lY <= anchorMatrixBiggerThanThis has no
// anchors; otherwise the MUM chain of the pair, and (recursiveMums) one non-recursive level of getAlignedMums2 into every gap
// of the chain -- before the first MUM, between two MUMs, after the last -- whose area exceeds the threshold.
#pragma once
#include <stdint.h>
#include <string.h>
#include <string>
#include <utility>
#include <vector>

namespace barb200 {
namespace mum {

static const int kMaxK = 64;       // k-mer lengths the key packing supports (kMaxWords words of >= 9 symbols)
static const int kMaxWords = 8;

struct MumParams {
    int64_t k, u, bigger;          // anchorMatrixBiggerThanThis, squared as bar.c:25-26
    int recursive;
};

inline std::string check_params(const MumParams &P) {
    if (P.k < 1 || P.k > kMaxK) return "MUM anchors: k = " + std::to_string((long long)P.k) + " is outside 1.." + std::to_string(kMaxK);
    if (P.u < 0) return "MUM anchors: u must be >= 0";
    if (P.bigger < 0) return "MUM anchors: anchorMatrixBiggerThanThis must be >= 0";
    return "";
}

// The bytes the pair-HMM batch takes: NUL-free 7-bit ASCII (the reference compares tolower() bytes, which is locale-free only
// there). Returns "" or a message naming the first bad byte.
inline std::string check_bytes(const char *s, int64_t n, const char *which) {
    for (int64_t i = 0; i < n; ++i) {
        const unsigned char c = (unsigned char)s[i];
        if (c == 0 || c >= 128) return std::string("MUM anchors: byte ") + std::to_string((int)c) + " at position " + std::to_string((long long)i) +
                                       " of " + which + " is not a NUL-free ASCII symbol";
    }
    return "";
}

inline unsigned char lower(unsigned char c) { return (c >= 'A' && c <= 'Z') ? (unsigned char)(c + 32) : c; }

// A pair's symbol codes: cmpKmers compares tolower() bytes, so each lower-cased byte present in X or Y gets its rank among
// them. Codes preserve the byte order, hence k-mer keys built from them compare as the reference's k-mers do.
struct Alphabet {
    uint8_t code[128];
    int bits = 1;                  // bits per symbol
    int per_word = 64;             // symbols per 64-bit key word
    int words = 1;                 // key words per k-mer
};

inline void make_alphabet(const char *sx, int64_t lx, const char *sy, int64_t ly, int64_t k, Alphabet &a) {
    bool seen[128] = {false};
    for (int64_t i = 0; i < lx; ++i) seen[lower((unsigned char)sx[i]) & 127] = true;
    for (int64_t i = 0; i < ly; ++i) seen[lower((unsigned char)sy[i]) & 127] = true;
    int d = 0;
    for (int c = 0; c < 128; ++c) { a.code[c] = (uint8_t)d; if (seen[c]) ++d; }
    for (int c = 'A'; c <= 'Z'; ++c) a.code[c] = a.code[c + 32];
    a.bits = 1;
    while ((1 << a.bits) < d) ++a.bits;
    a.per_word = 64 / a.bits;
    a.words = (int)((k + a.per_word - 1) / a.per_word);
}

inline int64_t kmers(int64_t len, int64_t k) { return len - k + 1 > 0 ? len - k + 1 : 0; }

// Device bytes of one pair in a chunk (mum_anchor.cu's buffers): symbol codes, the keys of every X and Y k-mer, the two sort
// buffers of Y, the match per X position, the MUM records and the sweep line per X position, the chain and its dense copy.
inline int64_t pair_bytes(int64_t lx, int64_t ly, int64_t k, int words) {
    const int64_t nx = kmers(lx, k), ny = kmers(ly, k);
    return lx + ly + 16 + (nx + ny) * words * 8 + ny * 8 + nx * (8 + 24 + 4 + 12 + 12) + 256;
}

// Consecutive chunks [first, second) whose bytes stay within budget; a pair larger than the budget is a chunk of its own (the
// caller rejects it if it does not fit the device).
inline std::vector<std::pair<int64_t, int64_t>> plan_chunks(const std::vector<int64_t> &bytes, int64_t budget) {
    std::vector<std::pair<int64_t, int64_t>> out;
    const int64_t n = (int64_t)bytes.size();
    int64_t i0 = 0;
    while (i0 < n) {
        int64_t i1 = i0, b = 0;
        while (i1 < n && (i1 == i0 || b + bytes[i1] <= budget)) b += bytes[i1++];
        out.push_back(std::make_pair(i0, i1));
        i0 = i1;
    }
    return out;
}

// One MUM search: X[x0, x1) against Y[y0, y1) of pair `pair` (coordinates in the pair). Offsets into the chunk's buffers.
struct Problem {
    int32_t pair, x0, x1, y0, y1;
    int32_t pad;
    int64_t ny_off;                // sort buffers: kmers(y1 - y0) entries
    int64_t nx_off;                // match / MUM / sweep buffers: kmers(x1 - x0) entries
};

// A MUM of a chain: (x, y) start in the pair, length.
struct ChainMum { int32_t x, y, len; };

// The gaps of a pair's chain (first to last) that the recursion searches: (x0, y0, x1, y1) in the pair. An empty chain has no
// gaps: its only gap would be the whole pair, whose non-recursive search repeats the one that found nothing.
inline void gap_table(const ChainMum *c, int64_t n, int32_t lx, int32_t ly, int64_t bigger, std::vector<int32_t> &gaps) {
    gaps.clear();
    if (n == 0) return;
    int64_t px = 0, py = 0;
    for (int64_t i = 0; i <= n; ++i) {
        const int64_t ex = i < n ? c[i].x : lx, ey = i < n ? c[i].y : ly;
        if ((ex - px) * (ey - py) > bigger) { gaps.push_back((int32_t)px); gaps.push_back((int32_t)py); gaps.push_back((int32_t)ex); gaps.push_back((int32_t)ey); }
        if (i < n) { px = (int64_t)c[i].x + c[i].len; py = (int64_t)c[i].y + c[i].len; }
    }
}

// The anchors of one pair in the reference's order. chain = the pair's MUMs first to last; sub[g] = the chain of gap g of
// gap_table (recursive only). Recursive: tracebackMums appends each gap's pairs (last to first) before the MUM that precedes
// it and reverses the whole list at the top level, so the result is every MUM base and every gap's MUM bases in increasing
// x (and y). Non-recursive: the list is not reversed -- last MUM first, each MUM's bases backwards.
inline int64_t splice(const ChainMum *chain, int64_t n, const std::vector<int32_t> &gaps, const std::vector<std::vector<ChainMum>> &sub,
                      bool recursive, int64_t *out) {
    int64_t m = 0;
    auto emit = [&](const ChainMum &c) { for (int32_t i = 0; i < c.len; ++i) { out[2 * m] = (int64_t)c.x + i; out[2 * m + 1] = (int64_t)c.y + i; ++m; } };
    if (!recursive) {
        for (int64_t i = n - 1; i >= 0; --i)
            for (int32_t j = chain[i].len - 1; j >= 0; --j) { out[2 * m] = (int64_t)chain[i].x + j; out[2 * m + 1] = (int64_t)chain[i].y + j; ++m; }
        return m;
    }
    size_t g = 0;
    for (int64_t i = 0; i <= n; ++i) {
        const int64_t ex = i < n ? chain[i].x : INT64_MAX;
        if (g < sub.size() && gaps[4 * g + 2] <= ex) { for (const ChainMum &c : sub[g]) emit(c); ++g; }
        if (i < n) emit(chain[i]);
    }
    return m;
}

inline int64_t chain_bases(const std::vector<ChainMum> &c) { int64_t s = 0; for (const ChainMum &m : c) s += m.len; return s; }

}  // namespace mum
}  // namespace barb200
