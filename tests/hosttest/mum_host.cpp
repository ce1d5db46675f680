// mum_host.cpp -- TEST-ONLY host build of K5 (cactus_b200/csrc/mum_anchor.cuh + mum_plan.h): the product's key packing, match
// search, sweep-line chaining, gap table and splice run on the CPU, one problem at a time, in the order mum_anchor.cu runs them.
// The k-mer sort is std::sort on the same keys (the kernels' bitonic / merge sort is checked on the GPU); tie_seed != 0 shuffles
// every run of equal k-mers after it, which must not change the result (mum_anchor.cuh, "Equal k-mers in any order").
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <random>
#include <vector>
#include "../../cactus_b200/csrc/mum_anchor.cuh"

using namespace barb200::mum;

namespace {

// one problem of a pair: the chain of X[x0, x1) against Y[y0, y1)
std::vector<ChainMum> host_problem(const KeyView &K, int32_t x0, int32_t x1, int32_t y0, int32_t y1, int64_t u, std::mt19937_64 *tie) {
    const int32_t ny = n_kmers(y1 - y0, K.k), nx = n_kmers(x1 - x0, K.k);
    std::vector<int32_t> sorted(ny);
    for (int32_t i = 0; i < ny; ++i) sorted[i] = y0 + i;
    std::sort(sorted.begin(), sorted.end(), [&](int32_t a, int32_t b) { return key_less(K.y(a), K.y(b), K.words); });
    if (tie) {
        for (int32_t a = 0; a < ny;) {
            int32_t b = a + 1;
            while (b < ny && !key_less(K.y(sorted[a]), K.y(sorted[b]), K.words)) ++b;
            std::shuffle(sorted.begin() + a, sorted.begin() + b, *tie);
            a = b;
        }
    }
    std::vector<int32_t> my(std::max(nx, 1)), ml(std::max(nx, 1));
    for (int32_t i = 0; i < nx; ++i) {
        int len = 0;
        const int32_t j = longest_unique_match(K, sorted.data(), ny, x0 + i, u, &len);
        my[i] = j >= 0 ? sorted[j] : -1;
        ml[i] = len;
    }
    std::vector<MumRec> mums(std::max(nx, 1));
    std::vector<int32_t> sweep(std::max(nx, 1));
    std::vector<ChainMum> chain(std::max(nx, 1));
    chain.resize(chain_problem(x0, x1, y0, K.k, my.data(), ml.data(), mums.data(), sweep.data(), chain.data()));
    return chain;
}

}  // namespace

// anchors of one pair as barb200_pecan_anchor_pairs_batch computes them; returns n (x, y) pairs in *out (malloc'd) or -1 for
// parameters / bytes the product rejects
extern "C" int64_t hosttest_mum_anchor_pairs(const char *sx, int64_t lx, const char *sy, int64_t ly, int64_t k, int64_t u, int64_t bigger,
                                             int recursive, uint64_t tie_seed, int64_t **out) {
    *out = nullptr;
    const MumParams P{k, u, bigger, recursive};
    if (!check_params(P).empty() || !check_bytes(sx, lx, "sX").empty() || !check_bytes(sy, ly, "sY").empty()) return -1;
    if (lx * ly <= bigger) { *out = (int64_t *)malloc(16); return 0; }
    Alphabet A;
    make_alphabet(sx, lx, sy, ly, k, A);
    std::vector<uint8_t> codes(lx + ly);
    for (int64_t i = 0; i < lx; ++i) codes[i] = A.code[(unsigned char)sx[i]];
    for (int64_t i = 0; i < ly; ++i) codes[lx + i] = A.code[(unsigned char)sy[i]];
    const int32_t nx = n_kmers((int32_t)lx, (int)k), ny = n_kmers((int32_t)ly, (int)k);
    std::vector<uint64_t> keys((size_t)(nx + ny) * A.words + 1);
    for (int32_t i = 0; i < nx; ++i) make_key(&codes[i], (int)k, A.bits, A.per_word, A.words, &keys[(size_t)i * A.words]);
    for (int32_t i = 0; i < ny; ++i) make_key(&codes[lx + i], (int)k, A.bits, A.per_word, A.words, &keys[(size_t)(nx + i) * A.words]);
    KeyView K; K.keys = keys.data(); K.y_base = nx; K.k = (int)k; K.bits = A.bits; K.per_word = A.per_word; K.words = A.words;
    std::mt19937_64 rng(tie_seed);
    std::mt19937_64 *tie = tie_seed ? &rng : nullptr;
    const std::vector<ChainMum> top = host_problem(K, 0, (int32_t)lx, 0, (int32_t)ly, u, tie);
    std::vector<int32_t> gaps;
    std::vector<std::vector<ChainMum>> sub;
    if (recursive) {
        gap_table(top.data(), (int64_t)top.size(), (int32_t)lx, (int32_t)ly, bigger, gaps);
        for (size_t g = 0; g < gaps.size(); g += 4) sub.push_back(host_problem(K, gaps[g], gaps[g + 2], gaps[g + 1], gaps[g + 3], u, tie));
    }
    int64_t m = chain_bases(top);
    for (const auto &c : sub) m += chain_bases(c);
    int64_t *o = (int64_t *)malloc(16 * (size_t)std::max<int64_t>(m, 1));
    const int64_t n = splice(top.data(), (int64_t)top.size(), gaps, sub, recursive != 0, o);
    *out = o;
    return n;
}

extern "C" void hosttest_mum_free(void *p) { free(p); }

// the planning code, for tests: plan_chunks over per-pair bytes (out: 2 * n_chunks entries), pair_bytes, gap_table
extern "C" int64_t hosttest_mum_plan_chunks(const int64_t *bytes, int64_t n, int64_t budget, int64_t *out) {
    const auto c = plan_chunks(std::vector<int64_t>(bytes, bytes + n), budget);
    for (size_t i = 0; i < c.size(); ++i) { out[2 * i] = c[i].first; out[2 * i + 1] = c[i].second; }
    return (int64_t)c.size();
}
extern "C" int64_t hosttest_mum_pair_bytes(int64_t lx, int64_t ly, int64_t k, int words) { return pair_bytes(lx, ly, k, words); }
extern "C" int hosttest_mum_key_words(const char *sx, int64_t lx, const char *sy, int64_t ly, int64_t k) {
    Alphabet A; make_alphabet(sx, lx, sy, ly, k, A); return A.words;
}
// chain: n (x, y, len) triples first to last; out: 4 * gaps entries (x0, y0, x1, y1)
extern "C" int64_t hosttest_mum_gap_table(const int32_t *chain, int64_t n, int32_t lx, int32_t ly, int64_t bigger, int32_t *out) {
    std::vector<ChainMum> c(n);
    for (int64_t i = 0; i < n; ++i) c[i] = ChainMum{chain[3 * i], chain[3 * i + 1], chain[3 * i + 2]};
    std::vector<int32_t> g;
    gap_table(c.data(), n, lx, ly, bigger, g);
    memcpy(out, g.data(), 4 * g.size());
    return (int64_t)g.size() / 4;
}
