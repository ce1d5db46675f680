// synth.cpp -- WORKLOAD GENERATOR (not part of the engine: built into workload/libbarsynth.so so that the reference arm of
// bench.py maps no product library). Seeded synthetic BAR ends of BASELINE.json's "N ends x K seqs x L bp" shape (SURVEY.md section 8d).
// For end e: xoshiro256** seeded (through splitmix64) with seed + e; parent = L uniform ACGT; K descendants, each base
// deleted with probability `del`, substituted by a uniformly chosen different base with probability `sub`, and followed by
// a uniformly random inserted base with probability `ins`; rows sorted by length, longest first (stable), which is the
// order get_end_sequences hands them to the aligner (bar/impl/poaBarAligner.c:1073-1081).
#include <stdint.h>
#include <algorithm>
#include <numeric>
#include <vector>

namespace {
struct Xoshiro {
    uint64_t s[4];
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    explicit Xoshiro(uint64_t seed) {
        for (int i = 0; i < 4; ++i) {   // splitmix64
            uint64_t z = (seed += 0x9e3779b97f4a7c15ULL);
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL; z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL; s[i] = z ^ (z >> 31);
        }
    }
    uint64_t next() {
        const uint64_t r = rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rotl(s[3], 45);
        return r;
    }
    double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};
}  // namespace

extern "C" int64_t barsynth_end(uint64_t seed, uint64_t end_index, int K, int L, double sub, double ins, double del,
                                     uint8_t *codes_out, int *lens_out) {
    if (K <= 0 || L <= 0 || !codes_out || !lens_out) return -1;
    Xoshiro rng(seed + end_index);
    std::vector<uint8_t> parent((size_t)L);
    for (int i = 0; i < L; ++i) parent[i] = (uint8_t)(rng.next() >> 62);
    std::vector<std::vector<uint8_t>> rows((size_t)K);
    for (int k = 0; k < K; ++k) {
        std::vector<uint8_t> &r = rows[k];
        r.reserve((size_t)L + 16);
        for (int i = 0; i < L && (int)r.size() < 2 * L + 8; ++i) {
            const double u = rng.uniform();
            if (u >= del) r.push_back(u < del + sub ? (uint8_t)((parent[i] + 1 + rng.next() % 3) & 3) : parent[i]);
            if (rng.uniform() < ins) r.push_back((uint8_t)(rng.next() >> 62));
        }
        if (r.empty()) r.push_back(parent[0]);
    }
    std::vector<int> idx((size_t)K);
    std::iota(idx.begin(), idx.end(), 0);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return rows[a].size() > rows[b].size(); });
    int64_t o = 0;
    for (int k = 0; k < K; ++k) {
        const std::vector<uint8_t> &r = rows[idx[k]];
        std::copy(r.begin(), r.end(), codes_out + o);
        lens_out[k] = (int)r.size(); o += (int64_t)r.size();
    }
    return o;
}

// Seeded synthetic sequence PAIR for the cPecan-mode benchmark: two descendants of one random parent (same event model as
// above) as ASCII, plus anchor pairs placed the way cPecan's MUM anchoring places them on similar sequences: every
// position of every run of >= k_anchor identical, co-linear bases of the true alignment (getAlignedMums emits one anchor
// per base of each maximal unique match of length >= k, submodules/cPecan/impl/pairwiseAligner.c:2032-2059; Cactus
// configures k = 50, :1389). sx_out / sy_out: at least 2*L+16 bytes each; anchors_out: at least 2*L (x, y) int64 pairs.
extern "C" int64_t barsynth_pair(uint64_t seed, uint64_t pair_index, int L, double sub, double ins, double del, int k_anchor,
                                      char *sx_out, int64_t *lx_out, char *sy_out, int64_t *ly_out, int64_t *anchors_out) {
    if (L <= 0 || k_anchor <= 0 || !sx_out || !sy_out || !lx_out || !ly_out || !anchors_out) return -1;
    Xoshiro rng(seed * 0x9e3779b97f4a7c15ULL + pair_index + 0x5eed);
    std::vector<uint8_t> parent((size_t)L);
    for (int i = 0; i < L; ++i) parent[i] = (uint8_t)(rng.next() >> 62);
    static const char B[4] = {'A', 'C', 'G', 'T'};
    // pos[s][i] = position in descendant s of the unchanged copy of parent base i, or -1
    std::vector<int> pos[2] = {std::vector<int>((size_t)L, -1), std::vector<int>((size_t)L, -1)};
    char *outs[2] = {sx_out, sy_out};
    int64_t lens[2] = {0, 0};
    for (int s = 0; s < 2; ++s) {
        int64_t n = 0;
        for (int i = 0; i < L && n < 2 * (int64_t)L + 8; ++i) {
            const double u = rng.uniform();
            if (u >= del) {
                if (u < del + sub) outs[s][n++] = B[(parent[i] + 1 + rng.next() % 3) & 3];
                else { pos[s][i] = (int)n; outs[s][n++] = B[parent[i]]; }
            }
            if (rng.uniform() < ins) outs[s][n++] = B[rng.next() >> 62];
        }
        if (n == 0) outs[s][n++] = B[parent[0]];
        lens[s] = n;
    }
    *lx_out = lens[0]; *ly_out = lens[1];
    int64_t na = 0, run0 = 0, runlen = 0;     // runs of consecutive (x+1, y+1) columns among the shared unchanged bases
    std::vector<std::pair<int, int>> cols;
    for (int i = 0; i < L; ++i) if (pos[0][i] >= 0 && pos[1][i] >= 0) cols.emplace_back(pos[0][i], pos[1][i]);
    for (size_t c = 0; c <= cols.size(); ++c) {
        const bool cont = c < cols.size() && runlen > 0 && cols[c].first == cols[c - 1].first + 1 && cols[c].second == cols[c - 1].second + 1;
        if (cont) { ++runlen; continue; }
        if (runlen >= k_anchor)
            for (int64_t q = 0; q < runlen; ++q) { anchors_out[2 * na] = cols[run0 + q].first; anchors_out[2 * na + 1] = cols[run0 + q].second; ++na; }
        run0 = (int64_t)c; runlen = c < cols.size() ? 1 : 0;
    }
    return na;
}

// FNV-1a over (msa_len, bytes) of a K x msa_len alignment matrix: the per-end hash bench.py's parity gate compares between the
// GPU arm and the CPU arm (same function as oracle/ref_harness.c: msa_hash)
extern "C" uint64_t barsynth_msa_hash(const uint8_t *m, int64_t n, int msa_len) {
    uint64_t h = 1469598103934665603ULL ^ (uint64_t)(uint32_t)msa_len;
    h *= 1099511628211ULL;
    for (int64_t k = 0; k < n; ++k) { h ^= m[k]; h *= 1099511628211ULL; }
    return h;
}

// plain 64-bit FNV-1a over n bytes: the anchor and triple hashes of a cPecan harvest record (shim/cactus_pecan_harvest.c)
extern "C" uint64_t barsynth_fnv1a(const uint8_t *b, int64_t n) {
    uint64_t h = 0xcbf29ce484222325ULL;
    for (int64_t k = 0; k < n; ++k) { h ^= b[k]; h *= 0x100000001b3ULL; }
    return h;
}
