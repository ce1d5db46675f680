// pecan_plan.h -- host-side planning of pair-HMM jobs: splitting a sequence pair at large anchor gaps, the anchor band,
// and the forward/traceback schedule (which only depends on the band geometry) that sizes the device buffers.
// Re-stated from submodules/cPecan/impl/pairwiseAligner.c: getSplitPoints :1241-1292, the sub-anchor selection of
// getPosteriorProbsWithBandingSplittingAlignmentsByLargeGaps :1308-1363, band_construct :193-244 with
// band_setCurrentDiagonal :104-132, and the traceback conditions of getPosteriorProbsWithBanding :798-803, 817.
#pragma once
#include <stdint.h>
#include <string>
#include <utility>
#include <vector>

namespace barb200 {
namespace pecan {

struct PlanParams {
    double threshold;
    int64_t min_diags, tb_diags, expansion, split_bigger;
};

struct SubJob {
    int64_t pair = 0;              // index of the sequence pair this sub-matrix belongs to
    int64_t x1 = 0, y1 = 0;        // offset of the sub-matrix in the pair
    int lx = 0, ly = 0;
    int ragged = 0;                // bit 0 left, bit 1 right
    std::vector<int64_t> anchors;  // (x, y) relative to (x1, y1)
    // plan
    std::vector<int> bandL;        // xmyL of diagonals 0..D
    std::vector<int> coff;         // cells before diagonal d, D+2 entries
    std::vector<int> foff;         // cells of MARKED diagonals before diagonal d, D+2 entries (see plan_subjob)
    int64_t cells = 0;             // sum of diagonal widths
    int64_t span_cells = 0;        // most forward cells alive at once (between two tracebacks)
    int64_t span_full_cells = 0;   // most cells of marked diagonals alive at once
    std::vector<int> tb_from;      // the diagonal each traceback starts emitting posteriors from (ascending)
    int max_w = 0;
    int ring_center = 0;           // cell-weighted mean of the absolute ring coordinate ((xmy + parity) / 2 + ly) over the band
    int out_cap = 0;
};

// Returns "" or an error message (the reference asserts on the same conditions).
std::string check_params(const PlanParams &P);
std::string check_anchors(const int64_t *anchors, int64_t n, int64_t lx, int64_t ly);

// getSplitPoints + sub-anchor lists: appends the sub-jobs of one pair (anchors: n (x, y) pairs, 0-based).
void split_pair(const PlanParams &P, int64_t pair, int64_t lx, int64_t ly, const int64_t *anchors, int64_t n_anchor,
                bool ragged_left, bool ragged_right, std::vector<SubJob> &out);

// band_construct: fills bandL / coff / cells / max_w; then the schedule: which spans of diagonals are alive together
// (span_cells) and which diagonals a traceback needs COMPLETE forward cells of (marked in foff): the ones the total
// probability is recomputed on (every 10th posterior diagonal, pairwiseAligner.c:840-848) with their predecessors, and
// the two diagonals the forward sweep resumes from after an intermediate traceback. Returns "" or an error.
std::string plan_subjob(const PlanParams &P, SubJob &j);

// A batch over ndev devices: whole pairs by cost (a pair-HMM pair: the planned cells of its sub-jobs; a MUM-anchor pair: its
// device bytes), largest first to the least-loaded device (ties: the lower device; equal costs: the earlier pair), every share
// in caller order. One device takes every pair in caller order. Returns ndev shares of indices into `cost`.
std::vector<std::vector<int64_t>> deal_pairs(const std::vector<int64_t> &cost, int ndev);

// The reference's order of emission inside one sub-matrix (getPosteriorProbsWithBanding): tracebacks in increasing order of
// their start diagonal, inside a traceback diagonals x+y downwards, inside a diagonal x - y (hence x) upwards.
// Sort key of the candidate (0-based x, y) of sub-job j; ascending (first, second) = order of emission.
inline std::pair<uint64_t, uint32_t> emission_key(const SubJob &j, int x, int y) {
    const uint32_t t = (uint32_t)x + (uint32_t)y + 2u;
    size_t seg = 0, hi = j.tb_from.size();          // first traceback with tb_from >= t
    while (seg < hi) { const size_t mid = (seg + hi) / 2; if ((uint32_t)j.tb_from[mid] >= t) hi = mid; else seg = mid + 1; }
    return std::make_pair(((uint64_t)seg << 32) | (uint64_t)(0xffffffffu - t), (uint32_t)x);
}

}  // namespace pecan
}  // namespace barb200
