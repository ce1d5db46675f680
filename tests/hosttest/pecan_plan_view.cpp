// pecan_plan_view.cpp -- TEST-ONLY host build of the product's split and plan of one cPecan pair (cactus_b200/csrc/pecan_plan.cpp:
// split_pair, plan_subjob) behind a C symbol, for the tests that pin the edges of a pair-HMM launch plan.
// tests/test_pecan_edges_cpu.py compiles this file with pecan_plan.cpp into a temporary directory; never shipped, never loaded by
// cactus_b200.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../cactus_b200/csrc/pecan_plan.h"

// the layout of tests/_reflib.py: PecanParams
struct PlanViewParams { double threshold; int64_t minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion; };

enum { kPlanCols = 12 };

// Per sub-job of the pair, kPlanCols values: x1, y1, lx, ly, ragged, cells, max_w, span_cells, span_full_cells, ring_center, the
// number of tracebacks, and the output room a stage gives it (pecan.cu: stage_build). Returns the number of sub-jobs with *out
// malloc'd (free it with hosttest_pecan_plan_free), -1 for parameters or anchors the product rejects, -2 for a band it rejects.
extern "C" int64_t hosttest_pecan_plan(int64_t lX, int64_t lY, const int64_t *anchors, int64_t n_anchor, int ragged_left, int ragged_right,
                                       const PlanViewParams *pp, int64_t split_bigger, int64_t **out) {
    namespace pc = barb200::pecan;
    const pc::PlanParams P{pp->threshold, pp->minDiagsBetweenTraceBack, pp->traceBackDiagonals, pp->diagonalExpansion, split_bigger};
    *out = nullptr;
    if (!pc::check_params(P).empty() || !pc::check_anchors(anchors, n_anchor, lX, lY).empty()) return -1;
    std::vector<pc::SubJob> subs;
    pc::split_pair(P, 0, lX, lY, anchors, n_anchor, ragged_left != 0, ragged_right != 0, subs);
    std::vector<int64_t> v;
    for (pc::SubJob &s : subs) {
        if (!pc::plan_subjob(P, s).empty()) return -2;
        const int64_t row[kPlanCols] = {s.x1, s.y1, s.lx, s.ly, s.ragged, s.cells, s.max_w, s.span_cells, s.span_full_cells, s.ring_center,
                                        (int64_t)s.tb_from.size(), std::min<int64_t>(s.cells, (int64_t)s.lx + s.ly + 64)};
        v.insert(v.end(), row, row + kPlanCols);
    }
    *out = (int64_t *)malloc(sizeof(int64_t) * std::max<size_t>(v.size(), 1));
    if (!v.empty()) memcpy(*out, v.data(), sizeof(int64_t) * v.size());
    return (int64_t)subs.size();
}

extern "C" void hosttest_pecan_plan_free(void *p) { free(p); }
