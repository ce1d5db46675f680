// pred_rows.cpp -- TEST-ONLY: the host build of hosttest.cpp with a count of the predecessor rows every DP sweep sees.
// Each sweep's row table (poa_graph.cuh: RowRec / pre_row, built by the topological sort) is read just after the sweep, before
// the alignment is fused, so the counts describe exactly the rows the kernel's sweep of the same job walks: how many rows have
// a predecessor at r - d, how many have row 0 as a predecessor at row 2, and how many have 3 or 4 predecessors. Compiled by
// tests/test_far_rows_cpu.py.
#include "../../cactus_b200/csrc/poa_graph.cuh"

struct PredRowCounts {
    long long rows;            // rows swept (1 .. R-1 of every sweep)
    long long dist[65];        // predecessors at r - d (d >= 64 counted at 64)
    long long row0_at_row2;    // row 2 has row 0 as a predecessor
    long long npre[5];         // rows with 1, 2, 3, >= 4 predecessors (index 4 = 4 or more)
};
static PredRowCounts g_counts;

static void count_rows_then_best_cell(const barb200::Graph &g, const barb200::RowTables &rt, barb200::DpState &d,
                                      const barb200::PoaParams &P, int L) {
    const int R = g.node_n - 1;
    for (int r = 1; r < R; ++r) {
        const int np = rt.rec[r].base_npre >> 8, off = rt.rec[r].pre_off;
        ++g_counts.rows;
        ++g_counts.npre[np < 4 ? np : 4];
        for (int k = 0; k < np; ++k) {
            const int p = rt.pre_row[off + k], dd = r - p;
            ++g_counts.dist[dd < 64 ? dd : 64];
            if (r == 2 && p == 0) ++g_counts.row0_at_row2;
        }
    }
    barb200::dp_best_cell(g, rt, d, P, L);
}
#define dp_best_cell count_rows_then_best_cell
#include "hosttest.cpp"

extern "C" void pred_rows_reset() { memset(&g_counts, 0, sizeof g_counts); }
extern "C" const long long *pred_rows_counts() { return &g_counts.rows; }
