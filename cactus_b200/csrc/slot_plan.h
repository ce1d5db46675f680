// slot_plan.h -- the arithmetic of a stage's device-memory plan (stage_plan.h: fit_stage) and the layout of the memory it plans:
// a POA slot, a guide-tree scratch slot. CUDA-free, so that the CPU suite runs the product's graph and guide-tree code on the
// same layout (tests/hosttest) and checks the plan for a given device size.
#pragma once
#include <stdint.h>
#include <algorithm>
#include "poa_types.h"
#include "guide_tree.cuh"

namespace barb200 {

inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// byte ranges carved one after the other from one block, each starting at a multiple of `align`
struct BumpOffsets {
    int64_t align, end = 0;
    int64_t take(int64_t bytes) { const int64_t r = end; end = align_up(end + bytes, align); return r; }
};

// ---- a POA slot: one resident CTA's graph, row tables, band table, cigar and traceback scratch; its DP planes lie apart ----
// Byte offsets of every per-slot array from the slot base; the arrays' element types and counts are those of Graph, RowTables
// and DpState (poa_types.h).
struct SlotLayout {
    int64_t slot_bytes;
    int node_cap, in_pool, out_pool, W, cigar_cap, fc_cap;
    int64_t plane_cap;   // ints per slot
    int64_t o_base, o_aln_n, o_aln_id, o_in_off, o_in_n, o_in_cap, o_out_off, o_out_n, o_out_cap;
    int64_t o_in_id, o_in_w, o_out_id, o_out_w, o_out_rid;
    int64_t o_index_to_node, o_node_to_index, o_remain, o_msa_rank, o_tmp0, o_tmp1;
    int64_t o_row_rec, o_pre_row;
    int64_t o_row_off, o_row_info, o_cigar, o_fc;
};

// What a slot must hold: the largest of the jobs it may run.
struct SlotNeeds {
    int64_t nodes = 4, edges = 4, max_len = 1, K = 1, plane_ints = 0;
    // a job of K sequences, `sum` bases in all, the longest `ml`, whose planes are planned at `planes` ints: at worst every base
    // is a new node besides source and sink, and every read's path adds an edge per base plus one
    void add_job(int64_t k, int64_t sum, int64_t ml, int64_t planes) {
        nodes = std::max(nodes, sum + 2); edges = std::max(edges, sum + k); max_len = std::max(max_len, ml); K = std::max(K, k);
        plane_ints = std::max(plane_ints, planes);
    }
};

// Capacities and offsets of a slot for `n`. The edge pools hold 4x the edges: an edge list that grows moves to a fresh chunk
// of twice its size (poa_types.h: Graph). Arrays 16-byte aligned, the slot a multiple of 256 bytes.
inline SlotLayout plan_slot(const SlotNeeds &n) {
    SlotLayout Y{};
    Y.node_cap = (int)n.nodes; Y.in_pool = (int)(4 * n.edges + 64); Y.out_pool = Y.in_pool;
    Y.W = (int)(1 + ((n.K - 1) >> 6)); Y.cigar_cap = (int)(n.max_len + n.nodes + 16); Y.fc_cap = (int)(n.max_len + 2);
    Y.plane_cap = align_up(n.plane_ints, 8);
    BumpOffsets o{16};
    const int64_t N = Y.node_cap, E = Y.in_pool;
    Y.o_base = o.take(N); Y.o_aln_n = o.take(N); Y.o_aln_id = o.take(N * 16);
    Y.o_in_off = o.take(N * 4); Y.o_in_n = o.take(N * 4); Y.o_in_cap = o.take(N * 4);
    Y.o_out_off = o.take(N * 4); Y.o_out_n = o.take(N * 4); Y.o_out_cap = o.take(N * 4);
    Y.o_in_id = o.take(E * 4); Y.o_in_w = o.take(E * 4);
    Y.o_out_id = o.take(E * 4); Y.o_out_w = o.take(E * 4);
    Y.o_out_rid = o.take(E * 8 * Y.W);
    Y.o_index_to_node = o.take(N * 4); Y.o_node_to_index = o.take(N * 4); Y.o_remain = o.take(N * 4); Y.o_msa_rank = o.take(N * 4);
    Y.o_tmp0 = o.take(N * 4); Y.o_tmp1 = o.take(N * 4);
    Y.o_row_rec = o.take(N * 16); Y.o_pre_row = o.take(E * 4);
    Y.o_row_off = o.take(N * 8); Y.o_row_info = o.take(N * 16);
    Y.o_cigar = o.take((int64_t)Y.cigar_cap * 8);
    Y.o_fc = o.take((int64_t)Y.fc_cap * 8);
    Y.slot_bytes = align_up(o.end, 256);
    return Y;
}

// The graph, row-table and DP views of the slot at `b` whose planes start at `planes`. What describes the job in them (node_n,
// W, the pools' use) graph_reset sets.
HD void slot_views(const SlotLayout &Y, uint8_t *b, int *planes, Graph &g, RowTables &rt, DpState &d) {
    g.node_cap = Y.node_cap; g.in_pool = Y.in_pool; g.out_pool = Y.out_pool;
    g.base = b + Y.o_base; g.aln_n = b + Y.o_aln_n; g.aln_id = (int *)(b + Y.o_aln_id);
    g.in_off = (int *)(b + Y.o_in_off); g.in_n = (int *)(b + Y.o_in_n); g.in_cap = (int *)(b + Y.o_in_cap);
    g.out_off = (int *)(b + Y.o_out_off); g.out_n = (int *)(b + Y.o_out_n); g.out_cap = (int *)(b + Y.o_out_cap);
    g.in_id = (int *)(b + Y.o_in_id); g.in_w = (int *)(b + Y.o_in_w);
    g.out_id = (int *)(b + Y.o_out_id); g.out_w = (int *)(b + Y.o_out_w); g.out_rid = (uint64_t *)(b + Y.o_out_rid);
    g.index_to_node = (int *)(b + Y.o_index_to_node); g.node_to_index = (int *)(b + Y.o_node_to_index);
    g.remain = (int *)(b + Y.o_remain); g.msa_rank = (int *)(b + Y.o_msa_rank);
    g.tmp0 = (int *)(b + Y.o_tmp0); g.tmp1 = (int *)(b + Y.o_tmp1);
    rt.rec = (RowRec *)(b + Y.o_row_rec); rt.pre_row = (int *)(b + Y.o_pre_row);
    d.planes = planes; d.plane_cap = Y.plane_cap;
    d.row_off = (int64_t *)(b + Y.o_row_off); d.info = (RowInfo *)(b + Y.o_row_info);
    d.cigar = (uint64_t *)(b + Y.o_cigar); d.cigar_cap = Y.cigar_cap; d.n_cigar = 0;
    d.fc = (int *)(b + Y.o_fc); d.fc_cap = Y.fc_cap; d.fc_row = -1; d.fc_hi = -1;
}

// ---- a guide-tree scratch slot: one guide_tree_kernel CTA's arrays of GtScratch (guide_tree.cuh) ----
struct GtLayout {
    int64_t slot_bytes;
    int64_t o_keys, o_gx, o_hit, o_jac, o_score;
    int key_cap;                     // a power of two: the sort pads to one
    int64_t base_cap, seq_cap;       // bases and sequences of the largest job
};

// What a scratch slot must hold: the largest of the jobs whose read order comes from a guide tree.
struct GtNeeds {
    int64_t keys = 64, bases = 8, K = 1;
    // Minimizer keys: about 2 / (w + 1) per base, but ties in repeats can push it up to 2 w per base. Below the worst case the
    // keys are planned optimistically like the DP planes, and a job that outgrows them is retried with more (grow, worst_case).
    void add_job(int progressive, int64_t k, int64_t sum, int w, double grow, bool worst_case) {
        if (!(progressive && k > 2)) return;
        const int64_t worst = 2 * (int64_t)w * sum + k;
        keys = std::max(keys, worst_case ? worst : std::min<int64_t>(worst, (int64_t)(grow * (double)(sum / 2 + 64))));
        bases = std::max(bases, sum); K = std::max(K, k);
    }
};

inline GtLayout plan_gt_scratch(const GtNeeds &n) {
    GtLayout Y{};
    int64_t kc = 64; while (kc < n.keys) kc <<= 1;
    Y.key_cap = (int)kc; Y.base_cap = n.bases; Y.seq_cap = n.K;
    BumpOffsets o{16};
    const int64_t K = n.K;
    Y.o_keys = o.take(kc * 8); Y.o_gx = o.take(n.bases * 8); Y.o_hit = o.take(K * (K + 1) / 2 * 4); Y.o_jac = o.take(K * (K - 1) / 2 * 8 + 8);
    Y.o_score = o.take(K * 8);
    Y.slot_bytes = align_up(o.end, 256);
    return Y;
}

// The global-memory arrays of the scratch slot at `b`; the caller adds n_keys and the sort's tile (shared memory on the device).
HD GtScratch gt_views(const GtLayout &Y, uint8_t *b) {
    GtScratch G{};
    G.keys = (uint64_t *)(b + Y.o_keys); G.key_cap = Y.key_cap; G.gx = (uint64_t *)(b + Y.o_gx);
    G.hit = (int *)(b + Y.o_hit); G.jac = (double *)(b + Y.o_jac); G.score = (double *)(b + Y.o_score);
    return G;
}

// DP-plane ints one slot plans for a job of K sequences, `sum` bases in all, the longest `ml`. grow / worst_case: the capacity
// retries. Rows the graph can reach: worst case every base a new node; optimistic: the longest read plus a share of the rest.
// Columns a row stores: the adaptive band is [min(maxL, d) - w, max(maxR, d) + w] (abpoa_align_simd.c:946-960), i.e. 2w plus
// however far the best columns of the predecessors have drifted from the row's diagonal d; a quarter of 2w is allowed for that
// before the geometric retries take over. Only windows longer than ~2.5 kbp are narrower than the whole row (w = 1000 + 0.1 L):
// a 10 kbp window plans 0.77 GB of planes instead of 1.53 GB.
// Optimistic rows of a job's graph: the longest read plus an eighth of the other bases, plus a margin.
inline int64_t optimistic_rows(int64_t sum, int64_t ml) { return ml + (sum - ml) / 8 + 256; }

inline int64_t plane_ints_for_job(int wb, double wf, int64_t K, int64_t sum, int64_t ml, double grow, bool worst_case) {
    (void)K;
    int64_t rows = sum + 2;
    if (!worst_case) rows = std::min<int64_t>(rows, (int64_t)(grow * (double)optimistic_rows(sum, ml)));
    int64_t width = ml + 1;
    if (!worst_case) {
        const int64_t w = (int64_t)wb + (int64_t)(wf * (double)ml);
        width = std::min<int64_t>(width, (int64_t)(grow * (2.5 * (double)w + 64.0)));
    }
    return rows * (TB / CPT) * ((width + CPT - 1) / CPT * CPT + CPT);
}

// Words of a job's trace region (the trace kernels, poa_kernel.cu: trace_record): K records of 6 header words, the cigar and two
// words per row. At the worst case from the bounds of a slot planned for the job alone: rows = node_n - 1 < node_cap, and a cigar
// holds at most cigar_cap ops (the traceback fails the job beyond that). Optimistic: plane_ints_for_job's row estimate for every
// alignment, and a cigar of one op per query base and row; grow: the capacity retries, as for the planes.
inline int64_t trace_words_for_job(int64_t K, int64_t sum, int64_t ml, double grow, bool worst_case) {
    const int64_t node_cap = sum + 2, cigar_cap = ml + node_cap + 16;   // plan_slot of SlotNeeds::add_job(K, sum, ml, ...)
    const int64_t worst = K * (6 + cigar_cap + 2 * node_cap);
    if (worst_case) return worst;
    const int64_t rows = optimistic_rows(sum, ml);
    return std::min<int64_t>(worst, (int64_t)(grow * (double)(K * (6 + ml + 3 * rows))));
}

// Device bytes a lane may plan a stage with: a fraction of what is free plus what the lane's arena already holds, minus the
// stage's own block; once lanes are shared (the end queue runs), at most its share of the device.
inline double lane_budget_bytes(double free_b, double total_b, double arena_b, double block_b, double frac, bool shared, int lanes) {
    double budget = (free_b + arena_b) * frac - block_b;
    if (shared && lanes > 1) budget = std::min(budget, total_b * frac / lanes - block_b);
    return budget;
}

// A capacity retry (grow > 1 or worst case) whose single-slot plan exceeds the budget: its plane estimate is an upper bound, so
// the planes are cut to what the budget leaves after the slots' fixed part (the kernel checks every row against the cut capacity
// and flags a job that really outgrows it). Returns the factor to apply to every bucket's plane capacity, 0 if even the fixed
// part does not fit.
inline double retry_plane_scale(double budget, double fixed_bytes, double plane_bytes) {
    if (plane_bytes <= 0 || fixed_bytes >= budget) return 0.0;
    return std::min(1.0, (budget - fixed_bytes) / plane_bytes);
}

}  // namespace barb200
