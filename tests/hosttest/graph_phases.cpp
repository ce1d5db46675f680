// graph_phases.cpp -- TEST-ONLY: the host build of hosttest.cpp (incremental order) with the product's shared-memory forms of the
// graph phases (cactus_b200/csrc/graph_phases.cuh) run after every fusion, the CTA's T threads one after the other, and compared
// with the serial forms: the order splice with hosttest's incremental_order, the edge sort + max_remain + row tables with
// graph_sort_node_edges + graph_bfs_remain + graph_build_rows. A difference fails the job (JOB_ERR_TOPO). Compiled by
// tests/test_graph_phases_cpu.py.
#include <vector>
#include "../../cactus_b200/csrc/graph_phases.cuh"

struct GraphPhaseStats { long long splice_smem, splice_global, topo_smem, topo_global, mismatches; };
static GraphPhaseStats g_stats;
static int g_scr_bytes = 1 << 20, g_threads = 128;

// Called where hosttest's incremental path runs graph_bfs_remain: the new nodes are spliced into the order (incremental_order)
// and every edge list is sorted.
static void check_phases_then_bfs_remain(barb200::Graph &g, barb200::RowTables &rt, const barb200::DpState &d, const uint8_t *q, int L,
                                         int n_old) {
    using namespace barb200;
    const int n = g.node_n;
    std::vector<uint64_t> scr_words((size_t)g_scr_bytes / 8 + 2);
    unsigned char *scr = reinterpret_cast<unsigned char *>(scr_words.data());
    int ws[32];
    bool same = true;
    // ---- the order splice, from the order before the fusion (the old nodes in the spliced order) ----
    const std::vector<int> s_i2n(g.index_to_node, g.index_to_node + n), s_n2i(g.node_to_index, g.node_to_index + n);
    std::vector<int> node_of;                                  // node of every query base: the fused alignment replayed
    int next_new = n_old;
    for (int c = 0; c < d.n_cigar; ++c) {
        const int op = (int)(d.cigar[c] & 0xf);
        if (op == CMATCH) {
            const int node_id = (int)((d.cigar[c] >> 34) & 0x3fffffff), qi = (int)((d.cigar[c] >> 4) & 0x3fffffff);
            const int v = g.base[node_id] == q[qi] ? node_id : graph_aligned_with_base(g, node_id, q[qi]);
            if (v >= n_old) ++next_new;
            node_of.push_back(v);
        } else if (op == CINS) {
            for (int k = 0; k < (int)((d.cigar[c] >> 4) & 0x3fffffff); ++k) node_of.push_back(next_new++);
        }
    }
    if ((int)node_of.size() != L || next_new != n) same = false;
    if (same && splice_smem_fits(L, n_old, n, g_scr_bytes)) {
        ++g_stats.splice_smem;
        for (int i = 0, k = 0; i < n; ++i) if (s_i2n[i] < n_old) { g.index_to_node[k] = s_i2n[i]; g.node_to_index[s_i2n[i]] = k; ++k; }
        splice_order_smem(g, node_of.data(), L, n_old, n - n_old, scr, ws, g_threads);
        for (int i = 0; i < n; ++i) same = same && g.index_to_node[i] == s_i2n[i] && g.node_to_index[i] == s_n2i[i];
        std::copy(s_i2n.begin(), s_i2n.end(), g.index_to_node); std::copy(s_n2i.begin(), s_n2i.end(), g.node_to_index);
    } else ++g_stats.splice_global;
    // ---- edge sort, max_remain, row tables ----
    if (topo_smem_fits(n, g_scr_bytes)) {
        ++g_stats.topo_smem;
        int n_pre = 0;
        for (int v = 0; v < n; ++v) n_pre += g.in_n[v];
        const std::vector<int> in_id(g.in_id, g.in_id + g.in_used), in_w(g.in_w, g.in_w + g.in_used);
        const std::vector<int> out_id(g.out_id, g.out_id + g.out_used), out_w(g.out_w, g.out_w + g.out_used);
        topo_rows_smem(g, rt, scr, ws, g_threads);
        same = same && std::equal(in_id.begin(), in_id.end(), g.in_id) && std::equal(in_w.begin(), in_w.end(), g.in_w) &&
               std::equal(out_id.begin(), out_id.end(), g.out_id) && std::equal(out_w.begin(), out_w.end(), g.out_w);
        const std::vector<int> remain(g.remain, g.remain + n), pre_row(rt.pre_row, rt.pre_row + n_pre);
        const std::vector<RowRec> rec(rt.rec, rt.rec + n);
        (graph_bfs_remain)(g);
        graph_build_rows(g, rt);
        for (int v = 0; v < n; ++v) same = same && remain[v] == g.remain[v];
        for (int r = 0; r < n; ++r)
            same = same && rec[r].base_npre == rt.rec[r].base_npre && rec[r].rd == rt.rec[r].rd && rec[r].pre_off == rt.rec[r].pre_off && rec[r].pre0 == rt.rec[r].pre0;
        for (int k = 0; k < n_pre; ++k) same = same && pre_row[k] == rt.pre_row[k];
    } else {
        ++g_stats.topo_global;
        (graph_bfs_remain)(g);
    }
    if (!same) { ++g_stats.mismatches; g.err = JOB_ERR_TOPO; }
}
#define graph_bfs_remain(g) check_phases_then_bfs_remain(g, rt, d, q, L, n_old)
#include "hosttest.cpp"

extern "C" void graph_phases_config(int scr_bytes, int threads) { g_scr_bytes = scr_bytes; g_threads = threads; memset(&g_stats, 0, sizeof g_stats); }
extern "C" const long long *graph_phases_stats() { return &g_stats.splice_smem; }
