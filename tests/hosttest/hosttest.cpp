// hosttest.cpp -- TEST-ONLY build (never shipped, never loaded by cactus_b200): compiles the product's
// __host__ __device__ graph / traceback code (cactus_b200/csrc/poa_graph.cuh) and its guide tree (guide_tree.cuh, the
// CTA program with its threads run one after the other) with g++ so that the CPU suite can check them against the oracle
// in a container without a GPU.
// The DP sweep itself is CUDA-only; here it is stood in for by a scalar emulation of the kernel's per-row
// formulation (gathered band, prefix-maximum form of F) writing the same plane layout, which also pins that
// formulation's arithmetic. The real kernel is checked on the GPU by tests/test_gpu_*.py.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include <math.h>
#include "../../cactus_b200/csrc/poa_graph.cuh"
#include "../../cactus_b200/csrc/guide_tree.cuh"
#include "../../cactus_b200/csrc/slot_plan.h"
#include "../../cactus_b200/csrc/host_api.h"

using namespace barb200;

struct HtParams { int wb; float wf; int o1, e1, o2, e2; int mat[25]; int k, w, min_w; int progressive, disable_seeding; };

static long long emulate_sweep(const Graph &g, const RowTables &rt, DpState &d, const PoaParams &P, const uint8_t *q, int L) {
    const int node_n = g.node_n, R = node_n - 1, NEG = P.inf_min, e1 = P.e1, e2 = P.e2, oe1 = P.o1 + P.e1, oe2 = P.o2 + P.e2;
    const int w = P.wb + (int)(P.wf * L), pn = reference_lane_count(P, L, node_n);
    long long cur_off = 0, cells = 0;
    for (int r = 0; r < R; ++r) {
        int beg, end;
        const int b = row_base(rt, r), p0 = rt.rec[r].pre_off, p1 = p0 + row_npre(rt, r), dd = L - rt.rec[r].rd;
        if (r == 0) { beg = 0; end = std::min(L, std::max(0, dd) + w); }
        else {
            int maxL = node_n, maxR = 0, min_pre_beg = 0x7fffffff;
            for (int k = p0; k < p1; ++k) { const int p = rt.pre_row[k]; maxL = std::min(maxL, d.info[p].left + 1); maxR = std::max(maxR, d.info[p].right + 1); min_pre_beg = std::min(min_pre_beg, d.info[p].beg); }
            beg = std::max(0, std::min(maxL, dd) - w); end = std::min(L, std::max(maxR, dd) + w);
            if (beg / pn < min_pre_beg / pn) beg = min_pre_beg;
        }
        if (cur_off + row_ints(beg, end) > d.plane_cap) return -1;
        int *rowp = d.planes + cur_off;
        // the row maximum starts below every value, as in the kernel (inf_min minus a constant wraps when both extensions are <= 1)
        int P1 = NEG + beg * e1, P2 = NEG + beg * e2, tmax = INT32_MIN, tl = 0, tr = r == 0 ? 0 : -1;
        for (int j = beg / CPT * CPT; j <= (end / CPT) * CPT + CPT - 1; ++j) {
            int h, x1, x2, f1, f2;
            if (r == 0) {
                if (j == 0) { h = 0; x1 = -oe1; x2 = -oe2; f1 = f2 = NEG; }
                else if (j <= end) { f1 = -P.o1 - e1 * j; f2 = -P.o2 - e2 * j; h = std::max(f1, f2); x1 = x2 = NEG; }
                else h = x1 = x2 = f1 = f2 = NEG;
            } else {
                int m = NEG; x1 = NEG; x2 = NEG;
                for (int k = p0; k < p1; ++k) {
                    const int p = rt.pre_row[k];
                    m = std::max(m, plane_cell(d, NEG, p, 0, j - 1)); x1 = std::max(x1, plane_cell(d, NEG, p, 1, j)); x2 = std::max(x2, plane_cell(d, NEG, p, 2, j));
                }
                const int s = (j >= 1 && j <= L) ? P.mat[5 * b + q[j - 1]] : 0;
                int hme;
                if (j < beg || j > end) { hme = NEG; x1 = NEG; x2 = NEG; } else hme = std::max(std::max(m + s, x1), x2);
                const int A1 = hme - oe1 + (j + 1) * e1, A2 = hme - oe2 + (j + 1) * e2;
                f1 = P1 - j * e1; f2 = P2 - j * e2;
                P1 = std::max(P1, A1); P2 = std::max(P2, A2);
                if (j < beg || j > end) { h = NEG; f1 = NEG; f2 = NEG; }
                else {
                    h = std::max(std::max(hme, f1), f2);
                    x1 = std::max(x1 - e1, h - oe1); x2 = std::max(x2 - e2, h - oe2);
                    if (h > tmax) { tmax = h; tl = tr = j; } else if (h == tmax) tr = j;
                }
            }
            // the sweep's plane layout: H and the two E values as 16-bit distances below H (poa_types.h); F is not stored.
            // In-band cells of rows >= 1 must encode exactly (e <= H - E' <= oe), which this emulation asserts.
            const int c1 = e_encode(h, x1), c2 = e_encode(h, x2);
            if (r > 0 && j >= beg && j <= end && (e_decode(h, c1, NEG) != x1 || e_decode(h, c2, NEG) != x2)) return -2;
            (void)f1; (void)f2;
            rowp[plane_index(beg, end, 0, j)] = h; rowp[plane_index(beg, end, 1, j)] = c1 | (c2 << 16);
        }
        // the reference counts only cells above inf_min as a row maximum (simd_abpoa_max_in_row starts at inf_min), the kernel every
        // cell. They agree because every row a band reaches has a cell above inf_min (the band holds a predecessor's argmax column
        // or the one right of it), which this emulation asserts
        if (r > 0 && tmax <= NEG) return -2;
        RowInfo ri; ri.beg = beg; ri.end = end; ri.left = r == 0 ? 0 : tl; ri.right = r == 0 ? 0 : tr;
        d.info[r] = ri; d.row_off[r] = cur_off;
        cur_off += row_ints(beg, end); cells += end - beg + 1;
    }
    return cells;
}


// TEST-ONLY serial statement of the incremental topological order the device uses instead of re-running the BFS
// (poa_cta.cuh: cta_fuse_alignment): the previous order stays valid for old nodes; a new node aligned to x is appended
// to x's block of aligned nodes, an inserted (unaligned) new node opens a block right after the block of the previous
// path node. Called AFTER graph_fuse_alignment; replays the cigar to find the node of every query base.
static void incremental_order(Graph &g, const uint8_t *seq, const uint64_t *cigar, int n_cigar, int first_new, int n_old) {
    std::vector<int> path;                                   // node of query base q
    int next_new = first_new;
    for (int c = 0; c < n_cigar; ++c) {
        const int op = (int)(cigar[c] & 0xf);
        if (op == CMATCH) {
            const int node_id = (int)((cigar[c] >> 34) & 0x3fffffff), q = (int)((cigar[c] >> 4) & 0x3fffffff);
            int v = node_id;
            if (g.base[node_id] != seq[q]) v = graph_aligned_with_base(g, node_id, seq[q]);
            if (v >= first_new) ++next_new;
            path.push_back(v);
        } else if (op == CINS) {
            const int len = (int)((cigar[c] >> 4) & 0x3fffffff);
            for (int k = 0; k < len; ++k) path.push_back(next_new++);
        }
    }
    auto block_end = [&](int v) {                            // last old index of v's block of aligned nodes, -1 if none
        int e = v < first_new ? g.node_to_index[v] : -1;
        for (int k = 0; k < g.aln_n[v]; ++k) { const int a = g.aln_id[v * 4 + k]; if (a < first_new) e = std::max(e, g.node_to_index[a]); }
        return e;
    };
    std::vector<std::vector<int>> after(n_old);              // new nodes to place after old index i, in path order
    int anchor = 0;                                          // SRC's index
    for (size_t q = 0; q < path.size(); ++q) {
        const int v = path[q], e = block_end(v);
        if (e >= 0) anchor = std::max(anchor, e);
        if (v >= first_new) after[anchor].push_back(v);
    }
    std::vector<int> order;
    for (int i = 0; i < n_old; ++i) { order.push_back(g.index_to_node[i]); for (int v : after[i]) order.push_back(v); }
    for (size_t k = 0; k < order.size(); ++k) { g.index_to_node[k] = order[k]; g.node_to_index[order[k]] = (int)k; }
    // the order must be topological for every edge AND for the quotient by aligned groups (a later fusion may move a
    // path onto an aligned sibling): all members of a block are contiguous
    if ((int)order.size() != g.node_n) g.err = JOB_ERR_TOPO;
    for (int v = 0; v < g.node_n; ++v) {
        for (int k = 0; k < g.out_n[v]; ++k) if (g.node_to_index[v] >= g.node_to_index[g.out_id[g.out_off[v] + k]]) g.err = JOB_ERR_TOPO;
        int lo = g.node_to_index[v], hi = lo;
        for (int k = 0; k < g.aln_n[v]; ++k) { lo = std::min(lo, g.node_to_index[g.aln_id[v * 4 + k]]); hi = std::max(hi, g.node_to_index[g.aln_id[v * 4 + k]]); }
        if (hi - lo != g.aln_n[v]) g.err = JOB_ERR_TOPO;
    }
}

// slot memory as the device has it: 256-byte aligned blocks (slot_plan.h)
struct alignas(256) HtBlock { uint8_t b[256]; };

// same word layout as oracle/ref_harness.c:ref_poa_msa_trace; returns malloc'd words
extern "C" int64_t *hosttest_poa_msa_trace(const HtParams *hp, int n_seq, const int *lens, const uint8_t *flat, int64_t *n_words, int *status) {
    const PoaParams P = poa_params(hp->mat, hp->o1, hp->e1, hp->o2, hp->e2, hp->wb, hp->wf);
    std::vector<const uint8_t *> seqs(n_seq); int64_t sum = 0; int maxl = 0;
    for (int i = 0; i < n_seq; ++i) { seqs[i] = flat + sum; sum += lens[i]; maxl = std::max(maxl, lens[i]); }
    std::vector<int> order(n_seq);
    {   // the product's guide tree (guide_tree.cuh) on the product's scratch layout at its worst case, a block of 64 emulated threads
        GtNeeds need;
        need.add_job(hp->progressive, n_seq, sum, hp->w, 1.0, true);
        const GtLayout Y = plan_gt_scratch(need);
        std::vector<HtBlock> scratch((size_t)Y.slot_bytes / sizeof(HtBlock));
        std::vector<uint64_t> tile(256);       // a small tile: the global-stride passes run too
        int n_keys = 0; double wsv[33]; long long wsi[33];
        GtScratch G = gt_views(Y, scratch.data()->b);
        G.n_keys = &n_keys; G.tile = tile.data(); G.tile_cap = (int)tile.size();
        const GuideTreeParams GP{hp->k, hp->w};
        if (cta_guide_tree(GP, hp->progressive, n_seq, [&](int i) { return seqs[i]; }, lens, order.data(), G, wsv, wsi, 64) != 0) { *status = JOB_ERR_GT_CAP; *n_words = 0; return nullptr; }
    }
    // the product's slot layout for this one job, its planes at the product's worst case (capped at 2^31 ints)
    SlotNeeds need;
    need.add_job(n_seq, sum, maxl, std::min<int64_t>(plane_ints_for_job(P.wb, P.wf, n_seq, sum, maxl, 1.0, true), (int64_t)1 << 31));
    const SlotLayout Y = plan_slot(need);
    std::vector<HtBlock> slot((size_t)Y.slot_bytes / sizeof(HtBlock));
    std::vector<int> planes((size_t)Y.plane_cap);
    Graph g; RowTables rt; DpState d;
    slot_views(Y, slot.data()->b, planes.data(), g, rt, d);
    graph_reset(g, n_seq);
    std::vector<int64_t> w;
    w.push_back(n_seq); w.push_back(0); w.push_back(0);
    for (int i = 0; i < n_seq; ++i) w.push_back(order[i]);
    long long cells = 0;
    for (int a = 0; a < n_seq && !g.err; ++a) {
        const int read = order[a], L = lens[read]; const uint8_t *q = seqs[read];
        const int node_n = g.node_n; int n_rows = 0; d.n_cigar = 0; d.best_score = 0;
        if (a == 0) graph_add_first_sequence(g, q, L, read);
        else {
            long long c = emulate_sweep(g, rt, d, P, q, L);
            if (c < 0) { g.err = c == -2 ? JOB_ERR_BACKTRACK : JOB_ERR_PLANE_CAP; break; }
            cells += c; n_rows = node_n - 1;
            dp_best_cell(g, rt, d, P, L); dp_backtrack(g, rt, d, P, q, L);
        }
        w.push_back(read); w.push_back(L); w.push_back(node_n); w.push_back(d.n_cigar); w.push_back(a == 0 ? 0 : d.best_score); w.push_back(n_rows);
        for (int c = 0; c < d.n_cigar; ++c) w.push_back((int64_t)d.cigar[c]);
        for (int r = 0; r < n_rows; ++r) w.push_back(d.info[r].beg);
        for (int r = 0; r < n_rows; ++r) w.push_back(d.info[r].end);
        if (g.err) break;
        const int n_old = g.node_n;
        if (a > 0) graph_fuse_alignment(g, q, d.cigar, d.n_cigar, read);
        if (g.err) break;
        if (a > 0 && getenv("HOSTTEST_INCREMENTAL_ORDER")) {
            // keep the previous order, splice the new nodes in; then the order independent parts of the sort
            incremental_order(g, q, d.cigar, d.n_cigar, n_old, n_old);
            for (int v = 0; v < g.node_n; ++v) graph_sort_node_edges(g, v);
            graph_bfs_remain(g);
            if (!g.err) graph_build_rows(g, rt);
        } else graph_topo_sort_serial(g, rt);
    }
    *status = g.err;
    int msa_len = 0; std::vector<uint8_t> msa;
    if (!g.err) {
        msa_len = graph_msa_rank(g);
        msa.assign((size_t)n_seq * msa_len, GAP_CODE);
        for (int v = 2; v < g.node_n; ++v) graph_msa_fill_node(g, v, msa.data(), msa_len);
    }
    w[1] = msa_len; w[2] = cells;
    const size_t nb = msa.size(), nw = (nb + 7) / 8, base_w = w.size();
    w.resize(base_w + nw, 0);
    if (nb) memcpy(w.data() + base_w, msa.data(), nb);
    int64_t *out = (int64_t *)malloc(sizeof(int64_t) * w.size());
    memcpy(out, w.data(), sizeof(int64_t) * w.size());
    *n_words = (int64_t)w.size();
    return out;
}

extern "C" void hosttest_free(void *p) { free(p); }

// ---------------------------------------------------------------------------------------------------------
// cPecan mode: the product's block program (cactus_b200/csrc/pecan_cta.cuh) with the T threads of every phase run one
// after the other, on top of the product's host planning (pecan_plan.cpp). The exp / threshold / floor step mirrors
// finish_pairs in pecan.cu. Same output as oracle_pecan_aligned_pairs.
// ---------------------------------------------------------------------------------------------------------
#include <math.h>
#include "../../cactus_b200/csrc/pecan_plan.h"
#include "../../cactus_b200/csrc/pecan_cta.cuh"

struct HtPecanParams { double threshold; int64_t minDiagsBetweenTraceBack, traceBackDiagonals, diagonalExpansion; };

static int g_pecan_threads = 32, g_pecan_ring_w = 0, g_pecan_ring_extra = 0;
extern "C" void hosttest_pecan_set_ring_extra(int e) { g_pecan_ring_extra = e; }
extern "C" void hosttest_pecan_set_threads(int t) { g_pecan_threads = t; }
extern "C" void hosttest_pecan_set_ring_width(int w) { g_pecan_ring_w = w; }

extern "C" int64_t hosttest_pecan_aligned_pairs(const char *csx, int64_t lX, const char *csy, int64_t lY, const int64_t *anchors, int64_t n_anchor,
                                                int ragged_left, int ragged_right, const HtPecanParams *pp, int64_t split_bigger,
                                                int64_t **trip, double **post, int64_t *cells_out) {
    namespace pc = barb200::pecan;
    pc::PlanParams P{pp->threshold, pp->minDiagsBetweenTraceBack, pp->traceBackDiagonals, pp->diagonalExpansion, split_bigger};
    *trip = nullptr; *post = nullptr;
    if (!pc::check_params(P).empty() || !pc::check_anchors(anchors, n_anchor, lX, lY).empty()) return -1;
    std::vector<pc::SubJob> subs;
    pc::split_pair(P, 0, lX, lY, anchors, n_anchor, ragged_left != 0, ragged_right != 0, subs);
    pc::Consts C; pc::fill_constants(C);
    pc::Params dp; dp.log_thr_lo = P.threshold > 0 ? log(P.threshold) - 1e-9 : -INFINITY;
    dp.min_diags = (int)P.min_diags; dp.tb_diags = (int)P.tb_diags; dp.expansion = (int)P.expansion;
    std::vector<int64_t> t; std::vector<double> po;
    int64_t cells = 0;
    for (pc::SubJob &s : subs) {
        if (!pc::plan_subjob(P, s).empty()) return -2;
        cells += s.cells;
        std::vector<uint8_t> sym((size_t)s.lx + s.ly + 1);
        auto code = [](char c) { switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; } };
        for (int k = 0; k < s.lx; ++k) sym[k] = (uint8_t)code(csx[s.x1 + k]);
        for (int k = 0; k < s.ly; ++k) sym[s.lx + k] = (uint8_t)code(csy[s.y1 + k]);
        unsigned capM = 1024; while (capM < (uint64_t)std::max<int64_t>(s.span_cells, 1)) capM <<= 1;
        unsigned capF = 1024; while (capF < 5 * (uint64_t)std::max<int64_t>(s.span_full_cells, 1)) capF <<= 1;
        // ring: modulus RW >= the widest diagonal, the first RWs positions in "shared memory", the rest in the overflow block
        const int RW = std::max(s.max_w, 1) + g_pecan_ring_extra, RWs = g_pecan_ring_w > 0 ? std::min(g_pecan_ring_w, RW) : RW;
        std::vector<double> fm(capM, NAN), ff(capF, NAN), ring(10 * (size_t)RWs, NAN), ring_o(10 * (size_t)(RW - RWs) + 1, NAN), tbuf((size_t)RWs, NAN), tbuf_o((size_t)(RW - RWs) + 1, NAN);
        double total = NAN; int n_out = 0;
        pc::CtaMem cm; cm.ring = ring.data(); cm.ring_o = ring_o.data(); cm.tbuf = tbuf.data(); cm.tbuf_o = tbuf_o.data(); cm.total = &total; cm.n_out = &n_out;
        cm.RW = RW; cm.RWs = RWs; cm.FM = fm.data(); cm.maskM = capM - 1; cm.FF = ff.data(); cm.maskF = capF - 1; cm.T = g_pecan_threads;
        pc::Job J; J.sx_off = 0; J.sy_off = s.lx; J.band_off = 0; J.out_off = 0; J.lx = s.lx; J.ly = s.ly; J.ragged = s.ragged; J.pad_ = 0;
        J.ring_shift = s.ring_center - RWs / 2;
        J.out_cap = (int)std::min<int64_t>(s.cells, (int64_t)s.lx + s.ly + 64);
        std::vector<pc::DiagMeta> meta((size_t)s.lx + s.ly + 2);
        for (int d = 0; d <= s.lx + s.ly + 1; ++d) meta[d] = pc::DiagMeta{d <= s.lx + s.ly ? s.bandL[d] : 0, s.coff[d], s.foff[d], 0};
        std::vector<pc::Pair> out((size_t)std::max(J.out_cap, 1));
        int n = pc::run_job(J, sym.data(), meta.data(), cm, dp, C.v, out.data());
        if (n > J.out_cap) {              // the product's retry: room for every cell
            J.out_cap = (int)s.cells; out.assign((size_t)std::max(J.out_cap, 1), pc::Pair());
            n = pc::run_job(J, sym.data(), meta.data(), cm, dp, C.v, out.data());
            if (n > J.out_cap) return -3;
        }
        // candidates arrive in no particular order within a diagonal (here: scrambled on purpose); restore the order of emission
        out.resize((size_t)n);
        for (int q = 0; q + 1 < n; q += 2) std::swap(out[q], out[q + 1]);
        std::sort(out.begin(), out.end(), [&](const pc::Pair &a, const pc::Pair &b) { return pc::emission_key(s, a.x, a.y) < pc::emission_key(s, b.x, b.y); });
        for (int q = n - 1; q >= 0; --q) {
            double p = exp(out[q].lp);
            if (!(p >= P.threshold)) continue;
            po.push_back(p);
            if (p > 1.0) p = 1.0;
            t.push_back((int64_t)floor(p * 10000000.0)); t.push_back(out[q].x + s.x1); t.push_back(out[q].y + s.y1);
        }
    }
    const int64_t n = (int64_t)po.size();
    *trip = (int64_t *)malloc(sizeof(int64_t) * 3 * (size_t)std::max<int64_t>(n, 1));
    *post = (double *)malloc(sizeof(double) * (size_t)std::max<int64_t>(n, 1));
    if (n) { memcpy(*trip, t.data(), sizeof(int64_t) * 3 * n); memcpy(*post, po.data(), sizeof(double) * n); }
    if (cells_out) *cells_out = cells;
    return n;
}

// ---------------------------------------------------------------------------------------------------------
// group commit (cactus_b200/csrc/group_commit.h): `threads` callers submit `iters` requests each to a fake device that
// squares numbers and takes a moment per batch. Returns the number of wrong answers; *merged = batches wider than one request,
// *batches = batches run, *overlaps = times two batches were inside exec at once (must stay 0).
// ---------------------------------------------------------------------------------------------------------
#include <atomic>
#include <chrono>
#include <thread>
#include "../../cactus_b200/csrc/group_commit.h"

struct HtReq { bool done = false; int rc = 0; int key = 0; std::vector<long long> in, out; };

extern "C" long long hosttest_group_commit_stress(int threads, int iters, long long *merged, long long *batches, long long *overlaps) {
    barb200::GroupCommit<HtReq> gc;
    std::atomic<long long> wrong(0), nmerged(0), nbatches(0), inside(0), noverlap(0);
    auto worker = [&](int tid) {
        for (int it = 0; it < iters; ++it) {
            HtReq r; r.key = (tid + it) % 2;
            for (int k = 0; k < 1 + (tid * 7 + it) % 5; ++k) r.in.push_back(1000LL * tid + it * 10 + k);
            gc.submit(&r, [](const HtReq &a, const HtReq &b) { return a.key == b.key; },
                      [&](std::vector<HtReq *> &batch) {
                          if (inside.fetch_add(1) != 0) ++noverlap;
                          ++nbatches; if (batch.size() > 1) ++nmerged;
                          if (batch.front()->in[0] % 97 == 13) { inside.fetch_sub(1); throw std::bad_alloc(); }     // a failing batch must not wedge the queue
                          for (HtReq *q : batch) if (q->key != batch.front()->key) ++wrong;       // only mergeable requests share a batch
                          std::vector<long long> all;                                               // the "device" works on the concatenation
                          for (HtReq *q : batch) all.insert(all.end(), q->in.begin(), q->in.end());
                          for (long long &v : all) v = v * v;
                          std::this_thread::sleep_for(std::chrono::microseconds(200));
                          size_t o = 0;
                          for (HtReq *q : batch) { q->out.assign(all.begin() + o, all.begin() + o + q->in.size()); o += q->in.size(); }
                          inside.fetch_sub(1);
                      });
            if (r.rc == -2) { if (!r.out.empty()) ++wrong; continue; }          // its batch "ran out of memory": reported, nothing delivered
            if (!r.done || r.out.size() != r.in.size()) { ++wrong; continue; }
            for (size_t k = 0; k < r.in.size(); ++k) if (r.out[k] != r.in[k] * r.in[k]) ++wrong;
        }
    };
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; ++t) ts.emplace_back(worker, t);
    for (auto &t : ts) t.join();
    *merged = nmerged; *batches = nbatches; *overlaps = noverlap;
    return wrong;
}

// ---------------------------------------------------------------------------------------------------------
// batch_merge.h: the plumbing that turns the requests of concurrent callers into one device batch, driven with stand-in
// "device" (cPecan: one triple (lx, ly, n_anchor) per pair). Returns the number
// of callers that got a wrong answer; *merged = batches wider than one request.
// ---------------------------------------------------------------------------------------------------------
#include <string>
#include "../../cactus_b200/csrc/batch_merge.h"

extern "C" long long hosttest_batch_merge_stress(int threads, int iters, long long *merged) {
    barb200::GroupCommit<barb200::PecanRequest> gpec;
    std::atomic<long long> wrong(0), nmerged(0);
    auto pec_impl = [&](const barb200_pecan_params *p, int64_t n, const char *const *sx, const int64_t *lx, const char *const *sy, const int64_t *ly,
                        const int64_t *const *an, const int64_t *na, const uint8_t *rl, const uint8_t *rr, int64_t **trip, int64_t *n_out, double **post,
                        int64_t *cells) -> int {
        for (int64_t i = 0; i < n; ++i) {
            trip[i] = (int64_t *)malloc(3 * sizeof(int64_t));
            trip[i][0] = lx[i] * 1000 + (sx[i] ? sx[i][0] : 0); trip[i][1] = ly[i] + (rl ? rl[i] : 0) * 7 + (rr ? rr[i] : 0) * 11; trip[i][2] = (na ? na[i] : 0) + ((an && an[i]) ? an[i][0] : 0);
            n_out[i] = 1;
            if (post) { post[i] = (double *)malloc(sizeof(double)); post[i][0] = p->threshold + (double)lx[i]; }
            if (cells) cells[i] = lx[i] * ly[i];
        }
        std::this_thread::sleep_for(std::chrono::microseconds(100));
        return 0;
    };
    auto worker = [&](int tid) {
        for (int it = 0; it < iters; ++it) {
            {   // cPecan request: 1..4 pairs, two parameter sets, with / without posteriors and optional arrays
                const int np = 1 + (tid * 3 + it) % 4;
                std::vector<std::string> xs(np), ys(np); std::vector<const char *> sx(np), sy(np); std::vector<int64_t> lx(np), ly(np), na(np), n_out(np, -1), cells(np, -1);
                std::vector<std::vector<int64_t>> an(np); std::vector<const int64_t *> anp(np); std::vector<uint8_t> rl(np), rr(np);
                std::vector<int64_t *> trip(np, nullptr); std::vector<double *> post(np, nullptr);
                for (int i = 0; i < np; ++i) {
                    xs[i] = std::string((size_t)(2 + (tid + i) % 5), (char)('A' + (tid + i) % 20)); ys[i] = std::string((size_t)(1 + (it + i) % 7), 'C');
                    sx[i] = xs[i].c_str(); sy[i] = ys[i].c_str(); lx[i] = (int64_t)xs[i].size(); ly[i] = (int64_t)ys[i].size();
                    na[i] = (tid + it + i) % 2; an[i] = {(int64_t)(tid + i), 0}; anp[i] = na[i] ? an[i].data() : nullptr; rl[i] = (uint8_t)((tid + i) & 1); rr[i] = (uint8_t)((it + i) & 1);
                }
                const bool want_post = (tid + it) % 3 == 0, with_flags = (tid + it) % 5 != 0;
                barb200::PecanRequest r; memset(&r.p, 0, sizeof(r.p)); r.p.min_diags_between_traceback = 1000; r.p.traceback_diagonals = 40;
                r.p.diagonal_expansion = 20; r.p.split_matrix_bigger_than_this = 9000000; r.p.threshold = (tid % 2) ? 0.01 : 0.2;
                r.n = np; r.sx = sx.data(); r.lx = lx.data(); r.sy = sy.data(); r.ly = ly.data(); r.anchors = anp.data(); r.n_anchor = na.data();
                r.ragged_left = with_flags ? rl.data() : nullptr; r.ragged_right = with_flags ? rr.data() : nullptr;
                r.triples_out = trip.data(); r.n_out = n_out.data(); r.posteriors_out = want_post ? post.data() : nullptr; r.cells_out = cells.data();
                gpec.submit(&r, barb200::pecan_can_merge, [&](std::vector<barb200::PecanRequest *> &b) { if (b.size() > 1) ++nmerged; barb200::run_pecan_group(b, pec_impl); });
                bool ok = r.rc == 0;
                for (int i = 0; ok && i < np; ++i) {
                    ok = trip[i] && n_out[i] == 1 && trip[i][0] == lx[i] * 1000 + xs[i][0] && trip[i][1] == ly[i] + (with_flags ? rl[i] * 7 + rr[i] * 11 : 0) &&
                         trip[i][2] == na[i] + (na[i] ? an[i][0] : 0) && cells[i] == lx[i] * ly[i] && (!want_post || (post[i] && post[i][0] == r.p.threshold + (double)lx[i]));
                }
                if (!ok) ++wrong;
                for (int i = 0; i < np; ++i) { free(trip[i]); free(post[i]); }
            }
        }
    };
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; ++t) ts.emplace_back(worker, t);
    for (auto &t : ts) t.join();
    *merged = nmerged;
    return wrong;
}


// ---------------------------------------------------------------------------------------------------------
// one device batch on the CPU: the product's job table and stage order (stage_plan.h), every job computed by
// hosttest_poa_msa_trace in the stage's internal order and its result written at the caller's index. The stand-in device
// (standin_device.cpp) and hosttest_flowers run their batches through it, so they reject what the product rejects.
// ---------------------------------------------------------------------------------------------------------
#include "../../cactus_b200/csrc/stage_plan.h"

int hosttest_device_batch(const HtParams &hp, int threads_per_block, const std::vector<HostJob> &jobs, std::vector<JobResult> &res, std::string &err) {
    res.assign(jobs.size(), JobResult());
    barb200_params p;
    params_default(&p);
    p.wb = hp.wb; p.wf = hp.wf; p.w = hp.w; p.progressive_poa = hp.progressive; p.threads_per_block = threads_per_block;
    JobTable T;
    err = build_table(p, 4, (int64_t)jobs.size(), [&](int64_t j, int64_t, int64_t) { return jobs[j]; }, T);
    if (!err.empty()) return BARB200_EINVAL;
    const StagePlan S = plan_stage_order(T, all_jobs((int64_t)jobs.size()), p, 1.0, false, 1, true);
    for (const int64_t c : S.perm) {
        HtParams q = hp; q.progressive = T.jobs[c].progressive;
        int64_t nw = 0; int status = 0;
        int64_t *w = hosttest_poa_msa_trace(&q, jobs[c].n_seq, jobs[c].lens, jobs[c].seqs, &nw, &status);
        if (status) { free(w); err = "stand-in device: job failed"; return BARB200_EJOB; }
        const int ml = (int)w[1];
        const size_t nb = (size_t)jobs[c].n_seq * ml, nwm = (nb + 7) / 8;
        res[c].msa.assign((const uint8_t *)(w + (nw - (int64_t)nwm)), (const uint8_t *)(w + (nw - (int64_t)nwm)) + nb);
        res[c].msa_len = ml; res[c].cells = w[2];
        free(w);
    }
    return BARB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// end_queue.h + bar_windows.h: the product's end queue (tickets, lane workers, window rounds, trimming, stitching, cross-end
// consistency) driven by application threads, with a stand-in device: every job's MSA comes from the host build of the
// product's graph code above (hosttest_poa_msa_trace). flowers: n_flowers tickets; flat description as in the arguments.
// Returns 0, or a negative code; col_out[e] / msa_out[e] (malloc'd, seq_no x column_no) per end, in submission order.
// ---------------------------------------------------------------------------------------------------------
#include "../../cactus_b200/csrc/end_queue.h"

extern "C" int hosttest_flowers(const HtParams *hp, int n_lanes, int n_threads, int64_t max_jobs, int fail_every, int64_t n_flowers, const int64_t *end_no,
                                const int64_t *end_lengths, const char *strings, const int64_t *string_lens, const int64_t *rei, const int64_t *reri,
                                const int64_t *ov, int64_t window_size, int64_t max_prog_rows, double max_prog_length_diff,
                                int64_t *col_out, uint8_t **msa_out, int64_t *batches_out, int *ticket_rc) {
    std::atomic<long long> calls(0);
    barb200::EndQueue::Exec exec = [&](int, const std::vector<barb200::HostJob> &jobs, std::vector<barb200::JobResult> &res, std::string &err) -> int {
        const long long c = ++calls;
        if (fail_every > 0 && jobs.size() > 2 && c % fail_every == 0) { err = "stand-in device: injected batch failure"; return -2; }
        return hosttest_device_batch(*hp, 0, jobs, res, err);
    };
    barb200::EndQueue q(n_lanes, exec, max_jobs, 1e18);
    // flat -> per-flower pointer tables
    std::vector<int64_t> f_end0(n_flowers + 1, 0);
    for (int64_t f = 0; f < n_flowers; ++f) f_end0[f + 1] = f_end0[f] + end_no[f];
    const int64_t n_ends = f_end0[n_flowers];
    std::vector<int64_t> e_str0(n_ends + 1, 0);
    for (int64_t e = 0; e < n_ends; ++e) e_str0[e + 1] = e_str0[e] + end_lengths[e];
    const int64_t n_str = e_str0[n_ends];
    std::vector<int64_t> s_off(n_str + 1, 0);
    for (int64_t k = 0; k < n_str; ++k) s_off[k + 1] = s_off[k] + string_lens[k];
    std::vector<std::unique_ptr<barb200::Ticket>> tickets(n_flowers);
    std::atomic<int> bad(0);
    auto worker = [&](int tid) {
        // submit every flower of this thread first, then collect them in order (as the shim's bar() does)
        for (int64_t f = tid; f < n_flowers; f += n_threads) {
            std::unique_ptr<barb200::Ticket> t(new barb200::Ticket());
            t->n_ends = end_no[f]; t->window_size = window_size; t->max_prog_rows = max_prog_rows; t->max_prog_length_diff = max_prog_length_diff;
            t->default_progressive = hp->progressive; t->consistent = rei != nullptr;
            t->ends.resize((size_t)end_no[f]);
            for (int64_t e = 0; e < end_no[f]; ++e) {
                const int64_t ge = f_end0[f] + e, K = end_lengths[ge];
                std::vector<char *> sp(K); std::vector<int> sl(K);
                for (int64_t i = 0; i < K; ++i) { sp[i] = (char *)strings + s_off[e_str0[ge] + i]; sl[i] = (int)string_lens[e_str0[ge] + i]; }
                if (!barb200::barwin::end_init(t->ends[e], K, sp.data(), sl.data()).empty()) ++bad;
                if (rei) {
                    t->right_end_indexes.emplace_back(rei + e_str0[ge], rei + e_str0[ge] + K);
                    t->right_end_row_indexes.emplace_back(reri + e_str0[ge], reri + e_str0[ge] + K);
                    t->overlaps.emplace_back(ov + e_str0[ge], ov + e_str0[ge] + K);
                }
            }
            q.submit(t.get());
            tickets[f] = std::move(t);
        }
        for (int64_t f = tid; f < n_flowers; f += n_threads) {
            barb200::Ticket &t = *tickets[f];
            q.wait(&t);
            if (ticket_rc) ticket_rc[f] = t.rc;
            if (t.rc) { for (int64_t e = 0; e < t.n_ends; ++e) { col_out[f_end0[f] + e] = -1; msa_out[f_end0[f] + e] = nullptr; } continue; }
            std::vector<barb200_msa *> ms((size_t)t.n_ends);
            for (int64_t e = 0; e < t.n_ends; ++e) ms[e] = barb200::barwin::end_stitch(t.ends[e]);
            if (t.consistent && !barb200::barwin::consistency_trim(t.n_ends, ms.data(), t.right_end_indexes, t.right_end_row_indexes, t.overlaps)) ++bad;
            for (int64_t e = 0; e < t.n_ends; ++e) {
                col_out[f_end0[f] + e] = ms[e]->column_no; msa_out[f_end0[f] + e] = ms[e]->msa;
                free(ms[e]->seq_lens); free(ms[e]);
            }
        }
    };
    std::vector<std::thread> ts;
    for (int t = 0; t < n_threads; ++t) ts.emplace_back(worker, t);
    for (auto &t : ts) t.join();
    int64_t nb = 0, nj = 0; q.stats(&nb, &nj);
    if (batches_out) *batches_out = nb;
    return bad ? -1 : 0;
}

// ---- the device-memory plan of a stage (slot_plan.h), for a given device size ----
// the slot layout for one job: slot_bytes, the 7 capacities (node_cap, in_pool, out_pool, W, cigar_cap, fc_cap, plane_cap),
// then the 26 offsets in SlotLayout's order
extern "C" void hosttest_slot_layout(int64_t K, int64_t sum, int64_t ml, int64_t plane_ints, int64_t out[34]) {
    SlotNeeds need;
    need.add_job(K, sum, ml, plane_ints);
    const SlotLayout Y = plan_slot(need);
    const int64_t v[34] = {Y.slot_bytes, Y.node_cap, Y.in_pool, Y.out_pool, Y.W, Y.cigar_cap, Y.fc_cap, Y.plane_cap,
                           Y.o_base, Y.o_aln_n, Y.o_aln_id, Y.o_in_off, Y.o_in_n, Y.o_in_cap, Y.o_out_off, Y.o_out_n, Y.o_out_cap,
                           Y.o_in_id, Y.o_in_w, Y.o_out_id, Y.o_out_w, Y.o_out_rid,
                           Y.o_index_to_node, Y.o_node_to_index, Y.o_remain, Y.o_msa_rank, Y.o_tmp0, Y.o_tmp1,
                           Y.o_row_rec, Y.o_pre_row, Y.o_row_off, Y.o_row_info, Y.o_cigar, Y.o_fc};
    memcpy(out, v, sizeof(v));
}
// the guide-tree scratch for one job: slot_bytes, key_cap, base_cap, seq_cap, then the 5 offsets in GtLayout's order
extern "C" void hosttest_gt_layout(int progressive, int64_t K, int64_t sum, int w, double grow, int worst_case, int64_t out[9]) {
    GtNeeds need;
    need.add_job(progressive, K, sum, w, grow, worst_case != 0);
    const GtLayout Y = plan_gt_scratch(need);
    const int64_t v[9] = {Y.slot_bytes, Y.key_cap, Y.base_cap, Y.seq_cap, Y.o_keys, Y.o_gx, Y.o_hit, Y.o_jac, Y.o_score};
    memcpy(out, v, sizeof(v));
}
extern "C" int64_t hosttest_plane_ints_for_job(int wb, double wf, int64_t K, int64_t sum, int64_t ml, double grow, int worst_case) {
    return barb200::plane_ints_for_job(wb, wf, K, sum, ml, grow, worst_case != 0);
}
extern "C" double hosttest_lane_budget_bytes(double free_b, double total_b, double arena_b, double block_b, double frac, int shared, int lanes) {
    return barb200::lane_budget_bytes(free_b, total_b, arena_b, block_b, frac, shared != 0, lanes);
}
extern "C" double hosttest_retry_plane_scale(double budget, double fixed_bytes, double plane_bytes) {
    return barb200::retry_plane_scale(budget, fixed_bytes, plane_bytes);
}

// ---- the plan of a stage (stage_plan.h) ----
static int plan_error(const std::string &e, int rc, char *err, int err_len) { snprintf(err, err_len, "%s", e.c_str()); return rc; }

// A stage of n jobs (caller order; lengths and bases back to back) under Cactus' band and `threads_per_block`, sized for (grow,
// worst_case); with per_sm > 0 also fitted to per_sm CTAs per SM of every class on sm_count SMs within `budget` bytes. Out: cost[n]
// in caller order; perm, msa_off, msa_stride [n] in internal order; buckets[6 x 6] = threads, job_base, n_jobs, slots, plane ints
// per slot, slot bytes. Returns the number of buckets, or the BARB200_* code of a rejection with its message in err.
extern "C" int hosttest_stage_plan(int64_t n, const int *n_seq, const int *lens, const uint8_t *seqs, int threads_per_block, double grow, int worst_case,
                                   int per_sm, int sm_count, double budget, double *cost, int64_t *perm, int64_t *msa_off, int64_t *msa_stride,
                                   int64_t *buckets, char *err, int err_len) {
    barb200_params p;
    params_default(&p);
    p.threads_per_block = threads_per_block;
    JobTable T;
    std::string e = table_of_arrays(p, 4, n, n_seq, lens, seqs, nullptr, T);
    if (!e.empty()) return plan_error(e, BARB200_EINVAL, err, err_len);
    StagePlan S = plan_stage_order(T, all_jobs(n), p, grow, worst_case != 0, sm_count, true);
    if (per_sm > 0 && !(e = fit_stage(S, std::vector<int>(S.buckets.size(), per_sm), sm_count, budget)).empty()) return plan_error(e, BARB200_ENOMEM, err, err_len);
    for (int64_t j = 0; j < n; ++j) { cost[j] = T.jobs[j].cost; perm[j] = S.perm[j]; msa_off[j] = S.desc[j].msa_off; msa_stride[j] = S.desc[j].msa_stride; }
    for (size_t b = 0; b < S.buckets.size(); ++b) {
        const PlanBucket &B = S.buckets[b];
        const int64_t v[6] = {B.T, B.job_base, B.n_jobs, B.slots, B.lay.plane_cap, B.lay.slot_bytes};
        memcpy(buckets + 6 * b, v, sizeof(v));
    }
    return (int)S.buckets.size();
}
// The capacity retry after a round of a stage over the caller's jobs perm[n], sized for (grow, worst_case) with plane_cap ints of
// planes per slot, whose jobs ended with status[n]: 0 with redo[*n_redo] and the next (grow, worst_case), or BARB200_EJOB and err.
extern "C" int hosttest_retry_round(int64_t n, const int *status, const int64_t *perm, double grow, int worst_case, int64_t plane_cap, int64_t *redo,
                                    int64_t *n_redo, double *next_grow, int *next_worst, char *err, int err_len) {
    StagePlan S;
    S.grow = grow; S.worst_case = worst_case != 0; S.perm.assign(perm, perm + n);
    S.buckets.resize(1); S.buckets[0].lay.plane_cap = plane_cap;
    RetryRound next;
    const std::string e = retry_round(S, std::vector<int>(status, status + n), next);
    if (!e.empty()) return plan_error(e, BARB200_EJOB, err, err_len);
    *n_redo = (int64_t)next.jobs.size(); std::copy(next.jobs.begin(), next.jobs.end(), redo);
    *next_grow = next.grow; *next_worst = next.worst_case;
    return 0;
}
// where the device batches of n jobs of sum_len[n] bases end; returns their number
extern "C" int64_t hosttest_chunk_ends(int64_t n, const int64_t *sum_len, int64_t *ends) {
    JobTable T;
    T.jobs.resize(n);
    for (int64_t j = 0; j < n; ++j) T.jobs[j].sum_len = sum_len[j];
    const std::vector<size_t> e = chunk_ends(T, all_jobs(n));
    std::copy(e.begin(), e.end(), ends);
    return (int64_t)e.size();
}
// n jobs of cost[n] dealt over ndev devices: counts[ndev] and every device's share back to back in jobs[n]
extern "C" void hosttest_deal_jobs(int64_t n, const double *cost, int ndev, int64_t *counts, int64_t *jobs) {
    JobTable T;
    T.jobs.resize(n);
    for (int64_t j = 0; j < n; ++j) T.jobs[j].cost = cost[j];
    for (const std::vector<int64_t> &s : deal_jobs(T, ndev)) { *counts++ = (int64_t)s.size(); jobs = std::copy(s.begin(), s.end(), jobs); }
}
