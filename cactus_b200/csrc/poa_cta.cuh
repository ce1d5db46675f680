// poa_cta.cuh -- CTA-cooperative forms of the graph phases between two DP sweeps (device only).
//
// The reference performs these steps serially per added sequence (abPOA src/abpoa_graph.c). On the device a
// single thread walking global memory costs ~1 us per dependent step, which would dwarf the DP sweep, so each
// step is restated in the form that exposes its parallelism while producing the SAME graph:
//   * first sequence / fusing an alignment (abpoa_graph.c:573-593, 689-774): a path visits every node at most
//     once and never two nodes of one aligned group, so the per-base updates of one fusion touch disjoint edge lists
//     and aligned groups; only the ids of new nodes are order dependent (query order) -> one prefix sum;
//   * topological order (abpoa_graph.c:221-266): inherently one dependent step per node; run by one thread on a
//     compact copy of the out-edge lists in SHARED memory (~10x lower latency per step) while the other warps
//     sort the edge lists in global memory (abpoa_graph.c:192-219);
//   * max_remain (abpoa_graph.c:268-309): remain[v] = remain[heaviest out neighbour] + 1 is a list ranking
//     -> pointer jumping, log2(n) parallel rounds;
//   * row tables: prefix sum over in-degrees, then one row per thread.
#pragma once
#include <cuda_runtime.h>
#include "poa_graph.cuh"
#include "graph_phases.cuh"

namespace barb200 {

// ---- edge lists with atomic pool allocation (same lists as graph_add_edge; chunk placement in the pool differs) ----
__device__ __forceinline__ bool grow_in_par(Graph &g, int t) {
    if (g.in_n[t] < g.in_cap[t]) return true;
    const int ncap = g.in_cap[t] ? g.in_cap[t] * 2 : 2;
    const int noff = atomicAdd(&g.in_used, ncap);
    if (noff + ncap > g.in_pool) { g.err = JOB_ERR_EDGE_CAP; return false; }
    for (int i = 0; i < g.in_n[t]; ++i) { g.in_id[noff + i] = g.in_id[g.in_off[t] + i]; g.in_w[noff + i] = g.in_w[g.in_off[t] + i]; }
    g.in_off[t] = noff; g.in_cap[t] = ncap;
    return true;
}
__device__ __forceinline__ bool grow_out_par(Graph &g, int f) {
    if (g.out_n[f] < g.out_cap[f]) return true;
    const int ncap = g.out_cap[f] ? g.out_cap[f] * 2 : 2;
    const int noff = atomicAdd(&g.out_used, ncap);
    if (noff + ncap > g.out_pool) { g.err = JOB_ERR_EDGE_CAP; return false; }
    const int W = g.W;
    for (int i = 0; i < g.out_n[f]; ++i) {
        g.out_id[noff + i] = g.out_id[g.out_off[f] + i]; g.out_w[noff + i] = g.out_w[g.out_off[f] + i];
        for (int w = 0; w < W; ++w) g.out_rid[(int64_t)(noff + i) * W + w] = g.out_rid[(int64_t)(g.out_off[f] + i) * W + w];
    }
    for (int i = g.out_n[f]; i < ncap; ++i) for (int w = 0; w < W; ++w) g.out_rid[(int64_t)(noff + i) * W + w] = 0;
    g.out_off[f] = noff; g.out_cap[f] = ncap;
    return true;
}
// abpoa_add_graph_edge (abpoa_graph.c:480-556) for concurrent callers that own `from`'s out list and `to`'s in list
__device__ __forceinline__ void graph_add_edge_par(Graph &g, int from, int to, int check_edge, int read_id) {
    int out_i = -1;
    if (check_edge) {
        const int io = g.in_off[to], in = g.in_n[to];
        for (int i = 0; i < in; ++i) if (g.in_id[io + i] == from) { g.in_w[io + i] += 1; break; }
        const int oo = g.out_off[from], on = g.out_n[from];
        for (int i = 0; i < on; ++i) if (g.out_id[oo + i] == to) { g.out_w[oo + i] += 1; out_i = i; break; }
    }
    if (out_i < 0) {
        if (!grow_in_par(g, to) || !grow_out_par(g, from)) return;
        const int ip = g.in_off[to] + g.in_n[to]; g.in_id[ip] = from; g.in_w[ip] = 1; g.in_n[to]++;
        out_i = g.out_n[from];
        const int op = g.out_off[from] + out_i; g.out_id[op] = to; g.out_w[op] = 1; g.out_n[from]++;
    }
    g.out_rid[(int64_t)(g.out_off[from] + out_i) * g.W + (read_id >> 6)] |= 1ULL << (read_id & 63);
}

// abpoa_add_graph_sequence (abpoa_graph.c:573-593) on an empty graph: SRC -> b0 -> ... -> SINK. All threads.
__device__ void cta_add_first_sequence(Graph &g, const uint8_t *seq, int len, int read_id) {
    const int tid = threadIdx.x, T = blockDim.x, W = g.W;
    if (len + 2 > g.node_cap) { if (tid == 0) g.err = JOB_ERR_NODE_CAP; __syncthreads(); return; }
    if (2 * (len + 1) > g.in_pool || 2 * (len + 1) > g.out_pool) { if (tid == 0) g.err = JOB_ERR_EDGE_CAP; __syncthreads(); return; }
    const int rw = read_id >> 6; const uint64_t rb = 1ULL << (read_id & 63);
    // in list of node 2+i: chunk [2i, 2i+2); out list of node 2+i: chunk [2(i+1), 2(i+1)+2); SRC out: [0,2); SINK in: [2len, 2len+2)
    for (int i = tid; i <= len; i += T) {
        const int to = i < len ? 2 + i : SINK_ID, from = i == 0 ? SRC_ID : 1 + i;
        g.in_off[to] = 2 * i; g.in_n[to] = 1; g.in_cap[to] = 2; g.in_id[2 * i] = from; g.in_w[2 * i] = 1;
        g.out_off[from] = 2 * i; g.out_n[from] = 1; g.out_cap[from] = 2; g.out_id[2 * i] = to; g.out_w[2 * i] = 1;
        for (int w = 0; w < W; ++w) { g.out_rid[(int64_t)(2 * i) * W + w] = w == rw ? rb : 0; g.out_rid[(int64_t)(2 * i + 1) * W + w] = 0; }
        if (i < len) { g.base[to] = seq[i]; g.aln_n[to] = 0; }
        // topological order of the chain: SRC, 2, 3, ..., len+1, SINK
        g.index_to_node[i + 1] = to; g.node_to_index[to] = i + 1;
    }
    if (tid == 0) { g.index_to_node[0] = SRC_ID; g.node_to_index[SRC_ID] = 0; }
    if (tid == 0) { g.node_n = len + 2; g.in_used = 2 * (len + 1); g.out_used = 2 * (len + 1); }
    __syncthreads();
}

// abpoa_add_subgraph_alignment(SRC, SINK, inc_both_ends = 1), abpoa_graph.c:689-774. All threads.
// Scratch: g.tmp0[q] = node that query base q ends up on, g.tmp1[q] = 1 if that node is new. ws: >= 32 ints shared.
// scr / scr_bytes: dynamic shared memory for the order splice (graph_phases.cuh), unused by the caller meanwhile.
__device__ void cta_fuse_alignment(Graph &g, const uint8_t *seq, int L, const uint64_t *cigar, int n_cigar, int read_id, int *ws,
                                   unsigned char *scr, int scr_bytes) {
    const int tid = threadIdx.x, T = blockDim.x;
    if (n_cigar == 0) return;
    int *node_of = g.tmp0, *is_new = g.tmp1;
    // (1) classify every cigar entry; entries know their query positions (abpoa_align.h:58-78)
    for (int c = tid; c < n_cigar; c += T) {
        const uint64_t cg = cigar[c];
        const int op = (int)(cg & 0xf);
        if (op == CMATCH) {
            const int node_id = (int)((cg >> 34) & 0x3fffffff), q = (int)((cg >> 4) & 0x3fffffff);
            const uint8_t b = seq[q];
            if (g.base[node_id] == b) { node_of[q] = node_id; is_new[q] = 0; }
            else {
                const int a = graph_aligned_with_base(g, node_id, b);
                if (a != -1) { node_of[q] = a; is_new[q] = 0; } else { node_of[q] = -1 - node_id; is_new[q] = 1; }   // new node aligned to node_id
            }
        } else if (op == CINS) {
            const int qe = (int)((cg >> 34) & 0x3fffffff), len = (int)((cg >> 4) & 0x3fffffff);
            for (int q = qe - len + 1; q <= qe; ++q) { node_of[q] = INT32_MIN; is_new[q] = 1; }                          // plain new node
        }
    }
    __syncthreads();
    // (2) ids of the new nodes in query order. is_new becomes the exclusive prefix count; keep the flag in node_of's sign
    const int first_new = g.node_n;            // (read before the scan's barriers: thread 0 moves node_n below)
    const int n_new = cta_excl_scan(is_new, L, ws);
    if (first_new + n_new > g.node_cap) { if (tid == 0) g.err = JOB_ERR_NODE_CAP; __syncthreads(); return; }
    // (3) create the new nodes (+ aligned-group links for mismatch columns)
    for (int q = tid; q < L; q += T) {
        const int m = node_of[q];
        if (m >= 0) { is_new[q] = 0; continue; }
        const int nid = first_new + is_new[q];
        g.base[nid] = seq[q]; g.aln_n[nid] = 0;
        g.in_off[nid] = 0; g.in_n[nid] = 0; g.in_cap[nid] = 0; g.out_off[nid] = 0; g.out_n[nid] = 0; g.out_cap[nid] = 0;
        if (m != INT32_MIN) graph_add_aligned(g, -1 - m, nid);
        node_of[q] = nid; is_new[q] = 1;
    }
    if (tid == 0) g.node_n = first_new + n_new;
    __syncthreads();
    if (g.err) return;
    // (3b) topological order WITHOUT re-running abPOA's BFS (abpoa_graph.c:221-266): the DP, the traceback and the MSA
    // do not depend on which topological order the rows are swept in (bands, scores and tie-breaks are per node / per
    // in-edge order; tests/test_host_graph_code.py pins this against the reference), so the previous order is kept for
    // the old nodes and the new ones are spliced in: a new node aligned to x goes to the end of x's block of aligned
    // nodes (blocks stay contiguous, so the order stays topological for the quotient by aligned groups, which later
    // fusions rely on when they move a path onto an aligned sibling), an inserted new node opens a block right after
    // the block of the previous path node. Anchors are non-decreasing along the path, so the new node with rank m
    // (in query order) and anchor A lands at A + 1 + m, and old index i moves up by the number of anchors < i.
    // In the shared-memory scratch where it fits (graph_phases.cuh: splice_order_smem), else on global scratch arrays.
    if (splice_smem_fits(L, first_new, first_new + n_new, scr_bytes)) splice_order_smem(g, node_of, L, first_new, n_new, scr, ws, T);
    else {
        int *anc = g.remain, *cnt = g.msa_rank, *new_i2n = g.tmp1;
        const int n_old = first_new;
        for (int q = tid; q < L; q += T) {
            const int v = node_of[q];
            int e = v < first_new ? g.node_to_index[v] : -1;
            for (int k = 0; k < g.aln_n[v]; ++k) { const int a = g.aln_id[v * 4 + k]; if (a < first_new) e = max(e, g.node_to_index[a]); }
            anc[q] = e;
        }
        for (int i = tid; i < n_old; i += T) cnt[i] = 0;
        __syncthreads();
        cta_incl_max_scan(anc, L, ws);
        for (int q = tid; q < L; q += T) if (node_of[q] >= first_new) atomicAdd(&cnt[max(anc[q], 0)], 1);
        __syncthreads();
        cta_excl_scan(cnt, n_old, ws);                                   // cnt[i] = number of new nodes anchored before old index i
        for (int i = tid; i < n_old; i += T) new_i2n[i + cnt[i]] = g.index_to_node[i];
        for (int q = tid; q < L; q += T) { const int v = node_of[q]; if (v >= first_new) new_i2n[max(anc[q], 0) + 1 + (v - first_new)] = v; }
        __syncthreads();
        for (int k = tid; k < first_new + n_new; k += T) { const int v = new_i2n[k]; g.index_to_node[k] = v; g.node_to_index[v] = k; }
        __syncthreads();
    }
    // (4) the L+1 edges of the path; check_edge = neither end is new (abpoa_graph.c:731-766)
    for (int q = tid; q <= L; q += T) {
        const int from = q == 0 ? SRC_ID : node_of[q - 1], to = q == L ? SINK_ID : node_of[q];
        const int fresh = (q > 0 && from >= first_new) || (q < L && to >= first_new);
        graph_add_edge_par(g, from, to, fresh ? 0 : 1, read_id);
    }
    __syncthreads();
}


// ---- traceback (simd_abpoa_cg_backtrack, abpoa_align_simd.c:309-458) by ONE WARP -------------------------------
// The walk is a chain of dependent lookups in planes that live in HBM (~1 us per lookup while the other CTAs sweep).
//  * Most of it is runs of MATCH ops along first predecessors, and in the ALL state the M test has priority over everything
//    else (:319-336), so a run can be verified for 31 cells at once: lane k takes the cell (c_k, j-k) on the
//    first-predecessor chain c_0 = i, c_{k+1} = first pred of c_k, all lanes load their H in parallel, lane k tests
//    H[c_{k+1}][j-k-1] + s == H[c_k][j-k], and the leading run of hits is emitted as MATCH ops in one go. The rows 32 further
//    down the chain guess are prefetched into L2 meanwhile.
//  * Wherever the run stops (gap, other predecessor, band edge) warp_backtrack_step applies the general rule once, the lanes
//    probing the predecessors side by side.
// The result is the serial walk's cigar (dp_backtrack, poa_graph.cuh), entry for entry.
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// One iteration of the reference's loop (:319-450; serial form: backtrack_step) by the 32 lanes of a warp, uniformly.
// Insertions are taken whole. The sweep does not store F1 / F2, and the walk does not need them: with
// F[j] = max_t H[i][j-t] - oe - (t-1) e (:1060-1075) and H[i][j] >= F[j],
//   H[i][j] == F1[j]  <=>  some t >= 1 has H[i][j-t] == H[i][j] + oe1 + (t-1) e1,
// the smallest such t is where the reference's walk leaves the F1 state (it tests "open" before "extend" at every column,
// :401-415), i.e. the length of the insertion, and because H[i][j] >= F2[j] bounds H[i][j-t] <= H[i][j] + oe2 + (t-1) e2 the F1
// equation has no solution beyond t1_max = (oe2 - oe1) / (e1 - e2) + 1 columns (27 with Cactus' 400/30, 1200/1). F2 is
// scanned leftwards until it is found (its insertion length) or the band ends (no op explains the cell: -1, as :448).
// States with F always carry M here (ALL, or M|F after a deletion), since an insertion is never left half walked.
__device__ int warp_backtrack_step(const RowTables &rt, const DpState &d, const PoaParams &P, const int *smat8, const uint8_t *q,
                                   int &i, int &j, int &cur_op, int &len) {
    const unsigned FULLM = 0xffffffffu;
    const int lane = threadIdx.x & 31, inf = P.inf_min, e1 = P.e1, e2 = P.e2, oe1 = P.o1 + P.e1, oe2 = P.o2 + P.e2;
    len = 1;
    const RowRec rc = rt.rec[i];
    const RowInfo ri = d.info[i];
    const int *rowi = d.planes + d.row_off[i];
    const int npre = rc.base_npre >> 8;
    const int s = smat8[8 * (rc.base_npre & 0xff) + q[j - 1]];
    int hij = inf; unsigned cij = (unsigned)E_NEG16 | (unsigned)E_NEG16 << 16;
    if (j >= ri.beg && j <= ri.end) { hij = __ldcg(rowi + plane_index(ri.beg, ri.end, 0, j)); cij = (unsigned)__ldcg(rowi + plane_index(ri.beg, ri.end, 1, j)); }
    // the first 32 columns left of j in row i (for the F tests), in flight together with the predecessor probes
    int hk0 = inf;
    if ((cur_op & OP_F) && j - 1 - lane >= ri.beg && j - 1 - lane <= ri.end) hk0 = __ldcg(rowi + plane_index(ri.beg, ri.end, 0, j - 1 - lane));
    // the lane's predecessor of a chunk of 32: row, H[j-1], H[j], E1[j], E2[j]
    int pi = -1, pm = inf, ph = inf, pe1 = inf, pe2 = inf; bool m_in = false, e_in = false;
    auto probe = [&](int kb) {
        const int k = kb + lane;
        pi = -1; m_in = false; e_in = false;
        if (k >= npre) return;
        pi = k == 0 ? rc.pre0 : rt.pre_row[rc.pre_off + k];
        const RowInfo pin = d.info[pi];
        const int *prow = d.planes + d.row_off[pi];
        m_in = (cur_op & OP_M) && j - 1 >= pin.beg && j - 1 <= pin.end;
        e_in = (cur_op & OP_E) && j >= pin.beg && j <= pin.end;
        if (m_in) pm = __ldcg(prow + plane_index(pin.beg, pin.end, 0, j - 1));
        if (e_in) {
            ph = __ldcg(prow + plane_index(pin.beg, pin.end, 0, j));
            const unsigned code = (unsigned)__ldcg(prow + plane_index(pin.beg, pin.end, 1, j));
            pe1 = e_decode(ph, (int)(code & 0xffffu), inf); pe2 = e_decode(ph, (int)(code >> 16), inf);
        }
    };
    if (cur_op & OP_M) {                                                       // :319-336
        for (int kb = 0; kb < npre; kb += 32) {
            probe(kb);
            const unsigned hit = __ballot_sync(FULLM, m_in && pm + s == hij);
            if (hit) { i = __shfl_sync(FULLM, pi, __ffs(hit) - 1); --j; cur_op = OP_ALL; return CMATCH; }
        }
    }
    if (cur_op & OP_E) {                                                       // :337-392, per predecessor E1 then E2
        const int own_e1 = e_decode(hij, (int)(cij & 0xffffu), inf), own_e2 = e_decode(hij, (int)(cij >> 16), inf);
        for (int kb = 0; kb < npre; kb += 32) {
            if (npre > 32 || !(cur_op & OP_M)) probe(kb);                      // (else the M loop's single probe is still in the registers)
            const bool ok1 = e_in && (cur_op & OP_E1) && ((cur_op & OP_M) ? hij == pe1 : own_e1 == pe1 - e1);
            const bool ok2 = e_in && (cur_op & OP_E2) && ((cur_op & OP_M) ? hij == pe2 : own_e2 == pe2 - e2);
            const unsigned hit = __ballot_sync(FULLM, ok1 || ok2);
            if (hit) {
                const int f = __ffs(hit) - 1;
                const int nop = ok1 ? ((ph - oe1 == pe1) ? (OP_M | OP_F) : OP_E1) : ((ph - oe2 == pe2) ? (OP_M | OP_F) : OP_E2);
                cur_op = __shfl_sync(FULLM, nop, f); i = __shfl_sync(FULLM, pi, f);
                return CDEL;
            }
        }
    }
    if (cur_op & OP_F) {                                                       // :393-428
        if (!(cur_op & OP_M)) return -1;                                       // (never the case, see above)
        const int avail = j - ri.beg;                                          // columns of the row left of j
        int t1_max;
        if (e1 > e2) t1_max = oe2 >= oe1 ? (oe2 - oe1) / (e1 - e2) + 1 : 0;
        else t1_max = (e1 < e2 || oe1 <= oe2) ? avail : 0;
        if (t1_max > avail) t1_max = avail;
        for (int which = 0; which < 2; ++which) {
            if (!(cur_op & (which ? OP_F2 : OP_F1))) continue;
            const int oe = which ? oe2 : oe1, e = which ? e2 : e1, tmax = which ? avail : t1_max;
            for (int t0 = 0; t0 < tmax; t0 += 32) {
                const int t = t0 + lane + 1;
                int hk = hk0;
                if (t0 > 0) { hk = inf; if (t <= avail) hk = __ldcg(rowi + plane_index(ri.beg, ri.end, 0, j - t)); }
                const unsigned hit = __ballot_sync(FULLM, t <= tmax && hk == hij + oe + (t - 1) * e);
                if (hit) { len = __ffs(hit); len += t0; j -= len; cur_op = OP_M | OP_E; return CINS; }
            }
        }
    }
    return -1;
}

__device__ void warp_backtrack(Graph &g, const RowTables &rt, DpState &d, const PoaParams &P, const int *smat8, const uint8_t *q, int L) {
    const unsigned FULLM = 0xffffffffu;
    const int lane = threadIdx.x & 31, inf = P.inf_min;
    if (lane == 0) { dp_best_cell(g, rt, d, P, L); d.fc_row = -1; d.fc_hi = -1; }
    __syncwarp();
    int i = d.best_i, j = d.best_j, cur_op = OP_ALL, nc = 0, last_op = -1;
    uint64_t *cg = d.cigar; const int cap = d.cigar_cap;
    int fail = 0;
    auto push = [&](int op, int len, int node_id, int query_id) {               // abpoa_push_cigar, abpoa_align.h:58-78
        if (nc == 0 || op != CINS || last_op != CINS) {
            if (nc >= cap) { fail = JOB_ERR_CIGAR_CAP; return; }
            if (lane == 0) {
                const uint64_t n_id = (uint64_t)(int64_t)node_id, q_id = (uint64_t)(int64_t)query_id, l = (uint64_t)len;
                cg[nc] = op == CMATCH ? (n_id << 34 | q_id << 4 | (uint64_t)op) : op == CINS ? (q_id << 34 | l << 4 | (uint64_t)op) : (n_id << 34 | l << 4 | (uint64_t)op);
            }
            ++nc;
        } else if (lane == 0) cg[nc - 1] += (uint64_t)len << 4;
        last_op = op;
    };
    if (j < L) push(CINS, L - j, -1, L - 1);
#ifdef BT_PROFILE
    long long pf_t0 = clock64(), pf_run_t = 0, pf_step_t = 0; int pf_iters = 0, pf_runs = 0, pf_cells = 0, pf_steps = 0, pf_ins = 0;
#endif
    while (i > 0 && j > 0 && !fail) {
        int run = 0;
#ifdef BT_PROFILE
        long long pf_a = clock64();
#endif
        if (cur_op == OP_ALL) {
            // rows of the first-predecessor chain: start from the linear guess i-k and re-base after each jump; every table entry
            // of a row is fetched in the same round trip
            int c = i - lane, pre = -1, base = 0, n_ok = 0, node = 0;
            RowInfo ric; ric.beg = 0; ric.end = -1; ric.left = 0; ric.right = 0;
            int64_t ro = 0;
            bool fresh = true;
#pragma unroll 1
            for (int it = 0; it < 4; ++it) {
                if (fresh) {
                    pre = -1;
                    if (c > 0) { const RowRec rc = rt.rec[c]; base = rc.base_npre & 0xff; pre = (rc.base_npre >> 8) ? rc.pre0 : -1; node = g.index_to_node[c]; }
                    if (c >= 0) { ric = d.info[c]; ro = d.row_off[c]; }
                }
                const int nxt = __shfl_down_sync(FULLM, c, 1);
                const bool ok = lane < 31 && pre >= 0 && pre == nxt;
                n_ok = __ffs(~__ballot_sync(FULLM, ok)) - 1;               // lanes 0..n_ok hold true chain rows
                if (n_ok >= 31 || it == 3) break;
                const int pre_b = __shfl_sync(FULLM, pre, n_ok);
                if (pre_b < 0) break;                                        // the chain ends at lane n_ok
                fresh = lane > n_ok;
                if (fresh) c = pre_b - (lane - n_ok - 1);
            }
            const int jj = j - lane;
            int hv = inf, inb = 0;
            if (lane <= n_ok && c >= 0 && jj >= 0) {
                inb = jj >= ric.beg && jj <= ric.end;
                if (inb) hv = __ldcg(d.planes + ro + plane_index(ric.beg, ric.end, 0, jj));
            }
            // the same diagonal 32 rows on: table entries now (they are back long before the end of the iteration), the plane line
            // from there
            const int cl = c - 32, jl = jj - 32;
            RowInfo ril; ril.beg = 0; ril.end = -1; ril.left = 0; ril.right = 0;
            int64_t rol = 0;
            if (cl >= 0 && jl >= 0) { ril = d.info[cl]; rol = d.row_off[cl]; prefetch_l2(rt.rec + cl); prefetch_l2(g.index_to_node + cl); }
            const int h_next = __shfl_down_sync(FULLM, hv, 1), inb_next = __shfl_down_sync(FULLM, inb, 1);
            bool hit = false;
            if (lane < n_ok && c > 0 && jj >= 1 && inb_next) hit = h_next + smat8[8 * base + q[jj - 1]] == hv;
            run = __ffs(~__ballot_sync(FULLM, hit)) - 1;
            if (run > 0) {
                if (nc + run > cap) fail = JOB_ERR_CIGAR_CAP;
                else {
                    if (lane < run) cg[nc + lane] = (uint64_t)node << 34 | (uint64_t)(jj - 1) << 4 | (uint64_t)CMATCH;
                    nc += run; last_op = CMATCH;
                    i = __shfl_sync(FULLM, c, run); j -= run;               // cur_op stays ALL
                }
            }
            if (cl >= 0 && jl >= 0 && jl <= ril.end) prefetch_l2(d.planes + rol + plane_index(ril.beg, ril.end, 0, jl < ril.beg ? ril.beg : jl));
        }
#ifdef BT_PROFILE
        long long pf_b = clock64(); if (cur_op == OP_ALL) { pf_run_t += pf_b - pf_a; ++pf_iters; if (run) { ++pf_runs; pf_cells += run; } }
#endif
        if (run == 0 && !fail) {
            const int id = g.index_to_node[i], jq = j - 1;
            int len = 1;
            const int op = warp_backtrack_step(rt, d, P, smat8, q, i, j, cur_op, len);
            if (op < 0) fail = JOB_ERR_BACKTRACK; else push(op, len, id, jq);
#ifdef BT_PROFILE
            pf_step_t += clock64() - pf_b; ++pf_steps; if (op == CINS) ++pf_ins;
#endif
        }
    }
#ifdef BT_PROFILE
    if (lane == 0 && blockIdx.x == 0) printf("bt L=%d total=%lld run_t=%lld step_t=%lld iters=%d runs=%d cells=%d steps=%d ins=%d\n", L, clock64() - pf_t0, pf_run_t, pf_step_t, pf_iters, pf_runs, pf_cells, pf_steps, pf_ins);
#endif
    if (!fail && j > 0) push(CINS, j, -1, j - 1);
    if (fail) { if (lane == 0) g.err = fail; return; }
    if (lane == 0) d.n_cigar = nc;
    __syncwarp();
    for (int a = lane; a < nc >> 1; a += 32) { const uint64_t t = cg[a]; cg[a] = cg[nc - 1 - a]; cg[nc - 1 - a] = t; }
    __syncwarp();
}

// ---- topological sort (abpoa_topological_sort, abpoa_graph.c:322-357) --------------------------------------
// Shared-memory copy of what abpoa_BFS_set_node_index walks: CSR of out edges (pre-sort order), in-degrees, sizes of
// the aligned groups, the FIFO (= index_to_node).
struct BfsScratch { uint32_t *optr; uint16_t *odst, *queue, *indeg; uint8_t *alnn; };

__device__ __forceinline__ size_t bfs_scratch_bytes(int n, int E) { return (size_t)4 * (n + 1) + (size_t)2 * E + 4 * (size_t)n + n + 16; }

__device__ void bfs_index_smem(Graph &g, const BfsScratch &B) {      // one thread
    const int n = g.node_n;
    int head = 0, tail = 0;
    B.queue[tail++] = SRC_ID;
    while (head < tail) {
        const int cur = B.queue[head++];
        if (cur == SINK_ID) {
            if (head != n) g.err = JOB_ERR_TOPO;       // every node must have been numbered before SINK
            return;
        }
        const uint32_t o0 = B.optr[cur], o1 = B.optr[cur + 1];
        for (uint32_t i = o0; i < o1; ++i) {
            const int o = B.odst[i];
            const int left = (int)B.indeg[o] - 1; B.indeg[o] = (uint16_t)left;
            if (left == 0) {
                const int an = B.alnn[o];
                bool ok = true;
                for (int j = 0; j < an; ++j) if (B.indeg[g.aln_id[o * 4 + j]] != 0) { ok = false; break; }
                if (!ok) continue;
                B.queue[tail++] = (uint16_t)o;
                for (int j = 0; j < an; ++j) B.queue[tail++] = (uint16_t)g.aln_id[o * 4 + j];
            }
        }
    }
    g.err = JOB_ERR_TOPO;
}

// All threads. scr/scr_bytes: dynamic shared memory scratch; ws: >= 32 ints shared.
// have_order: index_to_node / node_to_index already hold a valid topological order (cta_fuse_alignment keeps it up to
// date), so only the edge sort, max_remain and the row tables are (re)built: in the shared-memory scratch where the graph fits
// (graph_phases.cuh: topo_rows_smem), else by the global-memory form below.
__device__ void cta_topo_sort(Graph &g, RowTables &rt, unsigned char *scr, int scr_bytes, int *ws, bool have_order) {
    const int tid = threadIdx.x, T = blockDim.x, n = g.node_n;
    if (have_order && topo_smem_fits(n, scr_bytes)) { topo_rows_smem(g, rt, scr, ws, T); return; }
    if (have_order) {
        for (int v = tid; v < n; v += T) graph_sort_node_edges(g, v);
        __syncthreads();
    } else {
    // ---- (1) BFS index + edge sort ----
    for (int v = tid; v < n; v += T) g.tmp0[v] = g.out_n[v];
    __syncthreads();
    const int E = cta_excl_scan(g.tmp0, n, ws);
    if (n < 65536 && bfs_scratch_bytes(n, E) <= (size_t)scr_bytes) {
        BfsScratch B;
        B.optr = reinterpret_cast<uint32_t *>(scr);
        B.odst = reinterpret_cast<uint16_t *>(B.optr + n + 1);
        B.queue = B.odst + E; B.indeg = B.queue + n;
        B.alnn = reinterpret_cast<uint8_t *>(B.indeg + n);
        for (int v = tid; v < n; v += T) {
            const uint32_t o = (uint32_t)g.tmp0[v];
            B.optr[v] = o;
            const int oo = g.out_off[v], on = g.out_n[v];
            for (int i = 0; i < on; ++i) B.odst[o + i] = (uint16_t)g.out_id[oo + i];
            B.indeg[v] = (uint16_t)g.in_n[v]; B.alnn[v] = g.aln_n[v];
        }
        if (tid == 0) B.optr[n] = (uint32_t)E;
        __syncthreads();
        // one thread numbers the nodes from the shared-memory copy; everybody else sorts edge lists meanwhile
        if (T > 32) {
            if (tid == 0) bfs_index_smem(g, B);
            else if (tid >= 32) for (int v = tid - 32; v < n; v += T - 32) graph_sort_node_edges(g, v);
        } else {
            if (tid == 0) bfs_index_smem(g, B);
            __syncwarp();
            for (int v = tid; v < n; v += T) graph_sort_node_edges(g, v);
        }
        __syncthreads();
        if (g.err) return;
        for (int k = tid; k < n; k += T) { const int v = B.queue[k]; g.index_to_node[k] = v; g.node_to_index[v] = k; }
    } else {
        if (tid == 0) graph_bfs_index(g);
        __syncthreads();
        if (g.err) return;
        for (int v = tid; v < n; v += T) graph_sort_node_edges(g, v);
    }
    __syncthreads();
    }
    // ---- (2) max_remain by pointer jumping: d[v] = #steps to SINK along the first heaviest out edge ----
    int *nx[2] = {g.tmp0, g.tmp1}, *dd[2] = {g.remain, g.msa_rank};
    for (int v = tid; v < n; v += T) {
        int nxt = SINK_ID, dist = 0;
        if (v != SINK_ID) {
            int max_w = -1;
            const int oo = g.out_off[v], on = g.out_n[v];
            for (int i = 0; i < on; ++i) if (g.out_w[oo + i] > max_w) { max_w = g.out_w[oo + i]; nxt = g.out_id[oo + i]; }
            dist = 1;
        }
        nx[0][v] = nxt; dd[0][v] = dist;
    }
    __syncthreads();
    int cur = 0;
    for (int span = 1; span < n; span <<= 1, cur ^= 1) {
        for (int v = tid; v < n; v += T) {
            const int nv = nx[cur][v];
            dd[cur ^ 1][v] = dd[cur][v] + dd[cur][nv];
            nx[cur ^ 1][v] = nx[cur][nv];
        }
        __syncthreads();
    }
    if (cur == 0) { for (int v = tid; v < n; v += T) g.remain[v] -= 1; }
    else { for (int v = tid; v < n; v += T) g.remain[v] = g.msa_rank[v] - 1; }
    __syncthreads();
    // ---- (3) row tables: CSR offsets of the predecessor lists by topological index, then one row per thread ----
    for (int r = tid; r < n; r += T) g.tmp0[r] = g.in_n[g.index_to_node[r]];
    __syncthreads();
    cta_excl_scan(g.tmp0, n, ws);
    for (int r = tid; r < n; r += T) graph_build_row(g, rt, r, g.tmp0[r]);
    __syncthreads();
}


// abpoa_DFS_set_msa_rank (abpoa_graph.c:359-410) + msa_len (abpoa_output.c:157) on a shared-memory copy of the out-edge
// CSR (one thread walks; the rest stage and write back). Falls back to the global-memory walk when the graph does not
// fit the scratch. All threads; *msa_len_out is in shared memory.
__device__ void cta_msa_rank(Graph &g, unsigned char *scr, int scr_bytes, int *ws, int *msa_len_out) {
    const int tid = threadIdx.x, T = blockDim.x, n = g.node_n;
    for (int v = tid; v < n; v += T) g.tmp0[v] = g.out_n[v];
    __syncthreads();
    const int E = cta_excl_scan(g.tmp0, n, ws);
    if (n < 65535 && bfs_scratch_bytes(n, E) + 2 * (size_t)n <= (size_t)scr_bytes) {
        BfsScratch B;
        B.optr = reinterpret_cast<uint32_t *>(scr);
        B.odst = reinterpret_cast<uint16_t *>(B.optr + n + 1);
        B.queue = B.odst + E; B.indeg = B.queue + n;
        uint16_t *rk = B.indeg + n;
        B.alnn = reinterpret_cast<uint8_t *>(rk + n);
        for (int v = tid; v < n; v += T) {
            const uint32_t o = (uint32_t)g.tmp0[v];
            B.optr[v] = o;
            const int oo = g.out_off[v], on = g.out_n[v];
            for (int i = 0; i < on; ++i) B.odst[o + i] = (uint16_t)g.out_id[oo + i];
            B.indeg[v] = (uint16_t)g.in_n[v]; B.alnn[v] = g.aln_n[v];
        }
        if (tid == 0) B.optr[n] = (uint32_t)E;
        __syncthreads();
        if (tid == 0) {
            uint16_t *st = B.queue;
            int sp = 0, rank = 0, len = -1;
            st[sp++] = SRC_ID; rk[SRC_ID] = 0xffff;
            while (sp > 0) {
                const int cur = st[--sp];
                if (rk[cur] == 0xffff) {
                    rk[cur] = (uint16_t)rank;
                    for (int i = 0; i < B.alnn[cur]; ++i) rk[g.aln_id[cur * 4 + i]] = (uint16_t)rank;
                    ++rank;
                }
                if (cur == SINK_ID) { len = (int)rk[SINK_ID] - 1; break; }
                const uint32_t o0 = B.optr[cur], o1 = B.optr[cur + 1];
                for (uint32_t i = o0; i < o1; ++i) {
                    const int o = B.odst[i];
                    const int left = (int)B.indeg[o] - 1; B.indeg[o] = (uint16_t)left;
                    if (left == 0) {
                        const int an = B.alnn[o];
                        bool ok = true;
                        for (int j = 0; j < an; ++j) if (B.indeg[g.aln_id[o * 4 + j]] != 0) { ok = false; break; }
                        if (!ok) continue;
                        st[sp++] = (uint16_t)o; rk[o] = 0xffff;
                        for (int j = 0; j < an; ++j) { const int a = g.aln_id[o * 4 + j]; st[sp++] = (uint16_t)a; rk[a] = 0xffff; }
                    }
                }
            }
            if (len < 0) g.err = JOB_ERR_TOPO;
            *msa_len_out = len;
        }
        __syncthreads();
        if (g.err) return;
        for (int v = tid; v < n; v += T) g.msa_rank[v] = rk[v];
    } else {
        if (tid == 0) *msa_len_out = graph_msa_rank(g);
    }
    __syncthreads();
}

}  // namespace barb200
