// graph_phases.cuh -- the graph phases between two DP sweeps that run on compact copies in the CTA's shared-memory scratch.
//
// Between sweeps the dynamic shared memory of a CTA is idle (during a sweep it holds the row ring), and at 4 CTAs per SM the
// graph phases' chains of dependent global-memory loads wait behind the other CTAs' plane stores. So where the graph fits, the
// per-node state these phases compute stays on chip and the global arrays are written once:
//   * the order splice of a fusion (poa_cta.cuh: cta_fuse_alignment, step 3b): anchors, counts and the new order;
//   * max_remain by pointer jumping, then the row tables (poa_cta.cuh: cta_topo_sort, the have_order path).
// Graphs that do not fit, or whose node ids need more than 16 bits, take the global-memory forms in poa_cta.cuh.
// __host__ __device__: tests/hosttest runs the same source with the CTA's T threads one after the other (GT_THREADS) and checks
// every result against the serial forms of poa_graph.cuh.
#pragma once
#include "poa_graph.cuh"

// the two phases are cold, latency-bound code: kept out of line so that they do not change how the kernels' DP sweep is compiled
#if defined(__CUDACC__)
#define HD_COLD __host__ __device__ __noinline__
#else
#define HD_COLD inline
#endif

namespace barb200 {

// exclusive prefix sum of a[0..n) in place (global or shared memory); returns the total. All threads of the CTA.
// ws: >= 32 ints of shared memory.
HD int cta_excl_scan(int *a, int n, int *ws) {
#if defined(__CUDA_ARCH__)
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = T >> 5;
    const int chunk = (n + T - 1) / T, b = min(n, tid * chunk), e = min(n, b + chunk);
    int s = 0;
    for (int i = b; i < e; ++i) s += a[i];
    int inc = s;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, off); if (lane >= off) inc += v; }
    __syncthreads();                       // ws may still be read by a previous call
    if (lane == 31) ws[warp] = inc;
    __syncthreads();
    int woff = 0, total = 0;
    for (int k = 0; k < nw; ++k) { const int v = ws[k]; if (k < warp) woff += v; total += v; }
    int run = woff + inc - s;
    for (int i = b; i < e; ++i) { const int v = a[i]; a[i] = run; run += v; }
    __syncthreads();
    return total;
#else
    (void)ws;
    int run = 0;
    for (int i = 0; i < n; ++i) { const int v = a[i]; a[i] = run; run += v; }
    return run;
#endif
}

// inclusive prefix maximum of a[0..n) in place. All threads of the CTA. ws: >= 32 ints of shared memory.
HD void cta_incl_max_scan(int *a, int n, int *ws) {
#if defined(__CUDA_ARCH__)
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = T >> 5;
    const int chunk = (n + T - 1) / T, b = min(n, tid * chunk), e = min(n, b + chunk);
    int s = INT32_MIN;
    for (int i = b; i < e; ++i) s = max(s, a[i]);
    int inc = s;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, off); if (lane >= off) inc = max(inc, v); }
    int run = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) run = INT32_MIN;
    __syncthreads();
    if (lane == 31) ws[warp] = inc;
    __syncthreads();
    for (int k = 0; k < nw; ++k) if (k < warp) run = max(run, ws[k]);
    for (int i = b; i < e; ++i) { run = max(run, a[i]); a[i] = run; }
    __syncthreads();
#else
    (void)ws;
    int run = INT32_MIN;
    for (int i = 0; i < n; ++i) { run = imax(run, a[i]); a[i] = run; }
#endif
}

HD void cta_atomic_inc(int *p) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, 1);
#else
    ++*p;
#endif
}

// ---- the order splice of a fusion (cta_fuse_alignment, step 3b; see there for why it gives a topological order) ----
// Scratch: anc[L], cnt[n_old] (int32), then the new order new_i2n[n] (uint16).
HD size_t splice_smem_bytes(int L, int n_old, int n) { return 4 * ((size_t)L + n_old) + 2 * (size_t)n; }
HD bool splice_smem_fits(int L, int n_old, int n, int scr_bytes) { return n < 65536 && splice_smem_bytes(L, n_old, n) <= (size_t)scr_bytes; }

// node_of[q]: the node query base q ends up on; the nodes first_new .. first_new + n_new - 1 are new, numbered in query order.
// Moves every old node up by the number of new nodes anchored before it and writes index_to_node / node_to_index once. All threads.
HD_COLD void splice_order_smem(Graph &g, const int *node_of, int L, int first_new, int n_new, unsigned char *scr, int *ws, int T) {
    const int n_old = first_new, n = first_new + n_new;
    int *anc = reinterpret_cast<int *>(scr), *cnt = anc + L;
    uint16_t *new_i2n = reinterpret_cast<uint16_t *>(cnt + n_old);
    // anchor of base q: the last old index of its node's block of aligned nodes (-1: none)
    GT_THREADS(tid, T) {
        for (int q = tid; q < L; q += T) {
            const int v = node_of[q];
            int e = v < first_new ? g.node_to_index[v] : -1;
            for (int k = 0; k < g.aln_n[v]; ++k) { const int a = g.aln_id[v * 4 + k]; if (a < first_new) e = imax(e, g.node_to_index[a]); }
            anc[q] = e;
        }
        for (int i = tid; i < n_old; i += T) cnt[i] = 0;
    }
    GT_SYNC();
    cta_incl_max_scan(anc, L, ws);
    GT_THREADS(tid, T) for (int q = tid; q < L; q += T) if (node_of[q] >= first_new) cta_atomic_inc(&cnt[imax(anc[q], 0)]);
    GT_SYNC();
    cta_excl_scan(cnt, n_old, ws);                                   // cnt[i] = number of new nodes anchored before old index i
    GT_THREADS(tid, T) {
        for (int i = tid; i < n_old; i += T) new_i2n[i + cnt[i]] = (uint16_t)g.index_to_node[i];
        for (int q = tid; q < L; q += T) { const int v = node_of[q]; if (v >= first_new) new_i2n[imax(anc[q], 0) + 1 + (v - first_new)] = (uint16_t)v; }
    }
    GT_SYNC();
    GT_THREADS(tid, T) for (int k = tid; k < n; k += T) { const int v = new_i2n[k]; g.index_to_node[k] = v; g.node_to_index[v] = k; }
    GT_SYNC();
}

// ---- edge sort, max_remain and the row tables (cta_topo_sort when the order is already known) ----
// Scratch: next[2][n], dist[2][n] (uint16, the pointer jumping's double buffers), then off[n] (int32, each row's offset into
// pre_row). Once the jumping is done, next[] holds index_to_node / node_to_index.
HD size_t topo_smem_bytes(int n) { return (size_t)12 * n; }
HD bool topo_smem_fits(int n, int scr_bytes) { return n < 65536 && topo_smem_bytes(n) <= (size_t)scr_bytes; }

constexpr int TOPO_ROWS_PER_THREAD = 4;     // rows whose global loads a thread has in flight together

// Same results as graph_sort_node_edges on every node, graph_bfs_remain and graph_build_rows, with index_to_node a topological
// order. All threads.
HD_COLD void topo_rows_smem(Graph &g, RowTables &rt, unsigned char *scr, int *ws, int T) {
    const int n = g.node_n;
    uint16_t *nx = reinterpret_cast<uint16_t *>(scr), *dd = nx + 2 * n;
    int *off = reinterpret_cast<int *>(scr + 8 * (size_t)n);
    // the sort orders out edges by weight, descending, so a node's first out edge is the first heaviest one, the edge
    // graph_bfs_remain follows; d = steps to SINK along those edges
    GT_THREADS(tid, T) for (int v = tid; v < n; v += T) {
        graph_sort_node_edges(g, v);
        const int on = g.out_n[v];
        nx[v] = (uint16_t)(v == SINK_ID || on == 0 ? SINK_ID : g.out_id[g.out_off[v]]);
        dd[v] = (uint16_t)(v != SINK_ID);
    }
    GT_SYNC();
    // pointer jumping (list ranking): log2(n) rounds; d stays below n, so 16 bits hold it
    int cur = 0;
    for (int span = 1; span < n; span <<= 1, cur ^= 1) {
        const uint16_t *nc = nx + cur * n, *dc = dd + cur * n;
        uint16_t *nn = nx + (cur ^ 1) * n, *dn = dd + (cur ^ 1) * n;
        GT_THREADS(tid, T) for (int v = tid; v < n; v += T) { const int w = nc[v]; dn[v] = (uint16_t)(dc[v] + dc[w]); nn[v] = nc[w]; }
        GT_SYNC();
    }
    const uint16_t *dist = dd + cur * n;                 // remain + 1
    uint16_t *i2n = nx, *n2i = nx + n;
    GT_THREADS(tid, T) for (int k = tid; k < n; k += T) {
        g.remain[k] = (int)dist[k] - 1;
        const int v = g.index_to_node[k];
        i2n[k] = (uint16_t)v; n2i[v] = (uint16_t)k; off[k] = g.in_n[v];
    }
    GT_SYNC();
    cta_excl_scan(off, n, ws);
    const int rd0 = (int)dist[SINK_ID];                  // rd = remain[v] - remain[SINK] - 1 = dist[v] - dist[SINK] - 1
    constexpr int RB = TOPO_ROWS_PER_THREAD;
    GT_THREADS(tid, T) for (int r0 = tid; r0 < n; r0 += RB * T) {
        // every global load of RB rows is issued before any of their stores (the stores could alias them for the compiler)
        int io[RB], in[RB], b[RB], p0[RB];
#pragma unroll
        for (int u = 0; u < RB; ++u) {
            in[u] = 0; io[u] = 0; b[u] = 0;
            const int r = r0 + u * T;
            if (r < n) { const int v = i2n[r]; io[u] = g.in_off[v]; in[u] = g.in_n[v]; b[u] = g.base[v]; }
        }
#pragma unroll
        for (int u = 0; u < RB; ++u) p0[u] = in[u] ? g.in_id[io[u]] : -1;
#pragma unroll
        for (int u = 0; u < RB; ++u) {
            const int r = r0 + u * T;
            if (r >= n) break;
            const int o = off[r], v = i2n[r];
            RowRec rec;
            rec.base_npre = b[u] | (in[u] << 8);
            rec.rd = (int)dist[v] - rd0 - 1;
            rec.pre_off = o;
            rec.pre0 = in[u] ? (int)n2i[p0[u]] : -1;
            rt.rec[r] = rec;
            if (in[u]) rt.pre_row[o] = rec.pre0;
            for (int k = 1; k < in[u]; ++k) rt.pre_row[o + k] = n2i[g.in_id[io[u] + k]];
        }
    }
    GT_SYNC();
}

}  // namespace barb200
