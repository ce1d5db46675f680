// poa_types.h -- plain-old-data shared by the CUDA kernels and the host orchestration of libbarb200.
//
// One *job* is one abpoa_msa() call of the reference (one sliding window of one end,
// bar/impl/poaBarAligner.c:609): K sequences in, a K x msa_len byte matrix out.
// One *slot* is the device workspace a resident CTA uses while it works through a job:
// the partial-order graph, the banded DP planes of the current alignment, the cigar.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define HD __host__ __device__ __forceinline__
#else
#define HD inline
#endif

// The threads of a CTA program written once for both targets (guide_tree.cuh, graph_phases.cuh): on the device every thread runs
// the body once with its own tid; on the host (tests/hosttest) the body runs for tid = 0 .. T-1 one after the other, and the barrier
// between two such loops is the loop's end.
#if defined(__CUDA_ARCH__)
#define GT_THREADS(tid, T) for (int tid = (int)threadIdx.x, _gt_once = 1; _gt_once; _gt_once = 0)
#define GT_SYNC() __syncthreads()
#else
#define GT_THREADS(tid, T) for (int tid = 0; tid < (T); ++tid)
#define GT_SYNC() ((void)0)
#endif

namespace barb200 {

constexpr int SRC_ID = 0;    // ABPOA_SRC_NODE_ID  (abPOA include/abpoa.h:27)
constexpr int SINK_ID = 1;   // ABPOA_SINK_NODE_ID (abPOA include/abpoa.h:28)
constexpr int GAP_CODE = 5;  // abpt->m, the gap byte of msa_base (abpoa_output.c:160-163)

constexpr int OP_M = 0x1, OP_E1 = 0x2, OP_E2 = 0x4, OP_E = 0x6, OP_F1 = 0x8, OP_F2 = 0x10, OP_F = 0x18, OP_ALL = 0x1f;
constexpr int CMATCH = 0, CINS = 1, CDEL = 2;

enum JobStatus : int {
    JOB_OK = 0,
    JOB_ERR_NODE_CAP = 1,    // graph outgrew the slot's node arrays
    JOB_ERR_EDGE_CAP = 2,    // edge pools exhausted
    JOB_ERR_PLANE_CAP = 3,   // DP planes outgrew the slot (host retries with a larger slot)
    JOB_ERR_CIGAR_CAP = 4,
    JOB_ERR_MSA_CAP = 5,     // msa_len larger than the job's output stride (host retries)
    JOB_ERR_TOPO = 6,        // "Failed to set node index" in the reference (abpoa_graph.c:265)
    JOB_ERR_BACKTRACK = 7,   // "Error in cg_backtrack" in the reference (abpoa_align_simd.c:448)
    JOB_ERR_ALIGNED_CAP = 8,
    JOB_ERR_QUERY_LEN = 9,   // query longer than 16 x threads per CTA (host sizing bug)
    JOB_ERR_GT_CAP = 10,     // minimizer keys of the guide tree outgrew the slot (host retries with a larger slot)
    JOB_ERR_TRACE_CAP = 11   // a trace kernel's alignment records outgrew the job's trace region (host retries with a larger one)
};

// Scoring / banding parameters: what abpoaParamaters_constructFromCactusParams builds
// (bar/impl/poaBarAligner.c:24-81) reduced to what the DP reads.
struct PoaParams {
    int mat[25];          // 5x5 substitution matrix, row = graph base, col = query base
    int o1, e1, o2, e2;   // convex gap: min(o1 + k*e1, o2 + k*e2)
    int wb; float wf;     // adaptive band: w = wb + (int)(wf * qlen)  (abpoa_align_simd.c:474)
    int max_mat, min_mis; // derived, used for the int16/int32 lane-count rule (abpoa_align_simd.c:1293-1302)
    int inf_min;          // the reference's int32 "minus infinity" (abpoa_align_simd.c:1299)
};

// Per-job descriptor (device resident, written by the host before launch).
struct JobDesc {
    int n_seq;            // K
    int64_t seq_off;      // offset of the job's first base in the packed sequence buffer
    int64_t len_off;      // offset into the lens / order arrays
    int64_t msa_off;      // offset of the job's output block in the msa buffer
    int msa_stride;       // column capacity of the output block (rows are msa_stride apart)
    int progressive;      // abpt->progressive_poa of this job (poaBarAligner.c:567-571): read order from the guide tree
};

// The partial-order graph of one job (abPOA include/abpoa.h:96-116), SoA in the slot workspace.
// Edge lists are small arrays carved from bump-allocated pools; growing one copies it to a fresh chunk of
// twice the size (same observable behaviour as the reference's realloc, abpoa_graph.c:49-85).
struct Graph {
    int node_n, node_cap;
    int W;                              // 64-bit words per read-id set = 1 + ((K-1) >> 6)  (abpoa_graph.c:692)
    int in_used, in_pool, out_used, out_pool;
    int err;
    uint8_t *base;                      // [node_cap]
    uint8_t *aln_n;                     // [node_cap]   number of aligned nodes (<= 4: one per other base)
    int *aln_id;                        // [node_cap*4]
    int *in_off, *in_n, *in_cap;        // [node_cap]
    int *out_off, *out_n, *out_cap;     // [node_cap]
    int *in_id, *in_w;                  // [in_pool]
    int *out_id, *out_w;                // [out_pool]
    uint64_t *out_rid;                  // [out_pool * W] read ids per out edge (abpoa_graph.c:525-544)
    int *index_to_node, *node_to_index; // [node_cap] topological (BFS) order
    int *remain;                        // [node_cap] max_remain (abpoa_graph.c:268-309)
    int *msa_rank;                      // [node_cap]
    int *tmp0, *tmp1;                   // [node_cap] scratch: degree counters, queues
};

// Row-major view of the sorted graph that the DP sweeps (built after every topological sort): one 16-byte record
// per topological index r, fetched with a single load per row.
struct alignas(16) RowRec {
    int base_npre;       // base of the node at index r | (number of predecessors << 8)
    int rd;              // remain[v] - remain[SINK] - 1  (GET_AD_DP_BEGIN/END, abpoa_align.h:34-35)
    int pre_off;         // CSR offset into pre_row
    int pre0;            // first predecessor row (the only one for ~90 % of rows), -1 if none
};
struct RowTables {
    RowRec *rec;         // [node_cap]
    int *pre_row;        // [in_pool]   predecessor rows in in_id order (abpoa_align_simd.c:550-558)
};

// Per-row band bookkeeping of the current alignment.
struct alignas(16) RowInfo {
    int beg, end;        // dp_beg / dp_end (abpoa_align_simd.c:946-960)
    int left, right;     // left/right-most argmax of H in the row (abpoa_align_simd.c:1107-1119)
};

// Banded DP planes of the current alignment.
// Column ownership is fixed: thread t of the CTA owns columns [CPT*t, CPT*t + CPT) of EVERY row, so the values of the
// previous row stay in that thread's registers. A row with band [beg, end] covers the threads t0 = beg/CPT .. t1 = end/CPT
// and is stored at planes + row_off[r] as row_blocks(beg, end) thread blocks of TB = 2*CPT ints, starting at thread
// row_t0(beg): the stored range is widened to an even first thread and an even count, so that it has at most one
// padding block at either end (written with out-of-band values, never read). The row is "chunk-major": 8 chunk planes of
// 4 ints each -- H columns 0-3, 4-7, 8-11, 12-15 of every block, then the same four for D -- and stored block b's chunk c
// sits at int offset (c * nblk + b) * 4. A warp's 128-bit access to one chunk thus covers 512 contiguous bytes, and the even
// start and count keep every such run 32 B aligned (whole sectors only).
//
// What is stored, and why it is enough for the reference's traceback (abpoa_align_simd.c:309-458) -- 8 bytes per cell
// instead of the reference's five int32 planes (20 bytes):
//   H  the cell score, int32.
//   D  the two E values kept for later rows, as 16-bit DISTANCES below H: D = (H - E1) | (H - E2) << 16. For every row but
//      the first, E' = max(E_in - e, H - oe) with E_in <= H, so e <= H - E' <= oe: exact in 16 bits for any gap open + extend
//      below 65535 (barb200_create checks). 0xffff encodes "minus infinity" (row 0, where E does not derive from H);
//      cells outside the band hold H = inf_min, D = 0.
//   F1 / F2 are NOT stored: the traceback reads them only at the few cells where an insertion starts or continues, and they
//      are a pure function of the row's H' = max(M + s, E1, E2), which the predecessor rows' H / D give back. The warp traceback
//      decides "H == F" and the insertion's length from the row's own H values (poa_cta.cuh: warp_backtrack_step); the serial form
//      (host build, debug mode) recomputes the row prefix it needs (poa_graph.cuh: row_f_cache).
constexpr int CPT = 16;
constexpr int E_NEG16 = 0xffff;
struct DpState {
    int *planes; int64_t plane_cap;     // ints
    int64_t *row_off;                   // [node_cap]
    RowInfo *info;                      // [node_cap]
    uint64_t *cigar; int n_cigar, cigar_cap;
    int best_i, best_j, best_score;
    int *fc;                            // [2 * fc_cap] F1 / F2 of the cached row prefix (traceback scratch)
    int fc_cap, fc_row, fc_hi;          // columns per plane; cached row (-1: none) and its highest computed column
};

// Row layout (see DpState). j must lie in a stored thread's range.
constexpr int TB = 2 * CPT;   // ints per thread block of a row
constexpr int CHUNK = 4;      // ints per chunk (one 128-bit access)
HD int row_t0(int beg) { return (beg / CPT) & ~1; }                                   // first stored thread
HD int row_blocks(int beg, int end) { return ((end / CPT - row_t0(beg)) | 1) + 1; }   // stored blocks (even)
// int offset of chunk c (0-3: H, 4-7: D) of stored block b in a row of nblk blocks
HD int64_t chunk_index(int nblk, int b, int c) { return ((int64_t)c * nblk + b) * CHUNK; }
// int offset of column j of `plane` (0: H, 1: D) inside the row
HD int64_t plane_index(int beg, int end, int plane, int j) {
    return chunk_index(row_blocks(beg, end), j / CPT - row_t0(beg), plane * (CPT / CHUNK) + j % CPT / CHUNK) + j % CHUNK;
}
HD int64_t row_ints(int beg, int end) { return (int64_t)TB * row_blocks(beg, end); }
// E value from H and its 16-bit distance code
HD int e_decode(int h, int code, int inf_min) { return code == E_NEG16 ? inf_min : h - code; }
HD int e_encode(int h, int e) { const int d = h - e; return (d >= 0 && d < E_NEG16) ? d : E_NEG16; }

HD int imax(int a, int b) { return a > b ? a : b; }
HD int imin(int a, int b) { return a < b ? a : b; }

// The DP's parameters from the substitution matrix, the two gap pairs and the band, with the fields derived from them
inline PoaParams poa_params(const int mat[25], int o1, int e1, int o2, int e2, int wb, float wf) {
    PoaParams P;
    P.o1 = o1; P.e1 = e1; P.o2 = o2; P.e2 = e2; P.wb = wb; P.wf = wf;
    P.max_mat = 0; P.min_mis = 0;
    for (int i = 0; i < 25; ++i) { P.mat[i] = mat[i]; P.max_mat = imax(P.max_mat, mat[i]); P.min_mis = imax(P.min_mis, -mat[i]); }
    // the reference's int32 minus infinity, abpoa_align_simd.c:1299
    P.inf_min = imax(imax(INT32_MIN + P.min_mis, INT32_MIN + o1 + e1), INT32_MIN + o2 + e2) + 512 * imax(e1, e2);
    return P;
}

}  // namespace barb200
